"""Range scans on readers (dbeel_reader_scan): key ranges read the fences, the leaves their bound searches end in and the
records of the spans, and return what the seek oracle (tests/seek_oracle.py) returns -- which on sorted tables with no
stop is dbeel_scan_stream's result byte for byte; hash ranges return dbeel_scan_stream's result on the reader's snapshot."""
import ctypes
import os

import numpy as np
import pytest

import seek_oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS, assert_run_equal
from scan_cases import DAMAGES, damage, hash_ranges, key_ranges, random_tree

pytestmark = pytest.mark.gpu

EVERYTHING = [(b"", b"\xff" * 80)]


@pytest.fixture
def tiny_engine(monkeypatch):
    """An engine whose partitions and leaf groups are 4 KB."""
    monkeypatch.setenv("DBEEL_PARTITION_KB", "4")
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    e = capi.Engine(0)
    yield e
    e.close()


def _keys(tables):
    out = set()
    for d, i in tables:
        d, ix = bytes(d), bytes(i)
        for r in range(len(ix) // 16):
            off = int.from_bytes(ix[16 * r:16 * r + 8], "little")
            if off + 8 <= len(d):
                klen = int.from_bytes(d[off:off + 8], "little")
                if off + 8 + klen <= len(d):
                    out.add(d[off + 8:off + 8 + klen])
    return sorted(out)


def random_ranges(rng, tables, n):
    """Bounds that are present keys, absent keys (a present key with a byte added or dropped), keys over 64 bytes, empty
    and inverted ranges, overlapping ranges."""
    keys = _keys(tables) or [b"k"]

    def bound():
        k = keys[int(rng.integers(0, len(keys)))]
        style = int(rng.integers(0, 5))
        if style == 1:
            return k + b"\x00"
        if style == 2:
            return k[:-1]
        if style == 3:
            return k + b"\x7f" * 70
        return k
    out = []
    for j in range(n):
        a, b = bound(), bound()
        style = j % 5
        if style == 0:
            out.append((a, a))
        elif style == 1:
            out.append((max(a, b), min(a, b)))
        else:
            out.append((min(a, b), max(a, b)))
    return out


def check(e, reader, tables, ranges, sorted_clean=False):
    out, stop = reader.scan(ranges)
    st, reads = e.stats(), reader.last_stream_reads
    want, wstop = seek_oracle.reader_scan(tables, ranges)
    assert stop == wstop
    for d, (g, w) in enumerate(zip(out, want)):
        assert_run_equal(g, w, f"range {d}")
    assert st["input_bytes"] == sum(r[3] for r in reads)
    assert st["output_bytes"] == sum(g[0].size + g[1].size for g in out)
    for t, kind, off, size in reads:
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    if sorted_clean and stop[0] < 0:
        for ref in (e.scan_stream(tables, ranges, capi.SCAN_KEY), e.scan(tables, ranges, capi.SCAN_KEY)):
            assert ref[1] == stop
            for g, w in zip(out, ref[0]):
                assert_run_equal(g, w, "reader scan vs scan_stream / scan")
    return out, stop, reads, st


def _sorted(tables):
    """random_tree's tables with the shuffled one dropped: keys strictly ascend in each."""
    return [t for j, t in enumerate(tables) if j != 1 or len(tables) < 2]


@pytest.mark.parametrize("setting", ["default", "tiny_partitions", "depth0"])
def test_parity_on_random_trees(engine, tiny_engine, setting):
    e = tiny_engine if setting == "tiny_partitions" else engine
    fence_bytes = 1 if setting == "depth0" else 0
    for seed in range(12):
        rng = np.random.default_rng(700 + seed)
        tables = random_tree(rng, 1 + seed % 6, max_entries=120, big=seed == 5)
        for tbs, clean in ((tables, False), (_sorted(tables), True)):
            with e.open_reader([(d, i, None) for d, i in tbs], fence_bytes=fence_bytes) as r:
                for ranges in (key_ranges(tbs), random_ranges(rng, tbs, 9), EVERYTHING, random_ranges(rng, tbs, 256)):
                    check(e, r, tbs, ranges, sorted_clean=clean)


@pytest.mark.parametrize("kind", [k for k in DAMAGES if k != "ragged_index"])
def test_damage_inside_outside_and_on_the_search_path(engine, kind):
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    base = [(np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy())]
    other = random_tree(np.random.default_rng(3), 1)[0]
    inside = [(b"key-%06d" % 1400, b"key-%06d" % 1600)]
    outside = [(b"key-%06d" % 100, b"key-%06d" % 120)]
    clean = {}
    for ranges in (inside, outside):
        with engine.open_reader([(d_, i_, None) for d_, i_ in base + [other]]) as r:
            clean[str(ranges)] = r.scan(ranges)
    for rec in (1500, 1000):  # 1500 lies inside `inside`'s span only; 1000 is the root probe of every search
        # a table with no index record (a ragged one the reader rejects at open)
        bad = ([(base[0][0], base[0][1][:0])] if kind == "empty_table" else damage(base, kind, 0, rec)) + [other]
        with engine.open_reader([(d_, i_, None) for d_, i_ in bad]) as r:
            for ranges in (inside, outside, EVERYTHING):
                out, stop, _, _ = check(engine, r, bad, ranges)
                if rec == 1500 and ranges is outside and kind != "empty_table":
                    assert stop == (-1, 0, 0)
                    for g, w in zip(out, clean[str(ranges)][0]):
                        assert_run_equal(g, w, "damage outside every span")
                if rec == 1500 and ranges is inside and kind != "empty_table":
                    assert stop[0] == 0 and stop[2] == 1500
    # a probe the search cannot read: the table contributes nothing and the stop is at that record
    bad = [base[0], other]
    ix = bad[0][1].copy()
    ix[16 * 1000:16 * 1000 + 8] = np.array([bad[0][0].size + 1], "<u8").view(np.uint8)
    bad = [other, (bad[0][0], ix)]
    with engine.open_reader([(d_, i_, None) for d_, i_ in bad]) as r:
        out, stop, _, _ = check(engine, r, bad, outside)
        assert stop == (1, capi.SCAN_STOP_PANIC, 1000)


def _table_20000():
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(20000)]
    d, i = sstable.build_run(ents)
    return np.asarray(d, np.uint8), np.asarray(i, np.uint8)


def test_reads(engine):
    d, i = _table_20000()
    tables = [(d, i)]
    narrow = [(b"key-%06d" % 7000, b"key-%06d" % 7020)]
    with engine.open_reader([(d, i, None)]) as r:
        _, _, first, st1 = check(engine, r, tables, narrow, sorted_clean=True)
        _, _, second, st2 = check(engine, r, tables, narrow, sorted_clean=True)
        # the fences were read by the first call only: the second reads a subset of the first's reads, fewer bytes
        assert set(second) <= set(first) and len(second) < len(first)
        assert st2["input_bytes"] < st1["input_bytes"] and st2["input_bytes"] < 0.01 * (d.size + i.size)
        assert st2["entries_in"] == 20 and st2["entries_out"] == 20
        # every .index read of the span plan lies in the span or in a touched leaf near a bound
        for t, kind, off, size in second:
            if kind == 2:
                assert 16 * 6900 <= off and off + size <= 16 * 7100
        # a range key over the frame cap: fences are read for this call, every call
        wide = [(b"key-%06d" % 7000 + b"\x00" * 70, b"key-%06d" % 7020)]
        _, _, w1, _ = check(engine, r, tables, wide, sorted_clean=True)
        _, _, w2, _ = check(engine, r, tables, wide, sorted_clean=True)
        assert sorted(w1) == sorted(w2) and len(w2) > len(second)
        # a whole-key-space range reads the whole files once more than the seek
        _, _, wr, stw = check(engine, r, tables, EVERYTHING, sorted_clean=True)
        assert stw["entries_in"] == 20000


def test_hash_ranges_equal_scan_stream(engine, tiny_engine):
    for e in (engine, tiny_engine):
        for seed in range(6):
            rng = np.random.default_rng(40 + seed)
            tables = random_tree(rng, 1 + seed, max_entries=100, big=seed == 2)
            if seed == 4:
                tables = damage(tables, "timestamp", 2, 5)
            ranges = hash_ranges(rng, 7)
            with e.open_reader([(d, i, None) for d, i in tables]) as r:
                out, stop = r.scan(ranges, capi.SCAN_HASH)
                ref, rstop = e.scan_stream(tables, ranges, capi.SCAN_HASH)
                assert stop == rstop
                for g, w in zip(out, ref):
                    assert_run_equal(g, w, "hash ranges")


def test_tree_reader_snapshot(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(31)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    kr = [(b"t00500", b"t01800"), (b"t02990", b"u"), (b"a", b"t00010")]
    hr = hash_ranges(rng, 5)
    snap = tree.sstable_indices_and_sizes()
    a = tree.open_reader()
    rec = {k: tree.scan(rg, k) for k, rg in ((capi.SCAN_KEY, kr), (capi.SCAN_HASH, hr))}
    for k, rg in ((capi.SCAN_KEY, kr), (capi.SCAN_HASH, hr)):
        out, stop = a.scan(rg, k)
        assert stop == rec[k][1]
        for g, w in zip(out, rec[k][0]):
            assert_run_equal(g, w, "tree reader")
        sizes, stop2 = a.scan(rg, k, write=lambda *args: 0)
        assert stop2 == stop and sizes == [(g[0].size, g[1].size, g[1].size // 16) for g in out]
    tree.flush(sstable.build_run([(b"t00600", b"new", BASE_TS + 10 ** 6)]))
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    for k, rg in ((capi.SCAN_KEY, kr), (capi.SCAN_HASH, hr)):
        out, stop = a.scan(rg, k)  # the snapshot, its files unlinked
        assert stop == rec[k][1]
        for g, w in zip(out, rec[k][0]):
            assert_run_equal(g, w, "tree reader after the compaction")
    c = tree.open_reader()
    for k, rg in ((capi.SCAN_KEY, kr), (capi.SCAN_HASH, hr)):
        out, stop = c.scan(rg, k)
        now = tree.scan(rg, k)
        assert stop == now[1]
        for g, w in zip(out, now[0]):
            assert_run_equal(g, w, "a reader opened after the compaction")
    a.close()
    c.close()
    tree.close()


def test_errors_leave_the_reader_usable(engine):
    d, i = _table_20000()
    tables = [(d, i)]
    narrow = [(b"key-%06d" % 7000, b"key-%06d" % 7100)]
    with engine.open_reader([(d, i, None)]) as r:
        want = check(engine, r, tables, narrow)[0]
        n_reads = len(r.last_stream_reads)
    for at in (0, 1, n_reads - 1):  # a fence read (first call), a leaf read, a span read
        with engine.open_reader([(d, i, None)]) as r:
            with pytest.raises(capi.DbeelError) as ex:
                r.scan(narrow, fail_read_at=at)
            assert ex.value.code == 4242
            out, stop, _, _ = check(engine, r, tables, narrow)
            for g, w in zip(out, want):
                assert_run_equal(g, w, f"after a failed read {at}")
    with engine.open_reader([(d, i, None)]) as r:
        with pytest.raises(capi.DbeelError) as ex:
            r.scan(narrow, write=lambda *args: 777)
        assert ex.value.code == 777
        check(engine, r, tables, narrow)
        for bad in ([], [(b"a", b"b")] * 257):
            with pytest.raises(capi.DbeelError) as ex:
                r.scan(bad)
            assert ex.value.code == capi.ERR_INVALID_ARG
        with pytest.raises(capi.DbeelError) as ex:
            r.scan([(1, 2)], kind=7)
        assert ex.value.code == capi.ERR_INVALID_ARG
        rptr, _keep = capi.pack_ranges(capi.SCAN_KEY, narrow)
        res = (capi.JobResult * 1)()
        stop = capi.ScanStop()
        rc = capi.lib().dbeel_reader_scan(r._h, capi.SCAN_KEY, rptr, 1, capi.SCAN_WRITE_FN(0), None, res, ctypes.byref(stop))
        assert rc == capi.ERR_INVALID_ARG
        check(engine, r, tables, narrow)
    with pytest.raises(ValueError):
        r.scan(narrow)


def test_span_past_4gib(engine):
    """.data past 4 GiB served by a callback and never held whole: 2,000 entries whose offsets all lie above 2^32 (the
    bytes below are never referenced), and a range of 20 keys among them."""
    pad = (1 << 32) + (300 << 20)
    ents = [(b"k%05d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    td, ti = sstable.build_run(ents)
    td, ti = bytes(np.asarray(td, np.uint8)), np.asarray(ti, np.uint8).reshape(-1, 16).copy()
    offs = ti[:, :8].copy().view("<u8").reshape(-1) + np.uint64(pad)
    ti[:, :8] = offs.astype("<u8").view(np.uint8).reshape(-1, 8)
    index = ti.reshape(-1).copy()
    data_len = pad + len(td)

    def read(t, kind, off, size):
        if kind == 2:
            return index[off:off + size].tobytes() if off + size <= index.size else 4243
        if off + size > data_len:
            return 4243
        out = bytearray(size)
        a, b = max(off, pad), off + size
        if a < b:
            out[a - off:b - off] = td[a - pad:b - pad]
        return bytes(out)

    ranges = [(b"k01000", b"k01020")]
    with engine.open_reader([(data_len, index.size, None)], read=read) as r:
        for _ in range(2):
            out, stop = r.scan(ranges)
            reads = r.last_stream_reads
            assert stop == (-1, 0, 0)
            assert_run_equal(out[0], sstable.build_run(ents[1000:1020]), "span above 2^32")
            assert any(kind == 1 and off > 1 << 32 for _, kind, off, _ in reads)
        assert sum(size for _, _, _, size in reads) < 64 << 10
