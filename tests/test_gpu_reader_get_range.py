"""Range reads on readers (dbeel_reader_get_range): per key range the newest version of every key, merged on the device,
against the range oracle (tests/range_oracle.py) -- the raw scan of tests/seek_oracle.py deduplicated, sorted and with
tombstones dropped unless asked for -- and, on sorted trees, against dbeel_flush of the raw scan and get_values."""
import ctypes
import os

import numpy as np
import pytest

import range_oracle
import seek_oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS, assert_run_equal
from scan_cases import DAMAGES, damage, key_ranges, random_tree

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
    """Present and absent bounds, bounds over 64 bytes, empty, inverted and overlapping ranges."""
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


def check(e, reader, tables, ranges, keep=False):
    """get_range against the oracle, and the read and stats contract; returns (out, stop, reads, stats) or None when the
    oracle says DBEEL_ERR_UNSORTED_RUN (which the call must then return)."""
    want = range_oracle.get_range(tables, ranges, keep)
    if want == range_oracle.UNSORTED:
        with pytest.raises(capi.DbeelError) as ex:
            reader.get_range(ranges, keep_tombstones=keep)
        assert ex.value.code == capi.ERR_UNSORTED_RUN
        return None
    out, stop = reader.get_range(ranges, keep_tombstones=keep)
    st, reads = e.stats(), reader.last_stream_reads
    assert stop == want[1]
    for d, (g, w) in enumerate(zip(out, want[0])):
        assert_run_equal(g, w, f"range {d}")
    assert st["input_bytes"] == sum(r[3] for r in reads)
    assert st["output_bytes"] == sum(g[0].size + g[1].size for g in out)
    assert st["entries_out"] == sum(g[1].size // 16 for g in out)
    if stop[0] < 0 and st["partitions"]:  # the range header copy, then the scan chain + the merge stage per partition
        assert st["kernel_launches"] == 1 + 20 * st["partitions"]
    for t, kind, off, size in reads:
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return out, stop, reads, st


def _sorted(tables):
    """random_tree's tables with the shuffled one dropped: keys strictly ascend in each."""
    return [t for j, t in enumerate(tables) if j != 1 or len(tables) < 2]


@pytest.mark.parametrize("setting", ["default", "tiny_partitions", "depth0", "page_cache"])
def test_parity_on_random_trees(engine, tiny_engine, setting):
    e = tiny_engine if setting == "tiny_partitions" else engine
    fence_bytes = 1 if setting == "depth0" else 0
    cache = e.open_page_cache(1 << 20) if setting == "page_cache" else None
    for seed in range(10):
        rng = np.random.default_rng(900 + seed)
        tables = random_tree(rng, 1 + seed % 6, max_entries=120, big=seed == 5)
        for tbs in (tables, _sorted(tables)):
            with e.open_reader([(d, i, None) for d, i in tbs], fence_bytes=fence_bytes) as r:
                if cache is not None:
                    r.attach_page_cache(cache)
                for ranges in (key_ranges(tbs), random_ranges(rng, tbs, 9), EVERYTHING, random_ranges(rng, tbs, 256)):
                    for keep in (False, True):
                        check(e, r, tbs, ranges, keep)
    if cache is not None:
        cache.close()


def test_sorted_trees_equal_flush_and_get_values(engine):
    for seed in range(6):
        rng = np.random.default_rng(1300 + seed)
        tables = _sorted(random_tree(rng, 2 + seed % 4, max_entries=150))
        ranges = random_ranges(rng, tables, 6) + [(b"", b"\xff" * 80)]
        with engine.open_reader([(d, i, None) for d, i in tables]) as r:
            kept, stop = r.get_range(ranges, keep_tombstones=True)
            live, _ = r.get_range(ranges)
            raw, rstop = r.scan(ranges)
            assert stop == rstop == (-1, 0, 0)
            for d, (g, s) in enumerate(zip(kept, raw)):
                if s[1].size:
                    fd, fi, _ = engine.flush(s)
                    assert_run_equal(g, (fd, fi), f"flush of S_{d}")
                else:
                    assert g[0].size == 0 and g[1].size == 0
            keys = _keys(tables)
            rows, gd, gi = r.get_values(keys, capi.LOOKUP_EXACT)
            found = {k: (v, ts) for k, v, ts in sstable.parse_run(gd, gi)}
            for g in live:
                for k, v, ts in sstable.parse_run(*g):
                    assert found[k] == (v, ts), "an output entry is get_values' row"
            for k, (v, ts) in found.items():
                d = next((j for j, (s, e_) in enumerate(ranges) if s <= k < e_), None)
                if d is not None and v:
                    assert k in {kk for kk, _, _ in sstable.parse_run(*live[d])}


def _long_prefix_tables(n_tables=3, n=400):
    prefix = b"P" * 80
    tables = []
    for t in range(n_tables):
        ents = [(prefix + b"%020d" % k, b"t%d-%d" % (t, k) if (k + t) % 7 else b"", BASE_TS + t)
                for k in range(t, n * (t + 1), t + 1)]
        d, i = sstable.build_run(ents)
        tables.append((np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy()))
    return tables


def test_many_partitions(tiny_engine):
    e = tiny_engine
    rng = np.random.default_rng(77)
    for tables in (_long_prefix_tables(), _sorted(random_tree(rng, 5, max_entries=300))):
        with e.open_reader([(d, i, None) for d, i in tables]) as r:
            keys = _keys(tables)
            wide = [(keys[len(keys) // 10], keys[-len(keys) // 10])]
            for ranges in (EVERYTHING, wide, [(b"", keys[len(keys) // 2]), (keys[len(keys) // 3], b"\xff" * 90)]):
                for keep in (False, True):
                    res = check(e, r, tables, ranges, keep)
                    assert res is not None and res[3]["partitions"] > 1


@pytest.mark.parametrize("kind", [k for k in DAMAGES if k != "ragged_index"])
def test_damage_inside_outside_and_on_the_search_path(engine, kind):
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    base = [(np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy())]
    other = random_tree(np.random.default_rng(3), 1)[0]
    inside = [(b"key-%06d" % 1400, b"key-%06d" % 1600)]
    outside = [(b"key-%06d" % 100, b"key-%06d" % 120)]
    clean_tables = base + [other]
    for rec in (1500, 1000):
        bad = ([(base[0][0], base[0][1][:0])] if kind == "empty_table" else damage(base, kind, 0, rec)) + [other]
        with engine.open_reader([(d_, i_, None) for d_, i_ in bad]) as r:
            for ranges in (inside, outside, EVERYTHING):
                res = check(engine, r, bad, ranges)
                if res is None:
                    continue
                out, stop = res[0], res[1]
                assert stop == seek_oracle.reader_scan(bad, ranges)[1]
                if stop[0] >= 0:
                    assert all(g[0].size == 0 and g[1].size == 0 for g in out)
            # the next clean call on the same reader is right
            if kind != "empty_table":
                check(engine, r, bad, outside)
    with engine.open_reader([(d_, i_, None) for d_, i_ in clean_tables]) as r:
        check(engine, r, clean_tables, inside)


def _table_20000():
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(20000)]
    d, i = sstable.build_run(ents)
    return np.asarray(d, np.uint8), np.asarray(i, np.uint8)


def test_reads_equal_scan_when_one_partition(engine):
    d, i = _table_20000()
    tables = [(d, i)]
    narrow = [(b"key-%06d" % 7000, b"key-%06d" % 7020)]
    for ranges in (narrow, EVERYTHING):
        with engine.open_reader([(d, i, None)]) as a, engine.open_reader([(d, i, None)]) as b:
            res = check(engine, a, tables, ranges)
            b.scan(ranges)
            assert res[3]["partitions"] == 1
            assert sorted(res[2]) == sorted(b.last_stream_reads)


def test_tree_reader_snapshot(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(31)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    kr = [(b"t00500", b"t01800"), (b"t02990", b"u"), (b"a", b"t00010")]
    snap = tree.sstable_indices_and_sizes()
    a = tree.open_reader()
    before = a.get_range(kr)
    assert before[1] == (-1, 0, 0)
    tree.flush(sstable.build_run([(b"t00600", b"new", BASE_TS + 10 ** 6)]))
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    after = a.get_range(kr)
    assert after[1] == before[1]
    for g, w in zip(after[0], before[0]):
        assert_run_equal(g, w, "tree reader snapshot")
    c = tree.open_reader()
    now, _ = c.get_range(kr)
    assert any(v == b"new" for k, v, _ in sstable.parse_run(*now[0]) if k == b"t00600")
    a.close()
    c.close()
    tree.close()


def test_errors_leave_the_reader_usable(engine):
    d, i = _table_20000()
    tables = [(d, i)]
    narrow = [(b"key-%06d" % 7000, b"key-%06d" % 7100)]
    cache = engine.open_page_cache(1 << 20)
    with engine.open_reader([(d, i, None)]) as r:
        want = check(engine, r, tables, narrow)[0]
        n_reads = len(r.last_stream_reads)
    for at in (0, 1, n_reads - 1):
        with engine.open_reader([(d, i, None)]) as r:
            r.attach_page_cache(cache)
            with pytest.raises(capi.DbeelError) as ex:
                r.get_range(narrow, fail_read_at=at)
            assert ex.value.code == 4242
            out = check(engine, r, tables, narrow)[0]
            for g, w in zip(out, want):
                assert_run_equal(g, w, f"after a failed read {at}")
    with engine.open_reader([(d, i, None)]) as r:
        r.attach_page_cache(cache)
        with pytest.raises(capi.DbeelError) as ex:
            r.get_range(narrow, write=lambda *args: 777)
        assert ex.value.code == 777
        check(engine, r, tables, narrow)
        for bad in ([], [(b"a", b"b")] * 257):
            with pytest.raises(capi.DbeelError) as ex:
                r.get_range(bad)
            assert ex.value.code == capi.ERR_INVALID_ARG
        rptr, _keep = capi.pack_ranges(capi.SCAN_KEY, narrow)
        res = (capi.JobResult * 1)()
        stop = capi.ScanStop()
        cb = capi.SCAN_WRITE_FN(lambda *args: 0)
        assert capi.lib().dbeel_reader_get_range(r._h, rptr, 1, 0x2, cb, None, res, ctypes.byref(stop)) == capi.ERR_INVALID_ARG
        assert capi.lib().dbeel_reader_get_range(r._h, rptr, 1, 0, capi.SCAN_WRITE_FN(0), None, res,
                                                 ctypes.byref(stop)) == capi.ERR_INVALID_ARG
        check(engine, r, tables, narrow)
        assert cache.stats()["capacity_pages"] > 0
    cache.close()


def test_inputs_past_4gib(engine):
    """.data past 4 GiB served by a callback: 2,000 entries above 2^32, and a newer table overriding keys near the end."""
    pad = (1 << 32) + (300 << 20)
    ents = [(b"k%05d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    td, ti = sstable.build_run(ents)
    td, ti = bytes(np.asarray(td, np.uint8)), np.asarray(ti, np.uint8).reshape(-1, 16).copy()
    offs = ti[:, :8].copy().view("<u8").reshape(-1) + np.uint64(pad)
    ti[:, :8] = offs.astype("<u8").view(np.uint8).reshape(-1, 8)
    index = ti.reshape(-1).copy()
    data_len = pad + len(td)
    newer = [(b"k%05d" % n, b"new%d" % n if n % 3 else b"", BASE_TS + 10 ** 6) for n in range(1990, 2010)]
    nd, ni = (bytes(np.asarray(x, np.uint8)) for x in sstable.build_run(newer))

    def read(t, kind, off, size):
        if t == 1:
            f = nd if kind == 1 else ni
            return f[off:off + size] if off + size <= len(f) else 4243
        if kind == 2:
            return index[off:off + size].tobytes() if off + size <= index.size else 4243
        if off + size > data_len:
            return 4243
        out = bytearray(size)
        a, b = max(off, pad), off + size
        if a < b:
            out[a - off:b - off] = td[a - pad:b - pad]
        return bytes(out)

    ranges = [(b"k01980", b"k02005")]
    with engine.open_reader([(data_len, index.size, None), (len(nd), len(ni), None)], read=read) as r:
        out, stop = r.get_range(ranges)
        assert stop == (-1, 0, 0)
        merged = {k: (v, ts) for k, v, ts in ents[1980:2000]}
        merged.update({k: (v, ts) for k, v, ts in newer if k < b"k02005"})
        want = [(k, v, ts) for k, (v, ts) in sorted(merged.items()) if v]
        assert_run_equal(out[0], sstable.build_run(want), "a range above 2^32 with a newer table")
        assert any(kind == 1 and off > 1 << 32 for t, kind, off, _ in r.last_stream_reads if t == 0)


def test_planner_failures_leave_the_reader_usable(tiny_engine):
    """A multi-partition call failing at reads spread over its whole read list -- the bound searches, the planner's
    .index pass, its sampled-key reads, the splitters' searches, its second .index pass and the partitions -- and at its
    write callback: the code comes back unchanged and the reader and its page cache stay right."""
    e = tiny_engine
    tables = _long_prefix_tables()
    with e.open_reader([(d, i, None) for d, i in tables]) as r:
        want, _, reads, st = check(e, r, tables, EVERYTHING)
    assert st["partitions"] > 1
    n = len(reads)
    keys = [j for j, (_, kind, _, size) in enumerate(reads) if kind == 1 and size <= 8 + 64]  # sampled keys
    picks = sorted(set(range(0, n, max(1, n // 40))) | set(keys[:2]) | set(keys[-2:]) | {n - 1})
    for at in picks:
        with e.open_reader([(d, i, None) for d, i in tables]) as r:
            with pytest.raises(capi.DbeelError) as ex:
                r.get_range(EVERYTHING, fail_read_at=at)
            assert ex.value.code == 4242
            out = check(e, r, tables, EVERYTHING)[0]
            for g, w in zip(out, want):
                assert_run_equal(g, w, f"after a failed read {at} of {n}")
    cache = e.open_page_cache(1 << 20)
    with e.open_reader([(d, i, None) for d, i in tables]) as r:
        r.attach_page_cache(cache)
        for fail_at in (0, 3):
            calls = [0]

            def write(*args):
                calls[0] += 1
                return 777 if calls[0] > fail_at else 0
            with pytest.raises(capi.DbeelError) as ex:
                r.get_range(EVERYTHING, write=write)
            assert ex.value.code == 777
            out, _, _, st2 = check(e, r, tables, EVERYTHING)
            assert st2["partitions"] > 1
            for g, w in zip(out, want):
                assert_run_equal(g, w, "after a failed write")
    cache.close()


def test_intervals_past_the_budget_are_not_staged(tiny_engine):
    """A shuffled table makes key intervals that would pass the budget: the call returns DBEEL_ERR_UNSORTED_RUN, or the
    raw scan's stop when the spans hold one, and stays usable."""
    e = tiny_engine
    tables = _long_prefix_tables()
    recs = tables[1][1].reshape(-1, 16).copy()
    np.random.default_rng(8).shuffle(recs)
    shuffled = [tables[0], (tables[1][0], recs.reshape(-1).copy()), tables[2]]
    for tbs in (shuffled, damage(shuffled, "timestamp", 2, 200), damage(shuffled, "full_size_zero", 0, 50)):
        with e.open_reader([(d, i, None) for d, i in tbs]) as r:
            for ranges in (EVERYTHING, [(b"", b"P" * 80 + b"%020d" % 300)]):
                check(e, r, tbs, ranges)
    with e.open_reader([(d, i, None) for d, i in tables]) as r:
        assert check(e, r, tables, EVERYTHING)[3]["partitions"] > 1
