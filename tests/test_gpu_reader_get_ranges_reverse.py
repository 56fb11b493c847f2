"""Range reads from the end (dbeel_reader_get_ranges_reverse): every row against the reverse statement of the limited range
oracle (tests/range_limit_rev_oracle.py) -- the last entries of G_q in descending key order on clean queries,
the top-down damage rule on damaged ones -- paging backward through a tree, and the read, stats, capacity and argument
contracts."""
import ctypes as C
import os

import numpy as np
import pytest

import range_limit_rev_oracle as rro
import seek_oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS
from scan_cases import DAMAGES, damage, key_ranges, random_tree
from test_gpu_reader_get_range import EVERYTHING, _sorted, random_ranges, tiny_engine  # noqa: F401 (a fixture)
from test_gpu_reader_get_ranges import _table, entries_of

pytestmark = pytest.mark.gpu


def check(e, reader, tables, ranges, limits, keep=False):
    rows, data, index = reader.get_ranges(ranges, limits, keep_tombstones=keep, reverse=True)
    st, reads = e.stats(), reader.last_stream_reads
    lim = [limits] * len(ranges) if isinstance(limits, int) else list(limits)
    first = 0
    for q, (rng_, row) in enumerate(zip(ranges, rows)):
        assert int(row["first"]) == first
        first += int(row["count"])
        rro.check_row(tables, rng_, lim[q], keep,
                      (row["first"], row["count"], row["flags"], (row["table"], row["reason"], row["record"])),
                      entries_of(data, index, row))
    assert index.size == 16 * first
    assert st["input_bytes"] == sum(r[3] for r in reads)
    assert st["entries_out"] == first and st["output_bytes"] == data.size + index.size
    for t, kind, off, size in reads:
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return rows, data, index, reads, st


def key_of(entry):
    kl = int(np.frombuffer(entry[:8], "<u8")[0])
    return bytes(entry[8:8 + kl])


@pytest.mark.parametrize("setting", ["default", "tiny_partitions", "depth0", "page_cache"])
def test_parity_on_random_trees(engine, tiny_engine, setting):
    e = tiny_engine if setting == "tiny_partitions" else engine
    fence_bytes = 1 if setting == "depth0" else 0
    cache = e.open_page_cache(1 << 20) if setting == "page_cache" else None
    for seed in range(6):
        rng = np.random.default_rng(2900 + seed)
        tables = random_tree(rng, 1 + seed % 6, max_entries=120, big=seed == 5)
        for tbs in (tables, _sorted(tables)):
            with e.open_reader([(d, i, None) for d, i in tbs], fence_bytes=fence_bytes) as r:
                if cache is not None:
                    r.attach_page_cache(cache)
                ranges = key_ranges(tbs) + random_ranges(rng, tbs, 40) + EVERYTHING
                ranges += ranges[:3]  # duplicates
                for limits in (1, 2, 7, [int(x) for x in rng.integers(1, 300, len(ranges))]):
                    for keep in (False, True):
                        check(e, r, tbs, ranges, limits, keep)
    if cache is not None:
        cache.close()


def test_many_versions(engine):
    rng = np.random.default_rng(8)
    keys = [b"key%06d" % j for j in range(3000)]
    tables = []
    for t in range(6):
        pick = sorted(rng.choice(len(keys), 1500, replace=False))
        tables.append(_table([keys[j] for j in pick], b"t%d" % t if t != 3 else b"", BASE_TS + t))
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        ranges = [(keys[j], keys[min(j + int(rng.integers(1, 400)), 2999)]) for j in rng.integers(0, 3000, 200)]
        for limits in (1, 10, 100):
            for keep in (False, True):
                check(engine, r, tables, ranges, limits, keep)


def test_tombstone_wall_at_the_top(engine):
    keys = [b"k%08d" % j for j in range(40000)]
    tables = [_table(keys), _table(keys[20000:], b"", BASE_TS + 1)]
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        rows, data, index, reads, st = check(engine, r, tables, EVERYTHING, 10)
        assert int(rows[0]["count"]) == 10 and int(rows[0]["flags"]) == rro.MORE
        got = entries_of(data, index, rows[0])
        assert [key_of(x) for x in got] == keys[19990:20000][::-1]
        # chunks of 11 double downward until they pass the 20,000 tombstones: about log2(20000 / 11) + 2 rounds
        assert 1 < st["partitions"] <= 14


def test_paging_backward_and_forward(engine):
    rng = np.random.default_rng(41)
    tables = _sorted(random_tree(rng, 4, max_entries=120))
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        for start, end in key_ranges(tables) + EVERYTHING:
            (whole,), stop = r.get_range([(start, end)])
            if stop[0] >= 0:
                continue
            want = entries_of(whole[0], whole[1], {"first": 0, "count": whole[1].size // 16})
            for lim in (1, 3, 7):
                back, hi = [], end
                while True:
                    rows, data, index = r.get_ranges([(start, hi)], lim, reverse=True)
                    got = entries_of(data, index, rows[0])
                    assert int(rows[0]["flags"]) & ~rro.MORE == 0 and len(got) <= lim
                    back += got
                    if not int(rows[0]["flags"]) & rro.MORE:
                        break
                    hi = key_of(got[-1])  # the previous page: end is exclusive
                assert back == want[::-1]
                fwd, lo = [], start
                while True:
                    rows, data, index = r.get_ranges([(lo, end)], lim)
                    got = entries_of(data, index, rows[0])
                    fwd += got
                    if not int(rows[0]["flags"]) & rro.MORE:
                        break
                    lo = key_of(got[-1]) + b"\x00"
                assert fwd[::-1] == back


def test_reads_and_cache(engine):
    rng = np.random.default_rng(12)
    keys = sorted({bytes(rng.integers(97, 123, 12, dtype=np.uint8)) for _ in range(50000)})
    tables = [_table([keys[j] for j in sorted(set(rng.integers(0, len(keys), 50000).tolist()))], b"x" * 40, BASE_TS + t)
              for t in range(4)]
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        whole = [(b"", b"\xff" * 16)]  # bounds the cached fences serve
        check(engine, r, tables, whole, 10)  # the first call loads the exact-mode fences
        _, _, _, reads, st = check(engine, r, tables, whole, 10)
        assert st["input_bytes"] < 64 * 1024, (st["input_bytes"], reads)
        for t, kind, off, size in reads:
            if kind != 2:
                continue
            d, ix = bytes(tables[t][0]), bytes(tables[t][1])
            lo, hi = seek_oracle.seek(d, ix, whole[0][0])[0], seek_oracle.seek(d, ix, whole[0][1])[0]
            assert 16 * lo <= off and off + size <= 16 * hi, (t, off, size, lo, hi)
        assert any(kind == 2 and off + size == len(tables[t][1]) for t, kind, off, size in reads)  # staged from the top
        with engine.open_page_cache(64 << 20) as cache:
            r.attach_page_cache(cache)
            ranges = [(keys[j], keys[j] + b"\xff") for j in rng.integers(0, len(keys), 64)]
            a = check(engine, r, tables, ranges, 10)
            b = check(engine, r, tables, ranges, 10)
            assert b[4]["input_bytes"] == 0, b[3]
            assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[0], b[0])
            r.attach_page_cache(None)


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage(engine, kind):
    rng = np.random.default_rng(310 + DAMAGES.index(kind))
    tables = _sorted(random_tree(rng, 3, max_entries=80))
    if kind == "ragged_index":  # a reader takes whole index records only
        return
    n1 = np.asarray(tables[1][1]).size // 16
    for rec in ((0,) if kind == "empty_table" else (0, 5, 40, n1 - 1)):
        bad = damage(tables, kind, 1, rec)
        with engine.open_reader([(d, i, None) for d, i in bad]) as r:
            ranges = key_ranges(bad) + random_ranges(rng, bad, 20) + EVERYTHING
            for limits in (1, 3, 1000):
                rows = check(engine, r, bad, ranges, limits)[0]
                if rec == n1 - 1 or kind == "empty_table":  # the last record of table 1's span of EVERYTHING
                    assert int(rows[len(ranges) - 1]["flags"]) & (rro.STOPPED | rro.UNSORTED), rows[len(ranges) - 1]


def test_capacity_errors_and_retry(engine):
    rng = np.random.default_rng(22)
    tables = _sorted(random_tree(rng, 3, max_entries=100))
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        ranges = key_ranges(tables) + EVERYTHING
        rows, data, index = r.get_ranges(ranges, 50, reverse=True)
        if data.size:
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, 50, caps=(data.size - 1, index.size), reverse=True)
            assert ex.value.code == capi.ERR_CAPACITY and ex.value.needed == (data.size, index.size)
            assert np.array_equal(ex.value.rows, rows)
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, 50, caps=(data.size, index.size - 16), reverse=True)
            assert ex.value.code == capi.ERR_CAPACITY and ex.value.needed == (data.size, index.size)
        rows2, data2, index2 = r.get_ranges(ranges, 50, caps=(data.size, index.size), reverse=True)
        assert np.array_equal(rows, rows2) and np.array_equal(data, data2) and np.array_equal(index, index2)
        n_reads = len(r.last_stream_reads)
        for k in sorted({0, n_reads // 2, n_reads - 1}):
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, 50, fail_read_at=k, reverse=True)
            assert ex.value.code == 4242
            again = r.get_ranges(ranges, 50, reverse=True)
            assert all(np.array_equal(x, y) for x, y in zip(again, (rows, data, index)))
        for bad_limits in (0, capi.RANGE_LIMIT_MAX + 1):
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, bad_limits, reverse=True)
            assert ex.value.code == capi.ERR_INVALID_ARG
        with pytest.raises(capi.DbeelError) as ex:
            r.get_ranges([(b"a", b"b")] * 65537, capi.RANGE_LIMIT_MAX, caps=(1, 16), reverse=True)
        assert ex.value.code == capi.ERR_INVALID_ARG
        with pytest.raises(capi.DbeelError) as ex:
            r.get_ranges([], 1, reverse=True)
        assert ex.value.code == capi.ERR_INVALID_ARG
        out = capi.Out()
        row = np.zeros(1, capi.RANGE_ROW_DTYPE)
        lim = np.ones(1, np.uint32)
        rptr, _keep = capi.pack_ranges(capi.SCAN_KEY, [(b"a", b"b")])
        fn = capi.lib().dbeel_reader_get_ranges_reverse
        assert fn(r._h, rptr, 1, lim.ctypes.data, 0x2, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert fn(r._h, None, 1, lim.ctypes.data, 0, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert fn(r._h, rptr, 1, None, 0, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert fn(r._h, rptr, 1, lim.ctypes.data, 0, None, row.ctypes.data) == capi.ERR_INVALID_ARG
        assert fn(r._h, rptr, 1, lim.ctypes.data, 0, C.byref(out), None) == capi.ERR_INVALID_ARG
        assert fn(None, rptr, 1, lim.ctypes.data, 0, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert all(np.array_equal(x, y) for x, y in zip(r.get_ranges(ranges, 50, reverse=True), (rows, data, index)))


def test_tree_reader_snapshot(engine, tmp_path):
    """A tree reader keeps answering its snapshot after a flush and a compaction unlink its inputs."""
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(32)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    kr = [(b"t00500", b"t01800"), (b"t02990", b"u"), (b"a", b"t00010"), (b"t00599", b"t00700")]
    snap = tree.sstable_indices_and_sizes()
    a = tree.open_reader()
    before = a.get_ranges(kr, 5, reverse=True)
    want = [a.get_range([x])[0][0] for x in kr]  # one call per range: the ranges overlap
    for q, (dd, ii) in enumerate(want):
        n = ii.size // 16
        assert int(before[0][q]["count"]) == min(n, 5) and bool(before[0][q]["flags"] & rro.MORE) == (n > 5)
        assert entries_of(before[1], before[2], before[0][q]) == entries_of(dd, ii, {"first": 0, "count": n})[::-1][:5]
    tree.flush(sstable.build_run([(b"t00699", b"new", BASE_TS + 10 ** 6)]))
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    after = a.get_ranges(kr, 5, reverse=True)
    assert all(np.array_equal(x, y) for x, y in zip(after, before))
    c = tree.open_reader()
    rows, data, index = c.get_ranges([(b"t00599", b"t00700")], 1, reverse=True)
    assert sstable.parse_run(data, index)[0][:2] == (b"t00699", b"new")
    a.close()
    c.close()
    tree.close()


def test_inputs_past_4gib(engine):
    """.data past 4 GiB served by a callback: 2,000 entries above 2^32, and a newer table overriding keys near the end --
    the first records a reverse read meets."""
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

    merged = {k: (v, ts) for k, v, ts in ents}
    merged.update({k: (v, ts) for k, v, ts in newer})
    live = [(k, v, ts) for k, (v, ts) in sorted(merged.items()) if v]
    ranges = [(b"k01980", b"k02005"), (b"k00100", b"z"), (b"k01995", b"z"), (b"k00100", b"k01992")]
    limits = [7, 3, 50, 4]
    with engine.open_reader([(data_len, index.size, None), (len(nd), len(ni), None)], read=read) as r:
        rows, data, index_out = r.get_ranges(ranges, limits, reverse=True)
        for q, ((s, e), lim) in enumerate(zip(ranges, limits)):
            want = [x for x in live if s <= x[0] < e][::-1]
            assert int(rows[q]["flags"]) == (rro.MORE if len(want) > lim else 0)
            f, n = int(rows[q]["first"]), int(rows[q]["count"])
            got = sstable.parse_run(data, index_out[16 * f:16 * (f + n)])
            assert [(k, v) for k, v, _ in got] == [(k, v) for k, v, _ in want[:lim]]
        assert any(kind == 1 and off > 1 << 32 for t, kind, off, _ in r.last_stream_reads if t == 0)
