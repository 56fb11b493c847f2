"""Range reads with a limit (dbeel_reader_get_ranges): every row against the limited range oracle
(tests/range_limit_oracle.py) -- G_q cut to the limit on clean queries, the damage rule on damaged ones -- and the read,
stats, capacity and argument contracts."""
import os

import numpy as np
import pytest

import range_limit_oracle as rlo
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS
from scan_cases import DAMAGES, damage, key_ranges, random_tree
from test_gpu_reader_get_range import EVERYTHING, _sorted, random_ranges, tiny_engine  # noqa: F401 (a fixture)

pytestmark = pytest.mark.gpu


def entries_of(data, index, row):
    ix = np.asarray(index, np.uint8).reshape(-1, 16)
    out = []
    for k in range(int(row["first"]), int(row["first"]) + int(row["count"])):
        off = int(ix[k, :8].view("<u8")[0])
        fs = int(ix[k, 12:16].view("<u4")[0])
        out.append(bytes(np.asarray(data[off:off + fs], np.uint8)))
    return out


def check(e, reader, tables, ranges, limits, keep=False):
    rows, data, index = reader.get_ranges(ranges, limits, keep_tombstones=keep)
    st, reads = e.stats(), reader.last_stream_reads
    lim = [limits] * len(ranges) if isinstance(limits, int) else list(limits)
    first = 0
    for q, (rng_, row) in enumerate(zip(ranges, rows)):
        assert int(row["first"]) == first
        first += int(row["count"])
        rlo.check_row(tables, rng_, lim[q], keep,
                      (row["first"], row["count"], row["flags"], (row["table"], row["reason"], row["record"])),
                      entries_of(data, index, row))
    assert index.size == 16 * first
    assert st["input_bytes"] == sum(r[3] for r in reads)
    assert st["entries_out"] == first and st["output_bytes"] == data.size + index.size
    for t, kind, off, size in reads:
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return rows, data, index, reads, st


@pytest.mark.parametrize("setting", ["default", "tiny_partitions", "depth0", "page_cache"])
def test_parity_on_random_trees(engine, tiny_engine, setting):
    e = tiny_engine if setting == "tiny_partitions" else engine
    fence_bytes = 1 if setting == "depth0" else 0
    cache = e.open_page_cache(1 << 20) if setting == "page_cache" else None
    for seed in range(6):
        rng = np.random.default_rng(1900 + seed)
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


def _table(keys, value=b"v", ts=BASE_TS):
    d, i = sstable.build_run([(k, value, ts) for k in keys])
    return np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy()


def test_tombstone_wall(engine):
    keys = [b"k%08d" % j for j in range(40000)]
    tables = [_table(keys), _table(keys[:20000], b"", BASE_TS + 1)]
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        rows, data, index, reads, st = check(engine, r, tables, EVERYTHING, 10)
        assert int(rows[0]["count"]) == 10 and int(rows[0]["flags"]) == rlo.MORE
        assert entries_of(data, index, rows[0])[0][8:17] == b"k00020000"
        # chunks of 11 double until they pass the 20,000 tombstones: about log2(20000 / 11) + 2 rounds
        assert 1 < st["partitions"] <= 14


def test_many_versions(engine):
    rng = np.random.default_rng(7)
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


def test_reads_and_cache(engine):
    rng = np.random.default_rng(11)
    keys = sorted({bytes(rng.integers(97, 123, 12, dtype=np.uint8)) for _ in range(50000)})
    tables = [_table([keys[j] for j in sorted(set(rng.integers(0, len(keys), 50000).tolist()))], b"x" * 40, BASE_TS + t)
              for t in range(4)]
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        whole = [(b"", b"\xff" * 16)]  # bounds the cached fences serve
        check(engine, r, tables, whole, 10)  # the first call loads the exact-mode fences
        _, _, _, reads, st = check(engine, r, tables, whole, 10)
        assert st["input_bytes"] < 64 * 1024, (st["input_bytes"], reads)
        with engine.open_page_cache(64 << 20) as cache:
            r.attach_page_cache(cache)
            ranges = [(keys[j], keys[j] + b"\xff") for j in rng.integers(0, len(keys), 64)]
            a = check(engine, r, tables, ranges, 10)
            b = check(engine, r, tables, ranges, 10)
            assert b[4]["input_bytes"] == 0, b[3]
            assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[0], b[0])
            r.attach_page_cache(None)


def test_scale(tiny_engine, monkeypatch):
    rng = np.random.default_rng(12)
    tables = _sorted(random_tree(rng, 4, max_entries=120))
    with tiny_engine.open_reader([(d, i, None) for d, i in tables]) as r:
        base = key_ranges(tables) + random_ranges(rng, tables, 59)
        ranges = [base[j % len(base)] for j in range(65536)]
        limits = [1 + j % 9 for j in range(65536)]
        rows, data, index = r.get_ranges(ranges, limits)
        memo = {}
        for q in range(0, 65536, 97):
            key = (ranges[q], limits[q])
            got = entries_of(data, index, rows[q])
            if key in memo:
                assert got == memo[key]
            memo[key] = got
            rlo.check_row(tables, ranges[q], limits[q], False,
                          (rows[q]["first"], rows[q]["count"], rows[q]["flags"],
                           (rows[q]["table"], rows[q]["reason"], rows[q]["record"])), got)


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage(engine, kind):
    rng = np.random.default_rng(300 + DAMAGES.index(kind))
    tables = _sorted(random_tree(rng, 3, max_entries=80))
    if kind == "ragged_index":  # a reader takes whole index records only
        return
    for rec in ((0,) if kind == "empty_table" else (0, 5, 40)):
        bad = damage(tables, kind, 1, rec)
        with engine.open_reader([(d, i, None) for d, i in bad]) as r:
            ranges = key_ranges(bad) + random_ranges(rng, bad, 20) + EVERYTHING
            for limits in (1, 3, 1000):
                rows = check(engine, r, bad, ranges, limits)[0]
                if rec == 0 and kind != "empty_table":  # damage at the first record of table 1's span of EVERYTHING
                    assert int(rows[len(ranges) - 1]["flags"]) & (rlo.STOPPED | rlo.UNSORTED), rows[len(ranges) - 1]


def test_capacity_errors_and_retry(engine):
    rng = np.random.default_rng(21)
    tables = _sorted(random_tree(rng, 3, max_entries=100))
    with engine.open_reader([(d, i, None) for d, i in tables]) as r:
        ranges = key_ranges(tables) + EVERYTHING
        rows, data, index = r.get_ranges(ranges, 50)
        if data.size:
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, 50, caps=(data.size - 1, index.size))
            assert ex.value.code == capi.ERR_CAPACITY and ex.value.needed == (data.size, index.size)
            assert np.array_equal(ex.value.rows, rows)
        rows2, data2, index2 = r.get_ranges(ranges, 50, caps=(data.size, index.size))
        assert np.array_equal(rows, rows2) and np.array_equal(data, data2) and np.array_equal(index, index2)
        n_reads = len(r.last_stream_reads)
        for k in sorted({0, n_reads // 2, n_reads - 1}):
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, 50, fail_read_at=k)
            assert ex.value.code == 4242
            again = r.get_ranges(ranges, 50)
            assert all(np.array_equal(x, y) for x, y in zip(again, (rows, data, index)))
        for bad_limits in (0, capi.RANGE_LIMIT_MAX + 1):
            with pytest.raises(capi.DbeelError) as ex:
                r.get_ranges(ranges, bad_limits)
            assert ex.value.code == capi.ERR_INVALID_ARG
        with pytest.raises(capi.DbeelError) as ex:
            r.get_ranges([(b"a", b"b")] * 65537, capi.RANGE_LIMIT_MAX, caps=(1, 16))
        assert ex.value.code == capi.ERR_INVALID_ARG
        with pytest.raises(capi.DbeelError) as ex:
            r.get_ranges([], 1)
        assert ex.value.code == capi.ERR_INVALID_ARG
        import ctypes as C
        out = capi.Out()
        row = np.zeros(1, capi.RANGE_ROW_DTYPE)
        lim = np.ones(1, np.uint32)
        rptr, _keep = capi.pack_ranges(capi.SCAN_KEY, [(b"a", b"b")])
        assert capi.lib().dbeel_reader_get_ranges(r._h, rptr, 1, lim.ctypes.data, 0x2, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert capi.lib().dbeel_reader_get_ranges(r._h, None, 1, lim.ctypes.data, 0, C.byref(out), row.ctypes.data) == capi.ERR_INVALID_ARG
        assert capi.lib().dbeel_reader_get_ranges(r._h, rptr, 1, lim.ctypes.data, 0, None, row.ctypes.data) == capi.ERR_INVALID_ARG
        assert all(np.array_equal(x, y) for x, y in zip(r.get_ranges(ranges, 50), (rows, data, index)))


def test_tree_reader_snapshot(engine, tmp_path):
    """A tree reader keeps answering its snapshot after a compaction unlinks its inputs."""
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(31)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    kr = [(b"t00500", b"t01800"), (b"t02990", b"u"), (b"a", b"t00010"), (b"t00599", b"t00700")]
    snap = tree.sstable_indices_and_sizes()
    a = tree.open_reader()
    before = a.get_ranges(kr, 5)
    want = [a.get_range([x])[0][0] for x in kr]  # one call per range: the ranges overlap
    for q, (dd, ii) in enumerate(want):
        n = ii.size // 16
        assert int(before[0][q]["count"]) == min(n, 5) and bool(before[0][q]["flags"] & rlo.MORE) == (n > 5)
        assert entries_of(before[1], before[2], before[0][q]) == entries_of(dd, ii, {"first": 0, "count": min(n, 5)})
    tree.flush(sstable.build_run([(b"t00600", b"new", BASE_TS + 10 ** 6)]))
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    after = a.get_ranges(kr, 5)
    assert all(np.array_equal(x, y) for x, y in zip(after, before))
    c = tree.open_reader()
    rows, data, index = c.get_ranges([(b"t00600", b"u")], 1)
    assert sstable.parse_run(data, index)[0][:2] == (b"t00600", b"new")
    a.close()
    c.close()
    tree.close()


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

    merged = {k: (v, ts) for k, v, ts in ents}
    merged.update({k: (v, ts) for k, v, ts in newer})
    live = [(k, v, ts) for k, (v, ts) in sorted(merged.items()) if v]
    ranges = [(b"k01980", b"k02005"), (b"k00100", b"z"), (b"k01995", b"z")]
    with engine.open_reader([(data_len, index.size, None), (len(nd), len(ni), None)], read=read) as r:
        rows, data, index_out = r.get_ranges(ranges, [7, 3, 50])
        for q, ((s, e), lim) in enumerate(zip(ranges, [7, 3, 50])):
            want = [x for x in live if s <= x[0] < e]
            assert int(rows[q]["flags"]) == (rlo.MORE if len(want) > lim else 0)
            f, n = int(rows[q]["first"]), int(rows[q]["count"])
            got = sstable.parse_run(data, index_out[16 * f:16 * (f + n)])
            assert [(k, v) for k, v, _ in got] == [(k, v) for k, v, _ in want[:lim]]
        assert any(kind == 1 and off > 1 << 32 for t, kind, off, _ in r.last_stream_reads if t == 0)
