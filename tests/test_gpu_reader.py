"""Readers (dbeel_reader_*, dbeel_tree_reader_open): batches on a fixed set of tables with the filters uploaded once and
each table's fences kept on the device after the first batch in a mode reaches it.  Every batch returns what
dbeel_get_values_stream (and dbeel_get_values) return for the same tables, keys and mode; from the second batch on, no
fence is read again."""
import os
from collections import Counter

import numpy as np
import pytest

from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS, assert_run_equal
from test_gpu_get_values import _rec, _set_u32
from test_gpu_get_values_stream import all_cases, case_compacted_with_filter, case_four_overlapping

pytestmark = pytest.mark.gpu

MODES = (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT)
NODE_BYTES = 2 * (16 + 8 + 80)  # one probe-tree node of cached fences, both modes (host/lookup_plan.h)


@pytest.fixture
def tiny_engine(monkeypatch):
    """An engine whose leaf groups are 4 KB: leaves spread over many groups."""
    monkeypatch.setenv("DBEEL_PARTITION_KB", "4")
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    e = capi.Engine(0)
    yield e
    e.close()


def same(e, reader, tables, keys, mode, ref_engine=None):
    """reader.get_values == get_values_stream == get_values on the same tables; input_bytes = what the callback
    delivered.  Returns (rows, data, index, reads, stats) of the reader and the stream's (reads, stats)."""
    rows, d, i = reader.get_values(keys, mode)
    st, reads = e.stats(), reader.last_stream_reads
    sr, sd, si = e.get_values_stream(tables, keys, mode)
    s_st, s_reads = e.stats(), e.last_stream_reads
    wr, wd, wi = (ref_engine or e).get_values(tables, keys, mode)
    assert np.array_equal(rows, sr) and np.array_equal(rows, wr)
    assert_run_equal((d, i), (sd, si), "reader vs stream")
    assert_run_equal((d, i), (wd, wi), "reader vs whole")
    assert st["entries_in"] == len(keys) and st["entries_out"] == i.size // 16 and st["output_bytes"] == d.size + i.size
    assert st["input_bytes"] == sum(r[3] for r in reads)
    for t, kind, off, size in reads:
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return rows, d, i, reads, st, s_reads, s_st


def max_depth(n):
    d = 0
    while d < 16 and (2 << d) <= n:
        d += 1
    return d


def reader_depth(n, fence_bytes=0):
    """D_t of a reader's only table (reader_depths with one table): the deepest level whose fences fit the budget."""
    b = fence_bytes or capi.DEFAULT_READER_FENCE_BYTES
    d = 0
    while d < max_depth(n) and NODE_BYTES << (d + 1) <= b:
        d += 1
    return d


def fence_positions(mode, n, depth):
    """The records the open internal nodes of the top `depth` levels probe (plan_probe_tree restated)."""
    def step(s, c):
        a, b, half, _ = s
        if mode == 0:
            a2 = half + 1 if c < 0 else a
            b2 = max(half, 1) - 1 if c > 0 else b
            h2 = (b2 + a2) // 2
            return (a2, b2, h2, half == 0 or half == n or a2 > b2)
        mid = a + (b - a) // 2
        a2, b2 = (mid + 1, b) if c < 0 else (a, mid)
        return (a2, b2, 0, a2 >= b2)

    def pos(s):
        return s[2] if mode == 0 else s[0] + (s[1] - s[0]) // 2
    root = (0, n - 1 if n else 0, n // 2, n == 0) if mode == 0 else (0, n, 0, n == 0)
    out, level = set(), [root] if not root[3] else []
    for _ in range(depth):
        nxt = []
        for s in level:
            out.add(pos(s))
            nxt += [c for c in (step(s, 1), step(s, -1)) if not c[3]]
        level = nxt
    return out


def table_20000():
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(20000)]
    d, i = sstable.build_run(ents)
    return (d, i, None), [k for k, _, _ in ents]


@pytest.mark.parametrize("budget", ["default", "tiny"])
def test_parity_on_every_case(engine, tiny_engine, budget):
    """Three different batches per mode on one reader, on every table set of the stream's tests."""
    e = engine if budget == "default" else tiny_engine
    rng = np.random.default_rng(21)
    for tables, keys in all_cases(engine):
        with e.open_reader(tables) as r:
            for mode in MODES:
                half = [keys[j] for j in rng.permutation(len(keys))[:len(keys) // 2]]
                for batch in (keys, half, keys[:7]):
                    same(e, r, tables, batch, mode, ref_engine=engine)


def test_damage_at_fences_and_inside_leaves(engine):
    """Corrupt records and bad entries at fence positions and inside leaves give the same rows and flags through the
    cached fences as through fences read per call."""
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    keys = [k for k, _, _ in ents[::7]] + [b"key-%06dx" % n for n in range(0, 2000, 13)]
    rng = np.random.default_rng(11)
    fences = sorted(fence_positions(0, 2000, 4) | fence_positions(1, 2000, 4))
    for r in list(rng.choice(2000, 6, replace=False)) + fences[:6] + [0, 1999]:
        off, ks, fs = _rec(i, int(r))
        for kind in range(4):
            bi, bd = i.copy(), d
            if kind == 0:  # offset past .data: corrupt
                bi[16 * r:16 * r + 8] = np.frombuffer((d.size - 4).to_bytes(8, "little"), np.uint8)
            elif kind == 1:  # a length prefix past .data: corrupt
                bd = d.copy()
                bd[off:off + 8] = np.frombuffer((1 << 50).to_bytes(8, "little"), np.uint8)
            elif kind == 2:  # key_size lies: a bad entry when hit
                _set_u32(bi, int(r), 8, ks + 3)
            else:  # the offset points into the middle of another entry
                bi[16 * r:16 * r + 8] = np.frombuffer((off + 5).to_bytes(8, "little"), np.uint8)
            tables = [(bd, bi, None)]
            with engine.open_reader(tables) as rd:
                for mode in MODES:
                    for _ in range(2):  # the batch that loads the fences, then one that uses them
                        same(engine, rd, tables, keys + [ents[int(r)][0]], mode)


def test_reads_from_the_second_batch_on(engine):
    tables, keys = case_compacted_with_filter(engine)
    _, gi, _ = tables[0]
    n = gi.size // 16
    starts = set(int(x) for x in gi.view("<u8").reshape(-1, 2)[:, 0])
    rng = np.random.default_rng(22)
    for mode in MODES:
        fences = fence_positions(mode, n, reader_depth(n))
        assert len(fences) > 1000
        with engine.open_reader(tables) as r:
            first = same(engine, r, tables, keys, mode)[3]
            again = same(engine, r, tables, keys, mode)[3]
            # the second run of the same batch reads what the first read, less the fence loads
            loads = Counter(first) - Counter(again)
            assert not Counter(again) - Counter(first) and loads
            for t, kind, off, size in loads:
                if kind == 2:
                    assert off % 16 == 0 and off // 16 in fences and (off + size) // 16 - 1 in fences
                else:
                    assert off in starts  # key frames start at a record's offset
            for b in range(3):
                batch = [keys[j] for j in rng.choice(len(keys), [1, 64, 2000][b], replace=False)]
                _, _, _, reads, st, _, s_st = same(engine, r, tables, batch, mode)
                # no .index read starts at a cached fence: leaf slices (merged or not) start inside a leaf
                assert not [x for x in reads if x[1] == 2 and x[2] // 16 in fences]
                assert st["input_bytes"] <= s_st["input_bytes"], (b, st["input_bytes"], s_st["input_bytes"])
    (d, i, _), keys20 = table_20000()
    tables = [(d, i, None)]
    for mode in MODES:
        with engine.open_reader(tables) as r:
            r.get_values(keys20[:100], mode)
            for k in keys20[::997] + [b"key-000500x", b"a", b"z"]:
                reads = same(engine, r, tables, [k], mode)[3]
                assert sum(1 for x in reads if x[1] == 2) <= 1, reads  # one leaf slice
                assert sum(1 for x in reads if x[1] == 1) <= 2, reads  # one window, one fence hit's entry


def fence_reads(reads, mode, n):
    """.index reads that start at a fence of the deepest probe tree a reader could cache.  Fences read per call start at
    one (the first of a merged run is a fence at the batch's depth, and so at every deeper one); a leaf slice of a batch
    that descends the cached fences never does (a leaf's records are not probed above it)."""
    fences = fence_positions(mode, n, reader_depth(n))
    return [x for x in reads if x[1] == 2 and x[2] // 16 in fences]


def test_fallbacks_read_fences_per_call(engine):
    """A key longer than the frame cap, or a batch that wants more depth than D_t: that table's fences are read for the
    batch exactly as get_values_stream reads them."""
    rng = np.random.default_rng(23)
    long_ents = [(b"%06d" % n + b"L" * 70, b"v%d" % n, BASE_TS + n) for n in range(5000)]
    d, i = sstable.build_run(long_ents)
    tables = [(d, i, None)]
    short = [k[:capi.READER_FRAME_CAP] for k, _, _ in long_ents[::50]] + [b"002500" + b"L" * 57 + b"M", b"9" * 64]
    longk = [long_ents[int(j)][0] for j in rng.choice(5000, 40, replace=False)]
    with engine.open_reader(tables) as r:
        for mode in MODES:
            same(engine, r, tables, short, mode)
            _, _, _, reads, st, s_reads, _ = same(engine, r, tables, short, mode)  # 64-byte keys: the cache serves
            assert Counter(reads) != Counter(s_reads) and not fence_reads(reads, mode, 5000)
            batch = longk + short
            _, _, _, reads, _, s_reads, _ = same(engine, r, tables, batch, mode)  # 76-byte keys: per call
            assert Counter(reads) == Counter(s_reads) and fence_reads(reads, mode, 5000)
    (d, i, _), keys20 = table_20000()
    tables = [(d, i, None)]
    assert reader_depth(20000, 4 * NODE_BYTES) == 2
    with engine.open_reader(tables, fence_bytes=4 * NODE_BYTES) as r:  # D_t = 2: every batch wants more
        for mode in MODES:
            for batch in ([keys20[7]], keys20[::13]):
                for _ in range(2):
                    _, _, _, reads, _, s_reads, _ = same(engine, r, tables, batch, mode)
                    assert Counter(reads) == Counter(s_reads) and fence_reads(reads, mode, 20000)


def test_callback_errors_and_capacity_leave_the_reader_usable(engine):
    tables, keys = case_four_overlapping(engine)
    mode = capi.LOOKUP_EXACT
    with engine.open_reader(tables) as r:
        with pytest.raises(capi.DbeelError) as ei:  # the first read of all: a fence load
            r.get_values(keys, mode, fail_read_at=0)
        assert ei.value.code == 4242
        same(engine, r, tables, keys, mode)
        rows, d, i, reads, _, _, _ = same(engine, r, tables, keys, mode)  # the reads of a batch after the fence loads
        for at in (0, len(reads) // 2, len(reads) - 1):
            with pytest.raises(capi.DbeelError) as ei:
                r.get_values(keys, mode, fail_read_at=at)
            assert ei.value.code == 4242
            same(engine, r, tables, keys, mode)
        for caps in ((d.size - 1, i.size), (d.size, i.size - 1)):
            with pytest.raises(capi.DbeelError) as ei:
                r.get_values(keys, mode, caps=caps)
            assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (d.size, i.size)
            r2, d2, i2 = r.get_values(keys, mode)
            assert np.array_equal(r2, rows) and np.array_equal(d2, d) and np.array_equal(i2, i)
    bad = [t for t in tables if t[2] is not None][0]
    with pytest.raises(capi.DbeelError) as ei:
        engine.open_reader([(bad[0], bad[1], bad[2][:-4])])
    assert ei.value.code == capi.ERR_BAD_BLOOM


def test_tree_reader_snapshots(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(24)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    keys = [b"t%05d" % n for n in range(0, 3100, 7)] + [b"t00001", b"t00001"]
    snap = tree.sstable_indices_and_sizes()
    saved = [sstable.read_run_files(d, idx) + (None,) for idx, _ in snap]
    a = tree.open_reader()
    before = {}
    for mode in MODES:
        before[mode] = a.get_values(keys, mode)
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert np.array_equal(before[mode][0], sr)
        assert_run_equal(before[mode][1:], (sd, si), "tree reader A")
    # B shares A's three tables; its own table holds one record (no fences): B's first batch per mode loads nothing
    tree.flush(sstable.build_run([(b"u", b"x", BASE_TS)]))
    b = tree.open_reader()
    for mode in MODES:
        r1, d1, i1 = b.get_values(keys, mode)
        first = engine.stats()["input_bytes"]
        r2, d2, i2 = b.get_values(keys, mode)
        assert engine.stats()["input_bytes"] == first
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert first < engine.stats()["input_bytes"]
        assert np.array_equal(r1, sr) and np.array_equal(r2, sr)
        assert_run_equal((d1, i1), (sd, si), "tree reader B")
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    c = tree.open_reader()
    for mode in MODES:
        ra, da, ia = a.get_values(keys, mode)  # A answers from its snapshot, its files unlinked
        assert np.array_equal(ra, before[mode][0])
        assert_run_equal((da, ia), before[mode][1:], "A after the compaction")
        wr, wd, wi = engine.get_values(saved, keys, mode)
        assert np.array_equal(ra, wr)
        assert_run_equal((da, ia), (wd, wi), "A vs the saved bytes")
        rc_, dc_, ic_ = c.get_values(keys, mode)
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert np.array_equal(rc_, sr)
        assert_run_equal((dc_, ic_), (sd, si), "reader C")
    for r in (a, b, c):
        r.close()
    tree.close()


def test_device_memory_is_the_filters_and_the_fence_budget(engine):
    """Device memory a reader holds: its filters plus at most fence_bytes, with 2 MiB of allocation granularity per
    device block (one per filter, one per table and mode with fences); all of it returns at close."""
    import torch
    tables, keys = case_four_overlapping(engine)
    t2, k2 = case_compacted_with_filter(engine)
    tables, keys = tables + t2, keys + k2
    for mode in MODES:  # the engine's own workspaces grow to this batch first
        engine.get_values_stream(tables, keys, mode)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    fence_bytes = 3 << 20
    blooms = sum(b.size for _, _, b in tables if b is not None)
    blocks = sum(1 for _, _, b in tables if b is not None) + 2 * len(tables)
    r = engine.open_reader(tables, fence_bytes=fence_bytes)
    for mode in MODES:
        for _ in range(2):
            r.get_values(keys, mode)
    used = free0 - torch.cuda.mem_get_info()[0]
    print(f"reader: {used / 1e6:.2f} MB of device memory; filters {blooms / 1e6:.2f} MB, fence budget {fence_bytes / 1e6:.2f} MB")
    assert used <= blooms + fence_bytes + (2 << 20) * blocks
    r.close()
    assert free0 - torch.cuda.mem_get_info()[0] <= 2 << 20


def test_engine_destroy_closes_open_readers():
    tables, keys = [table_20000()[0]], [b"key-000001"]
    e = capi.Engine(0)
    r = e.open_reader(tables)
    rows, _, _ = r.get_values(keys, capi.LOOKUP_EXACT)
    assert rows["table"][0] == 0
    e.close()
    r.close()  # a no-op: the engine closed it
