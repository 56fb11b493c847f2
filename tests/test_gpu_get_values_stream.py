"""Batched reads from SSTable files (dbeel_get_values_stream, row N2): the same rows, .data, .index and items as
dbeel_get_values on the same tables, while only the index records, key frames and entries the searches reach are read
through the callback."""
import resource

import numpy as np
import pytest

from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from dbeel_b200 import workloads as W
from helpers import BASE_TS, assert_run_equal, nasty_keys, random_runs
from test_gpu_get_values import SEED, TS_MAX, TS_MIN, _rec, _set_u32, keys_of

pytestmark = pytest.mark.gpu

MODES = (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT)


@pytest.fixture
def tiny_engine(monkeypatch):
    """An engine whose leaf groups are 4 KB: leaves spread over many groups."""
    monkeypatch.setenv("DBEEL_PARTITION_KB", "4")
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    e = capi.Engine(0)
    yield e
    e.close()


def same(engine, tables, keys, mode, ref_engine=None):
    """get_values_stream == get_values: rows, .data, .index, items; input_bytes = what the callback delivered."""
    rows, d, i = engine.get_values_stream(tables, keys, mode)
    st = engine.stats()
    reads = engine.last_stream_reads
    er, ed, ei = (ref_engine or engine).get_values(tables, keys, mode)
    assert np.array_equal(rows, er)
    assert_run_equal((d, i), (ed, ei), "stream vs whole")
    assert st["entries_in"] == len(keys) and st["entries_out"] == i.size // 16 and st["output_bytes"] == d.size + i.size
    assert st["input_bytes"] == sum(r[3] for r in reads)
    for t, kind, off, size in reads:  # every read inside its file
        f = tables[t][0] if kind == 1 else tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return rows, d, i, reads


def case_compacted_with_filter(engine):
    gd, gi, gb, n = engine.compact(W.make_merge_runs(W.scaled(W.CFG2, 20_000)), keep_tombstones=False, seed=SEED)
    table = (gd, gi, gb)
    present = keys_of(table)
    rng = np.random.default_rng(1)
    sample = [present[j] for j in rng.choice(len(present), 3000, replace=False)] + present[:40] + present[-40:]
    absent = [b"\xb0k%015d" % int(x) for x in rng.integers(0, 1 << 40, 1500)] + [b"", present[7] + b"\x00", present[9][:-1]]
    return [table], sample + absent + sample[:500]


def case_tiny_tables(engine):
    out = []
    for n in (1, 2, 3, 4, 5, 8, 33):
        d, i = sstable.build_run([(bytes([10 + 2 * j]), b"v" * j, BASE_TS + j) for j in range(n)])
        out.append(([(d, i, None)], [bytes([x]) for x in range(8, 12 + 2 * n)]))
    return out


def case_four_overlapping(engine):
    rng = np.random.default_rng(3)
    ents = [(b"\xb0k%015d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 90)), dtype=np.uint8)), BASE_TS + n)
            for n in range(9000)]
    tables = []
    for t, (lo, hi, step) in enumerate([(0, 6000, 1), (3000, 9000, 2), (100, 8000, 3), (5000, 5400, 1)]):
        d, i, b, _ = engine.compact([sstable.build_run(ents[lo:hi:step])], keep_tombstones=True,
                                    bloom_min_size=1000 if t != 2 else 1 << 40, seed=SEED)
        tables.append((d, i, b))
    keys = [ents[int(j)][0] for j in rng.integers(0, 9000, 2500)] + [b"\xb0k%015d" % n for n in range(9000, 9300)]
    return tables, keys


def case_big_entries(engine):
    rng = np.random.default_rng(4)
    pool = nasty_keys(rng, 600, max_len=50)
    runs = random_runs(rng, 3, 400, pool, max_doc=40, tombstone_frac=0.3)
    big = sorted(rng.choice(len(pool), 4, replace=False))
    runs.append(sstable.build_run(sorted((pool[j], bytes(rng.integers(0, 256, s, dtype=np.uint8)), BASE_TS + 999)
                                         for j, s in zip(big, [3 << 20, 5 << 20, 8191, 16385]))))
    gd, gi, gb, n = engine.compact(runs, keep_tombstones=True, bloom_min_size=1000, seed=SEED)
    ents = sstable.parse_run(gd, gi)
    return [(gd, gi, gb)], [k for k, _, _ in ents] + [pool[j] for j in big] * 3 + [b"\xfe\xfe-absent"]


def case_damaged(engine):
    ents = [(b"k%03d" % n, b"value-%d" % n, BASE_TS + n) for n in range(64)]
    ents[20] = (ents[20][0], b"t20", TS_MAX + 1)
    ents[21] = (ents[21][0], b"t21", TS_MIN - 1)
    ents[22] = (ents[22][0], b"t22", TS_MAX)
    ents[23] = (ents[23][0], b"t23", TS_MIN)
    d, i = sstable.build_run(ents)
    for r, field, delta in ((5, 8, 1), (6, 8, -1), (7, 12, -1), (8, 12, 1)):
        _set_u32(i, r, field, _rec(i, r)[1 if field == 8 else 2] + delta)
    _set_u32(i, 9, 12, _rec(i, 9)[1] - 1)
    keys = [k for k, _, _ in ents]
    broken = i.copy()
    broken[16 * 32:16 * 32 + 8] = np.frombuffer((1 << 40).to_bytes(8, "little"), np.uint8)
    return [([(d, i, None)], keys), ([(d[:-1].copy(), i, None)], keys[-3:]), ([(d, broken, None)], [b"k010", b"k050"] + keys)]


def all_cases(engine):
    d, i = sstable.build_run([(b"a%03d" % n, b"x" * n, BASE_TS) for n in range(100)])
    cases = [case_compacted_with_filter(engine), case_four_overlapping(engine), case_big_entries(engine)]
    cases += case_tiny_tables(engine) + case_damaged(engine)
    cases += [([(d, i, None)], [b"b%03d" % n for n in range(300)]), ([(d, i, None)], []), ([], [b"a001", b""])]
    return cases


@pytest.mark.parametrize("budget", ["default", "tiny"])
def test_parity_with_get_values_on_every_table_set(engine, tiny_engine, budget):
    e = engine if budget == "default" else tiny_engine
    for tables, keys in all_cases(engine):
        for mode in MODES:
            same(e, tables, keys, mode, ref_engine=engine)
    if budget == "tiny":
        tables, keys = case_compacted_with_filter(engine)
        same(e, tables, keys, capi.LOOKUP_EXACT, ref_engine=engine)
        assert e.stats()["partitions"] > 10


def test_damage_at_fences_and_inside_leaves(engine):
    """Corrupt records and bad entries at every record position of a 2000-entry table: some are fences, most inside
    leaves; and index records whose key_size or offset lie about where a key frame ends."""
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    keys = [k for k, _, _ in ents[::7]] + [b"key-%06dx" % n for n in range(0, 2000, 13)]
    rng = np.random.default_rng(11)
    for r in list(rng.choice(2000, 12, replace=False)) + [0, 999, 1000, 1999]:
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
            for mode in MODES:
                same(engine, [(bd, bi, None)], keys + [ents[int(r)][0]], mode)


def test_a_table_the_filter_rejects_is_not_read(engine):
    d0, i0 = sstable.build_run([(b"old-%05d" % n, b"x", BASE_TS) for n in range(5000)])
    gd, gi, gb, _ = engine.compact([sstable.build_run([(b"new-%05d" % n, b"y", BASE_TS) for n in range(5000)])],
                                   keep_tombstones=True, bloom_min_size=1, seed=SEED)
    assert gb is not None
    tables = [(d0, i0, None), (gd, gi, gb)]
    cand = [b"old-%05d" % n for n in range(0, 5000, 3)]
    rows = engine.get_many(tables, cand)
    keys = [k for k, j in zip(cand, rows["bloom_rejects"]) if j == 1]  # rejected by the newer table's filter
    assert len(keys) > 1000
    rows, _, _, reads = same(engine, tables, keys, capi.LOOKUP_EXACT)
    assert reads and all(t == 0 for t, _, _, _ in reads)


def test_sparse_batch_reads_a_small_share_and_a_dense_one_reads_data_once(engine):
    gd, gi, gb, n = engine.compact(W.make_merge_runs(W.scaled(W.CFG2, 25_000)), keep_tombstones=False, seed=SEED)
    table = (gd, gi, gb)
    present = keys_of(table)
    assert n > 150_000
    rng = np.random.default_rng(12)
    keys = [present[j] for j in rng.choice(n, 30, replace=False)] + [b"\xb0k%015d" % int(x) for x in rng.integers(0, 1 << 40, 30)]
    for mode in MODES:
        _, _, _, reads = same(engine, [table], keys, mode)
        got = sum(r[3] for r in reads)
        assert got < 0.06 * (gd.size + gi.size), (got, gd.size + gi.size)  # stated bound: under 6 % of the table
    keys = [present[j] for j in rng.choice(n, 60_000, replace=False)]
    rows, d, _, reads = same(engine, [table], keys, capi.LOOKUP_EXACT)
    assert (rows["table"] == 0).all()
    # Every .data byte is read at most once, apart from the fences' key frames: a fence frame is one read of exactly
    # [offset, offset + 8 + longest key) of some record; every other .data read (leaf windows, the entries of hits at
    # fences) is disjoint from all the others.  The answered entries come out of the leaf windows, not from a second read.
    frame = 8 + max(len(k) for k in keys)
    offsets = set(int(x) for x in gi.view("<u8").reshape(-1, 2)[:, 0])
    small = [(o, z) for t, k, o, z in reads if k == 1 and z <= frame]
    assert small and all(z == frame and o in offsets for o, z in small)
    big = sorted((o, o + z) for t, k, o, z in reads if k == 1 and z > frame)
    assert all(a[1] <= b[0] for a, b in zip(big, big[1:])), "two .data reads overlap"
    assert sum(z for t, k, o, z in reads if k == 1) <= gd.size + len(small) * frame


def test_callback_errors_and_capacity(engine):
    tables, keys = case_four_overlapping(engine)
    mode = capi.LOOKUP_EXACT
    rows, d, i, reads = same(engine, tables, keys, mode)
    for at in (0, 1, len(reads) // 2, len(reads) - 1):
        with pytest.raises(capi.DbeelError) as ei:
            engine.get_values_stream(tables, keys, mode, fail_read_at=at)
        assert ei.value.code == 4242
        r2, d2, i2 = engine.get_values_stream(tables, keys, mode)
        assert np.array_equal(r2, rows) and np.array_equal(d2, d) and np.array_equal(i2, i)
    for caps in ((d.size - 1, i.size), (d.size, i.size - 1)):
        with pytest.raises(capi.DbeelError) as ei:
            engine.get_values_stream(tables, keys, mode, caps=caps)
        assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (d.size, i.size)


# ---- a table larger than device memory, that exists only as a function of the record number
SYN_F = 1024                  # full_size of every entry: u64 16 | 16-byte key | u64 dlen | dlen bytes | i128 ts
SYN_V = SYN_F - 48
SYN_N = (96 << 30) // SYN_F   # 100 663 296 records, 96 GiB of .data
TS16 = np.frombuffer(int(BASE_TS).to_bytes(16, "little", signed=True), np.uint8)


def syn_key(r):
    return b"k%015d" % r


def syn_records(r0, r1):
    """Entries r0 .. r1 - 1 as one (count, SYN_F) byte array: the value's first 8 bytes hold r."""
    r = np.arange(r0, r1, dtype=np.uint64)
    e = np.zeros((r1 - r0, SYN_F), np.uint8)
    e[:, 0] = 16
    e[:, 8] = ord("k")
    digits = r.copy()
    for p in range(15):
        e[:, 23 - p] = (digits % 10).astype(np.uint8) + ord("0")
        digits //= 10
    e[:, 24:32] = np.frombuffer(np.uint64(SYN_V).tobytes(), np.uint8)
    e[:, 32:40] = r.view(np.uint8).reshape(-1, 8)
    e[:, SYN_F - 16:] = TS16
    return e


def syn_read(table, kind, off, size):
    if kind == 2:
        r0, r1 = off // 16, (off + size + 15) // 16
        rec = np.zeros((r1 - r0, 2), np.uint64)
        rec[:, 0] = np.arange(r0, r1, dtype=np.uint64) * SYN_F
        rec[:, 1] = np.uint64(24 | (SYN_F << 32))
        return rec.view(np.uint8).reshape(-1)[off - 16 * r0:off - 16 * r0 + size]
    r0, r1 = off // SYN_F, (off + size + SYN_F - 1) // SYN_F
    return syn_records(r0, r1).reshape(-1)[off - SYN_F * r0:off - SYN_F * r0 + size]


def ref_binary_search(key):
    """binary_search (lsm_tree.rs:605-670) restated on the synthetic table: the record found, or -1."""
    low, high, half = 0, SYN_N - 1, SYN_N // 2
    while low <= high:
        k = syn_key(half)
        if k == key:
            return half
        if k < key:
            low = half + 1
        else:
            high = max(half, 1) - 1
        if half == 0 or half == SYN_N:
            break
        half = (high + low) // 2
    return -1


def test_a_table_larger_than_device_memory(engine):
    import torch
    rng = np.random.default_rng(13)
    rec = sorted(int(x) for x in rng.integers(0, SYN_N, 500)) + [0, 1, SYN_N - 1, (1 << 32) // SYN_F + 1]
    keys = [syn_key(r) for r in rec] + [syn_key(r) + b"x" for r in rec[:250]] + [b"k", b"k999999999999999", b"a"]
    free0 = torch.cuda.mem_get_info()[0]
    for mode in MODES:
        rows, d, i = engine.get_values_stream([(SYN_N * SYN_F, SYN_N * 16, None)], keys, mode, read=syn_read)
        st = engine.stats()
        for q, k in enumerate(keys):
            want = -1
            if q < len(rec):
                want = rec[q] if mode == capi.LOOKUP_EXACT else ref_binary_search(k)
            elif mode == capi.LOOKUP_REFERENCE:
                want = ref_binary_search(k)
            assert rows["table"][q] == (0 if want >= 0 else -1), (q, k)
            if want >= 0:
                assert rows["record"][q] == want and rows["bloom_rejects"][q] == 0
        hits = [rec[q] for q in range(len(rec)) if rows["table"][q] == 0]
        assert i.size == 16 * len(hits) and d.size == SYN_F * len(hits)
        ents = d.reshape(-1, SYN_F)
        assert np.array_equal(ents[:, 32:40].copy().view(np.uint64).reshape(-1), np.array(hits, np.uint64))
        print(f"mode {mode}: {len(keys)} keys, {st['input_bytes'] / 1e6:.1f} MB read of {SYN_N * (SYN_F + 16) / 1e9:.1f} GB, "
              f"{st['partitions']} leaf groups, device memory in use {(free0 - torch.cuda.mem_get_info()[0]) / 1e9:.2f} GB more, "
              f"max RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6:.2f} GB")
        assert st["input_bytes"] < 4e9
    assert free0 - torch.cuda.mem_get_info()[0] < 4 << 30


def test_tree_get_values_stream_after_flush_and_compact(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine)
    rng = np.random.default_rng(14)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    keys = [b"t%05d" % n for n in range(0, 3100, 7)] + [b"t00001", b"t00001"]
    for step in ("flushed", "compacted"):
        for mode in MODES:
            rows, od, oi = tree.get_values_stream(keys, mode)
            er, ed, ei = tree.get_values(keys, mode)
            assert np.array_equal(rows, er)
            assert_run_equal((od, oi), (ed, ei), step)
        if step == "flushed":
            tree.compact([0, 2, 4], 5, True)
    tree.close()
