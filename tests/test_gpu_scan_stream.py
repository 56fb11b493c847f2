"""dbeel_scan_stream / dbeel_tree_scan_stream: the scan fed from files, one partition of the record sequence at a time.
Byte and stop parity with the scan oracle and with dbeel_scan on trees split into many partitions (small budgets), callback
errors, and device memory that does not grow with the tree."""
import numpy as np
import pytest

import oracle
import scan_oracle
from dbeel_b200 import capi, sstable, storage_engine as se
from helpers import BASE_TS, assert_run_equal
from scan_cases import DAMAGES, HASH, KEY, NONE, damage, eighths, hash_ranges, key_ranges, random_tree

pytestmark = pytest.mark.gpu


@pytest.fixture
def make_engine(monkeypatch):
    """Engines with their own partition budget (KB) and ring depth: small trees split into many partitions."""
    made = []

    def make(budget_kb: int, ring: int = 3):
        monkeypatch.setenv("DBEEL_PARTITION_KB", str(budget_kb))
        monkeypatch.setenv("DBEEL_STREAM_RING", str(ring))
        monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
        e = capi.Engine(0)
        made.append(e)
        return e

    yield make
    for e in made:
        e.close()


def _check(got, exp, what):
    (gr, gs), (er, es) = got, exp
    assert gs == es, f"{what}: stop {gs} != {es}"
    assert len(gr) == len(er)
    for j, (g, e) in enumerate(zip(gr, er)):
        assert_run_equal(g, e, f"{what} destination {j}")


def _all(stream_engine, tables, ranges, kind, what, engine=None):
    exp = scan_oracle.scan(tables, ranges, kind)
    got = stream_engine.scan_stream(tables, ranges, kind)
    _check(got, exp, what)
    st = stream_engine.stats()
    if st["partitions"]:  # the range header copy, then classify + split + carry + phase 2 per partition
        assert st["kernel_launches"] == 1 + 12 * st["partitions"], what
    if engine is not None:
        _check(engine.scan(tables, ranges, kind), exp, what + " (dbeel_scan)")
    return exp


def _tree_bytes(tables):
    return sum(d.size + i.size for d, i in tables)


@pytest.mark.parametrize("n_tables,big", [(1, False), (8, False), (37, False), (8, True)])
@pytest.mark.parametrize("ring", [2, 3])
def test_hash_ranges_match_oracle_and_dbeel_scan(engine, make_engine, n_tables, big, ring):
    rng = np.random.default_rng(n_tables * 10 + big)
    tables = random_tree(rng, n_tables, max_entries=200, big=big)
    eng = make_engine(4, ring)
    for ranges in (hash_ranges(rng, 1), hash_ranges(rng, 8), eighths(), hash_ranges(rng, 256),
                   [(0, 0xFFFFFFFF)], [(5, 5), (9, 3)], [(1 << 31, 1 << 31), (0, 1 << 30), (1 << 29, 1 << 31)]):
        _all(eng, tables, ranges, HASH, f"{n_tables} tables, {len(ranges)} ranges, ring {ring}", engine)
    assert eng.stats()["partitions"] > 1


@pytest.mark.parametrize("n_tables", [1, 8, 37])
def test_key_ranges_match_oracle(engine, make_engine, n_tables):
    rng = np.random.default_rng(500 + n_tables)
    tables = random_tree(rng, n_tables, max_entries=150)
    eng = make_engine(2)
    for ranges in (key_ranges(tables), [(b"", b"\xff" * 200)], [(b"", b"")], [(b"\xff", b"\xff\xff\xff\xff\xff\xff\xff\xff\xff\x00")],
                   [(b"common-prefix-that-is-quite-long/", b"common-prefix-that-is-quite-long/\x00\x01")]):
        _all(eng, tables, ranges, KEY, f"{n_tables} tables, key ranges {ranges[:1]}", engine)


def test_budgets_from_one_record_to_more_than_the_tree(engine, make_engine):
    rng = np.random.default_rng(31)
    tables = random_tree(rng, 8, max_entries=120)
    total_kb = _tree_bytes(tables) // 1024 + 1
    parts = []
    for kb in (1, 3, 16, total_kb, 4 * total_kb):
        eng = make_engine(kb)
        _all(eng, tables, eighths(), HASH, f"budget {kb} KB")
        _all(eng, tables, key_ranges(tables), KEY, f"budget {kb} KB, key ranges")
        parts.append(eng.stats()["partitions"])
    assert parts[0] > parts[2] > 1 and parts[-1] == 1


def _big_overlap_tree(copies: int):
    """One ~1 MiB entry listed `copies` times between small entries: larger than the budget, and an output many times
    the input."""
    ents = [(b"a", b"x" * 10, BASE_TS), (b"big", bytes(range(256)) * 4096, BASE_TS + 1), (b"z", b"y" * 7, BASE_TS + 2)]
    d, i = sstable.build_run(ents)
    recs = np.asarray(i, np.uint8).reshape(-1, 16)
    idx = np.concatenate([recs[:1]] + [recs[1:2]] * copies + [recs[2:]]).reshape(-1).copy()
    small = sstable.build_run([(b"k%d" % n, b"v" * n, BASE_TS) for n in range(50)])
    return [(np.asarray(d, np.uint8).copy(), idx), (np.asarray(small[0], np.uint8).copy(), np.asarray(small[1], np.uint8).copy())]


def test_entry_larger_than_the_budget_and_overlapping_records(engine, make_engine):
    tables = _big_overlap_tree(16)
    for kb in (64, 4096, 64 * 1024):
        eng = make_engine(kb)
        for ranges, kind in ((eighths(), HASH), ([(0, 0xFFFFFFFF)], HASH), ([(b"", b"\xff")], KEY)):
            exp = _all(eng, tables, ranges, kind, f"overlapping records, budget {kb} KB", engine)
        assert sum(d.size for d, _ in exp[0]) > 15 * sum(d.size for d, _ in tables)


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage_in_every_partition_position(engine, make_engine, kind):
    rng = np.random.default_rng(77)
    tables = random_tree(rng, 6, max_entries=120)
    eng = make_engine(2)
    eng.scan_stream(tables, eighths(), HASH)
    n_parts = eng.stats()["partitions"]
    assert n_parts >= 6
    flat = [(t, r) for t in range(len(tables)) for r in range(tables[t][1].size // 16)]
    # first partition, middle, last, and a sweep of consecutive records across several cuts (2 KB holds a handful)
    spots = [flat[0], flat[len(flat) // 2], flat[-1]] + flat[40:64]
    for t, rec in spots:
        bad = damage(tables, kind, t, rec)
        exp = _all(eng, bad, eighths(), HASH, f"{kind} at {t}/{rec}")
        if kind == "ragged_index":
            assert exp[1] == (-1, NONE, 0)
        else:
            assert exp[1][0] == t
    for t, rec in spots[:3]:
        bad = damage(tables, kind, t, rec)
        _all(eng, bad, key_ranges(tables), KEY, f"{kind} at {t}/{rec}, key ranges", engine)


@pytest.mark.parametrize("where", ["first_read", "mid_read", "first_write", "last_write"])
def test_callback_errors_come_back_and_the_engine_stays_usable(engine, make_engine, where):
    import torch
    rng = np.random.default_rng(21)
    tables = random_tree(rng, 8, max_entries=300)
    eng = make_engine(4)
    ok = eng.scan_stream(tables, eighths(), HASH)
    n_reads, n_writes = eng.last_stream_calls  # callback calls of a clean run: where the failures go
    assert n_reads > 4 and n_writes > 4
    at = {"first_read": ("r", 0), "mid_read": ("r", n_reads // 2), "first_write": ("w", 0), "last_write": ("w", n_writes - 1)}[where]
    with pytest.raises(capi.DbeelError) as ei:
        if at[0] == "r":
            eng.scan_stream(tables, eighths(), HASH, fail_read_at=at[1])
        else:
            eng.scan_stream(tables, eighths(), HASH, fail_write_at=at[1])
    assert ei.value.code == 4242
    # the same engine: a device scan and a streamed scan give the right bytes
    dev = torch.device("cuda:0")
    t_tabs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in tables]
    dc = sum(d.size for d, _ in tables) * 2
    ic = sum(i.size for _, i in tables)
    od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
    oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    rows, stop = eng.scan_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_tabs], eighths(),
                                 (od.data_ptr(), dc, oi.data_ptr(), ic), HASH)
    exp = scan_oracle.scan(tables, eighths(), HASH)
    assert stop == exp[1]
    d_all, i_all = od.cpu().numpy(), oi.cpu().numpy()
    for r, (ed, ei_) in zip(rows, exp[0]):
        assert_run_equal((d_all[r["data_off"]:r["data_off"] + r["data_len"]], i_all[r["index_off"]:r["index_off"] + r["index_len"]]),
                         (ed, ei_), "device scan after a callback error")
    _check(eng.scan_stream(tables, eighths(), HASH), exp, "streamed scan after a callback error")
    _check(ok, exp, "before the error")


def _scaled_tree(rng, copies: int):
    """`copies` tables of ~2 MB each with running offsets, like the writer's."""
    tables = []
    for c in range(copies):
        ents = [(b"key-%08d-%d" % (k, c), bytes(rng.integers(0, 256, 250, dtype=np.uint8)), BASE_TS + k) for k in range(7000)]
        d, i = sstable.build_run(ents)
        tables.append((np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy()))
    return tables


def test_device_memory_does_not_grow_with_the_tree(make_engine):
    import torch
    rng = np.random.default_rng(5)
    small, large = _scaled_tree(rng, 2), _scaled_tree(rng, 8)
    eng = make_engine(512)
    torch.cuda.synchronize()
    got = eng.scan_stream(small, eighths(), HASH)
    _check(got, scan_oracle.scan(small, eighths(), HASH), "tree S")
    p_small = eng.stats()["partitions"]
    free_small = torch.cuda.mem_get_info()[0]
    got = eng.scan_stream(large, eighths(), HASH)
    _check(got, scan_oracle.scan(large, eighths(), HASH), "tree 4S")
    p_large = eng.stats()["partitions"]
    free_large = torch.cuda.mem_get_info()[0]
    assert free_large == free_small, (free_small, free_large)
    assert 3.5 * p_small <= p_large <= 4.5 * p_small, (p_small, p_large)


def test_tree_scan_stream_on_files(engine, make_engine, tmp_path):
    """dbeel_tree_scan_stream over files written by flushes and a compaction gives dbeel_tree_scan's destinations."""
    d = str(tmp_path)
    eng = make_engine(1)
    tree = se.LSMTree.open_or_create(d, eng)
    rng = np.random.default_rng(3)
    writes = [(b"k%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 90)), dtype=np.uint8)), BASE_TS + n) for n in range(400)]
    writes += [(b"k00001", b"", BASE_TS + 1000), (b"k00004", b"", BASE_TS + 1001)]
    batch = sstable.build_run(writes)
    for sub_d, sub_i, _ in oracle.memtable_flushes(batch, capacity=64):
        tree.flush((sub_d, sub_i))
    for ranges, kind in ((eighths(), HASH), ([(b"k00001", b"k00200"), (b"", b"\xff")], KEY)):
        got = tree.scan_stream(ranges, kind)
        assert eng.stats()["partitions"] > 1
        _check(got, tree.scan(ranges, kind), f"tree, {len(ranges)} ranges")
    idx = [i for i, _ in tree.sstable_indices_and_sizes()]
    tree.compact(idx[:3], idx[-1] + 1, False)
    for ranges, kind in ((eighths(), HASH), ([(b"k00001", b"k00200"), (b"", b"\xff")], KEY)):
        _check(tree.scan_stream(ranges, kind), tree.scan(ranges, kind), f"after compaction, {len(ranges)} ranges")
    # the write callback's error code comes back
    rows, _ = tree.scan_stream(eighths(), HASH, write=lambda dest, kind, off, src, size: 0)
    assert sum(r[2] for r in rows) > 0
    with pytest.raises(capi.DbeelError) as ei:
        tree.scan_stream(eighths(), HASH, write=lambda dest, kind, off, src, size: 4242)
    assert ei.value.code == 4242
    _check(tree.scan_stream(eighths(), HASH), tree.scan(eighths(), HASH), "after a write error")


def test_compaction_after_streamed_scans_is_unchanged(make_engine):
    eng = make_engine(8)
    rng = np.random.default_rng(13)
    runs = [sstable.build_run(sorted(((int(k).to_bytes(2, "little") + bytes([r]), bytes(rng.integers(0, 256, 50, dtype=np.uint8)),
                                       BASE_TS + r) for k in range(2000)), key=lambda e: e[0])) for r in range(4)]
    seed = bytes(range(32))
    before = eng.compact(runs, False, bloom_min_size=1000, seed=seed)
    big = random_tree(rng, 37, max_entries=400)
    eng.scan_stream(big, hash_ranges(rng, 256), HASH)
    eng.scan_stream(big, key_ranges(big), KEY)
    after = eng.compact(runs, False, bloom_min_size=1000, seed=seed)
    exp = oracle.compact(runs, False, bloom_min_size=1000, seed=seed)
    for a, b, c in zip(before[:3], after[:3], exp[:3]):
        assert np.array_equal(a, b) and np.array_equal(a, c)
