"""dbeel_scan / dbeel_scan_device / dbeel_tree_scan (LSMTree::iter_filter's SSTable part) against the scan oracle:
byte-identical per destination, identical stop."""
import numpy as np
import pytest

import oracle
import scan_oracle
from dbeel_b200 import capi, sstable, storage_engine as se
from helpers import BASE_TS, assert_run_equal
from scan_cases import DAMAGES, HASH, KEY, NONE, damage, eighths, hash_ranges, key_ranges, random_tree

pytestmark = pytest.mark.gpu


def u16key(n: int) -> bytes:
    return int(n).to_bytes(2, "little")


def _check(got, exp, what):
    (gr, gs), (er, es) = got, exp
    assert gs == es, f"{what}: stop {gs} != {es}"
    assert len(gr) == len(er)
    for j, (g, e) in enumerate(zip(gr, er)):
        assert_run_equal(g, e, f"{what} destination {j}")


def _both(engine, tables, ranges, kind, what):
    exp = scan_oracle.scan(tables, ranges, kind)
    _check(engine.scan(tables, ranges, kind), exp, what)
    return exp


@pytest.mark.parametrize("n_tables,big", [(1, False), (8, False), (37, False), (8, True)])
def test_hash_ranges_match_oracle(engine, n_tables, big):
    rng = np.random.default_rng(n_tables * 10 + big)
    tables = random_tree(rng, n_tables, max_entries=200, big=big)
    for ranges in (hash_ranges(rng, 1), hash_ranges(rng, 8), eighths(), hash_ranges(rng, 256),
                   [(0, 0xFFFFFFFF)], [(5, 5), (9, 3)], [(1 << 31, 1 << 31), (0, 1 << 30), (1 << 29, 1 << 31)]):
        _both(engine, tables, ranges, HASH, f"{n_tables} tables, {len(ranges)} ranges")


@pytest.mark.parametrize("n_tables", [1, 8, 37])
def test_key_ranges_match_oracle(engine, n_tables):
    rng = np.random.default_rng(500 + n_tables)
    tables = random_tree(rng, n_tables, max_entries=150)
    for ranges in (key_ranges(tables), [(b"", b"\xff" * 200)], [(b"", b"")], [(b"\xff", b"\xff\xff\xff\xff\xff\xff\xff\xff\xff\x00")],
                   [(b"common-prefix-that-is-quite-long/", b"common-prefix-that-is-quite-long/\x00\x01")]):
        _both(engine, tables, ranges, KEY, f"{n_tables} tables, key ranges {ranges[:1]}")


@pytest.mark.parametrize("kind", DAMAGES)
def test_damaged_trees_stop_where_the_reference_stops(engine, kind):
    rng = np.random.default_rng(77)
    tables = random_tree(rng, 6, max_entries=120)
    for t, rec in [(0, 0), (2, 5), (3, 10 ** 6 + 7), (5, 119)]:
        bad = damage(tables, kind, t, rec)
        exp = _both(engine, bad, eighths(), HASH, f"{kind} at {t}/{rec}")
        if kind == "ragged_index":
            assert exp[1] == (-1, NONE, 0)
        else:
            assert exp[1][0] == t
        _both(engine, bad, key_ranges(tables), KEY, f"{kind} at {t}/{rec}, key ranges")


def test_host_and_device_entry_points_agree(engine):
    import torch
    rng = np.random.default_rng(9)
    tables = random_tree(rng, 8, max_entries=300)
    tables = damage(tables, "timestamp", 6, 40)
    ranges = hash_ranges(rng, 8)
    host = engine.scan(tables, ranges, HASH)
    dev = torch.device("cuda:0")
    t_tabs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in tables]
    dc = sum(d.size for d, _ in tables) * 2
    ic = sum(i.size for _, i in tables)
    od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
    oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    rows, stop = engine.scan_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_tabs], ranges,
                                    (od.data_ptr(), dc, oi.data_ptr(), ic), HASH)
    assert stop == host[1]
    d_all, i_all = od.cpu().numpy(), oi.cpu().numpy()
    for r, (hd, hi) in zip(rows, host[0]):
        assert r["bloom_len"] == 0 and r["items_written"] * 16 == r["index_len"]
        assert_run_equal((d_all[r["data_off"]:r["data_off"] + r["data_len"]], i_all[r["index_off"]:r["index_off"] + r["index_len"]]),
                         (hd, hi), "device vs host")


def test_output_feeds_dbeel_flush(engine):
    """A destination's stream is an arrival batch: dbeel_flush of it equals the oracle's memtable flushes."""
    rng = np.random.default_rng(11)
    tables = random_tree(rng, 8, max_entries=400)
    outs, _ = engine.scan(tables, eighths(), HASH)
    for d, i in outs:
        if i.size == 0:
            continue
        exp = oracle.memtable_flushes((d, i))  # fewer distinct keys than one memtable holds: one flush
        assert len(exp) == 1
        fd, fi, n = engine.flush((d, i))
        assert n == exp[0][2]
        assert_run_equal((fd, fi), exp[0][:2], "flush of a scan destination")


def test_capacity_and_arguments(engine):
    rng = np.random.default_rng(12)
    tables = random_tree(rng, 3)
    with pytest.raises(capi.DbeelError) as ei:
        engine.scan(tables, [], HASH)
    assert ei.value.code == capi.ERR_INVALID_ARG
    with pytest.raises(capi.DbeelError) as ei:
        engine.scan(tables, [(0, 1)] * 257, HASH)
    assert ei.value.code == capi.ERR_INVALID_ARG
    assert engine.scan([], [(0, 0xFFFFFFFF)], HASH)[1] == (-1, NONE, 0)


def test_compaction_after_scans_is_unchanged(engine):
    """The scan shares the engine's grow-only workspace with compaction."""
    rng = np.random.default_rng(13)
    runs = [sstable.build_run(sorted(((u16key(k) + bytes([r]), bytes(rng.integers(0, 256, 50, dtype=np.uint8)), BASE_TS + r)
                                      for k in range(2000)), key=lambda e: e[0])) for r in range(4)]
    seed = bytes(range(32))
    before = engine.compact(runs, False, bloom_min_size=1000, seed=seed)
    big = random_tree(rng, 37, max_entries=400)
    engine.scan(big, hash_ranges(rng, 256), HASH)
    engine.scan(big, key_ranges(big), KEY)
    after = engine.compact(runs, False, bloom_min_size=1000, seed=seed)
    exp = oracle.compact(runs, False, bloom_min_size=1000, seed=seed)
    for a, b, c in zip(before[:3], after[:3], exp[:3]):
        assert np.array_equal(a, b) and np.array_equal(a, c)


def test_tree_scan_on_files(engine, tmp_path):
    """dbeel_tree_scan over files written by dbeel_tree_flush / dbeel_tree_compact: get_after_compaction's range reads
    (lsm_tree.rs:1363-1397), and hash scans against the oracle over the same files."""
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine)
    writes = [(u16key(n), u16key(n), BASE_TS + n) for n in range(94)]
    writes += [(u16key(1), b"", BASE_TS + 1000), (u16key(4), b"", BASE_TS + 1001)]
    batch = sstable.build_run(writes)
    for sub_d, sub_i, _ in oracle.memtable_flushes(batch, capacity=32):
        tree.flush((sub_d, sub_i))
    assert [i for i, _ in tree.sstable_indices_and_sizes()] == [0, 2, 4]
    (out,), stop = tree.scan([(u16key(1), u16key(5))], KEY)
    assert stop == (-1, NONE, 0)
    assert [v for _, v, _ in sstable.parse_run(*out)] == [u16key(1), u16key(2), u16key(3), u16key(4), b"", b""]
    files = [sstable.read_run_files(d, i) for i in (0, 2, 4)]
    _check(tree.scan(eighths(), HASH), scan_oracle.scan(files, eighths(), HASH), "tree hash scan")
    tree.compact([0, 2, 4], 5, False)
    (out,), stop = tree.scan([(u16key(1), u16key(5))], KEY)
    assert stop == (-1, NONE, 0)
    assert [v for _, v, _ in sstable.parse_run(*out)] == [u16key(2), u16key(3)]
    _check(tree.scan(eighths(), HASH), scan_oracle.scan([sstable.read_run_files(d, 5)], eighths(), HASH), "after compaction")


def _big_overlap_tree(copies: int):
    """One ~1 MiB entry listed `copies` times in its table's .index, between small entries: the scan's output is many
    8 KB gather tiles larger than the tables' .data."""
    ents = [(b"a", b"x" * 10, BASE_TS), (b"big", bytes(range(256)) * 4096, BASE_TS + 1), (b"z", b"y" * 7, BASE_TS + 2)]
    d, i = sstable.build_run(ents)
    recs = np.asarray(i, np.uint8).reshape(-1, 16)
    idx = np.concatenate([recs[:1]] + [recs[1:2]] * copies + [recs[2:]]).reshape(-1).copy()
    small = sstable.build_run([(b"k%d" % n, b"v" * n, BASE_TS) for n in range(50)])
    return [(np.asarray(d, np.uint8).copy(), idx), (np.asarray(small[0], np.uint8).copy(), np.asarray(small[1], np.uint8).copy())]


def test_output_larger_than_the_inputs(engine):
    """Index records that share .data bytes: every copy is delivered (no dedupe), host and device entry points."""
    import torch
    tables = _big_overlap_tree(16)
    exp = scan_oracle.scan(tables, eighths(), HASH)
    assert sum(d.size for d, _ in exp[0]) > 15 * sum(d.size for d, _ in tables)
    for ranges, kind in ((eighths(), HASH), ([(0, 0xFFFFFFFF)], HASH), ([(b"", b"\xff")], KEY)):
        exp = _both(engine, tables, ranges, kind, f"overlapping records, {len(ranges)} ranges")
        dev = torch.device("cuda:0")
        t_tabs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in tables]
        dc = sum(d.size for d, _ in exp[0])
        ic = sum(i.size for _, i in tables)
        od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
        oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
        rows, stop = engine.scan_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_tabs], ranges,
                                        (od.data_ptr(), dc, oi.data_ptr(), ic), kind)
        assert stop == exp[1]
        d_all, i_all = od.cpu().numpy(), oi.cpu().numpy()
        for r, (ed, ei) in zip(rows, exp[0]):
            assert_run_equal((d_all[r["data_off"]:r["data_off"] + r["data_len"]], i_all[r["index_off"]:r["index_off"] + r["index_len"]]),
                             (ed, ei), "device, overlapping records")


def _raw_scan(engine, tables, kind, ranges_ptr, n_ranges, data_cap, index_cap, device=False, out_ptrs=None):
    import ctypes as C
    arr = (capi.Table * max(1, len(tables)))()
    for j, t in enumerate(tables):
        arr[j] = capi.Table(t[0], t[1], t[2], t[3], None, 0)
    od = np.empty(max(1, data_cap), np.uint8)
    oi = np.empty(max(16, index_cap), np.uint8)
    dp, ip = out_ptrs if out_ptrs else (od.ctypes.data, oi.ctypes.data)
    out = capi.Out(dp, data_cap, 0, ip, index_cap, 0, None, 0, 0, 0)
    res = (capi.JobResult * max(1, n_ranges))()
    for r in res:
        r.data_off = r.data_len = r.index_off = r.index_len = r.items_written = 12345
    stop = capi.ScanStop()
    f = capi.lib().dbeel_scan_device if device else capi.lib().dbeel_scan
    rc = f(engine._h, arr, len(tables), kind, ranges_ptr, n_ranges, C.byref(out), res, C.byref(stop))
    return rc, res, out


def test_error_paths(engine):
    import ctypes as C
    import torch
    tables = _big_overlap_tree(4)
    ptrs = [(d.ctypes.data, d.size, i.ctypes.data, i.size) for d, i in tables]
    hr = np.array([0, 0xFFFFFFFF], np.uint32)
    dsum, isum = sum(d.size for d, _ in tables), sum(i.size for _, i in tables)
    # the output (the big entry four times) exceeds caps sized by dbeel_scan_bound: DBEEL_ERR_CAPACITY, rows zeroed
    dc, ic = C.c_uint64(), C.c_uint64()
    arr = (capi.Table * 2)(*[capi.Table(p[0], p[1], p[2], p[3], None, 0) for p in ptrs])
    assert capi.lib().dbeel_scan_bound(arr, 2, C.byref(dc), C.byref(ic)) == 0 and (dc.value, ic.value) == (dsum, isum)
    rc, res, out = _raw_scan(engine, ptrs, capi.SCAN_HASH, hr.ctypes.data, 1, dc.value, ic.value)
    assert rc == capi.ERR_CAPACITY
    assert (res[0].data_len, res[0].index_len, res[0].items_written, out.data_len, out.index_len) == (0, 0, 0, 0, 0)
    # the same call with room for the output succeeds
    rc, res, out = _raw_scan(engine, ptrs, capi.SCAN_HASH, hr.ctypes.data, 1, 4 * dsum, isum)
    assert rc == 0 and out.data_len > dsum
    # more than DBEEL_MAX_RUNS tables, an unknown kind, key offsets that do not ascend
    assert _raw_scan(engine, [ptrs[1]] * 1025, capi.SCAN_HASH, hr.ctypes.data, 1, 1025 * dsum, 1025 * isum)[0] == capi.ERR_INVALID_ARG
    assert _raw_scan(engine, ptrs, 2, hr.ctypes.data, 1, 4 * dsum, isum)[0] == capi.ERR_INVALID_ARG
    keys = np.frombuffer(b"abcdef", np.uint8).copy()
    offs = np.array([0, 4, 2], np.uint64)
    kr = capi.KeyRanges(keys.ctypes.data, offs.ctypes.data)
    assert _raw_scan(engine, ptrs, capi.SCAN_KEY, C.addressof(kr), 1, 4 * dsum, isum)[0] == capi.ERR_INVALID_ARG
    offs[:] = [0, 2, 4]
    assert _raw_scan(engine, ptrs, capi.SCAN_KEY, C.addressof(kr), 1, 4 * dsum, isum)[0] == 0
    # device entry point: a .index or an output buffer that is not 16-byte aligned
    dev = torch.device("cuda:0")
    t_tabs = [(torch.from_numpy(d).to(dev), torch.from_numpy(np.concatenate([np.zeros(16, np.uint8), i])).to(dev)) for d, i in tables]
    od = torch.empty(4 * dsum + 64, dtype=torch.uint8, device=dev)
    oi = torch.empty(isum + 64, dtype=torch.uint8, device=dev)
    good = [(d.data_ptr(), d.numel(), i.data_ptr() + 16, i.numel() - 16) for d, i in t_tabs]
    bad = [(d.data_ptr(), d.numel(), i.data_ptr() + 8, i.numel() - 16) for d, i in t_tabs]
    assert _raw_scan(engine, good, capi.SCAN_HASH, hr.ctypes.data, 1, 4 * dsum, isum, True, (od.data_ptr(), oi.data_ptr()))[0] == 0
    assert _raw_scan(engine, bad, capi.SCAN_HASH, hr.ctypes.data, 1, 4 * dsum, isum, True, (od.data_ptr(), oi.data_ptr()))[0] == capi.ERR_INVALID_ARG
    assert _raw_scan(engine, good, capi.SCAN_HASH, hr.ctypes.data, 1, 4 * dsum, isum, True,
                     (od.data_ptr() + 4, oi.data_ptr()))[0] == capi.ERR_INVALID_ARG
    assert _raw_scan(engine, good, capi.SCAN_HASH, hr.ctypes.data, 1, 4 * dsum, isum, True,
                     (od.data_ptr(), oi.data_ptr() + 8))[0] == capi.ERR_INVALID_ARG
    # the engine still scans correctly afterwards
    _both(engine, tables, eighths(), HASH, "after the error paths")
