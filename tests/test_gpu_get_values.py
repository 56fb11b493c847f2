"""Batched reads that return the entries (dbeel_get_values*, row N2): rows, .data and .index byte for byte against the CPU
oracle (tests/get_values_oracle.c), and rows equal to dbeel_get_many's with the bad-entry bit masked."""
import numpy as np
import pytest

import get_values_oracle as gvo
import oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from dbeel_b200 import workloads as W
from helpers import BASE_TS, assert_run_equal, nasty_keys, random_runs

pytestmark = pytest.mark.gpu

SEED = bytes(range(32))
TS_MAX = 253402300799 * 10**9 + 999_999_999
TS_MIN = -377705116800 * 10**9


@pytest.fixture(scope="module")
def dev():
    import torch
    return torch.device("cuda:0")


def _rec(index, r):
    b = bytes(np.asarray(index[16 * r:16 * r + 16], np.uint8))
    return int.from_bytes(b[:8], "little"), int.from_bytes(b[8:12], "little"), int.from_bytes(b[12:], "little")


def _set_u32(index, r, field, v):
    index[16 * r + field:16 * r + field + 4] = np.frombuffer(int(v).to_bytes(4, "little"), np.uint8)


def stored_batch(tables, rows):
    """The answered rows' entries as stored, in query order, as an arrival batch (offsets from 0)."""
    d, ix = [], []
    pos = 0
    for t, j, r in zip(rows["table"], rows["bloom_rejects"], rows["record"]):
        if t < 0 or j & capi.LOOKUP_BAD_ENTRY:
            continue
        off, ks, fs = _rec(tables[t][1], int(r))
        d.append(bytes(np.asarray(tables[t][0][off:off + fs], np.uint8)))
        ix.append(pos.to_bytes(8, "little") + ks.to_bytes(4, "little") + fs.to_bytes(4, "little"))
        pos += fs
    return np.frombuffer(b"".join(d), np.uint8), np.frombuffer(b"".join(ix), np.uint8)


def check(engine, tables, keys, mode=capi.LOOKUP_REFERENCE, oracle_ok=True):
    """Host entry point: rows == get_many's (bit masked) and == the oracle's; the batch == the oracle's EntryWriter output
    (REFERENCE mode) and == the stored bytes of the answered rows (both modes)."""
    rows, d, i = engine.get_values(tables, keys, mode)
    st = engine.stats()
    many = engine.get_many(tables, keys, mode)
    masked = rows.copy()
    masked["bloom_rejects"] &= ~np.uint32(capi.LOOKUP_BAD_ENTRY)
    assert np.array_equal(masked, many)
    ed, ei = stored_batch(tables, rows)
    assert_run_equal((d, i), (ed, ei), "stored bytes")
    n_ans = int(((rows["table"] >= 0) & ((rows["bloom_rejects"] & capi.LOOKUP_BAD_ENTRY) == 0)).sum())
    assert st["entries_out"] == n_ans and st["entries_in"] == len(keys) and st["output_bytes"] == d.size + i.size
    assert st["kernel_launches"] == (0 if not keys else 5 if n_ans == 0 else 12)
    if mode == capi.LOOKUP_REFERENCE and oracle_ok:
        blob, off = capi.pack_keys(keys)
        et, er, ej, od, oi = gvo.get_values(tables, blob, off)
        assert np.array_equal(rows["table"], et) and np.array_equal(rows["bloom_rejects"], ej)
        assert np.array_equal(np.where(rows["table"] >= 0, rows["record"], 0), er)
        assert_run_equal((d, i), (od, oi), "oracle")
    return rows, d, i


def keys_of(table):
    return [k for k, _, _ in sstable.parse_run(table[0], table[1])]


def test_both_modes_on_a_compacted_table_with_a_filter(engine):
    c = W.scaled(W.CFG2, 20_000)
    gd, gi, gb, n = engine.compact(W.make_merge_runs(c), keep_tombstones=False, seed=SEED)
    assert gb is not None
    table = (gd, gi, gb)
    present = keys_of(table)
    rng = np.random.default_rng(1)
    sample = [present[j] for j in rng.choice(len(present), 3000, replace=False)] + present[:40] + present[-40:]
    absent = [b"\xb0k%015d" % int(x) for x in rng.integers(0, 1 << 40, 1500)] + [b"", present[7] + b"\x00", present[9][:-1]]
    keys = sample + absent + sample[:500]  # asked twice: returned twice
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        rows, d, i = check(engine, [table], keys, mode)
        if mode == capi.LOOKUP_EXACT:
            assert (rows["table"][:len(sample)] == 0).all()


def test_tiny_tables_and_the_reference_early_exit(engine):
    for n in (1, 2, 3, 4, 5, 8, 33):
        ents = [(bytes([10 + 2 * j]), b"v" * j, BASE_TS + j) for j in range(n)]
        d, i = sstable.build_run(ents)
        keys = [bytes([x]) for x in range(8, 12 + 2 * n)]
        for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
            check(engine, [(d, i, None)], keys, mode)


def test_four_overlapping_tables_newest_first(engine):
    rng = np.random.default_rng(3)
    ents = [(b"\xb0k%015d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 90)), dtype=np.uint8)), BASE_TS + n)
            for n in range(9000)]
    tables = []
    for t, (lo, hi, step) in enumerate([(0, 6000, 1), (3000, 9000, 2), (100, 8000, 3), (5000, 5400, 1)]):
        d, i, b, _ = engine.compact([sstable.build_run(ents[lo:hi:step])], keep_tombstones=True,
                                    bloom_min_size=1000 if t != 2 else 1 << 40, seed=SEED)
        assert (b is None) == (t == 2)
        tables.append((d, i, b))
    keys = [ents[int(j)][0] for j in rng.integers(0, 9000, 2500)] + [b"\xb0k%015d" % n for n in range(9000, 9300)]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        rows, _, _ = check(engine, tables, keys, mode)
        assert set(np.unique(rows["table"])) >= {-1, 0, 1, 2, 3}


def test_tombstones_empty_values_and_entries_larger_than_a_gather_tile(engine):
    rng = np.random.default_rng(4)
    pool = nasty_keys(rng, 600, max_len=50)
    runs = random_runs(rng, 3, 400, pool, max_doc=40, tombstone_frac=0.3)
    big = sorted(rng.choice(len(pool), 4, replace=False))
    sizes = [3 << 20, 5 << 20, 8191, 16385]
    runs.append(sstable.build_run(sorted((pool[j], bytes(rng.integers(0, 256, s, dtype=np.uint8)), BASE_TS + 999)
                                         for j, s in zip(big, sizes))))
    gd, gi, gb, n = engine.compact(runs, keep_tombstones=True, bloom_min_size=1000, seed=SEED)
    table = (gd, gi, gb)
    ents = sstable.parse_run(gd, gi)
    assert any(v == b"" for _, v, _ in ents) and max(len(v) for _, v, _ in ents) >= 5 << 20
    keys = [k for k, _, _ in ents] + [pool[j] for j in big] * 3 + [b"\xfe\xfe-absent"]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        rows, d, i = check(engine, [table], keys, mode)
    assert d.size > 24 << 20  # EXACT: every big entry four times


def test_nothing_found_no_keys_no_tables(engine):
    d, i = sstable.build_run([(b"a%03d" % n, b"x" * n, BASE_TS) for n in range(100)])
    rows, od, oi = check(engine, [(d, i, None)], [b"b%03d" % n for n in range(300)])
    assert (rows["table"] == -1).all() and od.size == 0 and oi.size == 0 and engine.stats()["entries_out"] == 0
    rows, od, oi = engine.get_values([(d, i, None)], [])
    assert len(rows) == 0 and od.size == 0 and oi.size == 0
    rows, od, oi = check(engine, [], [b"a001", b""])
    assert (rows["table"] == -1).all() and od.size == 0


def test_bad_entries_and_corrupt_records(engine):
    ents = [(b"k%03d" % n, b"value-%d" % n, BASE_TS + n) for n in range(64)]
    ents[20] = (ents[20][0], b"t20", TS_MAX + 1)
    ents[21] = (ents[21][0], b"t21", TS_MIN - 1)
    ents[22] = (ents[22][0], b"t22", TS_MAX)
    ents[23] = (ents[23][0], b"t23", TS_MIN)
    d, i = sstable.build_run(ents)
    for r, field, delta in ((5, 8, 1), (6, 8, -1), (7, 12, -1), (8, 12, 1)):
        _set_u32(i, r, field, _rec(i, r)[1 if field == 8 else 2] + delta)
    _set_u32(i, 9, 12, _rec(i, 9)[1] - 1)  # full_size < key_size
    keys = [k for k, _, _ in ents]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        rows, _, _ = check(engine, [(d, i, None)], keys, mode)
        bad = set(np.flatnonzero(rows["bloom_rejects"] & capi.LOOKUP_BAD_ENTRY))
        if mode == capi.LOOKUP_EXACT:
            assert bad == {5, 6, 7, 8, 9, 20, 21}
    # a value running past the end of .data (the last entry loses its last byte)
    check(engine, [(d[:-1].copy(), i, None)], keys[-3:], capi.LOOKUP_EXACT)
    rows, _, _ = check(engine, [(d[:-1].copy(), i, None)], keys[-1:], capi.LOOKUP_EXACT)
    assert rows["bloom_rejects"][0] & capi.LOOKUP_BAD_ENTRY
    # an index record that points past the end of .data: the CORRUPT bit as in get_many, no entry
    broken = i.copy()
    broken[16 * 32:16 * 32 + 8] = np.frombuffer((1 << 40).to_bytes(8, "little"), np.uint8)
    rows, od, oi = check(engine, [(d, broken, None)], [b"k010", b"k050"], oracle_ok=False)
    assert (rows["table"] == -1).all() and (rows["bloom_rejects"] & capi.LOOKUP_CORRUPT).all() and od.size == 0


def _device_table(dev, table):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) if a is not None else None for a in table]


def _guarded(dev, size, rng, shift=0):
    """(tensor, data pointer) with a 256-byte front guard and a gather tile + 64 bytes behind, seeded random bytes."""
    import torch
    front, back = 256 + shift, 16384 + 64
    buf = torch.from_numpy(rng.integers(0, 256, front + size + back, dtype=np.uint8)).to(dev)
    return buf, front


def test_device_entry_point_on_compact_device_output_with_guards_and_caps(engine, dev):
    import torch
    runs = W.make_merge_runs(W.scaled(W.CFG2, 50_000))
    t_runs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in runs]
    opts = capi.make_opts(False, seed=SEED)
    dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], opts)
    od, oi, ob = (torch.empty(c + 16, dtype=torch.uint8, device=dev) for c in (dc, ic, bc))
    dl, il, bl, n = engine.compact_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_runs],
                                          (od.data_ptr(), dc, oi.data_ptr(), ic, ob.data_ptr(), bc), opts)
    host = (od[:dl].cpu().numpy(), oi[:il].cpu().numpy(), ob[:bl].cpu().numpy())
    present = keys_of(host)
    rng = np.random.default_rng(6)
    keys = [present[j] for j in rng.choice(n, 20_000, replace=False)] + [b"\xb0k%015d" % int(x) for x in rng.integers(0, 1 << 40, 5000)]
    keys += keys[:300]
    blob, koff = capi.pack_keys(keys)
    d_keys, d_off = torch.from_numpy(blob.copy()).to(dev), torch.from_numpy(koff.view(np.int64)).to(dev)
    tab = [(od.data_ptr(), dl, oi.data_ptr(), il, ob.data_ptr(), bl)]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        want_rows, wd, wi = engine.get_values([host], keys, mode)
        need_d, need_i = wd.size, wi.size
        for k, (cd, ci) in enumerate([(need_d, need_i), (need_d - 1, need_i), (need_d, need_i - 1)]):
            d_res = torch.zeros(len(keys) * 2, dtype=torch.int64, device=dev)
            gd, fd = _guarded(dev, cd, rng, 16 * k)
            gi, fi = _guarded(dev, ci, rng, 48)
            gd0, gi0 = gd.cpu().numpy(), gi.cpu().numpy()
            torch.cuda.synchronize()
            if k == 0:
                got = engine.get_values_device(tab, d_keys.data_ptr(), d_off.data_ptr(), len(keys), d_res.data_ptr(),
                                               (gd.data_ptr() + fd, cd, gi.data_ptr() + fi, ci), mode)
                assert got == (need_d, need_i, need_i // 16)
                gdn, gin = gd.cpu().numpy(), gi.cpu().numpy()
                assert np.array_equal(gdn[fd:fd + cd], wd) and np.array_equal(gin[fi:fi + ci], wi)
                gdn[fd:fd + cd] = gd0[fd:fd + cd]
                gin[fi:fi + ci] = gi0[fi:fi + ci]
                assert np.array_equal(gdn, gd0) and np.array_equal(gin, gi0), "a guard byte changed"
            else:
                with pytest.raises(capi.DbeelError) as ei:
                    engine.get_values_device(tab, d_keys.data_ptr(), d_off.data_ptr(), len(keys), d_res.data_ptr(),
                                             (gd.data_ptr() + fd, cd, gi.data_ptr() + fi, ci), mode)
                assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (need_d, need_i)
                assert np.array_equal(gd.cpu().numpy(), gd0) and np.array_equal(gi.cpu().numpy(), gi0), "written on ERR_CAPACITY"
            assert np.array_equal(d_res.cpu().numpy().view(capi.LOOKUP_DTYPE), want_rows)
        with pytest.raises(capi.DbeelError) as ei:  # host entry point, one byte short
            engine.get_values([host], keys, mode, caps=(need_d - 1, need_i))
        assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (need_d, need_i)
        check(engine, [host], keys[:4000], mode)  # the same engine goes on


def test_device_inputs_from_flush_many_device_unaligned_data(engine, dev):
    import torch
    rng = np.random.default_rng(7)
    batches = []
    for b in range(3):
        ents = [(b"b%d-%05d" % (b, int(k)), bytes(rng.integers(0, 256, int(rng.integers(0, 37)), dtype=np.uint8)),
                 BASE_TS + int(rng.integers(100))) for k in rng.integers(0, 3000, 900)]
        batches.append(sstable.build_run(ents))
    tb = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in batches]
    dc, ic = sum(d.size for d, _ in batches), sum(i.size for _, i in batches)
    od, oi = torch.empty(dc + 16, dtype=torch.uint8, device=dev), torch.empty(ic + 16, dtype=torch.uint8, device=dev)
    _, _, _, table_rows = engine.flush_many_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in tb],
                                                   (od.data_ptr(), dc, oi.data_ptr(), ic))
    assert any(r["data_off"] % 16 for r in table_rows)  # a table whose .data does not start 16-byte aligned
    tabs = [(od.data_ptr() + r["data_off"], r["data_len"], oi.data_ptr() + r["index_off"], r["index_len"], 0, 0) for r in table_rows]
    host = [(od[r["data_off"]:r["data_off"] + r["data_len"]].cpu().numpy(), oi[r["index_off"]:r["index_off"] + r["index_len"]].cpu().numpy(),
             None) for r in table_rows]
    keys = [b"b%d-%05d" % (int(b), int(k)) for b, k in zip(rng.integers(0, 3, 4000), rng.integers(0, 3100, 4000))]
    blob, koff = capi.pack_keys(keys)
    d_keys, d_off = torch.from_numpy(blob.copy()).to(dev), torch.from_numpy(koff.view(np.int64)).to(dev)
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        want_rows, wd, wi = check(engine, host, keys, mode)
        d_res = torch.zeros(len(keys) * 2, dtype=torch.int64, device=dev)
        gd = torch.empty(wd.size + 16, dtype=torch.uint8, device=dev)
        gi = torch.empty(wi.size + 16, dtype=torch.uint8, device=dev)
        got = engine.get_values_device(tabs, d_keys.data_ptr(), d_off.data_ptr(), len(keys), d_res.data_ptr(),
                                       (gd.data_ptr(), wd.size, gi.data_ptr(), wi.size), mode)
        assert got == (wd.size, wi.size, wi.size // 16)
        assert np.array_equal(d_res.cpu().numpy().view(capi.LOOKUP_DTYPE), want_rows)
        assert_run_equal((gd[:wd.size].cpu().numpy(), gi[:wi.size].cpu().numpy()), (wd, wi), "device")


def test_output_is_an_arrival_batch_dbeel_flush_takes(engine):
    rng = np.random.default_rng(8)
    pool = nasty_keys(rng, 900, max_len=30)
    gd, gi, gb, n = engine.compact(random_runs(rng, 2, 700, pool, tombstone_frac=0.2), keep_tombstones=True, seed=SEED)
    keys = [pool[int(j)] for j in rng.integers(0, len(pool), 3000)]
    rows, d, i = check(engine, [(gd, gi, gb)], keys)
    assert i.size // 16 > 1000
    fd, fi, _ = engine.flush((d, i))
    (od, oi, _), = oracle.memtable_flushes((d, i))
    assert_run_equal((fd, fi), (od, oi), "flush of the returned batch")


def test_tree_get_values_after_flush_and_compact(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine)
    u16 = lambda n: int(n).to_bytes(2, "little")
    writes = [(u16(n), u16(n) * 3, BASE_TS + n) for n in range(94)] + [(u16(1), b"", BASE_TS + 1000)]
    for lo, hi in ((0, 32), (32, 64), (64, 95)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    keys = [u16(n) for n in range(0, 100, 3)] + [u16(1), u16(1)]
    for step in ("flushed", "compacted"):
        files = [sstable.read_run_files(d, idx) + (None,) for idx, _ in tree.sstable_indices_and_sizes()]
        for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
            rows, od, oi = tree.get_values(keys, mode)
            er, ed, ei = engine.get_values(files, keys, mode)
            assert np.array_equal(rows, er)
            assert_run_equal((od, oi), (ed, ei), step)
            blob, koff = capi.pack_keys(keys)
            et, _, ej, gd_, gi_ = gvo.get_values(files, blob, koff)
            if mode == capi.LOOKUP_REFERENCE:
                assert np.array_equal(rows["table"], et) and np.array_equal(rows["bloom_rejects"], ej)
                assert_run_equal((od, oi), (gd_, gi_), step + " oracle")
        if step == "flushed":
            tree.compact([0, 2, 4], 5, True)
    vals = {k: v for k, v, _ in sstable.parse_run(od, oi)}
    assert vals[u16(1)] == b"" and vals[u16(3)] == u16(3) * 3
    tree.close()
