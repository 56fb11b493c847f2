"""The device entry points at the edges of the caller's buffers.

include/dbeel_compact.h promises three things about caller memory: a run's `.data` may start anywhere (the tables that
dbeel_flush_many / dbeel_compact_many leave back to back are inputs as they lie), nothing is written past an output's
`*_cap`, and only the 16-byte alignments the entry points check are needed.  The host entry points stage through engine
buffers with slack, so an overrun there lands in engine scratch; through the device entry points it corrupts the caller's
next SSTable.  Here every output sits inside one allocation between a front and a back guard filled with a seeded random
pattern, at offsets 0, 16 and 48 mod 256, with caps equal to the ABI's bounds and inputs built so that the output fills
the bound exactly; inputs start at every byte offset with poison around them.  Outputs must equal the CPU oracle byte for
byte and both guards must be untouched."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import scan_oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import workloads as W
from helpers import BASE_TS, assert_run_equal, nasty_keys

pytestmark = pytest.mark.gpu

TILE = 8192  # the payload gather's output tile (kGatherTileBytes)
OFFSETS = (0, 16, 48)  # output placements mod 256: nothing may rely on 32- or 256-byte alignment
SHIFTS = list(range(16)) + [33, 255, 4097]  # byte offsets of the inputs' .data
POISONS = ("zeros", "ones", "entry")
SEED = bytes(range(32))
STEP = 1 << 29
ALL_HASHES = [(k * STEP, (k + 1) * STEP) for k in range(7)] + [(7 * STEP, 0)]  # eight ranges that take every hash


class Guarded:
    """One device allocation: a front guard of at least 256 bytes, the buffer (`n` bytes at `offset` mod 256), a back guard
    of one gather tile and 64 bytes.  All of it starts as a seeded random pattern."""
    FRONT = 256
    BACK = TILE + 64

    def __init__(self, n: int, offset: int = 0, seed: int = 0):
        self.n, self.start = int(n), self.FRONT + int(offset)
        self.pattern = np.random.default_rng(seed).integers(0, 256, self.start + self.n + self.BACK, dtype=np.uint8)
        self.t = torch.from_numpy(self.pattern).to("cuda:0")
        assert self.t.data_ptr() % 256 == 0
        torch.cuda.synchronize()  # the engine runs on its own stream

    @property
    def ptr(self) -> int:
        return self.t.data_ptr() + self.start

    def bytes(self, lo: int = 0, hi=None) -> np.ndarray:
        return self.t[self.start + lo:self.start + (self.n if hi is None else hi)].cpu().numpy()

    def check(self, what: str, untouched_from=None):
        """Both guards still hold the pattern; with untouched_from = k, so do the buffer's bytes [k, n)."""
        torch.cuda.synchronize()
        got = self.t.cpu().numpy()
        back = self.start + (self.n if untouched_from is None else int(untouched_from))
        for lo, hi, name in ((0, self.start, "front guard"), (back, got.size, "bytes at or past the end")):
            bad = np.flatnonzero(got[lo:hi] != self.pattern[lo:hi])
            if bad.size:
                first, last = lo + int(bad[0]) - self.start, lo + int(bad[-1]) - self.start
                raise AssertionError(f"{what}: {name} overwritten: {bad.size} bytes in buffer[{first}..{last}] "
                                     f"(buffer of {self.n} bytes)")


def outs(sizes, offset: int, seed: int):
    return [Guarded(n, OFFSETS[(offset + k) % 3], seed + k) for k, n in enumerate(sizes)]


def sized_entries(rng, total: int, n: int, tomb: float = 0.15):
    """Up to n entries (fewer when their keys alone would not fit) with distinct keys whose encoded sizes add up to exactly
    `total` bytes; about `tomb` of them are tombstones."""
    keys = nasty_keys(rng, n, max_len=24)
    while sum(sstable.ENTRY_OVERHEAD + len(k) for k in keys) > total:
        keys.pop()
    n = len(keys)
    budget = total - sum(sstable.ENTRY_OVERHEAD + len(k) for k in keys)
    w = rng.random(n) * (rng.random(n) >= tomb)
    w[int(rng.integers(n))] += 1.0
    dl = np.floor(w / w.sum() * budget).astype(np.int64)
    dl[int(np.argmax(w))] += budget - int(dl.sum())
    ents = [(k, bytes(rng.integers(0, 256, int(d), dtype=np.uint8)), BASE_TS + int(rng.integers(-999, 999)))
            for k, d in zip(keys, dl)]
    assert sum(len(sstable.encode_entry(*e)) for e in ents) == total
    return ents


def n_entries_for(total: int) -> int:
    return int(min(3000, max(40, total // 100)))


def sized_runs(rng, total: int, n_runs: int, n=None):
    """n_runs sorted runs of distinct keys, interleaved in key order, whose .data files add up to exactly `total` bytes."""
    ents = sized_entries(rng, total, n or n_entries_for(total))
    owner = np.concatenate([np.arange(n_runs), rng.integers(0, n_runs, len(ents) - n_runs)])
    rng.shuffle(owner)
    return [sstable.build_run(sorted((e for e, o in zip(ents, owner) if o == r), key=lambda e: e[0])) for r in range(n_runs)]


def arrivals(rng, total: int, n=None):
    """An arrival batch of distinct keys in random order: its flush is exactly as large as the batch."""
    ents = sized_entries(rng, total, n or n_entries_for(total))
    rng.shuffle(ents)
    return sstable.build_run(ents)


def to_dev(a: np.ndarray):
    return torch.from_numpy(np.ascontiguousarray(a, np.uint8)).to("cuda:0")


def dev_runs(runs, keep):
    """Runs copied to fresh device buffers (512-aligned): (data_ptr, data_len, index_ptr, index_len) per run."""
    ptrs = []
    for d, i in runs:
        td, ti = to_dev(np.concatenate([d, np.zeros(16, np.uint8)])), to_dev(np.concatenate([i, np.zeros(16, np.uint8)]))
        keep += [td, ti]
        ptrs.append((td.data_ptr(), d.size, ti.data_ptr(), i.size))
    torch.cuda.synchronize()
    return ptrs


def poison(kind: str, n: int) -> np.ndarray:
    if kind == "zeros":
        return np.zeros(n, np.uint8)
    if kind == "ones":
        return np.full(n, 0xFF, np.uint8)
    e = sstable.encode_entry(b"\x00poison", b"P" * 21, BASE_TS)  # a decodable 64-byte entry, over and over
    return np.frombuffer((e * (n // len(e) + 1))[:n], np.uint8).copy()


def placed_runs(runs, shift: int, kind: str, keep):
    """Every run's .data at byte offset 64 + shift of its allocation with poison before and after it; its .index (16-byte
    aligned) followed by a copy of its last record, which a kernel that reads one record too many would take as a
    duplicate key."""
    ptrs = []
    for d, i in runs:
        pre = 64 + shift
        td = to_dev(np.concatenate([poison(kind, pre), d, poison(kind, 64)]))
        ti = to_dev(np.concatenate([i, i[-16:]]))
        keep += [td, ti]
        ptrs.append((td.data_ptr() + pre, d.size, ti.data_ptr(), i.size))
    torch.cuda.synchronize()
    return ptrs


def raises(code: int, fn, *args, **kw):
    with pytest.raises(capi.DbeelError) as ei:
        fn(*args, **kw)
    assert ei.value.code == code, str(ei.value)


# ---------------------------------------------------------------------------------------------------------- the helper


def test_guards_catch_one_byte_on_either_side():
    """The check fails for a single byte written into the front guard, into the back guard, and (where nothing may be
    written) into the buffer itself; it passes on an untouched allocation."""
    for off in OFFSETS:
        g = Guarded(100, off, seed=off)
        assert (g.ptr - off) % 256 == 0
        g.check("untouched")
        g.check("untouched", untouched_from=0)
        for pos in (-1, -g.start, g.n, g.n + g.BACK - 1):
            g.t[g.start + pos] ^= 0x5A
            with pytest.raises(AssertionError, match=f"buffer\\[{pos}\\.\\.{pos}\\]"):
                g.check(f"byte {pos}")
            g.t[g.start + pos] ^= 0x5A
            g.check("restored")
        g.t[g.start + 40] ^= 1
        g.check("inside the buffer")
        with pytest.raises(AssertionError, match="at or past the end"):
            g.check("nothing may be written", untouched_from=0)
        with pytest.raises(AssertionError):
            g.check("nothing past byte 40", untouched_from=40)
        g.check("bytes before 41 may change", untouched_from=41)


# ------------------------------------------------------------------------------------------------------ compactions

# (runs, .data bytes): every residue mod 16, k * 8192 - 1, k * 8192 and k * 8192 + 1..16, a few megabytes
COMPACT_CASES = ([((1, 2, 9, 40)[r % 4], 4000 + r) for r in range(16)]
                 + [((1, 2, 9, 40)[j % 4], k * TILE + d) for k in (1, 3) for j, d in enumerate((-1, 0, 1, 7, 15, 16))]
                 + [(9, 5 * (1 << 20) + 3), (40, 3 * (1 << 20) + TILE - 1)])


@pytest.mark.parametrize("case", range(len(COMPACT_CASES)))
def test_compact_device_fills_exact_caps(engine, case):
    """dbeel_compact_device with data / index / bloom caps from dbeel_compact_bound and an output of exactly that size
    (distinct keys, tombstones kept): one run (five kernels), 2 and 9 runs (k_merge_final), 40 runs; every second case with
    a filter; both readers."""
    n_runs, total = COMPACT_CASES[case]
    rng = np.random.default_rng(1000 + case)
    runs = sized_runs(rng, total, n_runs)
    keep = []
    ptrs = dev_runs(runs, keep)
    bloom_min = 1 if case % 2 else 1 << 62
    exp = oracle.compact(runs, keep_tombstones=True, bloom_min_size=bloom_min, seed=SEED)
    for flags in (0, capi.FLAG_REFERENCE_READER):
        opts = capi.make_opts(True, bloom_min, seed=SEED, flags=flags)
        dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], opts)
        assert dc == total and (bc > 0) == bool(case % 2)
        od, oi, ob = outs((dc, ic, bc), case + flags, seed=case)
        dl, il, bl, n = engine.compact_device(ptrs, (od.ptr, dc, oi.ptr, ic, ob.ptr, bc), opts)
        what = f"{n_runs} runs, {total} bytes, flags {flags}"
        assert (dl, il, bl) == (dc, ic, bc) and n == exp[3], what
        for g, name in ((od, ".data"), (oi, ".index"), (ob, ".bloom")):
            g.check(f"{what}: {name}")
        assert_run_equal((od.bytes(), oi.bytes()), exp[:2], what)
        if bc:
            assert np.array_equal(ob.bytes(), exp[2]), f"{what}: .bloom differs"


@pytest.mark.parametrize("seed", range(3))
def test_compact_many_device_jobs_abut(engine, seed):
    """dbeel_compact_many_device: the jobs' outputs lie back to back in one stream with caps from
    dbeel_compact_many_bound, so an overrun of one job shows up as a corrupted neighbour."""
    rng = np.random.default_rng(2000 + seed)
    sizes = [int(rng.integers(2500, 5000)) for _ in range(5)] + [TILE - 1, TILE + 5, 2 * TILE + 16]
    if seed == 2:
        sizes.append(2 * (1 << 20) + 9)
    rng.shuffle(sizes)
    jobs = [(sized_runs(rng, s, int(rng.choice([1, 2, 5, 9]))), j % 4 != 3) for j, s in enumerate(sizes)]
    seeds = [bytes([(11 * j + k) % 256 for k in range(32)]) for j in range(len(jobs))]
    bloom_min = 4000
    hold = []
    ptrs = [(dev_runs(runs, hold), k) for runs, k in jobs]
    arr, _keep = capi.Engine._jobs_array(ptrs, seeds)
    dc, ic, bc = C.c_uint64(), C.c_uint64(), C.c_uint64()
    assert capi.lib().dbeel_compact_many_bound(arr, len(jobs), bloom_min, capi.DEFAULT_BLOOM_FP, C.byref(dc), C.byref(ic),
                                               C.byref(bc)) == 0
    assert dc.value == sum(sizes)
    od, oi, ob = outs((dc.value, ic.value, bc.value), seed, seed=50 + seed)
    rows = engine.compact_many_device(ptrs, (od.ptr, dc.value, oi.ptr, ic.value, ob.ptr, bc.value), bloom_min, seeds)
    for g, name in ((od, ".data"), (oi, ".index"), (ob, ".bloom")):
        g.check(f"compact-many {seed}: {name}")
    d_all, i_all, b_all = od.bytes(), oi.bytes(), ob.bytes()
    pos = 0
    for j, ((runs, keep_t), r) in enumerate(zip(jobs, rows)):
        ed, ei, eb, en = oracle.compact(runs, keep_tombstones=keep_t, bloom_min_size=bloom_min, seed=seeds[j])
        assert r["data_off"] == pos and r["items_written"] == en, f"job {j}"
        if keep_t:
            assert r["data_len"] == sizes[j], f"job {j}"
        pos += r["data_len"]
        assert_run_equal((d_all[r["data_off"]:pos], i_all[r["index_off"]:r["index_off"] + r["index_len"]]), (ed, ei), f"job {j}")
        assert (eb is None) == (r["bloom_len"] == 0), f"job {j}"
        if eb is not None:
            assert np.array_equal(b_all[r["bloom_off"]:r["bloom_off"] + r["bloom_len"]], eb), f"job {j}: .bloom"


# ----------------------------------------------------------------------------------------------------------- flushes

FLUSH_TOTALS = [3000 + r for r in range(16)] + [k * TILE + d for k in (1, 2) for d in (-1, 0, 1, 8, 16)] + [4 * (1 << 20) + 11]


@pytest.mark.parametrize("total", FLUSH_TOTALS)
def test_flush_device_fills_exact_caps(engine, total):
    rng = np.random.default_rng(total)
    batch = arrivals(rng, total)
    (ed, ei, en), = oracle.memtable_flushes(batch, capacity=1 << 20)
    hold = []
    (ptr,) = dev_runs([batch], hold)
    od, oi = outs((batch[0].size, batch[1].size), total, seed=total)
    dl, il, n = engine.flush_device(ptr, (od.ptr, od.n, oi.ptr, oi.n))
    assert (dl, il, n) == (total, batch[1].size, en)
    od.check(f"flush of {total} bytes: .data")
    oi.check(f"flush of {total} bytes: .index")
    assert_run_equal((od.bytes(), oi.bytes()), (ed, ei), f"flush of {total} bytes")


def _check_flush_rows(rows, od, oi, expect, what):
    d_all, i_all = od.bytes(), oi.bytes()
    pos = 0
    for k, (r, (ed, ei, en)) in enumerate(zip(rows, expect)):
        assert r["data_off"] == pos and r["items"] == en, f"{what}: memtable {k}"
        pos += r["data_len"]
        assert_run_equal((d_all[r["data_off"]:pos], i_all[r["index_off"]:r["index_off"] + r["index_len"]]), (ed, ei),
                         f"{what}: memtable {k}")
    assert pos == od.n


@pytest.mark.parametrize("seed", range(3))
def test_flush_many_device_fills_exact_caps(engine, seed):
    """dbeel_flush_many_device (otherwise only exercised inside the cfg5 pipeline): memtables of distinct keys, caps equal
    to the batches' sums, so the SSTables fill the buffers to the last byte."""
    rng = np.random.default_rng(3000 + seed)
    sizes = [int(rng.integers(2000, 6000)) for _ in range(6)] + [TILE - 1, TILE + 1, 3 * TILE + 13]
    if seed == 1:
        sizes.append(3 * (1 << 20) + 5)
    rng.shuffle(sizes)
    batches = [arrivals(rng, s) for s in sizes]
    expect = [oracle.memtable_flushes(b, capacity=1 << 20)[0] for b in batches]
    hold = []
    ptrs = dev_runs(batches, hold)
    od, oi = outs((sum(sizes), sum(b[1].size for b in batches)), seed, seed=60 + seed)
    dl, il, n, rows = engine.flush_many_device(ptrs, (od.ptr, od.n, oi.ptr, oi.n))
    od.check("flush-many: .data")
    oi.check("flush-many: .index")
    assert (dl, il) == (od.n, oi.n)
    _check_flush_rows(rows, od, oi, expect, "flush-many")


def _sparse_batches(rng, sizes):
    """Memtables whose index records are slices of one shared arrival buffer, interleaved the way a routed stream's are:
    (shared .data, [index slice per memtable], expected flush per memtable)."""
    per = [sized_entries(rng, s, n_entries_for(s)) for s in sizes]
    order = np.concatenate([np.full(len(p), b) for b, p in enumerate(per)])
    rng.shuffle(order)
    it = [iter(p) for p in per]
    data, index = sstable.build_run([next(it[b]) for b in order])
    recs = index.reshape(-1, 16)
    slices = [np.ascontiguousarray(recs[order == b]).reshape(-1) for b in range(len(sizes))]
    expect = [oracle.memtable_flushes(sstable.build_run(sstable.parse_run(data, s)), capacity=1 << 20)[0] for s in slices]
    return data, slices, expect


def _dev_sparse(data, slices, hold):
    td = to_dev(np.concatenate([poison("entry", 37), data, poison("entry", 64)]))
    ti = to_dev(np.concatenate([np.concatenate(slices), np.zeros(16, np.uint8)]))
    hold += [td, ti]
    torch.cuda.synchronize()
    base, ptrs = ti.data_ptr(), []
    for s in slices:
        ptrs.append((td.data_ptr() + 37, data.size, base, s.size))
        base += s.size
    return ptrs


@pytest.mark.parametrize("seed", range(2))
def test_flush_many_sparse_device_fills_exact_bound(engine, seed):
    rng = np.random.default_rng(4000 + seed)
    sizes = [int(rng.integers(1500, 5000)) for _ in range(7)] + [TILE + 3, 2 * TILE - 1]
    data, slices, expect = _sparse_batches(rng, sizes)
    hold = []
    ptrs = _dev_sparse(data, slices, hold)
    bound = sum(sizes)
    od, oi = outs((bound, sum(s.size for s in slices)), seed, seed=70 + seed)
    _, _, _, rows = engine.flush_many_sparse_device(ptrs, bound, (od.ptr, bound, oi.ptr, oi.n))
    od.check("sparse flush: .data")
    oi.check("sparse flush: .index")
    _check_flush_rows(rows, od, oi, expect, "sparse flush")


# (payload bound, true payload): the bound is not a multiple of the gather tile, the payload runs past the next tile edge
TOO_LOW = [(3 * TILE + 100, 5 * TILE + 100), (TILE + 1, 3 * TILE + 5), (2 * TILE - 16, 4 * TILE)]


@pytest.mark.parametrize("bound,total", TOO_LOW)
def test_flush_many_sparse_device_too_low_bound_writes_nothing_past_it(engine, bound, total):
    """A payload bound below the bytes the memtables hold: DBEEL_ERR_CAPACITY, and with out->data_cap == the bound not
    one byte at or past it may change ("nothing is written past it")."""
    assert bound % TILE and total > (bound // TILE + 1) * TILE
    rng = np.random.default_rng(bound)
    third = total // 3
    data, slices, _ = _sparse_batches(rng, [third, third, total - 2 * third])
    hold = []
    ptrs = _dev_sparse(data, slices, hold)
    od, oi = Guarded(bound, 16, seed=1), Guarded(sum(s.size for s in slices), 48, seed=2)
    raises(capi.ERR_CAPACITY, engine.flush_many_sparse_device, ptrs, bound, (od.ptr, bound, oi.ptr, oi.n))
    od.check(f"payload bound {bound} < {total}: .data")
    oi.check(f"payload bound {bound} < {total}: .index")


# --------------------------------------------------------------------------------------------------------------- WAL


@pytest.mark.parametrize("total", [3000, 3001, 3007, 3013, TILE - 1, TILE, TILE + 1, 2 * TILE + 9, 2 * (1 << 20) + 3])
def test_wal_flush_device_fills_exact_caps(engine, total):
    """Caps as the header gives them: the sum of the logged entries' sizes and 16 bytes per logged entry."""
    rng = np.random.default_rng(5000 + total)
    ents = sized_entries(rng, total, min(400, n_entries_for(total)))
    rng.shuffle(ents)
    wal = sstable.build_wal(ents, pad_byte=0xA5)
    ed, ei, en, _ = oracle.wal_flush(wal)
    d_wal = to_dev(np.concatenate([wal, poison("entry", 4096)]))
    od, oi = outs((total, 16 * len(ents)), total, seed=total)
    dl, il, n = engine.wal_flush_device(d_wal.data_ptr(), wal.size, (od.ptr, od.n, oi.ptr, oi.n))
    assert (dl, il, n) == (total, 16 * len(ents), en)
    od.check(f"log of {total} bytes: .data")
    oi.check(f"log of {total} bytes: .index")
    assert_run_equal((od.bytes(), oi.bytes()), (ed, ei), f"log of {total} bytes")


# -------------------------------------------------------------------------------------------------------------- scan


def _scan_device(engine, ptrs, ranges, od, oi, kind=capi.SCAN_HASH):
    return engine.scan_device(ptrs, ranges, (od.ptr, od.n, oi.ptr, oi.n), kind)


def _check_scan(rows, stop, exp, od, oi, what):
    assert stop == exp[1], what
    d_all, i_all = od.bytes(), oi.bytes()
    for j, (r, e) in enumerate(zip(rows, exp[0])):
        assert_run_equal((d_all[r["data_off"]:r["data_off"] + r["data_len"]], i_all[r["index_off"]:r["index_off"] + r["index_len"]]),
                         e, f"{what}: destination {j}")


@pytest.mark.parametrize("total", [4000 + r for r in range(0, 16, 3)] + [TILE - 1, TILE, TILE + 16, 3 * TILE + 1, 3 * (1 << 20) + 7])
def test_scan_device_fills_exact_caps(engine, total):
    """Caps from dbeel_scan_bound and ranges that take every entry: the destinations fill both buffers exactly."""
    rng = np.random.default_rng(6000 + total)
    tables = sized_runs(rng, total, int(rng.choice([1, 3, 8])))
    exp = scan_oracle.scan(tables, ALL_HASHES)
    hold = []
    ptrs = dev_runs(tables, hold)
    od, oi = outs((total, sum(i.size for _, i in tables)), total, seed=total)
    rows, stop = _scan_device(engine, ptrs, ALL_HASHES, od, oi)
    od.check(f"scan of {total} bytes: .data")
    oi.check(f"scan of {total} bytes: .index")
    assert sum(r["data_len"] for r in rows) == total
    _check_scan(rows, stop, exp, od, oi, f"scan of {total} bytes")


def test_scan_device_capacity_error_writes_nothing(engine):
    """DBEEL_ERR_CAPACITY, nothing written: a cap one byte short, and an output larger than dbeel_scan_bound (index records
    that share .data bytes) -- both buffers keep every byte."""
    rng = np.random.default_rng(61)
    tables = sized_runs(rng, 3 * TILE + 5, 3)
    hold = []
    ptrs = dev_runs(tables, hold)
    dsum, isum = sum(d.size for d, _ in tables), sum(i.size for _, i in tables)
    for dc, ic in ((dsum - 1, isum), (dsum, isum - 16)):
        od, oi = Guarded(dc, 16, seed=3), Guarded(ic, 48, seed=4)
        raises(capi.ERR_CAPACITY, _scan_device, engine, ptrs, ALL_HASHES, od, oi)
        od.check("scan cap short: .data", untouched_from=0)
        oi.check("scan cap short: .index", untouched_from=0)
    # one 200 KB entry listed six times: the output is several tiles larger than the bound
    big = sstable.build_run([(b"a", b"x" * 9, BASE_TS), (b"big", bytes(range(256)) * 800, BASE_TS), (b"z", b"y" * 3, BASE_TS)])
    recs = big[1].reshape(-1, 16)
    idx = np.concatenate([recs[:1]] + [recs[1:2]] * 6 + [recs[2:]]).reshape(-1).copy()
    ptrs = dev_runs([(big[0], idx)], hold)
    od, oi = Guarded(big[0].size, 0, seed=5), Guarded(idx.size, 16, seed=6)
    raises(capi.ERR_CAPACITY, _scan_device, engine, ptrs, [(1, 0)], od, oi)
    od.check("overlapping records: .data", untouched_from=0)
    oi.check("overlapping records: .index", untouched_from=0)


# ------------------------------------------------------------------------------------------------------------ routing


@pytest.mark.parametrize("n,n_shards", [(1, 8), (257, 3), (5000, 8), (20_000, 64)])
def test_route_device_exact_index_cap(engine, n, n_shards):
    rng = np.random.default_rng(n)
    batch = W.make_arrival_batch(n_writes=n, n_ids=max(64, n // 3), doc_bytes=int(rng.integers(20, 90)), seed=n)
    ring, _ = oracle.shard_ring(n_shards)
    exp_shard, _ = oracle.route(batch, ring)
    hold = []
    for k, kind in enumerate(POISONS):
        (ptr,) = placed_runs([batch], 2 * k + 7, kind, hold)
        out, owner, h64 = outs((16 * n, 4 * n, 8 * n), k, seed=n + 10 * k)
        counts, _ = engine.route_device(ptr, ring, out.ptr, out.n, owner.ptr, h64.ptr)
        for g, name in ((out, "routed index"), (owner, "shard_of"), (h64, "key hash64")):
            g.check(f"route {n} arrivals to {n_shards}: {name}")
        assert np.array_equal(owner.bytes().view(np.uint32), exp_shard)
        recs = batch[1].reshape(-1, 16)
        order = np.concatenate([np.flatnonzero(exp_shard == s) for s in range(n_shards)])
        assert np.array_equal(out.bytes().reshape(-1, 16), recs[order])
        assert list(counts) == [int((exp_shard == s).sum()) for s in range(n_shards)]
        ents = sstable.parse_run(*batch)
        keys = [ents[j][0] for j in order]
        ident = {}
        for key, h in zip(keys, h64.bytes().view(np.uint64).tolist()):
            assert ident.setdefault(key, h) == h, "one key, two identities"
        assert len(set(ident.values())) == len(ident), "two keys, one identity"


# ------------------------------------------------------------------------------------------------------ placed inputs


@pytest.mark.parametrize("shift", SHIFTS)
def test_inputs_placed_at_any_byte_with_poison_around(engine, shift):
    """Every run's .data at byte offset `shift` (mod 16 and a few odd ones), with 0x00, 0xFF or decodable-entry poison before
    and after it and a copy of its last index record behind its .index: compaction (with DBEEL_FLAG_VERIFY_SORTED, which
    turns one record too many into DBEEL_ERR_UNSORTED_RUN, and with the reference reader), flush, scan and lookups all
    equal the oracle."""
    rng = np.random.default_rng(7000 + shift)
    runs = sized_runs(rng, 3000 + 7 * shift, 3)
    batch = W.make_arrival_batch(n_writes=300, n_ids=120, doc_bytes=33 + shift, seed=shift)
    table = oracle.compact(runs, keep_tombstones=True, bloom_min_size=1, seed=SEED)
    present = [k for k, _, _ in sstable.parse_run(table[0], table[1])]
    keys = present[::2] + [k + b"\x00" for k in present[:20]] + [b"", b"\xff" * 30, b"zz"]
    blob, koff = capi.pack_keys(keys)
    d_keys, d_koff = to_dev(np.concatenate([blob, np.zeros(16, np.uint8)])), torch.from_numpy(koff.view(np.int64)).to("cuda:0")
    et, er, ej = oracle.get_many([table[:3]], blob, koff)
    for k, kind in enumerate(POISONS):
        what = f"shift {shift}, {kind} poison"
        hold = []
        ptrs = placed_runs(runs, shift, kind, hold)
        bloom_min = 1 if k == 1 else 1 << 62
        exp = oracle.compact(runs, keep_tombstones=True, bloom_min_size=bloom_min, seed=SEED)
        for flags in (capi.FLAG_VERIFY_SORTED, capi.FLAG_VERIFY_SORTED | capi.FLAG_REFERENCE_READER):
            opts = capi.make_opts(True, bloom_min, seed=SEED, flags=flags)
            dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], opts)
            od, oi, ob = outs((dc, ic, bc), shift + k, seed=k)
            dl, il, bl, n = engine.compact_device(ptrs, (od.ptr, dc, oi.ptr, ic, ob.ptr, bc), opts)
            for g, name in ((od, ".data"), (oi, ".index"), (ob, ".bloom")):
                g.check(f"{what}, flags {flags}: {name}")
            assert (dl, n) == (dc, exp[3])
            assert_run_equal((od.bytes(), oi.bytes()), exp[:2], f"{what}, flags {flags}")
            if bc:
                assert np.array_equal(ob.bytes(), exp[2]), f"{what}: .bloom"

        (bptr,) = placed_runs([batch], shift, kind, hold)
        (ed, ei, en), = oracle.memtable_flushes(batch, capacity=1 << 20)
        od, oi = outs((batch[0].size, batch[1].size), shift + k + 1, seed=k)
        dl, il, n = engine.flush_device(bptr, (od.ptr, od.n, oi.ptr, oi.n))
        od.check(f"{what}: flush .data")
        oi.check(f"{what}: flush .index")
        assert n == en
        assert_run_equal((od.bytes(0, dl), oi.bytes(0, il)), (ed, ei), f"{what}: flush")

        od, oi = outs((sum(d.size for d, _ in runs), sum(i.size for _, i in runs)), shift + k + 2, seed=k)
        rows, stop = _scan_device(engine, ptrs, ALL_HASHES, od, oi)
        od.check(f"{what}: scan .data")
        oi.check(f"{what}: scan .index")
        _check_scan(rows, stop, scan_oracle.scan(runs, ALL_HASHES), od, oi, f"{what}: scan")

        # the compacted table at the same offset, its filter 4-byte aligned; the result rows guarded
        (tptr,) = placed_runs([table[:2]], shift, kind, hold)
        tb = to_dev(np.concatenate([poison(kind, 4 * (1 + shift % 4)), table[2], poison(kind, 64)]))
        hold.append(tb)
        torch.cuda.synchronize()
        dev_table = (tptr[0], tptr[1], tptr[2], tptr[3], tb.data_ptr() + 4 * (1 + shift % 4), table[2].size)
        for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
            res = Guarded(16 * len(keys), OFFSETS[(shift + k + mode) % 3], seed=k)
            engine.get_many_device([dev_table], d_keys.data_ptr(), d_koff.data_ptr(), len(keys), res.ptr, mode)
            res.check(f"{what}: lookup results, mode {mode}")
            got = res.bytes().view(capi.LOOKUP_DTYPE)
            if mode == capi.LOOKUP_REFERENCE:
                assert np.array_equal(got["table"], et) and np.array_equal(got["bloom_rejects"], ej), what
                assert np.array_equal(np.where(got["table"] >= 0, got["record"], 0), er), what
            else:
                assert np.array_equal(got, engine.get_many([table[:3]], keys, mode)), what
