"""Every read entry point on a table past 2^32 records: record numbers, .data offsets and .index offsets with a nonzero
high word, in the searches, the leaf plans, the page cache and the results.

T_big (tests/reads_model.py) has N_BIG = 2^32 + 2^20 + 3 records of 48 bytes: 192 GiB of .data and 64 GiB of .index
that exist only as a read callback.  Record r holds key be64(2r + 1) and value le64(r) at .data offset 48 r, so
records 89478486 on have a .data offset past 2^32, records 2^28 on an .index offset past 2^32, and records 2^32 on a
record number past 2^32.  Point reads and range reads touch only fences, leaves and spans, so each call synthesises a
few hundred MB at most.  T_new is a small real table with newer versions (some tombstones) of records 2^32 - 2 ..
2^32 + 2, 2^32 + 2^19 - 1 .. 2^32 + 2^19 + 1 and N_BIG - 1, and new keys between T_big's.  T_bad is T_big with
scan_cases.damage's offset_eof defect at D1 = 2^32 + 12345 and its timestamp defect at D2 = 2^32 + 2^19 + 7.

Every result is compared with the closed-form model (rows, record numbers, entry bytes, stops), which
tests/test_reads_past_4gib_model.py checks against the oracles on materialised tables; equality between entry points is
an extra check.

The run-A tests at the end read real bytes back past 4 GiB: outputs of 4.8 GB whose .index offsets pass 2^32, compared
with the source bytes of run A (test_gpu_past_4gib.build_a).
"""
import resource
import threading
import time
from collections import Counter

import numpy as np
import pytest
import torch

import reads_model as M
from dbeel_b200 import capi, sstable
from scan_cases import ERR, PANIC
from test_gpu_reader import fence_positions
from test_gpu_reader_get_ranges import entries_of

pytestmark = pytest.mark.gpu

MODES = (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT)
N, T32 = M.N_BIG, M.TWO32
D1, D2 = T32 + 12345, T32 + (1 << 19) + 7
STRADDLE = [T32 // M.ENT, (1 << 33) // M.ENT]   # the records whose .data bytes cross 2^32 and 2^33
NEW_AT = [T32 - 2, T32 - 1, T32, T32 + 1, T32 + 2, T32 + (1 << 19) - 1, T32 + (1 << 19), T32 + (1 << 19) + 1, N - 1]
BETWEEN = [T32, T32 + 2, T32 + (1 << 19) + 3, N - 1]   # T_new's own keys: be64(2r), just below record r
EDGE = [0, 1, 2, (1 << 28) - 1, 1 << 28, STRADDLE[0] - 1, STRADDLE[0], STRADDLE[0] + 1, STRADDLE[1], STRADDLE[1] + 1,
        T32 - 3] + NEW_AT + [N - 2]
CACHE_BYTES = 64 << 20


@pytest.fixture(autouse=True)
def footprint(request):
    """Wall time, peak device memory in use (sampled every 20 ms) and peak host RSS of every test."""
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    peak = [total - free0]
    done = threading.Event()

    def sample():
        while not done.wait(0.02):
            peak[0] = max(peak[0], total - torch.cuda.mem_get_info()[0])
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    t0 = time.monotonic()
    yield
    done.set()
    th.join()
    print(f"\n[footprint] {request.node.name}: {time.monotonic() - t0:.1f} s, device memory in use at most "
          f"{peak[0] / 2**30:.2f} GiB (at start {(total - free0) / 2**30:.2f} GiB), "
          f"host max RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GiB")


@pytest.fixture(scope="module")
def env():
    ents = [(M.key_of(r), b"" if j % 3 == 1 else b"new-%d" % r, M.BIG_TS + 1 + j) for j, r in enumerate(NEW_AT)]
    ents += [(M.miss_below(r), b"between-%d" % r, M.BIG_TS + 7) for r in BETWEEN]
    nd, ni = sstable.build_run(sorted(ents))
    big, bad, new = M.SynTable(), M.SynTable(defects={D1: "offset_eof", D2: "timestamp"}), M.MemTable(nd, ni)

    def serve(*tables):
        return lambda t, kind, off, size: tables[t].read(kind, off, size)
    return {"big": big, "bad": bad, "new": new, "nd": nd, "ni": ni, "serve": serve,
            "files": lambda *ts: [(t.data_len, t.index_len, None) for t in ts]}


def batch(seed: int, n_random: int = 60):
    """About 130 keys in random order: the EDGE records, n_random records spread over the table, the misses just below
    and just above each edge record, and keys no record can hold."""
    rng = np.random.default_rng(seed)
    rs = EDGE + [int(x) for x in rng.integers(0, N, n_random)]
    keys = [M.key_of(r) for r in rs] + sorted({M.miss_below(r) for r in EDGE} | {M.miss_below(r + 1) for r in EDGE}) + [b"", b"\xff" * 9, M.key_of(T32)[:7]]
    return [keys[j] for j in rng.permutation(len(keys))]


def check_values(what, got, tables, keys, mode):
    """(rows, data, index) against the model; at least one row names a record past 2^32."""
    rows, d, i = got
    w = M.get_values(tables, keys, mode)
    M.compare_rows(what, rows, w[0])
    M.compare_out(what, d, i, w[1], w[2])
    assert (w[0]["record"] >> 32).max() == 1, f"{what}: no record past 2^32 in the batch"
    return w


def test_get_values_stream(engine, env):
    """dbeel_get_values_stream on [T_big, T_new] in both modes: rows with records 2^32 - 3 .. 2^32 + 2^19 + 1 and
    N_BIG - 1 (high word 1), T_new's versions and tombstones over them, entries read at .data offsets past 2^33; and on
    T_bad, D2's key answered with LOOKUP_BAD_ENTRY at record D2 and D1's key a miss, as the model says."""
    big, new, bad = env["big"], env["new"], env["bad"]
    keys = batch(1)
    for mode in MODES:
        got = engine.get_values_stream(env["files"](big, new), keys, mode, read=env["serve"](big, new))
        check_values(f"stream mode {mode}", got, [big, new], keys, mode)
        reads = engine.last_stream_reads
        assert any(k == 1 and t == 0 and off > 1 << 33 for t, k, off, _ in reads)
        assert any(k == 2 and t == 0 and off > T32 for t, k, off, _ in reads)
        bkeys = keys[:40] + [M.key_of(r) for r in (D1, D2, D1 - 1, D2 + 1)]
        got = engine.get_values_stream(env["files"](bad), bkeys, mode, read=env["serve"](bad))
        w = check_values(f"stream T_bad mode {mode}", got, [bad], bkeys, mode)
        q = len(bkeys) - 3
        assert (int(w[0]["table"][q]), int(w[0]["bloom_rejects"][q]), int(w[0]["record"][q])) == (0, M.BAD_ENTRY, D2)


def _same(engine, reader, env, tables, keys, mode):
    """reader.get_values == the model == get_values_stream on the same tables."""
    got = reader.get_values(keys, mode)
    reads, st = reader.last_stream_reads, engine.stats()
    check_values(f"reader mode {mode}", got, tables, keys, mode)
    sr, sd, si = engine.get_values_stream(env["files"](*tables), keys, mode, read=env["serve"](*tables))
    assert np.array_equal(got[0], sr)
    M.compare_out("reader vs stream", got[1], got[2], sd, si)
    assert st["input_bytes"] == sum(r[3] for r in reads)
    return got, reads


def test_reader_two_batches_per_mode(engine, env):
    """A reader on [T_big, T_new]: T_big's fences go 16 levels deep (2^16 - 1 index records, the deepest ones past
    .index offset 2^32), the first batch loads them, a repeat of it reads the same less the fences, and a second batch
    reads no fence; every batch equals the model and get_values_stream."""
    big, new = env["big"], env["new"]
    assert M.reader_depths([big.n, new.n], [big.data_len, new.data_len])[0] == 16
    with engine.open_reader(env["files"](big, new), read=env["serve"](big, new)) as r:
        for mode in MODES:
            fences = fence_positions(mode, N, 16)
            assert max(fences) > 1 << 28
            k1, k2 = batch(10 + mode), batch(20 + mode)
            _, first = _same(engine, r, env, [big, new], k1, mode)
            _, again = _same(engine, r, env, [big, new], k1, mode)
            loads = Counter(first) - Counter(again)
            assert not Counter(again) - Counter(first)
            big_loads = [x for x in loads if x[0] == 0 and x[1] == 2]
            assert len(big_loads) > 30000, len(big_loads)
            for t, kind, off, size in big_loads:
                assert off % 16 == 0 and off // 16 in fences and (off + size) // 16 - 1 in fences, (off, size)
            _, second = _same(engine, r, env, [big, new], k2, mode)
            assert not [x for x in second if x[0] == 0 and x[1] == 2 and x[2] // 16 in fences]


def test_readers_get_values(engine, env):
    """dbeel_readers_get_values: a T_big batch (exact), a batch on a small in-memory reader (reference), a second T_big
    batch (reference).  Each batch equals its solo reader.get_values and the model."""
    big, new, nd, ni = env["big"], env["new"], env["nd"], env["ni"]
    small_keys = [k for k, _, _ in sstable.parse_run(nd, ni)] + [M.key_of(5), M.miss_below(T32 + 1)]
    with engine.open_reader(env["files"](big, new), read=env["serve"](big, new)) as rb, \
            engine.open_reader([(nd, ni, None)]) as rs:
        jobs = [(rb, batch(30), capi.LOOKUP_EXACT), (rs, small_keys, capi.LOOKUP_REFERENCE),
                (rb, batch(31), capi.LOOKUP_REFERENCE)]
        got = engine.readers_get_values(jobs)
        for j, ((rd, keys, mode), g) in enumerate(zip(jobs, got)):
            solo = rd.get_values(keys, mode)
            assert np.array_equal(g[0], solo[0]), f"batch {j}: rows differ from the solo call"
            M.compare_out(f"batch {j} vs solo", g[1], g[2], solo[1], solo[2])
            tables = [big, new] if rd is rb else [new]
            w = M.get_values(tables, keys, mode)
            M.compare_rows(f"batch {j}", g[0], w[0])
            M.compare_out(f"batch {j}", g[1], g[2], w[1], w[2])
        assert (got[0][0]["record"] >> 32).max() == 1 and (got[2][0]["record"] >> 32).max() == 1


def test_page_cache(engine, env):
    """A 64 MiB page cache on a reader of [T_big, T_new]: the same results as uncached, every read page-aligned, pages
    read past 2^32 in .data and .index, and a repeated batch of keys around record 2^32 and the last record reads
    nothing."""
    big, new = env["big"], env["new"]
    files = env["files"](big, new)
    with engine.open_page_cache(CACHE_BYTES) as cache, \
            engine.open_reader(files, read=env["serve"](big, new)) as r:
        for mode in MODES:
            r.attach_page_cache(None)
            _same(engine, r, env, [big, new], batch(40), mode)   # the fences, uncached
            r.attach_page_cache(cache)
            for seed in (40, 41):
                _, reads = _same(engine, r, env, [big, new], batch(seed), mode)
                for t, kind, off, size in reads:
                    flen = files[t][0] if kind == 1 else files[t][1]
                    assert off % 4096 == 0 and ((off + size) % 4096 == 0 or off + size == flen), (t, kind, off, size)
                assert any(t == 0 and k == 1 and off > T32 for t, k, off, _ in reads)
                assert any(t == 0 and k == 2 and off > T32 for t, k, off, _ in reads)
            few = [M.key_of(r_) for r_ in (T32 - 2, T32, T32 + 1, N - 1, N - 2)] + [M.miss_below(T32)]
            _same(engine, r, env, [big, new], few, mode)
            s0 = cache.stats()
            _, reads = _same(engine, r, env, [big, new], few, mode)
            assert reads == [] and cache.stats()["misses"] == s0["misses"]
        r.attach_page_cache(None)


SCAN_RANGES = [(M.key_of(T32 - 1000), M.miss_below(T32 - 2)), (M.miss_below(T32 - 2), M.key_of(T32 + 3)),
               (M.key_of(T32 + 3), M.key_of(T32 + 1000)), (M.key_of(N - 300), b"\xff" * 9)]


def test_reader_scan(engine, env):
    """dbeel_reader_scan (SCAN_KEY) over records 2^32 - 1000 .. 2^32 + 999 in three ranges and the last 300 records: the
    entries the model writes, entries_in = the span records.  On T_bad a range over D1 stops at (0, PANIC, D1) and one
    over D2 at (0, ERR, D2), each record past 2^32."""
    big, bad = env["big"], env["bad"]
    with engine.open_reader(env["files"](big), read=env["serve"](big)) as r:
        for _ in range(2):
            out, stop = r.scan(SCAN_RANGES)
            st = engine.stats()
            want, wstop, n_span = M.reader_scan(big, SCAN_RANGES)
            M.compare_stop("scan", stop, wstop)
            for d, (g, w) in enumerate(zip(out, want)):
                M.compare_out(f"scan range {d}", g[0], g[1], w[0], w[1])
            assert st["entries_in"] == n_span == 2300
    with engine.open_reader(env["files"](bad), read=env["serve"](bad)) as r:
        for rg, want_stop in (((D1 - 500, D1 + 500), (0, PANIC, D1)), ((D2 - 500, D2 + 500), (0, ERR, D2)),
                              ((D1 - 100, D1 + 1), (0, PANIC, D1)), ((D2, D2 + 100), (0, ERR, D2))):
            ranges = [(M.key_of(rg[0]), M.key_of(rg[1]))]
            want, wstop, _ = M.reader_scan(bad, ranges)
            assert wstop == want_stop
            out, stop = r.scan(ranges)
            M.compare_stop(f"scan T_bad {rg}", stop, want_stop)
            M.compare_out(f"scan T_bad {rg}", out[0][0], out[0][1], want[0][0], want[0][1])


GET_RANGES = [(M.key_of(T32 - 10), M.key_of(T32 + 10)), (M.key_of(T32 + (1 << 19) - 5), M.key_of(T32 + (1 << 19) + 5)),
              (M.key_of(N - 10), b"\xff" * 9)]


def test_reader_get_range(engine, env):
    """dbeel_reader_get_range on [T_big, T_new]: per range the newest version of every key (T_new's over records 2^32 - 2
    .. 2^32 + 2 and the last record, its keys between T_big's), tombstones dropped or kept.  On T_bad the stop is the
    scan's, (0, PANIC, D1) and (0, ERR, D2)."""
    big, new, bad = env["big"], env["new"], env["bad"]
    with engine.open_reader(env["files"](big, new), read=env["serve"](big, new)) as r:
        for keep in (False, True):
            out, stop = r.get_range(GET_RANGES, keep_tombstones=keep)
            M.compare_stop("get_range", stop, (-1, 0, 0))
            for d, rg in enumerate(GET_RANGES):
                g, _ = M.get_range([big, new], rg, keep)
                assert len(g) > 5
                M.compare_out(f"get_range {d} keep={keep}", out[d][0], out[d][1], *M.pack(g))
    with engine.open_reader(env["files"](bad), read=env["serve"](bad)) as r:
        for rg, want in (((D1 - 50, D1 + 50), (0, PANIC, D1)), ((D2 - 50, D2 + 50), (0, ERR, D2))):
            out, stop = r.get_range([(M.key_of(rg[0]), M.key_of(rg[1]))])
            M.compare_stop(f"get_range T_bad {rg}", stop, want)
            assert all(o[0].size == 0 and o[1].size == 0 for o in out)


LIMITED = [(M.key_of(T32 - 3), M.key_of(T32 + 500)), (M.key_of(T32 - 1500), M.key_of(T32 + 5)),
           (M.miss_below(T32), M.key_of(T32 + 2)), (M.key_of(T32 + (1 << 19) - 20), M.key_of(T32 + (1 << 19) + 20)),
           (M.key_of(N - 2000), b"\xff" * 9), (M.key_of(T32 + 7), M.key_of(T32 + 7))]


@pytest.mark.parametrize("reverse", [False, True])
def test_reader_get_ranges(engine, env, reverse):
    """dbeel_reader_get_ranges(_reverse) with limits 1, 7 and 1000 on ranges that start or end at records 2^32 +- k (the
    reverse chunks of range 1 double downward across record 2^32, through T_new's tombstones): rows (first, count,
    MORE) and bytes equal the model.  On T_bad, the rows over D1 and D2 follow the damage rule, and some stop at
    exactly D1 (PANIC) and D2 (ERR)."""
    big, new, bad = env["big"], env["new"], env["bad"]
    with engine.open_reader(env["files"](big, new), read=env["serve"](big, new)) as r:
        for limit in (1, 7, 1000):
            for keep in (False, True):
                rows, data, index = r.get_ranges(LIMITED, limit, keep_tombstones=keep, reverse=reverse)
                first = 0
                for q, (rg, row) in enumerate(zip(LIMITED, rows)):
                    assert int(row["first"]) == first
                    first += int(row["count"])
                    assert M.check_limited_row([big, new], rg, limit, keep, reverse, row, entries_of(data, index, row)) is None
                assert index.size == 16 * first
    stops = set()
    dranges = [(M.key_of(a), M.key_of(b)) for a, b in ((D1 - 500, D1 + 500), (D1 - 100, D1 + 1), (D1 - 3, D1 + 3),
                                                       (D2 - 500, D2 + 500), (D2, D2 + 100), (D2 - 100, D2 + 1))]
    with engine.open_reader(env["files"](bad), read=env["serve"](bad)) as r:
        for limit in (1, 7, 1000):
            rows, data, index = r.get_ranges(dranges, limit, reverse=reverse)
            for rg, row in zip(dranges, rows):
                s = M.check_limited_row([bad], rg, limit, False, reverse, row, entries_of(data, index, row))
                if s is not None:
                    stops.add(s)
    assert (0, PANIC, D1) in stops and (0, ERR, D2) in stops, stops


# ------------------------------------------------------------------------------------------ run A: real bytes past 4 GiB
#
# Run A of test_gpu_past_4gib.py (4.83 GB of .data: small-entry clusters straddling 2^31 and 2^32, one entry starting
# 5 bytes before 2^32, 18 fillers of about 256 MiB none of which starts or ends on a 16-byte edge, filler words that hold
# their own position in .data).  Every batch lists the fillers first and cluster entries after them, so the outputs pass
# 4 GiB and the cluster entries' output .index offsets have a high word of 1.  The expected .data is A's source bytes,
# gathered lazily slice by slice; at most one large result is held at a time, and host-path calls run on engines of
# their own, closed after use, as an engine's partition stages only grow.

A_DEVICE_BYTES_NEEDED = 22 << 30   # measured peak 20.2 GiB: the 6 GiB page cache and an engine's stages over A
BIG_CACHE = 6 << 30                # holds all of A: slots past 2^20 put pool offsets past 2^32


class Gathered:
    """The concatenation of byte spans of `src`, sliced on demand (compare_data reads it 256 MiB at a time)."""

    def __init__(self, src, spans):
        self.src, self.spans = src, [(int(o), int(n)) for o, n in spans]
        self.starts = np.concatenate([[0], np.cumsum([n for _, n in self.spans], dtype=np.int64)])
        self.size = int(self.starts[-1])

    def __getitem__(self, s):
        lo, hi = s.start, min(s.stop, self.size)
        j = int(np.searchsorted(self.starts, lo, side="right")) - 1
        parts = []
        while lo < hi:
            o, n = self.spans[j]
            a = lo - int(self.starts[j])
            b = min(n, hi - int(self.starts[j]))
            parts.append(self.src[o + a:o + b])
            lo += b - a
            j += 1
        return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


@pytest.fixture(scope="module")
def run_a():
    from test_gpu_past_4gib import build_a
    free, _ = torch.cuda.mem_get_info(0)
    if free < A_DEVICE_BYTES_NEEDED:
        pytest.skip(f"needs {A_DEVICE_BYTES_NEEDED >> 30} GiB of free device memory, {free / 2**30:.1f} GiB free")
    a, marks = build_a(np.random.default_rng(4242))
    fl = marks["fillers"]
    cl = sorted(set(range(marks["straddle32"] - 30, marks["straddle32"] + 30)) | set(range(marks["straddle31"] - 5, marks["straddle31"] + 5)))
    misses = [a.keys[r] + b"\x00" for r in cl[::7]] + [a.keys[fl[3]] + b"\x00"]
    env = {"a": a, "marks": marks, "mem": M.MemTable(a.data, a.index), "pinned": torch.empty(256 << 20, dtype=torch.uint8, pin_memory=True),
           "keys": [a.keys[r] for r in fl] + [a.keys[r] for r in cl] + misses}
    assert sum(int(a.fs[r]) for r in fl) > T32 and len(fl) == 18
    yield env
    env.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def expect_values(env, keys, mode):
    """Model rows and the expected output: .index = running sums of full_size, .data = the answered records' bytes."""
    a = env["a"]
    rows, answered = M.lookup_rows([env["mem"]], keys, mode)
    recs = [r for _, r in answered]
    fs = a.fs[recs].astype(np.int64)
    idx = np.zeros((len(recs), 4), "<u4")
    idx[:, 0:2] = np.concatenate([[0], np.cumsum(fs)[:-1]]).astype("<u8").view("<u4").reshape(-1, 2)
    idx[:, 2] = [8 + len(a.keys[r]) for r in recs]
    idx[:, 3] = fs
    return rows, idx.view(np.uint8).reshape(-1), Gathered(a.data, [(a.off[r], a.fs[r]) for r in recs])


def check_a(what, rows, data_get, data_len, index, want):
    """Rows, .index and .data of one run-A result against expect_values; the .index holds offsets past 2^32."""
    from test_gpu_past_4gib import compare_data, compare_index
    M.compare_rows(what, rows, want[0])
    compare_index(what, index, want[1])
    offs = np.asarray(index).reshape(-1, 16)[:, :8].copy().view("<u8").ravel()
    assert data_len > T32 and int((offs >> np.uint64(32)).max()) == 1, f"{what}: the output does not pass 4 GiB"
    compare_data(what, data_get, want[2], data_len)


def test_run_a_get_values_and_get_values_device(run_a):
    """dbeel_get_values (A in host memory) and dbeel_get_values_device (A on the device), both modes: 18 fillers then the
    cluster entries around 2^31 and 2^32; the output passes 4 GiB and the cluster entries' offsets have high word 1."""
    from test_gpu_past_4gib import d2h
    a, keys = run_a["a"], run_a["keys"]
    eng = capi.Engine(0)
    try:
        for mode in MODES:
            want = expect_values(run_a, keys, mode)
            rows, d, i = eng.get_values([(a.data, a.index, None)], keys, mode)
            check_a(f"get_values mode {mode}", rows, lambda lo, hi: d[lo:hi], d.size, i, want)
            del d, i
    finally:
        eng.close()

    def dev(arr, extra=16):
        t = torch.empty(arr.size + extra, dtype=torch.uint8, device="cuda:0")
        for lo in range(0, arr.size, 256 << 20):
            t[lo:min(arr.size, lo + (256 << 20))].copy_(torch.from_numpy(arr[lo:lo + (256 << 20)]))
        t[arr.size:].zero_()
        return t
    eng = capi.Engine(0)
    try:
        ad, ai = dev(a.data), dev(a.index)
        blob, koff = capi.pack_keys(keys)
        dk, dko = dev(blob.copy()), torch.from_numpy(koff.view(np.int64)).to("cuda:0")
        res = torch.zeros(16 * len(keys), dtype=torch.uint8, device="cuda:0")
        cap = max(expect_values(run_a, keys, mode)[2].size for mode in MODES) + (1 << 20)
        out_d = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
        out_i = torch.empty(16 * len(keys), dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        for mode in MODES:
            want = expect_values(run_a, keys, mode)
            dl, il, items = eng.get_values_device([(ad.data_ptr(), a.data.size, ai.data_ptr(), a.index.size, 0, 0)], dk.data_ptr(),
                                                  dko.data_ptr(), len(keys), res.data_ptr(),
                                                  (out_d.data_ptr(), cap, out_i.data_ptr(), out_i.numel()), mode)
            torch.cuda.synchronize()
            rows = res.cpu().numpy().view(capi.LOOKUP_DTYPE)
            assert items == il // 16
            check_a(f"get_values_device mode {mode}", rows, lambda lo, hi: d2h(run_a, out_d, lo, hi).copy(), dl,
                    d2h(run_a, out_i, 0, il).copy(), want)
    finally:
        eng.close()
        ad = ai = dk = dko = res = out_d = out_i = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def test_run_a_stream_reader_and_page_caches(run_a):
    """get_values_stream, a reader, and readers with a 64 MiB page cache (smaller than one filler) and a 6 GiB one (all
    of A; slots past 2^20 sit at pool offsets past 2^32), over A served from host memory by the callback.  A repeat on
    the 6 GiB cache reads nothing and returns the same bytes."""
    a, keys = run_a["a"], run_a["keys"]
    tables = [(a.data, a.index, None)]
    eng = capi.Engine(0)
    try:
        for mode in MODES:
            want = expect_values(run_a, keys, mode)
            rows, d, i = eng.get_values_stream(tables, keys, mode)
            check_a(f"stream mode {mode}", rows, lambda lo, hi: d[lo:hi], d.size, i, want)
            del d, i
        for cache_bytes in (None, CACHE_BYTES, BIG_CACHE):
            cache = eng.open_page_cache(cache_bytes) if cache_bytes else None
            try:
                with eng.open_reader(tables) as r:
                    if cache is not None:
                        r.attach_page_cache(cache)
                    for mode in MODES:
                        want = expect_values(run_a, keys, mode)
                        for rep in range(2 if cache_bytes == BIG_CACHE else 1):
                            rows, d, i = r.get_values(keys, mode)
                            what = f"reader cache={cache_bytes} mode {mode} call {rep}"
                            check_a(what, rows, lambda lo, hi: d[lo:hi], d.size, i, want)
                            del d, i
                        if cache_bytes == BIG_CACHE:
                            assert r.last_stream_reads == [], "a repeat on the cache that holds A read something"
                            assert cache.stats()["resident_pages"] > (T32 >> 12)
            finally:
                if cache is not None:
                    cache.close()
    finally:
        eng.close()


def raw_readers_get_values(engine, batches, caps):
    """dbeel_readers_get_values called directly: the rows and the packed output before Engine.readers_get_values splits
    it per batch."""
    import ctypes as C
    arr = (capi.ReaderBatch * len(batches))()
    keep = []
    for j, (r, keys, mode) in enumerate(batches):
        blob, off = capi.pack_keys(keys)
        keep.append((blob, off))
        arr[j] = capi.ReaderBatch(r._h, blob.ctypes.data, off.ctypes.data, len(keys), mode, 0)
    rows = np.zeros(sum(len(k) for _, k, _ in batches), capi.LOOKUP_DTYPE)
    od, oi = np.empty(caps[0], np.uint8), np.empty(caps[1], np.uint8)
    out = capi.Out(od.ctypes.data, caps[0], 0, oi.ctypes.data, caps[1], 0, None, 0, 0, 0)
    engine._check(capi.lib().dbeel_readers_get_values(engine._h, arr, len(batches), C.byref(out), rows.ctypes.data),
                  "dbeel_readers_get_values")
    return rows, od[:out.data_len], oi[:out.index_len]


def test_run_a_readers_get_values(run_a):
    """Two readers of A: batch 0 asks for 10 fillers (about 2.5 GiB), batch 1 for the other 8 and the cluster entries.
    The raw output's .index offsets of batch 1 are shifted by batch 0's bytes, past 2^32; Engine.readers_get_values
    splits them back so that each batch equals the model from offset 0."""
    a, keys = run_a["a"], run_a["keys"]
    fl = run_a["marks"]["fillers"]
    k0, k1 = keys[:10], keys[10:]
    eng = capi.Engine(0)
    try:
        with eng.open_reader([(a.data, a.index, None)]) as r0, eng.open_reader([(a.data, a.index, None)]) as r1:
            jobs = [(r0, k0, capi.LOOKUP_EXACT), (r1, k1, capi.LOOKUP_REFERENCE)]
            w0, w1 = expect_values(run_a, k0, capi.LOOKUP_EXACT), expect_values(run_a, k1, capi.LOOKUP_REFERENCE)
            assert w0[2].size > 2 << 30 and w0[2].size + w1[2].size > T32
            rows, d, i = raw_readers_get_values(eng, jobs, (w0[2].size + w1[2].size, 16 * len(keys)))
            assert w0[2].spans == [(int(a.off[r]), int(a.fs[r])) for r in fl[:10]]
            idx = np.concatenate([w0[1], w1[1]]).reshape(-1, 16).copy()
            n0 = w0[1].size // 16
            shifted = idx[n0:, 0:8].copy().view("<u8") + np.uint64(w0[2].size)
            idx[n0:, 0:8] = shifted.view(np.uint8)
            assert int(shifted.max()) >> 32 == 1
            both = (np.concatenate([w0[0], w1[0]]), idx.reshape(-1), Gathered(a.data, w0[2].spans + w1[2].spans))
            check_a("raw readers_get_values", rows, lambda lo, hi: d[lo:hi], d.size, i, both)
            del d, i
            got = eng.readers_get_values(jobs)
            from test_gpu_past_4gib import compare_data, compare_index
            for j, ((gr, gd, gi), w) in enumerate(zip(got, (w0, w1))):
                M.compare_rows(f"batch {j}", gr, w[0])
                compare_index(f"batch {j}", gi, w[1])
                compare_data(f"batch {j}", lambda lo, hi: gd[lo:hi], w[2], gd.size)
            del got
    finally:
        eng.close()


class Sink:
    """A write callback for range reads into preallocated files, sized by the model: no 4 GiB bytearray copies."""

    def __init__(self, sizes):
        import ctypes as C
        self.C = C
        self.files = [{1: np.empty(max(1, ds), np.uint8), 2: np.empty(max(1, xs), np.uint8)} for ds, xs in sizes]

    def __call__(self, dest, kind, off, src, size):
        f = self.files[dest][kind]
        if off + size > f.size:
            return 4244
        self.C.memmove(f.ctypes.data + off, src, size)
        return 0


def test_run_a_range_reads(run_a):
    """reader_get_range (tombstones kept) and reader_scan (KEY) over [0x30, 0x80): every record from the first filler to
    the last, one destination of about 4.8 GB that is A's own bytes; reader_get_ranges forward and reverse (limit 64)
    over the three filler groups, 18 fillers in one output that passes 4 GiB, the reverse in descending key order."""
    from test_gpu_past_4gib import compare_data, compare_index
    a, fl = run_a["a"], run_a["marks"]["fillers"]
    lo, hi = fl[0], fl[-1] + 1
    assert all(a.keys[r][:1] in b"\x30\x40\x50\x60\x70" for r in range(lo, hi))
    want_d = a.data[int(a.off[lo]):int(a.off[hi - 1] + a.fs[hi - 1])]
    want_i = a.index[16 * lo:16 * hi].reshape(-1, 16).copy()
    want_i[:, 0:8] = (want_i[:, 0:8].copy().view("<u8") - np.uint64(a.off[lo])).view(np.uint8)
    want_i = want_i.reshape(-1)
    ranges = [(b"\x30", b"\x80")]
    eng = capi.Engine(0)
    try:
        with eng.open_reader([(a.data, a.index, None)]) as r:
            for name in ("get_range", "scan"):
                sink = Sink([(want_d.size, want_i.size)])
                if name == "scan":
                    res, stop = r.scan(ranges, write=sink)
                    assert eng.stats()["entries_in"] == hi - lo
                else:
                    res, stop = r.get_range(ranges, keep_tombstones=True, write=sink)
                M.compare_stop(name, stop, (-1, 0, 0))
                assert res[0][:2] == (want_d.size, want_i.size) and want_d.size > T32, (name, res)
                compare_index(name, sink.files[0][2][:want_i.size], want_i)
                compare_data(name, lambda x, y: sink.files[0][1][x:y], want_d, want_d.size)
                del sink
            groups = [[r_ for r_ in fl if a.keys[r_][:1] == p] for p in (b"\x30", b"\x50", b"\x70")]
            qs = [(p, p[:-1] + bytes([p[-1] + 1])) for p in (b"\x30", b"\x50", b"\x70")]
            for reverse in (False, True):
                order = [r_ for g in groups for r_ in (g[::-1] if reverse else g)]
                rows, d, i = r.get_ranges(qs, 64, reverse=reverse)
                assert [int(x) for x in rows["count"]] == [8, 8, 2] and [int(x) for x in rows["first"]] == [0, 8, 16]
                assert not rows["flags"].any() and (rows["table"] == -1).all()
                fs = a.fs[order].astype(np.int64)
                wi = np.zeros((len(order), 4), "<u4")
                wi[:, 0:2] = np.concatenate([[0], np.cumsum(fs)[:-1]]).astype("<u8").view("<u4").reshape(-1, 2)
                wi[:, 2] = [8 + len(a.keys[r_]) for r_ in order]
                wi[:, 3] = fs
                offs = wi[:, 0:2].copy().view("<u8").ravel().astype(np.int64)
                keys_out = [bytes(d[o + 8:o + int(ks)]) for o, ks in zip(offs, wi[:, 2])]
                assert keys_out == [a.keys[r_] for r_ in order]
                if reverse:
                    assert all(x > y for g in (keys_out[:8], keys_out[8:16], keys_out[16:]) for x, y in zip(g, g[1:]))
                compare_index(f"get_ranges reverse={reverse}", i, wi.view(np.uint8).reshape(-1))
                assert d.size > T32
                compare_data(f"get_ranges reverse={reverse}", lambda x, y: d[x:y],
                             Gathered(a.data, [(a.off[r_], a.fs[r_]) for r_ in order]), d.size)
                del d, i
    finally:
        eng.close()
