"""Every device entry point on files past 4 GiB: index offsets with a nonzero high word, in inputs and outputs.

An SSTable's .index record stores its .data offset as a u64, and the kernels carry 64-bit offsets through running sums,
tile clamps, rebases across jobs and partitions, and carried scans.  Below 2^32 bytes the high word of every offset is
zero, so a truncation to 32 bits anywhere on that path is invisible; past it, it gives wrong bytes, not a crash.

One module-scoped layout is built once and reused on the host and on the device:

* run A, about 4.6 GiB of .data, keys ascending: a cluster of small entries, ~256 MiB fillers, a cluster of small
  entries straddling 2^31, more fillers, a cluster straddling 2^32 (one entry starts a few bytes before it), more fillers,
  a tail of small entries.  No filler starts or ends on a 16-byte (or 8 KiB) edge.  Every aligned 8-byte word of a filler's payload holds its own absolute position in A's
  .data, so a copy from a wrong offset is caught, not only a copy of a wrong entry.
* run B, a few MB of small entries interleaving A's clusters: new keys, and keys equal to A's with higher, lower and
  equal timestamps, some of them tombstones, two of them equal to fillers.  B is tuned so that the A + B merge (keep
  tombstones) has an entry starting exactly at 2^32, and crosses 2^32 at a different key than A does.

The oracles' outputs for the big layout are first checked against an independent model (running sums of full_size, each
entry the bytes of its source); then every GPU output is compared with them byte for byte, in slices.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import scan_oracle
from dbeel_b200 import capi, sstable
from helpers import BASE_TS, nasty_keys

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
TWO31, TWO32 = 1 << 31, 1 << 32
FILL = 256 * MiB
POS_TAG = np.uint64(0xF1 << 56)  # top byte of every filler payload word; the rest is the word's position in A's .data
SLICE = 256 * MiB                # D2H / compare granule
SEED = bytes(range(32))
NO_BLOOM = 1 << 62
STEP = 1 << 29
EIGHTHS = [(k * STEP, (k + 1) * STEP) for k in range(7)] + [(7 * STEP, 0)]
DEVICE_BYTES_NEEDED = 22 * GiB   # the module's measured peak (A, B, one output stream and an engine's partition stages)


# ------------------------------------------------------------------------------------------------------------ the layout


class Table:
    """A run's files plus, per record in index order, what the model needs: key, timestamp, tombstone, offset, size."""

    def __init__(self, data, index, keys, ts, tomb):
        self.data, self.index = data, index
        self.keys, self.ts, self.tomb = keys, ts, tomb
        recs = index.reshape(-1, 16)
        self.off = recs[:, 0:8].copy().view("<u8").ravel().astype(np.int64)
        self.fs = recs[:, 12:16].copy().view("<u4").ravel().astype(np.int64)
        self.rec_of = {k: r for r, k in enumerate(keys)}

    def record_at(self, pos: int) -> int:
        """The record whose bytes hold .data position `pos`."""
        return int(np.searchsorted(self.off, pos, side="right")) - 1


def _entries(rng, prefix: bytes, keys, tomb_frac=0.15, max_doc=260):
    ents = []
    for k in sorted(prefix + k for k in keys):
        v = b"" if rng.random() < tomb_frac else bytes(rng.integers(0, 256, int(rng.integers(1, max_doc)), dtype=np.uint8))
        ents.append((k, v, BASE_TS + int(rng.integers(-10 ** 6, 10 ** 6))))
    return ents


def _off16(pos: int) -> int:
    """The smallest d >= 0 that puts pos + d off every 16-byte (and so every 8 KiB tile) edge."""
    return 3 if pos % 16 == 0 else 0


def _split(start: int, total: int, n: int):
    """n filler sizes near total / n that fill [start, start + total): every boundary between two of them lies off the
    16-byte and 8 KiB edges (the caller places start and start + total off them too)."""
    base = total // n
    sizes = [base + (4099 * (j + 1)) % 8191 - 4000 for j in range(n - 1)]
    pos = start
    for j in range(n - 1):
        sizes[j] += _off16(pos + sizes[j])
        pos += sizes[j]
    sizes.append(total - sum(sizes))
    bounds = np.cumsum([start] + sizes)
    assert sum(sizes) == total and all(b % 16 for b in bounds) and all(s < 2 ** 32 - 1 for s in sizes)
    return sizes


def build_a(rng):
    """Run A.  Returns (Table, {name: record}) where the names mark the records around 2^31 and 2^32."""
    pool = {p: nasty_keys(rng, n, max_len=28) for p, n in ((0x20, 3000), (0x40, 6000), (0x60, 30000), (0x80, 2000))}
    small = {p: _entries(rng, bytes([p]), ks) for p, ks in pool.items()}
    size = lambda ents: sum(sstable.ENTRY_OVERHEAD + len(k) + len(v) for k, v, _ in ents)  # noqa: E731
    c1, c2 = small[0x40], small[0x60]
    h1, h2 = len(c1) // 2, len(c2) // 2
    # record h1 starts d1 >= 5 bytes past 2^31, so h1 - 1 straddles it; record h2 starts d2 >= 5 bytes before 2^32 and ends
    # after it.  d1, d2 and the last fillers' sizes are nudged so that no filler starts or ends on a 16-byte edge.
    if size(small[0x20]) % 16 == 0:
        k, v, t = next(e for e in small[0x20] if e[1])
        small[0x20][small[0x20].index((k, v, t))] = (k, v + b"+", t)
    d1 = next(d for d in range(5, 40) if (TWO31 + d - size(c1[:h1])) % 16 and (TWO31 + d - size(c1[:h1]) + size(c1)) % 16)
    d2 = next(d for d in range(5, 40) if (TWO32 - d - size(c2[:h2])) % 16 and (TWO32 - d - size(c2[:h2]) + size(c2)) % 16)
    c1_start, c2_start = TWO31 + d1 - size(c1[:h1]), TWO32 - d2 - size(c2[:h2])
    c0_end = size(small[0x20])
    g1 = _split(c0_end, c1_start - c0_end, 8)
    g2 = _split(c1_start + size(c1), c2_start - (c1_start + size(c1)), 8)
    g3_start = c2_start + size(c2)
    g3 = _split(g3_start, 2 * FILL + 12345 + _off16(g3_start + 2 * FILL + 12345), 2)
    layout = ([("small", e) for e in small[0x20]]
              + [("fill", (bytes([0x30]) + b"fill-%02d" % j, s)) for j, s in enumerate(g1)]
              + [("small", e) for e in c1]
              + [("fill", (bytes([0x50]) + b"fill-%02d" % j, s)) for j, s in enumerate(g2)]
              + [("small", e) for e in c2]
              + [("fill", (bytes([0x70]) + b"fill-%02d" % j, s)) for j, s in enumerate(g3)]
              + [("small", e) for e in small[0x80]])
    total = sum(size([e]) if kind == "small" else e[1] for kind, e in layout)
    buf = np.empty((total + 7) // 8 * 8, np.uint8)
    words = buf.view("<u8")
    chunk = 16 * MiB
    for lo in range(0, words.size, chunk):   # every aligned word: its own position, tagged
        hi = min(words.size, lo + chunk)
        words[lo:hi] = np.arange(8 * lo, 8 * hi, 8, dtype=np.uint64) | POS_TAG
    data = buf[:total]
    n = len(layout)
    index = np.zeros((n, 4), "<u4")
    keys, ts, tomb = [], np.zeros(n, np.int64), np.zeros(n, bool)
    pos = 0
    for r, (kind, e) in enumerate(layout):
        if kind == "small":
            k, v, t = e
            rec = sstable.encode_entry(k, v, t)
            data[pos:pos + len(rec)] = np.frombuffer(rec, np.uint8)
            fs, tomb[r] = len(rec), not v
        else:
            k, fs = e
            t = BASE_TS + r
            dlen = fs - sstable.ENTRY_OVERHEAD - len(k)
            data[pos:pos + 8 + len(k) + 8] = np.frombuffer(len(k).to_bytes(8, "little") + k + dlen.to_bytes(8, "little"), np.uint8)
            data[pos + fs - 16:pos + fs] = np.frombuffer(t.to_bytes(16, "little", signed=True), np.uint8)
        index[r, 0:2] = np.array([pos], "<u8").view("<u4")
        index[r, 2], index[r, 3] = 8 + len(k), fs
        keys.append(k)
        ts[r] = t
        pos += fs
    assert pos == total
    a = Table(data, index.view(np.uint8).reshape(-1), keys, ts, tomb)
    n0, n1 = len(small[0x20]) + len(g1), len(small[0x20]) + len(g1) + len(c1) + len(g2)
    marks = {"straddle31": n0 + h1 - 1, "after31": n0 + h1, "straddle32": n1 + h2, "before32": n1 + h2 - 1,
             "fillers": [r for r, (kind, _) in enumerate(layout) if kind == "fill"]}
    assert TWO31 < a.off[marks["after31"]] < TWO31 + 40 and a.off[marks["straddle31"]] < TWO31
    s32 = marks["straddle32"]
    assert TWO32 - 40 < a.off[s32] < TWO32 and a.off[s32] + a.fs[s32] > TWO32
    for r in marks["fillers"]:
        assert a.off[r] % 16 and (a.off[r] + a.fs[r]) % 16, "a filler boundary on a 16-byte edge"
    return a, marks


def build_b(rng, a: Table, marks, grow: int = 0, grow_key=None):
    """Run B: new keys in every cluster and between fillers, keys of A with higher / lower / equal timestamps (some of
    them tombstones), one filler overwritten by a newer tombstone and one by an older entry.  `grow` bytes are added to
    the payload of the entry with key `grow_key` (a new key of B that wins)."""
    ents = {}
    for p in (0x20, 0x40, 0x60, 0x80):
        for k, v, t in _entries(rng, bytes([p]), nasty_keys(rng, 1500, max_len=30), tomb_frac=0.1, max_doc=300):
            if k not in a.rec_of:
                ents[k] = (v, t)
    for j in range(8):
        ents[bytes([0x30]) + b"fill-%02d\x00" % j] = (b"between fillers %d" % j, BASE_TS)
    same = rng.choice(len(a.keys), 6000, replace=False)
    for r in same.tolist() + [marks["straddle31"], marks["after31"], marks["before32"]]:
        if a.fs[r] > 4096:
            continue
        d = int(rng.integers(-1, 2))   # older, equal (B wins the tie: later run), newer
        v = b"" if rng.random() < 0.3 else bytes(rng.integers(0, 256, int(rng.integers(1, 90)), dtype=np.uint8))
        ents[a.keys[r]] = (v, int(a.ts[r]) + d)
    fl = marks["fillers"]
    ents[a.keys[fl[-1]]] = (b"", int(a.ts[fl[-1]]) + 1)          # a newer tombstone: the last filler is dropped
    ents[a.keys[fl[9]]] = (b"older than the filler", int(a.ts[fl[9]]) - 1)
    if grow:
        v, t = ents[grow_key]
        ents[grow_key] = (v + bytes(rng.integers(0, 256, grow, dtype=np.uint8)), t)
    keys = sorted(ents)
    data, index = sstable.build_run([(k, *ents[k]) for k in keys])
    return Table(data, index, keys, np.array([ents[k][1] for k in keys], np.int64),
                 np.array([ents[k][0] == b"" for k in keys], bool))


def merge_model(tables, keep: bool):
    """Appendix A.3 on record metadata: per key the max (timestamp, run position) record wins; a winning tombstone is
    dropped unless `keep`.  Returns the winners in key order as (run, record)."""
    best = {}
    for run, t in enumerate(tables):
        for r, k in enumerate(t.keys):
            cur = best.get(k)
            if cur is None or (int(t.ts[r]), run) > (int(tables[cur[0]].ts[cur[1]]), cur[0]):
                best[k] = (run, r)
    return [best[k] for k in sorted(best) if keep or not tables[best[k][0]].tomb[best[k][1]]]


def model_offsets(tables, srcs):
    fs = np.array([tables[t].fs[r] for t, r in srcs], np.int64)
    off = np.zeros(len(srcs) + 1, np.int64)
    np.cumsum(fs, out=off[1:])
    return off


def check_model(what, tables, srcs, data, index):
    """An oracle's output against the model: .index = running sums of full_size with key_size = 8 + key length, and each
    entry's bytes = its source record's bytes."""
    off = model_offsets(tables, srcs)
    recs = np.asarray(index).reshape(-1, 16)
    assert recs.shape[0] == len(srcs), f"{what}: {recs.shape[0]} records, model {len(srcs)}"
    assert data.size == off[-1], f"{what}: .data {data.size} bytes, model {off[-1]}"
    got_off = recs[:, 0:8].copy().view("<u8").ravel().astype(np.int64)
    assert np.array_equal(got_off, off[:-1]), f"{what}: offsets are not the running sums of full_size"
    ks = np.array([8 + len(tables[t].keys[r]) for t, r in srcs], np.uint32)
    fs = np.array([tables[t].fs[r] for t, r in srcs], np.uint32)
    assert np.array_equal(recs[:, 8:12].copy().view("<u4").ravel(), ks), f"{what}: key_size"
    assert np.array_equal(recs[:, 12:16].copy().view("<u4").ravel(), fs), f"{what}: full_size"
    for j, (t, r) in enumerate(srcs):
        src = tables[t]
        o, n = int(src.off[r]), int(src.fs[r])
        if not np.array_equal(data[off[j]:off[j] + n], src.data[o:o + n]):
            raise AssertionError(f"{what}: entry {j} (run {t} record {r}) is not its source's bytes")
    return off


@pytest.fixture(scope="module")
def big():
    """The shared layout, on the host and on the device, with the oracle outputs every case compares against."""
    free, _ = torch.cuda.mem_get_info(0)
    if free < DEVICE_BYTES_NEEDED:
        pytest.skip(f"needs {DEVICE_BYTES_NEEDED / GiB:.0f} GiB of free device memory, {free / GiB:.1f} GiB free")
    rng = np.random.default_rng(4242)
    a, marks = build_a(rng)
    hi = a.index.reshape(-1, 16)[:, 4:8].copy().view("<u4").ravel()
    assert int((hi > 0).sum()) > 1000 and a.data.size > TWO32 + 512 * MiB, "run A does not reach past 4 GiB"
    # tune B so that the kept merge has an entry starting exactly at 2^32
    state = rng.bit_generator.state
    b = build_b(rng, a, marks)
    srcs = merge_model([a, b], keep=True)
    off = model_offsets([a, b], srcs)
    k = int(np.searchsorted(off, TWO32, side="right")) - 1
    grow_key = next(key for key in b.keys[::-1] if key[0] == 0x40 and key not in a.rec_of and not b.tomb[b.rec_of[key]])
    assert TWO32 - off[k] < 4096, "2^32 falls outside the small entries of the merged output"
    rng.bit_generator.state = state
    b = build_b(rng, a, marks, grow=TWO32 - int(off[k]), grow_key=grow_key)
    keep_srcs = merge_model([a, b], keep=True)
    off = model_offsets([a, b], keep_srcs)
    k = int(np.searchsorted(off, TWO32))
    assert off[k] == TWO32, "no merged entry starts at 2^32"
    assert [a, b][keep_srcs[k - 1][0]].keys[keep_srcs[k - 1][1]] != a.keys[marks["straddle32"]], \
        "the merge crosses 2^32 at the same entry as run A"

    def dev(arr):
        t = torch.empty(arr.size + 16, dtype=torch.uint8, device="cuda:0")
        for lo in range(0, arr.size, SLICE):
            t[lo:min(arr.size, lo + SLICE)].copy_(torch.from_numpy(arr[lo:lo + SLICE]))
        t[arr.size:].zero_()
        return t

    env = {"a": a, "b": b, "marks": marks, "keep_srcs": keep_srcs, "drop_srcs": merge_model([a, b], keep=False)}
    env["a_dev"], env["ai_dev"] = dev(a.data), dev(a.index)
    env["b_dev"], env["bi_dev"] = dev(b.data), dev(b.index)
    out_cap = a.data.size + b.data.size + 8 * MiB
    env["out_d"] = torch.empty(out_cap, dtype=torch.uint8, device="cuda:0")
    env["out_i"] = torch.empty(a.index.size + b.index.size + MiB, dtype=torch.uint8, device="cuda:0")
    env["out_b"] = torch.empty(4 * MiB, dtype=torch.uint8, device="cuda:0")
    env["pinned"] = torch.empty(SLICE, dtype=torch.uint8, pin_memory=True)
    env["cache"] = {}
    torch.cuda.synchronize()
    yield env
    env.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def runs_ptrs(env, names=("a", "b")):
    return [(env[f"{n}_dev"].data_ptr(), env[n].data.size, env[f"{n}i_dev"].data_ptr(), env[n].index.size) for n in names]


def merged(env, keep: bool):
    """The oracle's A + B compaction (with a filter), checked against the model once; one result is held at a time."""
    key = ("merge", keep)
    cache = env["cache"]
    if key not in cache:
        cache.clear()
        a, b = env["a"], env["b"]
        res = oracle.compact([(a.data, a.index), (b.data, b.index)], keep_tombstones=keep, seed=SEED)
        check_model(f"oracle merge keep={keep}", [a, b], env["keep_srcs" if keep else "drop_srcs"], res[0], res[1])
        assert res[0].size > TWO32 and res[2] is not None
        cache[key] = res
    return cache[key]


# ------------------------------------------------------------------------------------------------------ the comparison


def d2h(env, t: torch.Tensor, lo: int, hi: int) -> np.ndarray:
    buf = env["pinned"][:hi - lo]
    buf.copy_(t[lo:hi])
    return buf.numpy()


def compare_data(what, get, exp: np.ndarray, n: int):
    """get(lo, hi) -> the output's bytes [lo, hi); compared slice by slice with `exp`."""
    assert n == exp.size, f"{what}: .data is {n} bytes, expected {exp.size}"
    for lo in range(0, n, SLICE):
        hi = min(n, lo + SLICE)
        g = get(lo, hi)
        if not np.array_equal(g, exp[lo:hi]):
            bad = lo + int(np.flatnonzero(g != exp[lo:hi])[0])
            raise AssertionError(f"{what}: .data differs at byte {bad} (0x{bad:x})")


def compare_index(what, got: np.ndarray, exp: np.ndarray):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.size == exp.size, f"{what}: .index is {got.size} bytes, expected {exp.size}"
    if not np.array_equal(got, exp):
        bad = int(np.flatnonzero(got != exp)[0])
        field = ("offset low word", "offset high word", "key_size", "full_size")[bad % 16 // 4]
        raise AssertionError(f"{what}: .index differs at record {bad // 16} ({field})")


def compare_dev(env, what, data_t, index_t, dl, il, exp_d, exp_i, data_off=0, index_off=0):
    compare_index(what, d2h(env, index_t, index_off, index_off + il).copy(), exp_i)
    compare_data(what, lambda lo, hi: d2h(env, data_t, data_off + lo, data_off + hi), exp_d, dl)


def max_offset(index) -> int:
    recs = np.asarray(index).reshape(-1, 16)
    return int(recs[:, 0:8].copy().view("<u8").max()) if recs.size else 0


# ---------------------------------------------------------------------------------------------------- the checker first


def test_layout_and_oracle_merge_match_the_model(big):
    """Run A's .index has records past 2^32; the oracle's merges equal the model (running sums, source bytes)."""
    a, m = big["a"], big["marks"]
    assert max_offset(a.index) > TWO32 and TWO32 - 40 < a.off[m["straddle32"]] < TWO32
    f = m["fillers"][11]
    lo = (int(a.off[f]) + 40 + 7) // 8 * 8
    words = a.data[lo:lo + 64].view("<u8")
    assert np.array_equal(words, np.arange(lo, lo + 64, 8, dtype=np.uint64) | POS_TAG), "filler words hold their positions"
    for keep in (True, False):   # merged() holds one result at a time: keep no reference to the previous one
        res = merged(big, keep)
        assert res[3] == len(big["keep_srcs" if keep else "drop_srcs"]) and max_offset(res[1]) > TWO32
        del res


# ----------------------------------------------------------------------------------------------------------- compactions


def _compact_device(engine, env, runs, keep, bloom_min, flags=0):
    opts = capi.make_opts(keep, bloom_min, seed=SEED, flags=flags)
    dc, ic, bc = capi.compact_bound([(r[1], r[3]) for r in runs], opts)
    assert dc <= env["out_d"].numel() and ic <= env["out_i"].numel() and bc <= env["out_b"].numel()
    return engine.compact_device(runs, (env["out_d"].data_ptr(), dc, env["out_i"].data_ptr(), ic, env["out_b"].data_ptr(), bc),
                                 opts)


def test_compact_device_a_alone(engine, big):
    """One run (the five-kernel path): keeping tombstones, the output is run A itself."""
    a = big["a"]
    dl, il, bl, n = _compact_device(engine, big, runs_ptrs(big, ("a",)), True, NO_BLOOM)
    assert n == len(a.keys) and bl == 0
    compare_dev(big, "A alone", big["out_d"], big["out_i"], dl, il, a.data, a.index)


def test_compact_device_keep(engine, big):
    d, i, _, n = merged(big, True)
    dl, il, bl, got_n = _compact_device(engine, big, runs_ptrs(big), True, NO_BLOOM)
    assert got_n == n and bl == 0 and dl > TWO32
    compare_dev(big, "A + B, keep", big["out_d"], big["out_i"], dl, il, d, i)


def test_compare_reports_host_side_corruption(engine, big):
    """The comparison sees a cleared high word in one index record past 2^32 and two swapped 8-byte words around it."""
    d, i, _, n = merged(big, True)
    dl, il, _, _ = _compact_device(engine, big, runs_ptrs(big), True, NO_BLOOM)
    got_i = d2h(big, big["out_i"], 0, il).copy()
    compare_index("untouched", got_i, i)
    r = int(np.flatnonzero(got_i.reshape(-1, 16)[:, 4:8].copy().view("<u4").ravel() > 0)[3])
    bad_i = got_i.copy()
    bad_i[16 * r + 4:16 * r + 8] = 0
    with pytest.raises(AssertionError, match=f"record {r} \\(offset high word\\)"):
        compare_index("high word cleared", bad_i, i)
    swap = {}
    lo = d2h(big, big["out_d"], TWO32 - 8, TWO32 + 8).copy()
    assert not np.array_equal(lo[:8], lo[8:]), "the two words are equal: swapping them would change nothing"
    swap.update({TWO32 - 8 + j: lo[8 + j] for j in range(8)})
    swap.update({TWO32 + j: lo[j] for j in range(8)})

    def swapped(lo_, hi_):
        g = d2h(big, big["out_d"], lo_, hi_).copy()
        for p, v in swap.items():
            if lo_ <= p < hi_:
                g[p - lo_] = v
        return g

    with pytest.raises(AssertionError, match=f"differs at byte {TWO32 - 8}"):
        compare_data("words swapped across 2^32", swapped, d, dl)
    compare_data("untouched", lambda lo_, hi_: d2h(big, big["out_d"], lo_, hi_), d, dl)


# The host entry points return their output in host memory.  Holding the oracle's output next to it would make three
# full copies (run A, the oracle's, the engine's), so these compare with the model, which the oracle's merge was checked
# against in test_layout_and_oracle_merge_match_the_model: the same bytes, entry by entry.  Each runs on an engine of its
# own: the pipelined path's device stages and the streaming path's page-locked rings are grow-only and sized by the
# largest partition (several GB here), and the session's engine would keep them for every later test.


def test_compact_host_pipelined(big):
    """dbeel_compact from host buffers: the pipelined path's key-range partitions carry out_offset_base past 2^32."""
    a, b = big["a"], big["b"]
    big["cache"].clear()
    eng = capi.Engine(0)
    try:
        gd, gi, gb, gn = eng.compact([(a.data, a.index), (b.data, b.index)], keep_tombstones=True, bloom_min_size=NO_BLOOM,
                                     seed=SEED)
        assert eng.stats()["partitions"] > 1
    finally:
        eng.close()
    assert gb is None and gd.size > TWO32
    check_model("dbeel_compact", [a, b], big["keep_srcs"], gd, gi)


def test_compact_stream(big):
    """dbeel_compact_stream with in-memory files, through the pipelined path (more than one partition, so the writer
    threads write each partition's pieces at offsets that pass 2^32)."""
    a, b = big["a"], big["b"]
    big["cache"].clear()
    eng = capi.Engine(0)
    try:
        gd, gi, gb, gn = eng.compact_stream([(a.data, a.index), (b.data, b.index)], keep_tombstones=True,
                                            bloom_min_size=NO_BLOOM, seed=SEED)
        assert eng.stats()["partitions"] > 1, "the job fell back to the one-piece path"
    finally:
        eng.close()
    assert gb is None and gd.size > TWO32
    check_model("dbeel_compact_stream", [a, b], big["keep_srcs"], gd, gi)


def test_compact_device_reference_reader_repairs_past_2_32(engine, big):
    """FLAG_REFERENCE_READER with the high word of one index record past 2^32 cleared: the job runs on the canonical
    index (k_ref_repair rebuilds the offsets across the boundary) and equals the oracle, which reads .data in order."""
    a, b = big["a"], big["b"]
    big["cache"].clear()
    r = a.record_at(TWO32 + 3 * MiB)
    bad = a.index.copy()
    bad[16 * r + 4:16 * r + 8] = 0
    d, i, _, n = oracle.compact([(a.data, bad), (b.data, b.index)], keep_tombstones=True, bloom_min_size=NO_BLOOM, seed=SEED)
    check_model("oracle merge, damaged record", [a, b], big["keep_srcs"], d, i)
    bad_dev = torch.from_numpy(bad).to("cuda:0")
    torch.cuda.synchronize()
    runs = [(big["a_dev"].data_ptr(), a.data.size, bad_dev.data_ptr(), bad.size)] + runs_ptrs(big, ("b",))
    dl, il, _, gn = _compact_device(engine, big, runs, True, NO_BLOOM, flags=capi.FLAG_REFERENCE_READER)
    assert engine.stats()["index_repaired"] == 1 and gn == n
    compare_dev(big, "reference reader, damaged record past 2^32", big["out_d"], big["out_i"], dl, il, d, i)


def test_compact_many_device_third_job_past_4gib(engine, big):
    """A small job, A + B, a small job in one output stream: the third job starts past 4 GiB of the stream and its file
    offsets restart at 0."""
    d, i, _, n = merged(big, True)
    rng = np.random.default_rng(7)
    smalls = []
    for j in range(2):
        ents = _entries(rng, b"\x55", nasty_keys(rng, 500 + 300 * j), max_doc=400)
        smalls.append(sstable.build_run(ents))
    hold = [torch.from_numpy(np.concatenate([x, np.zeros(16, np.uint8)])).to("cuda:0") for s in smalls for x in s]
    torch.cuda.synchronize()
    sp = [(hold[2 * j].data_ptr(), smalls[j][0].size, hold[2 * j + 1].data_ptr(), smalls[j][1].size) for j in range(2)]
    jobs = [([sp[0]], True), (runs_ptrs(big), True), ([sp[1]], False)]
    out = (big["out_d"].data_ptr(), big["out_d"].numel(), big["out_i"].data_ptr(), big["out_i"].numel(), 0, 0)
    rows = engine.compact_many_device(jobs, out, NO_BLOOM, seeds=[SEED] * 3)
    assert rows[2]["data_off"] > TWO32 and rows[1]["data_len"] > TWO32
    for j, (runs, keep) in enumerate(((smalls[0:1], True), (None, True), (smalls[1:2], False))):
        if runs is None:
            ed, ei, en = d, i, n
        else:
            ed, ei, _, en = oracle.compact(runs, keep_tombstones=keep, bloom_min_size=NO_BLOOM, seed=SEED)
        r = rows[j]
        assert r["items_written"] == en and r["bloom_len"] == 0, f"job {j}"
        compare_dev(big, f"compact-many job {j}", big["out_d"], big["out_i"], r["data_len"], r["index_len"], ed, ei,
                    r["data_off"], r["index_off"])


def test_compact_device_drop_with_filter(engine, big):
    """Tombstones dropped, a filter with a fixed seed."""
    d, i, bloom, n = merged(big, False)
    dl, il, bl, gn = _compact_device(engine, big, runs_ptrs(big), False, oracle.DEFAULT_BLOOM_MIN_SIZE)
    assert gn == n and dl > TWO32
    assert np.array_equal(d2h(big, big["out_b"], 0, bl), bloom), ".bloom differs"
    compare_dev(big, "A + B, drop, filter", big["out_d"], big["out_i"], dl, il, d, i)


# ---------------------------------------------------------------------------------------------------------------- flushes


def _oracle_flush(batch_data, batch_index):
    """One memtable flush in the oracle, into buffers of our own (no second copy of a 4 GiB output)."""
    arr, keep = oracle._mk_runs([(batch_data, batch_index)])
    out, (d, i, _) = oracle._mk_out(batch_data.size, batch_index.size, 0)
    consumed = C.c_uint64(0)
    assert oracle.lib().orc_memtable_flush(arr, 0, 1 << 20, 0, C.byref(out), C.byref(consumed)) == 0
    assert consumed.value == batch_index.size // 16
    return d[:out.data_len], i[:out.index_len], int(out.items_written)


def test_flush_device_and_flush_many_device(engine, big):
    """A batch of more than 4 GiB (run A's entries, distinct keys, tombstones kept): its flush is run A itself.  In
    dbeel_flush_many_device a second memtable starts past 4 GiB of the output stream."""
    a, b = big["a"], big["b"]
    big["cache"].clear()
    od, oi, on = _oracle_flush(a.data, a.index)
    assert on == len(a.keys)
    check_model("oracle flush of A", [a], [(0, r) for r in range(len(a.keys))], od, oi)
    del od, oi
    dl, il, n = engine.flush_device(runs_ptrs(big, ("a",))[0], (big["out_d"].data_ptr(), a.data.size, big["out_i"].data_ptr(),
                                                                a.index.size))
    assert n == len(a.keys)
    compare_dev(big, "flush of A", big["out_d"], big["out_i"], dl, il, a.data, a.index)

    ed, ei, en = _oracle_flush(b.data, b.index)
    caps = (big["out_d"].data_ptr(), a.data.size + b.data.size, big["out_i"].data_ptr(), a.index.size + b.index.size)
    _, _, _, rows = engine.flush_many_device(runs_ptrs(big, ("a", "b")), caps)
    assert rows[1]["data_off"] > TWO32 and rows[0]["items"] == len(a.keys) and rows[1]["items"] == en
    compare_dev(big, "flush-many memtable 0", big["out_d"], big["out_i"], rows[0]["data_len"], rows[0]["index_len"], a.data, a.index)
    compare_dev(big, "flush-many memtable 1", big["out_d"], big["out_i"], rows[1]["data_len"], rows[1]["index_len"], ed, ei,
                rows[1]["data_off"], rows[1]["index_off"])


def test_wal_flush_device(engine, big):
    """A write-ahead log of more than 4 GiB: 1.1 M logged writes to 6000 keys, one page each, so the replay's sparse
    offsets pass 2^32.  The last write of every key lies past 2^32 and every write's payload names its arrival, so a read
    through an offset truncated to 32 bits would return an older write.  (Repeated keys keep the memtable under the
    reference's capacity and the oracle's copies small.)"""
    big["cache"].clear()
    rng = np.random.default_rng(99)
    page, n_keys, klen, dlen = sstable.PAGE_SIZE, 6000, 16, 64
    keys = np.unique(rng.integers(0, 256, (n_keys + 100, klen), dtype=np.uint8), axis=0)[:n_keys]
    n = TWO32 // page + 60_000
    kid = rng.permutation(n_keys)[np.arange(n) % n_keys]
    ent = 32 + klen + dlen
    wal = np.full(n * page, 0xA5, np.uint8)
    rows_all = wal.reshape(n, page)
    for lo in range(0, n, 1 << 16):
        hi = min(n, lo + (1 << 16))
        j = np.arange(lo, hi, dtype=np.uint64)
        rows = np.empty((hi - lo, ent), np.uint8)
        rows[:, 0:8] = np.frombuffer(np.uint64(klen).tobytes(), np.uint8)
        rows[:, 8:8 + klen] = keys[kid[lo:hi]]
        rows[:, 8 + klen:16 + klen] = np.frombuffer(np.uint64(dlen).tobytes(), np.uint8)
        rows[:, 16 + klen:16 + klen + dlen] = (j[:, None] * np.uint64(dlen // 8) + np.arange(dlen // 8, dtype=np.uint64)
                                               | POS_TAG).view(np.uint8)
        ts = (np.int64(BASE_TS) + j.astype(np.int64)).astype("<i8")
        rows[:, ent - 16:ent - 8] = ts.view(np.uint8).reshape(-1, 8)
        rows[:, ent - 8:] = 0
        rows_all[lo:hi, :ent] = rows
    # the model: per key its last write, in key order
    last = np.zeros(n_keys, np.int64)
    last[kid] = np.arange(n)
    assert last.min() * page > TWO32
    order = np.lexsort(keys.T[::-1])
    exp_d = np.ascontiguousarray(rows_all[last[order], :ent]).reshape(-1)
    exp_i = np.zeros((n_keys, 4), "<u4")
    exp_i[:, 0:2] = (np.arange(n_keys, dtype=np.uint64) * np.uint64(ent)).view("<u4").reshape(-1, 2)
    exp_i[:, 2], exp_i[:, 3] = 8 + klen, ent
    exp_i = exp_i.view(np.uint8).reshape(-1)
    out, (od, oi, _) = oracle._mk_out(exp_d.size, exp_i.size, 0)
    seen = C.c_uint64(0)
    assert oracle.lib().orc_wal_flush(wal.ctypes.data, wal.size, capi.DEFAULT_TREE_CAPACITY, 0, C.byref(out), C.byref(seen)) == 0
    assert seen.value == n and out.items_written == n_keys
    assert np.array_equal(od[:out.data_len], exp_d) and np.array_equal(oi[:out.index_len], exp_i), "oracle WAL flush vs model"
    wal_dev = torch.empty(wal.size + 4096, dtype=torch.uint8, device="cuda:0")
    for lo in range(0, wal.size, SLICE):
        wal_dev[lo:min(wal.size, lo + SLICE)].copy_(torch.from_numpy(wal[lo:lo + SLICE]))
    wal_dev[wal.size:].zero_()
    torch.cuda.synchronize()
    wal_len = wal.size
    del wal, rows_all
    out_i = torch.empty(16 * n, dtype=torch.uint8, device="cuda:0")   # the cap: 16 bytes per logged entry
    try:
        dl, il, items = engine.wal_flush_device(wal_dev.data_ptr(), wal_len, (big["out_d"].data_ptr(), big["out_d"].numel(),
                                                                              out_i.data_ptr(), out_i.numel()))
        assert items == n_keys
        compare_dev(big, "WAL flush", big["out_d"], out_i, dl, il, od[:out.data_len], oi[:out.index_len])
    finally:
        del wal_dev, out_i
        torch.cuda.synchronize()
        torch.cuda.empty_cache()   # the log's 4.5 GB go back to the device, not to torch's cache


def test_route_and_sparse_flush(engine, big):
    """dbeel_route_device over run A as an arrival batch, then dbeel_flush_many_sparse_device of the routed streams: the
    routed records point into .data past 2^32."""
    a = big["a"]
    big["cache"].clear()
    ring, _ = oracle.shard_ring(8)
    exp_shard, _ = oracle.route((a.data, a.index), ring)
    out_idx = torch.empty(a.index.size + 16, dtype=torch.uint8, device="cuda:0")
    counts, _ = engine.route_device(runs_ptrs(big, ("a",))[0], ring, out_idx.data_ptr(), a.index.size)
    recs = a.index.reshape(-1, 16)
    order = np.concatenate([np.flatnonzero(exp_shard == s) for s in range(8)])
    assert np.array_equal(d2h(big, out_idx, 0, a.index.size).reshape(-1, 16), recs[order]), "routed index"
    batches, base = [], out_idx.data_ptr()
    for c in counts.tolist():
        batches.append((big["a_dev"].data_ptr(), a.data.size, base, 16 * int(c)))
        base += 16 * int(c)
    caps = (big["out_d"].data_ptr(), a.data.size, big["out_i"].data_ptr(), a.index.size)
    _, _, _, rows = engine.flush_many_sparse_device(batches, a.data.size, caps)
    assert max(r["data_off"] + r["data_len"] for r in rows) > TWO32
    far = 0
    for s, r in enumerate(rows):
        srcs = np.flatnonzero(exp_shard == s)   # distinct ascending keys: the flush is the routed entries in order
        fs = a.fs[srcs]
        off = np.zeros(srcs.size, np.int64)
        np.cumsum(fs[:-1], out=off[1:])
        ei = np.zeros((srcs.size, 4), "<u4")
        ei[:, 0:2] = off.astype("<u8").view("<u4").reshape(-1, 2)
        ei[:, 2] = recs[srcs, 8:12].copy().view("<u4").ravel()
        ei[:, 3] = fs
        ed = np.concatenate([a.data[int(a.off[q]):int(a.off[q] + a.fs[q])] for q in srcs])
        assert r["items"] == srcs.size
        far = max(far, int(a.off[srcs].max()))
        compare_dev(big, f"sparse flush shard {s}", big["out_d"], big["out_i"], r["data_len"], r["index_len"], ed,
                    ei.view(np.uint8).reshape(-1), r["data_off"], r["index_off"])
    assert far > TWO32


# ------------------------------------------------------------------------------------------------------------------ scans


def oracle_scan(tables, ranges, kind=scan_oracle.SCAN_HASH):
    """scan_oracle.scan without copying the outputs: views of buffers allocated (not touched) at the tables' size."""
    arr, keep = oracle._mk_runs([(t.data, t.index) for t in tables])
    dc = sum(int(t.fs.sum()) for t in tables)
    ic = sum(t.index.size for t in tables) + 16
    n = len(ranges)
    outs = (oracle._Out * n)()
    bufs = []
    for d in range(n):
        o, b = oracle._mk_out(dc, ic, 0)
        outs[d] = o
        bufs.append(b)
    if kind == scan_oracle.SCAN_HASH:
        hr = np.array(ranges, np.uint32).reshape(-1)
        blob, off = np.zeros(1, np.uint8), np.zeros(1, np.uint64)
    else:
        hr = np.zeros(1, np.uint32)
        parts = [bytes(k) for pair in ranges for k in pair]
        off = np.zeros(len(parts) + 1, np.uint64)
        off[1:] = np.cumsum([len(p) for p in parts])
        blob = np.frombuffer(b"".join(parts) + b"\0", np.uint8).copy()
    t, r, rec = C.c_int32(), C.c_uint32(), C.c_uint64()
    assert scan_oracle.lib().orc_scan(arr, len(keep), kind, hr.ctypes.data, blob.ctypes.data, off.ctypes.data, n, outs,
                                      C.byref(t), C.byref(r), C.byref(rec)) == 0
    return ([(bufs[d][0][:outs[d].data_len], bufs[d][1][:outs[d].index_len]) for d in range(n)],
            (int(t.value), int(r.value), int(rec.value)))


def scan_model(tables, ranges, upto=None):
    """Destination per record (hash ranges, first match), records in iteration order, up to (table, record) `upto`."""
    dests = [[] for _ in ranges]
    for ti, t in enumerate(tables):
        for r, k in enumerate(t.keys):
            if upto is not None and (ti, r) >= upto:
                return dests
            h = oracle.murmur3_32(k)
            d = next((j for j, (s, e) in enumerate(ranges) if scan_oracle.between_cmp(h, s, e)), None)
            if d is not None:
                dests[d].append((ti, r))
    return dests


def _scan_device(engine, env, tables_ptrs, ranges, kind=capi.SCAN_HASH):
    out = (env["out_d"].data_ptr(), env["out_d"].numel(), env["out_i"].data_ptr(), env["out_i"].numel())
    return engine.scan_device(tables_ptrs, ranges, out, kind)


def _check_scan_dev(env, what, rows, stop, exp):
    assert stop == exp[1], what
    for j, (r, (ed, ei)) in enumerate(zip(rows, exp[0])):
        compare_dev(env, f"{what}: destination {j}", env["out_d"], env["out_i"], r["data_len"], r["index_len"], ed, ei,
                    r["data_off"], r["index_off"])


def scan_expect(env, name):
    """Oracle scans of A + B, checked against the model once: hash eighths, and one key range that takes everything."""
    cache = env["cache"]
    if ("scan", name) not in cache:
        cache.clear()
        a, b = env["a"], env["b"]
        if name == "eighths":
            exp = oracle_scan([a, b], EIGHTHS)
            for d, (srcs, (ed, ei)) in enumerate(zip(scan_model([a, b], EIGHTHS), exp[0])):
                check_model(f"scan oracle, eighth {d}", [a, b], srcs, ed, ei)
        else:
            exp = oracle_scan([a, b], [(b"", b"\xff")], scan_oracle.SCAN_KEY)
            check_model("scan oracle, everything", [a, b], [(0, r) for r in range(len(a.keys))] + [(1, r) for r in range(len(b.keys))],
                        *exp[0][0])
        assert exp[1] == (-1, 0, 0)
        cache[("scan", name)] = exp
    return cache[("scan", name)]


def test_scan_device_hash_eighths(engine, big):
    exp = scan_expect(big, "eighths")   # each eighth's file is under 4 GiB; the shared output stream passes 2^32
    rows, stop = _scan_device(engine, big, runs_ptrs(big), EIGHTHS)
    assert rows[-1]["data_off"] > TWO32 or rows[-1]["data_off"] + rows[-1]["data_len"] > TWO32
    _check_scan_dev(big, "scan eighths", rows, stop, exp)


def test_scan_device_one_range_takes_everything(engine, big):
    exp = scan_expect(big, "all")
    assert max_offset(exp[0][0][1]) > TWO32
    rows, stop = _scan_device(engine, big, runs_ptrs(big), [(b"", b"\xff")], capi.SCAN_KEY)
    _check_scan_dev(big, "scan, one destination", rows, stop, exp)


def _damaged(env, r, how):
    a = env["a"]
    bad = a.index.copy()
    rec = bad[16 * r:16 * r + 16]
    if how == "err":   # one byte short of its entry: the entry does not decode
        rec[12:16] = np.array([a.fs[r] - 1], "<u4").view(np.uint8)
    else:              # past the end of .data, high word 2; truncated to 32 bits it would point at the record itself
        rec[0:8] = np.array([(2 << 32) | (int(a.off[r]) & 0xFFFFFFFF)], "<u8").view(np.uint8)
    t = Table(a.data, bad, a.keys, a.ts, a.tomb)
    dev = torch.from_numpy(np.concatenate([bad, np.zeros(16, np.uint8)])).to("cuda:0")
    torch.cuda.synchronize()
    return t, dev


@pytest.mark.parametrize("how,reason", [("err", capi.SCAN_STOP_ERR), ("panic", capi.SCAN_STOP_PANIC)])
def test_scan_device_stops_past_2_32(engine, big, how, reason):
    """An ERR stop at a record past 2^32, and a PANIC stop from an offset past the end of .data with a nonzero high word:
    what precedes the stop is delivered, nothing after it."""
    a, b = big["a"], big["b"]
    big["cache"].clear()
    r = a.record_at(TWO32 + 2 * MiB)
    assert a.off[r] > TWO32
    t, dev = _damaged(big, r, how)
    exp = oracle_scan([t, b], EIGHTHS)
    assert exp[1] == (0, reason, r)
    for d, (srcs, (ed, ei)) in enumerate(zip(scan_model([t, b], EIGHTHS, upto=(0, r)), exp[0])):
        check_model(f"scan oracle, {how} stop, eighth {d}", [t, b], srcs, ed, ei)
    tables = [(big["a_dev"].data_ptr(), a.data.size, dev.data_ptr(), a.index.size)] + runs_ptrs(big, ("b",))
    rows, stop = _scan_device(engine, big, tables, EIGHTHS)
    _check_scan_dev(big, f"scan, {how} stop", rows, stop, exp)


def _scan_stream_into(engine, tables, ranges, kind, sizes):
    """dbeel_scan_stream with in-memory files; every destination's files are preallocated at `sizes` ((data, index) per
    destination; a piece past them is an error), so no 4 GiB file is grown or copied."""
    keep = [(t.data, t.index) for t in tables]
    arr = (capi.Table * len(keep))()
    for j, (d, i) in enumerate(keep):
        arr[j] = capi.Table(None, d.size, None, i.size, None, 0)
    rptr, _rkeep = capi.pack_ranges(kind, ranges)
    n = len(ranges)
    outs = [{1: np.zeros(max(1, ds), np.uint8), 2: np.zeros(max(1, xs), np.uint8)} for ds, xs in sizes]

    def rd(_ctx, table, kind_, off, size, dst):
        src = keep[table][0] if kind_ == 1 else keep[table][1]
        if off + size > src.size:
            return 4243
        C.memmove(dst, src.ctypes.data + off, size)
        return 0

    def wr(_ctx, dest, kind_, off, src, size):
        if dest >= n or kind_ not in (1, 2) or off + size > outs[dest][kind_].size:
            return 4244
        C.memmove(outs[dest][kind_].ctypes.data + off, src, size)
        return 0

    io = capi.ScanIO(capi.STREAM_READ_FN(rd), capi.SCAN_WRITE_FN(wr), None)
    res = (capi.JobResult * n)()
    stop = capi.ScanStop()
    engine._check(capi.lib().dbeel_scan_stream(engine._h, arr, len(keep), kind, rptr, n, C.byref(io), res, C.byref(stop)),
                  "dbeel_scan_stream")
    return [(o[1][:r.data_len], o[2][:r.index_len]) for o, r in zip(outs, res[:n])], stop.as_tuple(), engine.stats()


@pytest.mark.parametrize("ring", [None, 2, 3])
def test_scan_stream(big, monkeypatch, ring):
    """dbeel_scan_stream at the default partition budget: windows start past 2^32 and the one destination's offsets cross
    it; rings of 2 and 3 slots.  The output is compared with the model (every record of A, then of B), which the scan
    oracle's output for the same range was checked against, so no oracle copy is held next to it."""
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    monkeypatch.delenv("DBEEL_PARTITION_KB", raising=False)
    if ring is None:
        monkeypatch.delenv("DBEEL_STREAM_RING", raising=False)
    else:
        monkeypatch.setenv("DBEEL_STREAM_RING", str(ring))
    a, b = big["a"], big["b"]
    big["cache"].clear()
    eng = capi.Engine(0)
    try:
        got, stop, st = _scan_stream_into(eng, [a, b], [(b"", b"\xff")], capi.SCAN_KEY,
                                          [(a.data.size + b.data.size, a.index.size + b.index.size)])
    finally:
        eng.close()
    assert st["partitions"] > 8 and stop == (-1, 0, 0)
    srcs = [(0, r) for r in range(len(a.keys))] + [(1, r) for r in range(len(b.keys))]
    check_model(f"scan stream, ring {ring}", [a, b], srcs, got[0][0], got[0][1])


# --------------------------------------------------------------------------------------------------------------- lookups


def test_get_many_device_around_the_boundaries(engine, big):
    """Keys of the entries on both sides of 2^31 and 2^32 and of fillers, and keys between them (most absent from both
    runs; B holds the ones that follow the 0x30 fillers), in both modes."""
    a, b, m = big["a"], big["b"], big["marks"]
    big["cache"].clear()
    near = []
    for c in (m["straddle31"], m["straddle32"]):
        near += list(range(c - 40, c + 40))
    near += m["fillers"] + [len(a.keys) - 1]
    between = [a.keys[r] + b"\x00" for r in near[::3]]
    keys = [a.keys[r] for r in near] + between + [b"", b"\xff" * 9, b"\x60"]
    assert sum(k not in a.rec_of and k not in b.rec_of for k in between) > 40
    blob, koff = capi.pack_keys(keys)
    et, er, ej = oracle.get_many([(a.data, a.index, None), (b.data, b.index, None)], blob, koff)
    assert any(int(a.off[a.rec_of[k]]) > TWO32 for k, t in zip(keys, et) if t == 0 and k in a.rec_of)
    d_keys = torch.from_numpy(np.concatenate([blob, np.zeros(16, np.uint8)])).to("cuda:0")
    d_koff = torch.from_numpy(koff.view(np.int64)).to("cuda:0")
    res = torch.zeros(16 * len(keys), dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    tables = [(p[0], p[1], p[2], p[3], 0, 0) for p in runs_ptrs(big)]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        engine.get_many_device(tables, d_keys.data_ptr(), d_koff.data_ptr(), len(keys), res.data_ptr(), mode)
        torch.cuda.synchronize()
        got = res.cpu().numpy().view(capi.LOOKUP_DTYPE)
        if mode == capi.LOOKUP_REFERENCE:
            assert np.array_equal(got["table"], et) and np.array_equal(got["bloom_rejects"], ej)
            assert np.array_equal(np.where(got["table"] >= 0, got["record"], 0), er)
        else:   # every present key is found, in the newest table that holds it
            for k, g in zip(keys, got):
                want = (1, b.rec_of[k]) if k in b.rec_of else (0, a.rec_of[k]) if k in a.rec_of else (-1, None)
                assert int(g["table"]) == want[0] and (want[1] is None or int(g["record"]) == want[1]), k
