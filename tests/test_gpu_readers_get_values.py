"""Batched reads across readers (dbeel_readers_get_values): the point-read batches of many readers in one call.  Every
batch's (rows, data, index) equal its solo Reader.get_values, the packed output equals their concatenation, each read
goes through its own reader's callback and page cache and lies inside what the solo calls read, and errors leave every
reader usable."""
import ctypes as C
import os
from collections import Counter

import numpy as np
import pytest

from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS, assert_run_equal
from test_gpu_get_values import _rec, _set_u32
from test_gpu_get_values_stream import all_cases, case_four_overlapping
from test_gpu_reader import fence_positions, reader_depth

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


def fence_reads(reads, mode, n):
    """.index reads that start at a fence of the deepest probe tree a reader could cache (test_gpu_reader.fence_reads):
    fences read per call start at one, a leaf slice of a batch that descends the cached fences never does."""
    fences = fence_positions(mode, n, reader_depth(n))
    return [x for x in reads if x[1] == 2 and x[2] // 16 in fences]


def raw_call(e, batches, caps=None):
    """dbeel_readers_get_values straight through ctypes: (rc, rows, data, index, out) with the packed output."""
    arr = (capi.ReaderBatch * len(batches))()
    keep = []
    for j, (r, keys, mode) in enumerate(batches):
        blob, off = capi.pack_keys(list(keys))
        keep.append((blob, off))
        arr[j] = capi.ReaderBatch(r._h, blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys), mode, 0)
    n = sum(len(k) for _, k, _ in batches)
    rows = np.zeros(max(1, n), capi.LOOKUP_DTYPE)
    dc, ic = caps or (64 << 20, 16 * n + 16)
    od, oi = np.full(max(1, dc), 0xAB, np.uint8), np.full(max(1, ic), 0xAB, np.uint8)
    out = capi.Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
    rc = capi.lib().dbeel_readers_get_values(e._h, arr, len(batches), C.byref(out), rows.ctypes.data)
    return rc, rows[:n], od, oi, out


def concat(solos):
    """The solo outputs packed as one call packs them: .data appended, .index offsets shifted."""
    data, index, base = [], [], 0
    for _, d, i in solos:
        ix = i.copy()
        ix.view("<u8")[0::2] += np.uint64(base)
        data.append(d)
        index.append(ix)
        base += d.size
    return (np.concatenate(data) if data else np.zeros(0, np.uint8)), (np.concatenate(index) if index else np.zeros(0, np.uint8))


def check(e, batches):
    """The multi call against the solo calls, batch by batch, and its packed output against their concatenation.
    Returns (solos, multi, multi stats)."""
    multi = e.readers_get_values(batches)
    st = e.stats()
    solos = [r.get_values(keys, mode) for r, keys, mode in batches]
    assert len(multi) == len(batches)
    for b, ((rows, d, i), (sr, sd, si)) in enumerate(zip(multi, solos)):
        assert np.array_equal(rows, sr), b
        assert_run_equal((d, i), (sd, si), f"batch {b}")
    n = sum(len(k) for _, k, _ in batches)
    rc, rows, od, oi, out = raw_call(e, batches)
    assert rc == 0
    cd, ci = concat(solos)
    assert np.array_equal(rows, np.concatenate([s[0] for s in solos]) if solos else rows)
    assert np.array_equal(od[:out.data_len], cd) and np.array_equal(oi[:out.index_len], ci)
    assert out.items_written == ci.size // 16
    assert st["entries_in"] == n and st["entries_out"] == ci.size // 16 and st["output_bytes"] == cd.size + ci.size
    return solos, multi, st


def version_stack(n_tables, n=600, seed=0):
    """n_tables overlapping tables of the same key space, newest last, with tombstone-free distinct values."""
    rng = np.random.default_rng(seed)
    tables = []
    for t in range(n_tables):
        ks = sorted(set(int(x) for x in rng.integers(0, 2 * n, n)))
        d, i = sstable.build_run([(b"s%05d" % k, b"t%d-%d" % (t, k) * int(rng.integers(1, 4)), BASE_TS + t) for k in ks])
        tables.append((d, i, None))
    return tables, [b"s%05d" % k for k in range(0, 2 * n, 3)] + [b"zz", b""]


@pytest.mark.parametrize("budget", ["default", "tiny"])
def test_parity_on_every_case(engine, tiny_engine, budget):
    """Every table set of the stream's tests as its own reader; one, two and all of them in one call, mixed modes, empty
    batches and keys asked twice, readers of one and of six tables together."""
    e = engine if budget == "default" else tiny_engine
    rng = np.random.default_rng(51)
    cases = all_cases(engine)
    six, six_keys = version_stack(6)
    one, one_keys = version_stack(1, seed=1)
    cases += [(six, six_keys), (one, one_keys)]
    readers = [e.open_reader(t) for t, _ in cases]
    try:
        def batch(j, mode=None):
            keys = cases[j][1]
            pick = [keys[x] for x in rng.permutation(len(keys))[:max(1, len(keys) // 2)]] if keys else []
            return readers[j], pick + pick[:3], int(rng.integers(0, 2)) if mode is None else mode
        for rnd in range(2):  # the call that loads fences, then one that uses them
            for j in range(len(cases)):
                check(e, [batch(j)])
            for j in range(len(cases) - 1):
                check(e, [batch(j, MODES[rnd]), batch(j + 1, MODES[1 - rnd])])
            many = [batch(j) for j in range(len(cases))]
            many.insert(3, (readers[0], [], capi.LOOKUP_EXACT))
            many.append((readers[-2], six_keys, capi.LOOKUP_REFERENCE))
            check(e, many)
    finally:
        for r in readers:
            r.close()


def test_damage_in_one_readers_table(engine):
    """The four damage kinds at fences and inside leaves of one reader's table: that batch's rows are its solo call's,
    and the healthy batches beside it are what they are alone."""
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    keys = [k for k, _, _ in ents[::7]] + [b"key-%06dx" % n for n in range(0, 2000, 13)]
    healthy, hkeys = version_stack(3, seed=5)
    rng = np.random.default_rng(52)
    fences = sorted(fence_positions(0, 2000, 4) | fence_positions(1, 2000, 4))
    with engine.open_reader(healthy) as h1, engine.open_reader([(d, i, None)]) as h2:
        for r in list(rng.choice(2000, 3, replace=False)) + fences[:4] + [0, 1999]:
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
                with engine.open_reader(healthy + [(bd, bi, None)]) as bad:
                    for mode in MODES:
                        for _ in range(2):
                            batches = [(h1, hkeys, mode), (bad, keys + [ents[int(r)][0]], mode), (h2, keys, 1 - mode)]
                            solos, _, _ = check(engine, batches)
                            # the healthy batches are unaffected: what they answer in a call of their own
                            alone = engine.readers_get_values([batches[0], batches[2]])
                            for a, s in zip(alone, (solos[0], solos[2])):
                                assert np.array_equal(a[0], s[0]) and np.array_equal(a[1], s[1]) and np.array_equal(a[2], s[2])


def test_shared_and_repeated_readers(engine, tmp_path):
    tables, keys = case_four_overlapping(engine)
    with engine.open_reader(tables) as r:
        for mode in MODES:
            check(engine, [(r, keys, mode), (r, keys[::2], 1 - mode), (r, keys, mode)])
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(53)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    tkeys = [b"t%05d" % n for n in range(0, 3100, 7)] + [b"t00001", b"t00001"]
    a = tree.open_reader()
    before = {m: a.get_values(tkeys, m) for m in MODES}
    tree.flush(sstable.build_run([(b"t00007", b"new", BASE_TS + 9000), (b"u", b"x", BASE_TS)]))
    b = tree.open_reader()  # shares A's three tables
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    c = tree.open_reader()
    try:
        for mode in MODES:
            solos, multi, _ = check(engine, [(a, tkeys, mode), (b, tkeys, mode), (c, tkeys, 1 - mode), (a, tkeys[:5], mode)])
            assert np.array_equal(multi[0][0], before[mode][0])
            assert_run_equal(multi[0][1:], before[mode][1:], "snapshot A")
    finally:
        for x in (a, b, c):
            x.close()
        tree.close()
    # from the second call on, no cached fence is read
    (d1, i1, _), k1 = (lambda ents: (sstable.build_run(ents) + (None,), [k for k, _, _ in ents]))(
        [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(20000)])
    with engine.open_reader([(d1, i1, None)]) as r1, engine.open_reader([(d1, i1, None)]) as r2:
        for mode in MODES:
            batches = [(r1, k1[::37], mode), (r2, k1[5::41], mode)]
            engine.readers_get_values(batches)
            for _ in range(2):
                engine.readers_get_values(batches)
                for r in (r1, r2):
                    assert not fence_reads(r.last_stream_reads, mode, 20000)


def test_reads_stay_inside_the_solo_calls_reads(engine, tiny_engine):
    """Fresh readers, twice: once for the solo calls in batch order, once for the multi call.  Every read of the multi call
    lies inside the union of the solo calls' reads of that reader's table and file kind, and input_bytes is at most
    their sum."""
    rng = np.random.default_rng(54)
    sets = [case_four_overlapping(engine), version_stack(6, n=3000, seed=7), version_stack(1, n=5000, seed=8)]
    for e in (engine, tiny_engine):
        for mode in MODES:
            batches_keys = []
            for t, keys in sets:
                pick = [keys[x] for x in rng.permutation(len(keys))[:max(1, len(keys) // 3)]]
                batches_keys.append((t, pick, mode if len(batches_keys) % 2 else 1 - mode))
            solo = [e.open_reader(t) for t, _, _ in batches_keys]
            union, total = [], 0
            for r, (_, keys, m) in zip(solo, batches_keys):
                r.get_values(keys, m)
                total += e.stats()["input_bytes"]
                union.append(list(r.last_stream_reads))
            multi = [e.open_reader(t) for t, _, _ in batches_keys]
            e.readers_get_values([(r, keys, m) for r, (_, keys, m) in zip(multi, batches_keys)])
            assert e.stats()["input_bytes"] <= total
            for b, r in enumerate(multi):
                for t, kind, off, size in r.last_stream_reads:
                    spans = sorted((o, o + s) for t2, k2, o, s in union[b] if t2 == t and k2 == kind)
                    covered, at = False, off
                    for lo, hi in spans:  # [off, off + size) inside the union of the solo spans
                        if lo <= at < hi:
                            at = hi
                        if at >= off + size:
                            covered = True
                            break
                    assert covered or size == 0, (b, t, kind, off, size)
            for r in solo + multi:
                r.close()


def test_page_caches(engine):
    """Readers sharing one cache, readers with caches of their own, and one reader with none: results equal the uncached
    ones, a repeat call reads nothing through a warm cache, and a cache smaller than one step's pages falls back to
    uncached reads for its readers only."""
    sets = [case_four_overlapping(engine), version_stack(3, n=2000, seed=9), version_stack(2, n=2000, seed=10)]
    plain = [engine.open_reader(t) for t, _ in sets]
    batches = lambda rs: [(r, keys, m) for r, (_, keys), m in zip(rs, sets, (0, 1, 0))]
    ref = engine.readers_get_values(batches(plain))
    with engine.open_page_cache(64 << 20) as big, engine.open_page_cache(64 << 20) as big2, engine.open_page_cache(8192) as small:
        for layout in ("shared", "own", "none_for_one", "small"):
            rs = [engine.open_reader(t) for t, _ in sets]
            caches = {"shared": (big, big, None), "own": (big, big2, None), "none_for_one": (big2, None, big),
                      "small": (small, big, None)}[layout]
            for r, c in zip(rs, caches):
                if c is not None:
                    r.attach_page_cache(c)
            for rnd in range(2):
                got = engine.readers_get_values(batches(rs))
                for g, w in zip(got, ref):
                    assert np.array_equal(g[0], w[0])
                    assert_run_equal(g[1:], w[1:], layout)
                if rnd == 0:
                    continue
                for r, c, w in zip(rs, caches, plain):
                    if c is None:
                        assert r.last_stream_reads  # uncached: reads again
                    elif c is small:  # each step outgrows its cache: read uncached, as the solo call does
                        r.get_values(sets[0][1], 0)
                        assert Counter(r.last_stream_reads)  # reads every time
                    else:
                        assert not r.last_stream_reads, layout  # a warm cache: nothing read
            for r in rs:
                r.close()
    for r in plain:
        r.close()


def test_capacity_callback_and_argument_errors(engine):
    sets = [case_four_overlapping(engine), version_stack(3, seed=11)]
    rs = [engine.open_reader(t) for t, _ in sets]
    batches = [(r, keys, capi.LOOKUP_EXACT) for r, (_, keys) in zip(rs, sets)]
    try:
        solos, multi, _ = check(engine, batches)
        cd, ci = concat(solos)
        for caps in ((cd.size - 1, ci.size), (cd.size, ci.size - 1)):
            rc, rows, od, oi, out = raw_call(engine, batches, caps)
            assert rc == capi.ERR_CAPACITY and (out.data_len, out.index_len) == (cd.size, ci.size)
            assert np.array_equal(rows, np.concatenate([s[0] for s in solos]))  # every row filled
            assert (od[:max(1, caps[0])] == 0xAB).all() and (oi[:max(1, caps[1])] == 0xAB).all()  # nothing written
            with pytest.raises(capi.DbeelError) as ei:
                engine.readers_get_values(batches, caps=caps)
            assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (cd.size, ci.size)
        # one reader's callback fails mid-call: its code comes back, and the next call on every reader is exact
        engine.readers_get_values(batches)
        n_reads = len(rs[1].last_stream_reads)
        for at in (0, n_reads // 2, max(0, n_reads - 1)):
            with pytest.raises(capi.DbeelError) as ei:
                engine.readers_get_values(batches, fail_read_at={rs[1]: at})
            assert ei.value.code == 4242
            check(engine, batches)
        with pytest.raises(capi.DbeelError) as ei:  # a fence load of a fresh reader
            fresh = engine.open_reader(sets[0][0])
            engine.readers_get_values([(fresh, sets[0][1], 0)] + batches, fail_read_at={fresh: 0})
        assert ei.value.code == 4242
        check(engine, [(fresh, sets[0][1], 0)] + batches)
        fresh.close()
        # invalid arguments, one per rule
        L = capi.lib()
        arr = (capi.ReaderBatch * 2)()
        blob, off = capi.pack_keys([b"k1", b"k2"])
        good = lambda r=rs[0]: capi.ReaderBatch(r._h, blob.ctypes.data, off.ctypes.data, 2, 0, 0)
        rows = np.zeros(4, capi.LOOKUP_DTYPE)
        od, oi = np.empty(4096, np.uint8), np.empty(4096, np.uint8)
        out = capi.Out(od.ctypes.data, 4096, 0, oi.ctypes.data, 4096, 0, None, 0, 0, 0)
        call = lambda a=arr, n=2, o=C.byref(out), res=rows.ctypes.data: L.dbeel_readers_get_values(engine._h, a, n, o, res)
        arr[0], arr[1] = good(), good(rs[1])
        assert call() == 0
        assert call(a=None) == capi.ERR_INVALID_ARG
        assert call(o=None) == capi.ERR_INVALID_ARG
        assert call(res=None) == capi.ERR_INVALID_ARG
        assert call(n=0) == capi.ERR_INVALID_ARG
        big = (capi.ReaderBatch * (capi.MAX_READER_BATCHES + 1))(*([good()] * (capi.MAX_READER_BATCHES + 1)))
        many_rows = np.zeros(2 * capi.MAX_READER_BATCHES + 2, capi.LOOKUP_DTYPE)
        od2, oi2 = np.empty(1 << 20, np.uint8), np.empty(1 << 20, np.uint8)
        out2 = capi.Out(od2.ctypes.data, od2.size, 0, oi2.ctypes.data, oi2.size, 0, None, 0, 0, 0)
        for nb, want in ((capi.MAX_READER_BATCHES + 1, capi.ERR_INVALID_ARG), (capi.MAX_READER_BATCHES, 0)):
            assert L.dbeel_readers_get_values(engine._h, big, nb, C.byref(out2), many_rows.ctypes.data) == want
        for field, value in (("reader", None), ("mode", 2), ("reserved", 1), ("key_offsets", None), ("keys", None)):
            arr[0], arr[1] = good(), good(rs[1])
            setattr(arr[1], field, value)
            assert call() == capi.ERR_INVALID_ARG, field
        huge = np.zeros(2, np.uint64)
        arr[0], arr[1] = good(), capi.ReaderBatch(rs[1]._h, None, huge.ctypes.data, (1 << 32) - 16, 0, 0)
        assert call() == capi.ERR_INVALID_ARG  # 2^32 - 16 keys in all (offsets never read: refused first)
        other = capi.Engine(0)
        try:
            foreign = other.open_reader(sets[0][0])
            arr[0], arr[1] = good(), good(foreign)
            assert call() == capi.ERR_INVALID_ARG
            foreign.close()
        finally:
            other.close()
        check(engine, batches + [(rs[0], [], capi.LOOKUP_REFERENCE)])
    finally:
        for r in rs:
            r.close()
