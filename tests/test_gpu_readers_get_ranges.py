"""Range reads across readers (dbeel_readers_get_ranges): the limited range-read batches of many readers, forward and
reverse, in one call.  Every batch's (rows, data, index) equal its solo Reader.get_ranges(..., reverse=...), the raw
output equals the solo outputs concatenated with .index offsets and `first` shifted, each read goes through its own
reader's callback and page cache and lies inside what the solo calls read, and errors leave every reader usable."""
import ctypes as C
import os

import numpy as np
import pytest

import range_limit_oracle as rlo
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS
from scan_cases import DAMAGES, damage, key_ranges, random_tree
from test_gpu_reader_get_range import EVERYTHING, _sorted, random_ranges

pytestmark = pytest.mark.gpu


@pytest.fixture
def small_engine(monkeypatch):
    """An engine whose partitions and leaf groups are 4 KB: seeks and rounds spread over many groups."""
    monkeypatch.setenv("DBEEL_PARTITION_KB", "4")
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    e = capi.Engine(0)
    yield e
    e.close()


def _limits(limits, n):
    return np.ascontiguousarray(np.full(n, limits, np.uint32) if isinstance(limits, (int, np.integer))
                                else np.array([int(x) for x in limits], np.uint32))


def raw_call(e, batches, caps=None):
    """dbeel_readers_get_ranges straight through ctypes, outputs behind 0xAB guard bytes: (rc, rows, od, oi, out)."""
    arr = (capi.RangeBatch * len(batches))()
    keep, n = [], 0
    for j, (r, ranges, limits, reverse, kt) in enumerate(batches):
        blob, off = capi.pack_keys([bytes(k) for pair in ranges for k in pair])
        lim = _limits(limits, len(ranges))
        keep.append((blob, off, lim))
        arr[j] = capi.RangeBatch(r._h, capi.KeyRanges(blob.ctypes.data if blob.size else None, off.ctypes.data),
                                 lim.ctypes.data, len(ranges), capi.RANGE_KEEP_TOMBSTONES if kt else 0, int(reverse), 0)
        n += len(ranges)
    rows = np.zeros(max(1, n), capi.RANGE_ROW_DTYPE)
    dc, ic = caps or (64 << 20, 16 << 20)
    od, oi = np.full(max(1, dc), 0xAB, np.uint8), np.full(max(1, ic), 0xAB, np.uint8)
    out = capi.Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
    rc = capi.lib().dbeel_readers_get_ranges(e._h, arr, len(batches), C.byref(out), rows.ctypes.data)
    return rc, rows[:n], od, oi, out


def concat(solos):
    """The solo outputs as one call packs them: rows' first and .index offsets shifted, .data appended."""
    rows, data, index, base, items = [], [], [], 0, 0
    for r, d, i in solos:
        r = r.copy()
        r["first"] += np.uint64(items)
        ix = i.copy()
        ix.view("<u8")[0::2] += np.uint64(base)
        rows.append(r)
        data.append(d)
        index.append(ix)
        base, items = base + d.size, items + i.size // 16
    cat = lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt)
    return cat(rows, capi.RANGE_ROW_DTYPE), cat(data, np.uint8), cat(index, np.uint8)


def solo(r, ranges, limits, reverse, kt):
    if not ranges:
        return np.zeros(0, capi.RANGE_ROW_DTYPE), np.zeros(0, np.uint8), np.zeros(0, np.uint8)
    return r.get_ranges(ranges, limits, keep_tombstones=kt, reverse=reverse)


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def check(e, batches):
    """The multi call against the solo calls, batch by batch, and its raw output against their concatenation.
    Returns (solos, multi, multi stats)."""
    multi = e.readers_get_ranges(batches)
    st = e.stats()
    solos = [solo(*b) for b in batches]
    assert len(multi) == len(batches)
    for b, (m, s) in enumerate(zip(multi, solos)):
        assert same(m, s), b
    rc, rows, od, oi, out = raw_call(e, batches)
    assert rc == 0
    cr, cd, ci = concat(solos)
    assert np.array_equal(rows, cr)
    assert np.array_equal(od[:out.data_len], cd) and np.array_equal(oi[:out.index_len], ci)
    assert (od[out.data_len:out.data_len + 64] == 0xAB).all() and (oi[out.index_len:out.index_len + 64] == 0xAB).all()
    assert out.items_written == ci.size // 16
    assert st["entries_out"] == ci.size // 16 and st["output_bytes"] == cd.size + ci.size
    return solos, multi, st


@pytest.mark.parametrize("setting", ["default", "small_partitions", "depth0", "shared_cache"])
def test_parity_on_random_trees(engine, small_engine, setting):
    """Readers of 1 to 6 tables, forward / reverse / mixed batches, keep_tombstones on some, empty batches, and one
    reader in several batches, in the same and opposite directions."""
    e = small_engine if setting == "small_partitions" else engine
    fence_bytes = 1 if setting == "depth0" else 0
    cache = e.open_page_cache(1 << 20) if setting == "shared_cache" else None
    rng = np.random.default_rng(4100)
    trees = [random_tree(rng, 1 + s % 6, max_entries=120, big=s == 5) for s in range(6)]
    trees = [t if s % 2 else _sorted(t) for s, t in enumerate(trees)]
    readers = [e.open_reader([(d, i, None) for d, i in t], fence_bytes=fence_bytes) for t in trees]
    try:
        if cache is not None:
            for r in readers[::2]:
                r.attach_page_cache(cache)
        qs = [key_ranges(t) + random_ranges(rng, t, 20) + EVERYTHING for t in trees]

        def batch(j, reverse, kt=None, limits=None):
            pick = [qs[j][x] for x in rng.permutation(len(qs[j]))[:int(rng.integers(1, len(qs[j]) + 1))]]
            lim = limits if limits is not None else [int(x) for x in rng.integers(1, 40, len(pick))]
            return readers[j], pick, lim, reverse, bool(rng.integers(0, 2)) if kt is None else kt

        for rnd in range(2):  # the call that loads the fences, then one on loaded fences
            for rev in (False, True):
                check(e, [batch(j, rev) for j in range(len(trees))])
            check(e, [batch(j, bool(j % 2)) for j in range(len(trees))])
            mixed = [batch(j, bool(rng.integers(0, 2))) for j in range(len(trees))]
            mixed.insert(2, (readers[1], [], 1, False, False))
            mixed.append((readers[0], [], 1, True, True))
            check(e, mixed)
            for lim in (1, 10, 100):
                check(e, [batch(0, False, limits=lim), batch(0, True, limits=lim), batch(5, True, False, lim),
                          batch(0, False, True, lim), batch(5, True, True, lim)])
    finally:
        for r in readers:
            r.close()
        if cache is not None:
            cache.close()


def _table(keys, value=b"v", ts=BASE_TS):
    d, i = sstable.build_run([(k, value, ts) for k in keys])
    return np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy()


def test_tombstone_wall_beside_one_round_batches(engine):
    """One batch whose merge a run of 20,000 tombstones holds back for many rounds, beside batches that finish in one:
    every row is its solo row, and the call runs fewer rounds than the solo calls together."""
    keys = [b"k%08d" % j for j in range(40000)]
    wall = [_table(keys), _table(keys[:20000], b"", BASE_TS + 1)]
    rng = np.random.default_rng(4101)
    small = [_sorted(random_tree(rng, 3, max_entries=80)) for _ in range(3)]
    with engine.open_reader([(d, i, None) for d, i in wall]) as w:
        others = [engine.open_reader([(d, i, None) for d, i in t]) for t in small]
        try:
            batches = [(w, EVERYTHING, 10, False, False)]
            batches += [(r, key_ranges(t) + EVERYTHING, 5, bool(j % 2), False) for j, (r, t) in enumerate(zip(others, small))]
            batches.append((w, [(b"k00019990", b"k00030000")], 10, True, False))
            solos, multi, st = check(engine, batches)
            rounds = 0
            for b in batches:
                solo(*b)
                rounds += engine.stats()["partitions"]
            assert int(multi[0][0][0]["count"]) == 10 and int(multi[0][0][0]["flags"]) == rlo.MORE
            assert st["partitions"] < rounds, (st["partitions"], rounds)
        finally:
            for r in others:
                r.close()


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage_in_one_readers_table(engine, kind):
    """Every damage kind of the solo tests in table 1 of one reader: that batch's rows are its solo rows, and the healthy
    batches beside it, in both directions, are what they are alone."""
    if kind == "ragged_index":  # a reader takes whole index records only
        return
    rng = np.random.default_rng(4200 + DAMAGES.index(kind))
    tables = _sorted(random_tree(rng, 3, max_entries=80))
    healthy = [_sorted(random_tree(rng, 2, max_entries=80)) for _ in range(2)]
    hr = [engine.open_reader([(d, i, None) for d, i in t]) for t in healthy]
    try:
        hb = [(r, key_ranges(t) + EVERYTHING, 7, bool(j), False) for j, (r, t) in enumerate(zip(hr, healthy))]
        alone = [solo(*b) for b in hb]
        for rec in ((0,) if kind == "empty_table" else (0, 5, 40)):
            bad = damage(tables, kind, 1, rec)
            with engine.open_reader([(d, i, None) for d, i in bad]) as r:
                ranges = key_ranges(bad) + random_ranges(rng, bad, 20) + EVERYTHING
                for limits in (1, 3, 1000):
                    for rev in (False, True):
                        _, multi, _ = check(engine, [hb[0], (r, ranges, limits, rev, False), hb[1]])
                        assert same(multi[0], alone[0]) and same(multi[2], alone[1])
                        if kind == "empty_table":  # only the batch of the reader with the empty table stops
                            assert (multi[1][0]["flags"] == rlo.STOPPED).all()
                            assert not (multi[0][0]["flags"] & rlo.STOPPED).any() and not (multi[2][0]["flags"] & rlo.STOPPED).any()
    finally:
        for r in hr:
            r.close()


def _covered(reads, union):
    """Every read [off, off + size) of (table, kind) lies inside the union of union's reads of that table and kind."""
    for t, kind, off, size in reads:
        spans = sorted((o, o + s) for t2, k2, o, s in union if t2 == t and k2 == kind)
        at = off
        for lo, hi in spans:
            if lo <= at < hi:
                at = max(at, hi)
            if at >= off + size:
                break
        assert at >= off + size or size == 0, (t, kind, off, size)


@pytest.mark.parametrize("budget", ["default", "small"])
def test_reads_stay_inside_the_solo_calls_reads(engine, small_engine, budget):
    """Fresh readers, twice: once for the solo calls in batch order, once for the multi call.  Every read of the multi
    call lies inside the union of the solo calls' reads of that reader, table and file kind, and input_bytes is at most
    their sum; then the same on loaded fences."""
    e = engine if budget == "default" else small_engine
    rng = np.random.default_rng(4300)
    trees = [_sorted(random_tree(rng, n, max_entries=150)) for n in (1, 4, 6)]
    batches_of = lambda rs: [(r, key_ranges(t) + random_ranges(np.random.default_rng(9 + j), t, 30) + EVERYTHING,
                              [1, 10, 100][j], bool(j % 2), j == 2) for j, (r, t) in enumerate(zip(rs, trees))]
    open_all = lambda: [e.open_reader([(d, i, None) for d, i in t]) for t in trees]
    first = open_all()
    union, total = [], 0
    for b in batches_of(first):
        solo(*b)
        total += e.stats()["input_bytes"]
        union.append(list(b[0].last_stream_reads))
    multi = open_all()
    e.readers_get_ranges(batches_of(multi))
    assert e.stats()["input_bytes"] <= total
    for r, u in zip(multi, union):
        _covered(r.last_stream_reads, u)
    # on loaded fences: the multi call reads what the solo calls on loaded fences read, no more
    union, total = [], 0
    for b in batches_of(first):
        solo(*b)
        total += e.stats()["input_bytes"]
        union.append(list(b[0].last_stream_reads))
    e.readers_get_ranges(batches_of(multi))
    assert e.stats()["input_bytes"] <= total
    for r, u in zip(multi, union):
        _covered(r.last_stream_reads, u)
    for r in first + multi:
        r.close()


def test_warm_page_cache_reads_nothing(engine):
    """Readers of short keys, whose loaded fences serve every bound, on one page cache: a repeated call reads nothing."""
    keys = [b"k%08d" % j for j in range(20000)]
    sets = [[_table(keys[j::3], b"x" * 40, BASE_TS + t) for t in range(n)] for j, n in enumerate((1, 4, 2))]
    rs = [engine.open_reader([(d, i, None) for d, i in t]) for t in sets]
    rng = np.random.default_rng(4301)
    whole = [(b"", b"\xff" * 16)]
    batches = [(r, whole + [(keys[j], keys[j] + b"\xff") for j in rng.integers(0, len(keys), 16)], 10, b == 1, False)
               for b, r in enumerate(rs)]
    try:
        for r in rs:  # the exact-mode fences, loaded before the cache is attached
            r.get_ranges(whole, 1)
        with engine.open_page_cache(64 << 20) as cache:
            for r in rs:
                r.attach_page_cache(cache)
            a = engine.readers_get_ranges(batches)
            b = engine.readers_get_ranges(batches)
            assert engine.stats()["input_bytes"] == 0 and not any(r.last_stream_reads for r in rs)
            assert all(same(x, y) for x, y in zip(a, b))
            for r in rs:
                r.attach_page_cache(None)
        check(engine, batches)
    finally:
        for r in rs:
            r.close()


def test_tree_reader_snapshots(engine, tmp_path):
    """Tree readers on snapshots before and after a flush and a compaction, in one call, both directions."""
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(4400)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    kr = [(b"t00500", b"t01800"), (b"t02990", b"u"), (b"a", b"t00010"), (b"t00599", b"t00700")]
    a = tree.open_reader()
    before = [a.get_ranges(kr, 5), a.get_ranges(kr, 5, reverse=True)]
    tree.flush(sstable.build_run([(b"t00600", b"new", BASE_TS + 10 ** 6)]))
    b = tree.open_reader()
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    c = tree.open_reader()
    try:
        batches = [(a, kr, 5, False, False), (b, kr, 5, True, False), (c, kr, 5, False, True), (a, kr, 5, True, False)]
        _, multi, _ = check(engine, batches)
        assert same(multi[0], before[0]) and same(multi[3], before[1])
        rows, data, index = multi[2]
        assert (b"t00600", b"new") in [(k, v) for k, v, _ in sstable.parse_run(data, index)]
    finally:
        for x in (a, b, c):
            x.close()
        tree.close()


def test_capacity_callback_and_argument_errors(engine):
    rng = np.random.default_rng(4500)
    trees = [_sorted(random_tree(rng, n, max_entries=100)) for n in (3, 2)]
    rs = [engine.open_reader([(d, i, None) for d, i in t]) for t in trees]
    batches = [(r, key_ranges(t) + EVERYTHING, 50, bool(j), False) for j, (r, t) in enumerate(zip(rs, trees))]
    try:
        solos, _, _ = check(engine, batches)
        cr, cd, ci = concat(solos)
        assert cd.size and ci.size
        for caps in ((cd.size - 1, ci.size), (cd.size, ci.size - 1)):
            rc, rows, od, oi, out = raw_call(engine, batches, caps)
            assert rc == capi.ERR_CAPACITY and (out.data_len, out.index_len) == (cd.size, ci.size)
            assert np.array_equal(rows, cr)  # every row filled
            assert (od == 0xAB).all() and (oi == 0xAB).all()  # nothing written
            with pytest.raises(capi.DbeelError) as ei:
                engine.readers_get_ranges(batches, caps=caps)
            assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (cd.size, ci.size)
        # one reader's callback fails mid-call: its code comes back, and every reader answers exactly afterwards
        engine.readers_get_ranges(batches)
        n_reads = len(rs[1].last_stream_reads)
        for at in sorted({0, n_reads // 2, max(0, n_reads - 1)}):
            with pytest.raises(capi.DbeelError) as ei:
                engine.readers_get_ranges(batches, fail_read_at={rs[1]: at})
            assert ei.value.code == 4242
            check(engine, batches)
        # invalid arguments, one per rule
        L = capi.lib()
        blob, off = capi.pack_keys([b"a", b"m", b"b", b"z"])
        lim = np.ones(2, np.uint32)
        good = lambda r=rs[0]: capi.RangeBatch(r._h, capi.KeyRanges(blob.ctypes.data, off.ctypes.data), lim.ctypes.data, 2, 0, 0, 0)
        arr = (capi.RangeBatch * 2)()
        rows = np.zeros(4, capi.RANGE_ROW_DTYPE)
        od, oi = np.empty(1 << 16, np.uint8), np.empty(1 << 16, np.uint8)
        out = capi.Out(od.ctypes.data, od.size, 0, oi.ctypes.data, oi.size, 0, None, 0, 0, 0)
        call = lambda a=arr, n=2, o=C.byref(out), res=rows.ctypes.data: L.dbeel_readers_get_ranges(engine._h, a, n, o, res)
        arr[0], arr[1] = good(), good(rs[1])
        assert call() == 0
        assert call(a=None) == capi.ERR_INVALID_ARG
        assert call(o=None) == capi.ERR_INVALID_ARG
        assert call(res=None) == capi.ERR_INVALID_ARG
        assert call(n=0) == capi.ERR_INVALID_ARG
        big = (capi.RangeBatch * (capi.MAX_READER_BATCHES + 1))(*([good()] * (capi.MAX_READER_BATCHES + 1)))
        many_rows = np.zeros(2 * capi.MAX_READER_BATCHES + 2, capi.RANGE_ROW_DTYPE)
        od2, oi2 = np.empty(1 << 20, np.uint8), np.empty(1 << 20, np.uint8)
        out2 = capi.Out(od2.ctypes.data, od2.size, 0, oi2.ctypes.data, oi2.size, 0, None, 0, 0, 0)
        for nb, want in ((capi.MAX_READER_BATCHES + 1, capi.ERR_INVALID_ARG), (capi.MAX_READER_BATCHES, 0)):
            assert L.dbeel_readers_get_ranges(engine._h, big, nb, C.byref(out2), many_rows.ctypes.data) == want
        bad_off = np.array([0, 2, 1, 3, 4], np.uint64)  # decreasing
        zero, over = np.array([1, 0], np.uint32), np.array([1, capi.RANGE_LIMIT_MAX + 1], np.uint32)
        for field, value in (("reader", None), ("limits", None), ("flags", 0x2), ("flags", 0x4), ("reverse", 2),
                             ("reserved", 1), ("limits", zero.ctypes.data), ("limits", over.ctypes.data),
                             ("ranges", capi.KeyRanges(blob.ctypes.data, None)),
                             ("ranges", capi.KeyRanges(None, off.ctypes.data)),
                             ("ranges", capi.KeyRanges(blob.ctypes.data, bad_off.ctypes.data))):
            arr[0], arr[1] = good(), good(rs[1])
            setattr(arr[1], field, value)
            assert call() == capi.ERR_INVALID_ARG, field
        # the limits of all batches sum to 2^32 - 16 or more
        huge_blob, huge_off = capi.pack_keys([b"a", b"b"] * 65536)
        huge_lim = np.full(65536, capi.RANGE_LIMIT_MAX, np.uint32)
        huge = lambda r: capi.RangeBatch(r._h, capi.KeyRanges(huge_blob.ctypes.data, huge_off.ctypes.data), huge_lim.ctypes.data,
                                         32768, 0, 0, 0)
        arr[0], arr[1] = huge(rs[0]), huge(rs[1])
        assert call() == capi.ERR_INVALID_ARG
        other = capi.Engine(0)
        try:
            foreign = other.open_reader([(d, i, None) for d, i in trees[0]])
            arr[0], arr[1] = good(), good(foreign)
            assert call() == capi.ERR_INVALID_ARG
            foreign.close()
        finally:
            other.close()
        # a batch of no ranges needs neither key_offsets nor limits
        arr[0], arr[1] = good(), capi.RangeBatch(rs[1]._h, capi.KeyRanges(None, None), None, 0, 0, 1, 0)
        assert call() == 0
        check(engine, batches + [(rs[0], [], 1, False, False)])
    finally:
        for r in rs:
            r.close()
