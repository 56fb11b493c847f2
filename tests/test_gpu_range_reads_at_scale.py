"""The reader's key-range reads at the sizes where their counting kernels change path, against the vectorised model of
tests/range_scale_model.py, byte for byte:

* k_range_tile_scan carries a running total across chunks of 1024 tiles of 1024 records: get_range spans and limit rounds
  of more than 2^20 records (one partition, one round -- each case asserts the size it reached from the stats);
* k_route_scan carries across chunks of 1024 blocks of 256 records: reader partitions of more than 262,144 records;
* k_range_flag / k_range_rank search across 256 uneven destination segments; k_limit_query / k_limit_rank run rounds of
  more than 256 queries;
* the shared-prefix key shape makes every 8-byte key prefix tie, so every comparison of those searches falls through to
  the full key comparison.

One engine with a 1 GiB partition budget serves the whole module, so a single partition or round holds several million
records; every large tree is built once per module."""
import os

import numpy as np
import pytest

import range_scale_model as m
from dbeel_b200 import capi
from helpers import assert_run_equal

pytestmark = pytest.mark.gpu

TILE_EDGE = 1 << 20        # 1024 tiles of 1024 records: k_range_tile_scan's second chunk
ROUTE_EDGE = 1024 * 256    # 1024 blocks of 256 records: k_route_scan's second chunk
SIZES = [1023, 1024, 1025, TILE_EDGE - 1, TILE_EDGE, TILE_EDGE + 1, 3 * TILE_EDGE + 5]


@pytest.fixture(scope="module")
def big_engine():
    """An engine whose partitions and range-read groups may hold 1 GiB: one partition takes more than 2^21 records."""
    saved = {k: os.environ.pop(k, None) for k in ("DBEEL_PARTITION_MB", "DBEEL_PARTITION_KB")}
    os.environ["DBEEL_PARTITION_MB"] = "1024"
    try:
        e = capi.Engine(0)
    finally:
        os.environ.pop("DBEEL_PARTITION_MB")
        for k, v in saved.items():
            if v is not None:
                os.environ[k] = v
    yield e
    e.close()


class Built:
    """A model tree, its tables' bytes and its cumulative record counts."""

    def __init__(self, tree: m.Tree, end: int):
        self.tree = tree
        self.tables = tree.built()
        self.end = end
        self.c = m.cumulative(tree, end)

    def reader(self, e):
        return e.open_reader([(d, i, None) for d, i in self.tables])

    def range_of(self, a: int, n: int):
        """A range of exactly n span records starting at or after a."""
        got = m.range_with(self.c, a, n)
        assert got is not None, (a, n)
        return got


def overlapping_tree(n_ids: int, prefix: bytes, seed: int) -> m.Tree:
    """Four tables over the integers [0, n_ids): a dense oldest one, then sparser newer ones that supersede its versions,
    with tombstones in every table."""
    rng = np.random.default_rng(seed)
    ids = np.arange(n_ids, dtype=np.uint64)
    tables = [(ids, ids % 11 == 0)]
    for frac, tomb in ((0.33, 0.2), (0.2, 0.3), (0.12, 0.5)):
        pick = ids[rng.random(n_ids) < frac]
        tables.append((pick, rng.random(pick.size) < tomb))
    return m.Tree(tables, prefix)


@pytest.fixture(scope="module")
def big():
    """~4 million records, default key shape: spans up to 3 * 2^20 + 5."""
    return Built(overlapping_tree(2_400_000, b"", 1), 2_400_000)


@pytest.fixture(scope="module")
def shared():
    """~1.65 million records whose keys all share their first 8 bytes: spans up to 2^20 + 1."""
    return Built(overlapping_tree(1_000_000, m.SHARED_PREFIX, 2), 1_000_000)


WALL_LO, WALL = 100_000, 2_000_000
WALL_END = WALL_LO + WALL + 100_000


@pytest.fixture(scope="module")
def wall():
    """An old table of WALL_END live keys and a newer one that tombstones WALL of them, from WALL_LO on."""
    old = np.arange(WALL_END, dtype=np.uint64)
    new = np.arange(WALL_LO, WALL_LO + WALL, dtype=np.uint64)
    return Built(m.Tree([(old, np.zeros(old.size, bool)), (new, np.ones(new.size, bool))]), WALL_END)


# ---- checks


def check_range(e, r, b: Built, ranges, keep, span_records):
    """get_range against the model, the stop, the stats, and one partition of exactly span_records records."""
    out, stop = r.get_range(b.tree.bounds(ranges), keep_tombstones=keep)
    st = e.stats()
    assert stop == (-1, 0, 0)
    want = b.tree.get_range(ranges, keep)
    for d, (g, w) in enumerate(zip(out, want)):
        assert_run_equal(g, w, f"get_range {d} of {len(ranges)} (keep={keep})")
    assert st["partitions"] == 1 and st["entries_in"] == span_records, (st["partitions"], st["entries_in"], span_records)
    assert st["entries_out"] == sum(g[1].size // 16 for g in out)
    assert st["output_bytes"] == sum(g[0].size + g[1].size for g in out)
    assert st["input_bytes"] == sum(x[3] for x in r.last_stream_reads)
    return out, st


def check_scan(e, r, b: Built, ranges, span_records):
    out, stop = r.scan(b.tree.bounds(ranges))
    st = e.stats()
    assert stop == (-1, 0, 0)
    for d, (g, w) in enumerate(zip(out, b.tree.reader_scan(ranges))):
        assert_run_equal(g, w, f"reader_scan {d} of {len(ranges)}")
    assert st["partitions"] == 1 and st["entries_in"] == span_records, (st["partitions"], st["entries_in"], span_records)
    return out


def check_rows(rows, data, index, want, what=""):
    """rows / data / index of a get_ranges call against the model's answer, byte for byte."""
    (first, count, flags), (wd, wi) = want
    assert np.array_equal(rows["first"].astype(np.int64), first), what
    assert np.array_equal(rows["count"].astype(np.int64), count), what
    assert np.array_equal(rows["flags"].astype(np.int64), flags), what
    assert (rows["table"] == -1).all() and (rows["reason"] == 0).all() and (rows["record"] == 0).all(), what
    assert_run_equal((data, index), (wd, wi), what)


def check_ranges(e, r, b: Built, ranges, limits, keep=False, reverse=False):
    """get_ranges / _reverse against the model, and the read, stats and offset contract of test_gpu_reader_get_ranges."""
    rows, data, index = r.get_ranges(b.tree.bounds(ranges), limits, keep_tombstones=keep, reverse=reverse)
    st, reads = e.stats(), r.last_stream_reads
    check_rows(rows, data, index, b.tree.get_ranges(ranges, limits, keep, reverse), f"get_ranges reverse={reverse}")
    assert index.size == 16 * int(rows["count"].sum())
    assert st["input_bytes"] == sum(x[3] for x in reads)
    assert st["entries_out"] == index.size // 16 and st["output_bytes"] == data.size + index.size
    for t, kind, off, size in reads:
        f = b.tables[t][0] if kind == 1 else b.tables[t][1]
        assert kind in (1, 2) and off + size <= len(f)
    return rows, data, index, st


def row_entries(rows, data, index, q):
    """Query q's entries, as the bytes of each."""
    f, c = int(rows["first"][q]), int(rows["count"][q])
    return entry_list(data, index[16 * f:16 * (f + c)])


def entry_list(data, index):
    ix = np.asarray(index, np.uint8).reshape(-1, 16)
    offs, sizes = ix[:, :8].copy().view("<u8").reshape(-1), ix[:, 12:16].copy().view("<u4").reshape(-1)
    return [bytes(data[int(o):int(o) + int(z)]) for o, z in zip(offs, sizes)]


def disjoint_batches(ranges, width=256):
    """The ranges, sorted, in batches of at most `width` pairwise disjoint ones."""
    batches = []
    for x in sorted(ranges):
        for bt in batches:
            if len(bt) < width and bt[-1][1] <= x[0]:
                bt.append(x)
                break
        else:
            batches.append([x])
    return batches


def cross_check(r, b: Built, ranges, rows, data, index, reverse=False):
    """Every query whose row holds its whole G_q (no MORE) returns exactly what get_range returns for its range alone
    (reversed, for a reverse row): the two merge chains against each other.  Returns how many rows were compared."""
    qs = [q for q in range(len(ranges)) if not int(rows["flags"][q]) and ranges[q][0] < ranges[q][1]]
    seen = {}
    for q in qs:
        seen.setdefault(ranges[q], []).append(q)
    for part in disjoint_batches(seen):
        out, stop = r.get_range(b.tree.bounds(part))
        assert stop == (-1, 0, 0)
        for rng_, (gd, gi) in zip(part, out):
            want = entry_list(gd, gi)
            if reverse:
                want = want[::-1]
            for q in seen[rng_]:
                assert row_entries(rows, data, index, q) == want, (q, rng_, reverse)
    return len(qs)


# ---- get_range: one destination at the tile-scan edges


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("shape", ["default", "shared_prefix"])
def test_get_range_span_sizes(big_engine, big, shared, shape, n):
    b = big if shape == "default" else shared
    if n > 2 * TILE_EDGE and shape == "shared_prefix":
        pytest.skip("the shared-prefix tree stops at 2^20 + 1 records")
    a, z = b.range_of(7 + n % 1000, n)
    with b.reader(big_engine) as r:
        for keep in (False, True):
            check_range(big_engine, r, b, [(a, z)], keep, n)
        if n <= 2048:
            rows, data, index, _ = check_ranges(big_engine, r, b, [(a, z)], capi.RANGE_LIMIT_MAX)
            assert cross_check(r, b, [(a, z)], rows, data, index) == 1


def test_get_range_page_cache(big_engine, big):
    """The 3 * 2^20 + 5 span with a page cache, twice: the same bytes, and the second call reads nothing the first did
    not (its bound searches come from the cache)."""
    n = SIZES[-1]
    a, z = big.range_of(100, n)
    with big_engine.open_page_cache(1 << 30) as cache, big.reader(big_engine) as r:
        r.attach_page_cache(cache)
        first, _ = check_range(big_engine, r, big, [(a, z)], False, n)
        reads1 = list(r.last_stream_reads)
        second, _ = check_range(big_engine, r, big, [(a, z)], False, n)
        assert set(r.last_stream_reads) <= set(reads1)
        assert cache.stats()["hits"] > 0
        for g, w in zip(second, first):
            assert_run_equal(g, w, "cached get_range")


# ---- 256 destinations


def uneven_ranges(b: Built, rng, n_ranges=256):
    """n_ranges disjoint ranges in shuffled order: empty ones (inverted, past every key), a 1-record one, segments at
    k * 1024 +- 1 and one above 2^20, the rest random; records in no range lie between them.  Returns (ranges, records)."""
    sizes = [1, 1023, 1024, 1025, 2047, 2048, 2049, 3071, 3072, 3073, TILE_EDGE + 3]
    sizes += [int(x) for x in rng.integers(1, 3000, n_ranges - len(sizes) - 2)]
    rng.shuffle(sizes)
    ranges, total, a = [], 0, 3
    for n in sizes:
        a, z = b.range_of(a, n)
        ranges.append((a, z))
        total += n
        a = z + int(rng.integers(1, 40))
    assert a < b.end
    ranges += [(b.end + 10, b.end + 20), (50, 50)]
    order = rng.permutation(len(ranges))
    return [ranges[j] for j in order], total


def test_256_destinations(big_engine, big):
    rng = np.random.default_rng(256)
    ranges, total = uneven_ranges(big, rng)
    assert len(ranges) == 256
    assert total > TILE_EDGE + ROUTE_EDGE
    with big.reader(big_engine) as r:
        for keep in (False, True):
            check_range(big_engine, r, big, ranges, keep, total)
        check_scan(big_engine, r, big, ranges, total)
        rows, data, index, _ = check_ranges(big_engine, r, big, ranges, capi.RANGE_LIMIT_MAX)
        assert cross_check(r, big, ranges, rows, data, index) >= 250
        for call in (r.get_range, r.scan):
            with pytest.raises(capi.DbeelError) as ex:
                call(big.tree.bounds(ranges + [(1, 2)]))
            assert ex.value.code == capi.ERR_INVALID_ARG
        check_range(big_engine, r, big, ranges[:3], False, sum(big.tree.count(*x) for x in ranges[:3]))


# ---- reader_scan past the route-scan carry


@pytest.mark.parametrize("n", [ROUTE_EDGE - 1, ROUTE_EDGE, ROUTE_EDGE + 1, 2_500_000])
def test_reader_scan_route_edges(big_engine, big, n):
    rng = np.random.default_rng(n)
    parts = 5
    sizes = [n // parts] * (parts - 1) + [n - (parts - 1) * (n // parts)]
    ranges, a = [], 11
    for s in sizes:
        a, z = big.range_of(a, s)
        ranges.append((a, z))
        a = z + int(rng.integers(1, 1000))
    with big.reader(big_engine) as r:
        check_scan(big_engine, r, big, ranges, n)
        check_range(big_engine, r, big, ranges, False, n)


# ---- get_ranges rounds past 2^20 staged records


@pytest.mark.parametrize("limit", [1, capi.RANGE_LIMIT_MAX])
def test_tombstone_wall(big_engine, wall, limit):
    """A newer table tombstones 2,000,000 consecutive keys: a query's chunks double until one round stages past the
    wall, more than 2^20 records of one query."""
    fwd = [(WALL_LO, WALL_END)]
    rev = [(0, WALL_LO + WALL)]
    with wall.reader(big_engine) as r:
        for ranges, reverse in ((fwd, False), (rev, True)):
            rows, data, index, st = check_ranges(big_engine, r, wall, ranges, limit, reverse=reverse)
            assert int(rows["count"][0]) == limit and int(rows["flags"][0]) == m.MORE
            # the round that finishes it stages the old table past the whole wall
            assert st["partitions"] > 1 and st["entries_in"] > WALL, (st["partitions"], st["entries_in"])
        rows, data, index, st = check_ranges(big_engine, r, wall, fwd, limit, keep=True)
        assert st["partitions"] == 1


def test_tombstone_wall_page_cache(big_engine, wall):
    ranges = [(WALL_LO, WALL_END), (0, WALL_LO + WALL)]
    with big_engine.open_page_cache(1 << 30) as cache, wall.reader(big_engine) as r:
        r.attach_page_cache(cache)
        for reverse in (False, True):
            a = check_ranges(big_engine, r, wall, ranges, 1000, reverse=reverse)
            b = check_ranges(big_engine, r, wall, ranges, 1000, reverse=reverse)
            assert b[3]["input_bytes"] == 0 and not r.last_stream_reads
            assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3]))


def test_24_queries_at_the_limit_in_one_round(big_engine, wall):
    """24 disjoint live ranges at RANGE_LIMIT_MAX on one table: one round stages 24 * 65,537 records."""
    old = Built(m.Tree([wall.tree.tables[0]]), WALL_END)
    ranges = [(j * 80_000 + 3, (j + 1) * 80_000) for j in range(24)]
    with old.reader(big_engine) as r:
        for reverse in (False, True):
            rows, _, _, st = check_ranges(big_engine, r, old, ranges, capi.RANGE_LIMIT_MAX, reverse=reverse)
            assert (rows["flags"] == m.MORE).all()
            assert st["partitions"] == 1 and st["entries_in"] == 24 * (capi.RANGE_LIMIT_MAX + 1) > TILE_EDGE, st


def test_24_queries_at_the_limit_on_overlapping_tables(big_engine, big):
    rng = np.random.default_rng(24)
    ranges, a = [], 0
    for _ in range(24):
        z = a + int(rng.integers(70_000, 95_000))
        ranges.append((a, z))
        a = z + int(rng.integers(0, 3))
    with big.reader(big_engine) as r:
        for reverse in (False, True):
            for keep in (False, True):
                _, _, _, st = check_ranges(big_engine, r, big, ranges, capi.RANGE_LIMIT_MAX, keep, reverse)
                assert st["entries_in"] > TILE_EDGE


def test_1000_queries_of_one_record(big_engine, big):
    """A round of 1,000 queries, most of one record: more queries than k_limit_query's one block and about as many
    records as queries (a live query stages at least one record)."""
    rng = np.random.default_rng(1000)
    ids = rng.integers(0, big.end + 500, 1000)
    ranges = [(int(i), int(i) + 1) for i in ids]
    ranges[::50] = [(int(i), int(i) + int(rng.integers(2, 300))) for i in ids[::50]]
    limits = [int(x) for x in rng.integers(1, 4, len(ranges))]
    staged = sum(big.tree.count(*x) for x in ranges)
    live = sum(1 for x in ranges if big.tree.count(*x))
    assert live > 256
    with big.reader(big_engine) as r:
        for reverse in (False, True):
            rows, data, index, st = check_ranges(big_engine, r, big, ranges, limits, reverse=reverse)
            if st["partitions"] == 1:  # every query finished in its first round: its chunks held its whole spans
                assert st["entries_in"] == staged
            assert cross_check(r, big, ranges, rows, data, index, reverse) > 900


# ---- readers_get_ranges


def test_readers_get_ranges(big_engine, big, shared, wall):
    rng = np.random.default_rng(3)
    ra = [(int(a), int(a) + int(rng.integers(1, 400_000))) for a in rng.integers(0, big.end, 12)]
    rs = [(int(a), int(a) + int(rng.integers(1, 200_000))) for a in rng.integers(0, shared.end, 12)]
    rw = [(WALL_LO - 3, WALL_END), (0, WALL_LO + WALL), (WALL_LO + 10, WALL_LO + 20)]
    la = [int(x) for x in rng.integers(1, capi.RANGE_LIMIT_MAX + 1, len(ra))]
    with big.reader(big_engine) as a, shared.reader(big_engine) as s, wall.reader(big_engine) as w:
        batches = [(a, ra, la, False, False), (s, rs, 5000, True, True), (w, rw, 7, True, False),
                   (a, ra, capi.RANGE_LIMIT_MAX, True, False), (w, rw, 2, False, True)]
        trees = [big, shared, wall, big, wall]
        got = big_engine.readers_get_ranges([(r, t.tree.bounds(x), lim, rev, keep)
                                             for (r, x, lim, rev, keep), t in zip(batches, trees)])
        for j, ((r, x, lim, rev, keep), t, (rows, data, index)) in enumerate(zip(batches, trees, got)):
            check_rows(rows, data, index, t.tree.get_ranges(x, lim, keep, rev), f"batch {j}")
            solo = r.get_ranges(t.tree.bounds(x), lim, keep_tombstones=keep, reverse=rev)
            assert all(np.array_equal(p, q) for p, q in zip((rows, data, index), solo)), j
