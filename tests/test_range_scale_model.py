"""The vectorised range-read model (tests/range_scale_model.py) against the existing oracles, on small trees of both key
shapes: its builder is sstable.build_run byte for byte, and its reader_scan, get_range and get_ranges (forward and
reverse) are seek_oracle.reader_scan, range_oracle.get_range, range_limit_oracle.clean and range_limit_rev_oracle.clean."""
import time

import numpy as np
import pytest

import range_limit_oracle as rlo
import range_limit_rev_oracle as rro
import range_oracle
import range_scale_model as m
import seek_oracle
from dbeel_b200 import sstable
from helpers import assert_run_equal

SHAPES = [b"", m.SHARED_PREFIX]


def small_tree(rng, n_tables, prefix, universe=300):
    tables = []
    for t in range(n_tables):
        ids = np.sort(rng.choice(universe, int(rng.integers(1, universe // 2)), replace=False)).astype(np.uint64)
        tables.append((ids, rng.random(ids.size) < 0.25))
    return m.Tree(tables, prefix)


def small_ranges(rng, n, universe=300):
    """Disjoint and overlapping ranges, empty and inverted ones, ranges past every key."""
    out = []
    for j in range(n):
        a, b = (int(x) for x in rng.integers(0, universe + 20, 2))
        out.append((a, b) if j % 7 else (b, a))
    out.append((0, universe + 50))
    out.append((universe + 10, universe + 30))
    return out


def entry_list(d, i):
    ix = np.asarray(i, np.uint8).reshape(-1, 16)
    return [bytes(d[int(r[:8].view("<u8")[0]):int(r[:8].view("<u8")[0]) + int(r[12:16].view("<u4")[0])]) for r in ix]


@pytest.mark.parametrize("prefix", SHAPES)
def test_builder_is_build_run(prefix):
    rng = np.random.default_rng(1 + len(prefix))
    ids = np.sort(rng.choice(1 << 32, 500, replace=False)).astype(np.uint64)
    tabs = rng.integers(0, 5, ids.size)
    for tomb in (np.zeros(ids.size, bool), rng.random(ids.size) < 0.3, np.ones(ids.size, bool)):
        want = sstable.build_run([(m.key(i, prefix), b"" if x else int(t).to_bytes(4, "little") + int(i).to_bytes(4, "little"),
                                   m.BASE_TS + int(t)) for i, t, x in zip(ids.tolist(), tabs.tolist(), tomb.tolist())])
        assert_run_equal(m.entries(ids, tabs, tomb, prefix), want, "entries")
    assert all(x.size == 0 for x in m.entries(ids[:0], 0, False, prefix))


def test_builder_is_vectorised():
    """Three million entries build in seconds: no per-entry Python loop."""
    ids = np.arange(3 << 20, dtype=np.uint64)
    t0 = time.perf_counter()
    d, i = m.entries(ids, 1, ids % 3 == 0)
    assert time.perf_counter() - t0 < 20
    assert i.size == 16 * ids.size and d.size == 48 * ids.size - 8 * ((ids.size + 2) // 3)


@pytest.mark.parametrize("prefix", SHAPES)
@pytest.mark.parametrize("seed", range(6))
def test_model_is_the_oracles(prefix, seed):
    rng = np.random.default_rng(4400 + seed)
    tree = small_tree(rng, 1 + seed % 4, prefix)
    tables = tree.built()
    ranges = small_ranges(rng, 12)
    bounds = tree.bounds(ranges)
    out, stop = seek_oracle.reader_scan(tables, bounds)
    assert stop == (-1, 0, 0)
    for d, (g, w) in enumerate(zip(tree.reader_scan(ranges), out)):
        assert_run_equal(g, w, f"reader_scan {d}")
    for keep in (False, True):
        want, stop = range_oracle.get_range(tables, bounds, keep)
        assert stop == (-1, 0, 0)
        for d, (g, w) in enumerate(zip(tree.get_range(ranges, keep), want)):
            assert_run_equal(g, w, f"get_range {d}")
        for reverse, oracle in ((False, rlo), (True, rro)):
            for limits in (1, 3, [int(x) for x in rng.integers(1, 200, len(ranges))]):
                (first, count, flags), (data, index) = tree.get_ranges(ranges, limits, keep, reverse)
                lim = np.broadcast_to(np.asarray(limits), (len(ranges),))
                got = entry_list(data, index)
                assert len(got) == int(count.sum())
                for q, (rng_, L) in enumerate(zip(bounds, lim.tolist())):
                    ents, more = oracle.clean(tables, rng_, L, keep)
                    f, c = int(first[q]), int(count[q])
                    assert (c, int(flags[q])) == (len(ents), m.MORE if more else 0), (q, reverse, keep)
                    assert got[f:f + c] == ents, (q, reverse, keep)
                    assert tree.group_size(*ranges[q], keep) == len(range_oracle._records(
                        *(bytes(x) for x in range_oracle.get_range(tables, [rng_], keep)[0][0])))


def test_range_with_finds_exact_counts():
    rng = np.random.default_rng(9)
    tree = small_tree(rng, 3, b"", universe=2000)
    c = m.cumulative(tree, 2000)
    for n in (1, 2, 17, 100, 500):
        a, b = m.range_with(c, int(rng.integers(0, 500)), n)
        assert tree.count(a, b) == n
