"""The restatement of dbeel_reader_scan's key ranges (tests/seek_oracle.py) checked on its own: seek_t against a plain
lower bound, equality with the scan oracle on sorted tables, and a hand-checked table whose index is shuffled."""
import numpy as np
import pytest

import seek_oracle
from dbeel_b200 import sstable
from helpers import BASE_TS
from scan_cases import ERR, KEY, NONE, PANIC, damage, key_ranges, py_scan, random_tree


def _sorted_tables(rng, n_tables):
    """random_tree's tables with strictly ascending keys (its shuffled table dropped)."""
    return [t for j, t in enumerate(random_tree(rng, n_tables + (n_tables >= 2))) if j != 1 or n_tables < 2][:n_tables]


def _keys(t):
    d, ix = bytes(t[0]), bytes(t[1])
    out = []
    for r in range(len(ix) // 16):
        off = int.from_bytes(ix[16 * r:16 * r + 8], "little")
        klen = int.from_bytes(d[off:off + 8], "little")
        out.append(d[off + 8:off + 8 + klen])
    return out


def _ranges(rng, tables, n):
    keys = sorted({k for t in tables for k in _keys(t)})
    pick = lambda: keys[int(rng.integers(0, len(keys)))] if keys and rng.random() < 0.6 else bytes(
        rng.integers(0, 256, int(rng.integers(0, 70)), dtype=np.uint8))
    return [(pick(), pick()) for _ in range(n)]


@pytest.mark.parametrize("seed", range(8))
def test_seek_is_the_lower_bound_on_sorted_tables(seed):
    rng = np.random.default_rng(seed)
    for t in _sorted_tables(rng, 3):
        keys = _keys(t)
        assert keys == sorted(set(keys))
        for start, _ in _ranges(rng, [t], 20):
            a, bad = seek_oracle.seek(bytes(t[0]), bytes(t[1]), start)
            assert bad is None and a == sum(k < start for k in keys)


@pytest.mark.parametrize("seed", range(10))
def test_equals_the_scan_on_sorted_tables(seed):
    rng = np.random.default_rng(100 + seed)
    tables = _sorted_tables(rng, int(rng.integers(1, 5)))
    for ranges in (key_ranges(tables), _ranges(rng, tables, 12), [(b"", b"\xff" * 80)], [(b"z", b"a")]):
        assert _same(seek_oracle.reader_scan(tables, ranges), py_scan(tables, ranges, KEY))


def _same(a, b):
    (oa, sa), (ob, sb) = a, b
    return sa == sb and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(oa, ob))


def test_a_shuffled_index_by_hand():
    """Keys a b c d stored in that order, index records listed c a d b: the probe path decides what is scanned."""
    ents = [(k, b"v" + k, BASE_TS) for k in (b"a", b"b", b"c", b"d")]
    d, i = sstable.build_run(ents)
    recs = np.asarray(i, np.uint8).reshape(-1, 16)
    table = (np.asarray(d, np.uint8), recs[[2, 0, 3, 1]].reshape(-1).copy())
    # seek(b) probes d (>, b = 2), then a (<, a = 2): 2; seek(d) probes d (=, b = 2), then a (<, a = 2): 2 -> no span
    assert seek_oracle.seek(bytes(table[0]), bytes(table[1]), b"b") == (2, None)
    assert seek_oracle.seek(bytes(table[0]), bytes(table[1]), b"d") == (2, None)
    out, stop = seek_oracle.reader_scan([table], [(b"b", b"d")])
    assert stop == (-1, NONE, 0) and out[0][1].size == 0
    # seek(a) = 0 (d >, a =, c >), seek(e) = 4 (d <, b <): every record, in index order c a d b
    out, stop = seek_oracle.reader_scan([table], [(b"a", b"e"), (b"", b"b")])
    assert stop == (-1, NONE, 0)
    assert _keys(out[0]) == [b"c", b"a", b"d", b"b"] and out[1][1].size == 0
    # random_tree's shuffled table: whatever the seek reaches is scanned in index order, entries in their ranges only
    rng = np.random.default_rng(5)
    tables = random_tree(rng, 3)
    ranges = key_ranges(tables)
    out, stop = seek_oracle.reader_scan(tables, ranges)
    sp, _ = seek_oracle.spans(tables, ranges)
    cut, _ = seek_oracle.cut(tables, sp)
    assert _same((out, stop), py_scan(cut, ranges, KEY))


def _point(table, rec, off, fs):
    d, i = table[0].copy(), table[1].copy()
    i[16 * rec:16 * rec + 8] = np.array([off], "<u8").view(np.uint8)
    i[16 * rec + 12:16 * rec + 16] = np.array([fs], "<u4").view(np.uint8)
    return d, i


def test_a_failed_seek_ends_the_scan_before_its_table():
    rng = np.random.default_rng(9)
    tables = _sorted_tables(rng, 3)
    n = tables[1][1].size // 16
    mid = n // 2  # the root probe of every search of table 1
    dl = tables[1][0].size
    everything = [(b"", b"\xff" * 80)]
    first, _ = py_scan(tables[:1], everything, KEY)
    # past the end of .data: the index alone shows it (PANIC); 4 bytes before the end: the index is fine but the length
    # prefix does not fit (ERR)
    for off, fs, reason in ((dl + 1, 40, PANIC), (dl - 4, 4, ERR)):
        bad = [tables[0], _point(tables[1], mid, off, fs), tables[2]]
        out, stop = seek_oracle.reader_scan(bad, everything)
        assert stop == (1, reason, mid)
        assert _same((out, stop), (first, stop))
    # a range that is empty or inverted is not searched: no failure
    bad = [tables[0], _point(tables[1], mid, dl + 1, 40), tables[2]]
    assert seek_oracle.reader_scan(bad, [(b"b", b"a")])[1] == (-1, NONE, 0)
    empty = [tables[0], (tables[1][0], tables[1][1][:0]), tables[2]]
    assert seek_oracle.reader_scan(empty, everything)[1] == (1, PANIC, 0)
