"""The scan oracle (tests/scan_oracle.c: LSMTree::iter_filter's SSTable part, lsm_tree.rs:210-281) against an
independent Python restatement, the reference's own expectations from get_after_compaction, and between_cmp's table."""
import numpy as np
import pytest

import oracle
import scan_oracle
from dbeel_b200 import sstable
from helpers import BASE_TS, assert_run_equal
from scan_cases import (DAMAGES, ERR, HASH, KEY, NONE, PANIC, damage, eighths, hash_ranges, key_ranges, py_between_cmp,
                        py_murmur3_32, py_scan, random_tree)


def u16key(n: int) -> bytes:
    return int(n).to_bytes(2, "little")


def _same(got, exp, what):
    (gr, gs), (er, es) = got, exp
    assert gs == es, f"{what}: stop {gs} != {es}"
    assert len(gr) == len(er)
    for j, (g, e) in enumerate(zip(gr, er)):
        assert_run_equal(g, e, f"{what} destination {j}")


def test_between_cmp_literal_table():
    M = 0xFFFFFFFF
    cases = [
        # (hash, start, end, expected)
        (5, 1, 10, True), (1, 1, 10, True), (10, 1, 10, False), (0, 1, 10, False),
        (7, 7, 7, False), (0, 0, 0, False), (M, M, M, False),  # start == end: nothing
        (0, 10, 1, True), (5, 10, 1, True), (10, 10, 1, True), (M, 10, 1, True), (1, 10, 1, True),  # end < start: everything
        (M, 0, M, False), (M - 1, 0, M, True), (0, 0, 1, True), (M, 1, 0, True),
    ]
    for h, a, b, want in cases:
        assert scan_oracle.between_cmp(h, a, b) == want, (h, a, b)
        assert py_between_cmp(h, a, b) == want, (h, a, b)
    rng = np.random.default_rng(3)
    for h, a, b in rng.integers(0, 1 << 32, (2000, 3), dtype=np.uint64):
        assert scan_oracle.between_cmp(int(h), int(a), int(b)) == py_between_cmp(int(h), int(a), int(b))


def test_python_murmur3_matches_oracle():
    rng = np.random.default_rng(4)
    for n in range(0, 40):
        b = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert py_murmur3_32(b) == oracle.murmur3_32(b)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_scan_matches_python_restatement(seed):
    rng = np.random.default_rng(100 + seed)
    tables = random_tree(rng, [1, 3, 8, 5, 2, 13][seed])
    for ranges in (hash_ranges(rng, 1), hash_ranges(rng, 8), eighths(), [(0, 0xFFFFFFFF)], [(9, 3)]):
        _same(scan_oracle.scan(tables, ranges, HASH), py_scan(tables, ranges, HASH), f"hash {ranges[:2]}")
    ranges = key_ranges(tables)
    _same(scan_oracle.scan(tables, ranges, KEY), py_scan(tables, ranges, KEY), "key")


@pytest.mark.parametrize("kind", DAMAGES)
def test_oracle_scan_damaged_trees(kind):
    rng = np.random.default_rng(7)
    tables = random_tree(rng, 4)
    for t, rec in [(0, 0), (1, 3), (2, 10 ** 6 + 5), (3, 17)]:
        bad = damage(tables, kind, t, rec)
        got = scan_oracle.scan(bad, eighths(), HASH)
        _same(got, py_scan(bad, eighths(), HASH), f"{kind} at {t}/{rec}")
        if kind == "ragged_index":
            assert got[1] == (-1, NONE, 0)
        else:
            assert got[1][0] == t and got[1][1] in (ERR, PANIC)
        if kind in ("offset_eof", "full_size_zero", "empty_table"):
            assert got[1][1] == PANIC
        if kind in ("klen", "timestamp"):
            assert got[1][1] == ERR


def test_stop_ends_the_scan_even_where_no_range_takes_the_entry():
    """read_one decodes before it filters (lsm_tree.rs:273): an undecodable record outside every range still ends it."""
    ents = [(u16key(n), b"v", BASE_TS) for n in range(10)]
    tables = [sstable.build_run(ents), sstable.build_run(ents)]
    bad = damage([(np.asarray(d), np.asarray(i)) for d, i in tables], "timestamp", 0, 4)
    (out,), stop = scan_oracle.scan(bad, [(u16key(0), u16key(2))], KEY)
    assert stop == (0, ERR, 4)
    assert [k for k, _, _ in sstable.parse_run(*out)] == [u16key(0), u16key(1)]


def _get_after_compaction_runs():
    """lsm_tree.rs:1400-1432: 94 u16-LE keys (value == key) at capacity 32 -> two automatic
    flushes, then deletes of [1,0] and [4,0], then a manual flush."""
    writes = [(u16key(n), u16key(n), BASE_TS + n) for n in range(32 * 3 - 2)]
    writes += [(u16key(1), b"", BASE_TS + 1000), (u16key(4), b"", BASE_TS + 1001)]
    batch = sstable.build_run(writes)
    return oracle.memtable_flushes(batch, capacity=32)


def test_get_after_compaction_range_reads():
    """validate_tree_iter_range (lsm_tree.rs:1363-1397) over [1,0]..[5,0]."""
    flushed = _get_after_compaction_runs()
    runs = [(d, i) for d, i, _ in flushed]  # tables 0, 2, 4
    (out,), stop = scan_oracle.scan(runs, [(u16key(1), u16key(5))], KEY)
    assert stop == (-1, NONE, 0)
    assert [v for _, v, _ in sstable.parse_run(*out)] == [u16key(1), u16key(2), u16key(3), u16key(4), b"", b""]
    d, i, _, _ = oracle.compact(runs, keep_tombstones=False)  # compact(&[0, 2, 4], 5, false)
    (out,), stop = scan_oracle.scan([(d, i)], [(u16key(1), u16key(5))], KEY)
    assert stop == (-1, NONE, 0)
    assert [v for _, v, _ in sstable.parse_run(*out)] == [u16key(2), u16key(3)]
