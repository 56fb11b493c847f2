"""The range-read oracle (tests/range_oracle.py) against an independent model on random sorted trees: for every key a
range takes, the newest table holding it, as get_entry walks the tables (newest first)."""
import struct

import numpy as np

import range_oracle
from scan_cases import damage, key_ranges, random_tree


def _sorted(tables):
    return [t for j, t in enumerate(tables) if j != 1 or len(tables) < 2]


def _table_entries(d, ix):
    d, ix = bytes(np.asarray(d, np.uint8)), bytes(np.asarray(ix, np.uint8))
    out = {}
    for r in range(len(ix) // 16):
        off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
        e = d[off:off + fs]
        klen = struct.unpack_from("<Q", e, 0)[0]
        out[e[8:8 + klen]] = e
    return out


def model(tables, ranges, keep_tombstones):
    per_table = [_table_entries(d, i) for d, i in tables]
    keys = sorted({k for t in per_table for k in t})
    outs = [[] for _ in ranges]
    for k in keys:
        for d, (s, e) in enumerate(ranges):
            if s <= k < e:
                newest = next(t[k] for t in reversed(per_table) if k in t)
                if keep_tombstones or struct.unpack_from("<Q", newest, 8 + len(k))[0]:
                    outs[d].append((k, newest))
                break
    return [range_oracle._pack(o) for o in outs]


def _ranges(rng, tables):
    keys = sorted({k for d, i in tables for k in _table_entries(d, i)}) or [b"k"]
    out = []
    for j in range(7):
        a, b = (keys[int(x)] for x in rng.integers(0, len(keys), 2))
        if j % 3 == 1:
            a = a + b"\x00"
        out.append((min(a, b), max(a, b)) if j % 4 else (max(a, b), min(a, b)))
    return out


def test_oracle_matches_newest_table_model():
    for seed in range(30):
        rng = np.random.default_rng(1200 + seed)
        tables = _sorted(random_tree(rng, 1 + seed % 6, max_entries=50))
        for ranges in (key_ranges(tables), _ranges(rng, tables), [(b"", b"\xff" * 80)]):
            for keep in (False, True):
                got, stop = range_oracle.get_range(tables, ranges, keep)
                assert stop == (-1, 0, 0)
                for g, w in zip(got, model(tables, ranges, keep)):
                    assert bytes(g[0]) == bytes(w[0]) and bytes(g[1]) == bytes(w[1])


def test_oracle_unsorted_and_stops():
    rng = np.random.default_rng(5)
    tables = random_tree(rng, 3, max_entries=60)  # table 1 is shuffled
    assert range_oracle.get_range(tables, [(b"", b"\xff" * 80)]) == range_oracle.UNSORTED
    st = _sorted(tables)
    bad = damage(st, "timestamp", 0, 3)
    got, stop = range_oracle.get_range(bad, [(b"", b"\xff" * 80)])
    assert stop[0] == 0 and all(g[0].size == 0 and g[1].size == 0 for g in got)
