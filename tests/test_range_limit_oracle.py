"""The limited range-read oracle (tests/range_limit_oracle.py) against an independent model: on sorted trees, for every
key a range takes, the newest table holding it (get_entry's walk, newest first), cut to the limit; on damaged trees, the
damage rule's A_q and damaged records against a walk of every table's records in key range."""
import struct

import numpy as np
import pytest

import range_limit_oracle as rlo
from scan_cases import DAMAGES, damage, key_ranges, random_tree
from test_range_oracle import _ranges, _sorted, _table_entries


def model(tables, rng_, limit, keep):
    per_table = [_table_entries(d, i) for d, i in tables]
    s, e = rng_
    out = []
    for k in sorted({k for t in per_table for k in t if s <= k < e}):
        newest = next(t[k] for t in reversed(per_table) if k in t)
        if keep or struct.unpack_from("<Q", newest, 8 + len(k))[0]:
            out.append(newest)
    return out[:limit], len(out) > limit


@pytest.mark.parametrize("seed", range(12))
def test_clean_answer_matches_the_newest_table_model(seed):
    rng = np.random.default_rng(4200 + seed)
    tables = _sorted(random_tree(rng, 1 + seed % 6, max_entries=50))
    for rng_ in key_ranges(tables) + _ranges(rng, tables):
        for limit in (1, 2, 7, 1000):
            for keep in (False, True):
                assert rlo.clean(tables, rng_, limit, keep) == model(tables, rng_, limit, keep)


@pytest.mark.parametrize("seed", range(6))
def test_damaged_merge_is_the_clean_answer_on_clean_trees(seed):
    rng = np.random.default_rng(4300 + seed)
    tables = _sorted(random_tree(rng, 1 + seed % 5, max_entries=40))
    for rng_ in key_ranges(tables):
        a, bad = rlo.damaged_merge(tables, rng_, False)
        assert not bad
        assert rlo.clean(tables, rng_, 10 ** 6, False) == (a, False)


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage_at_a_span_start_is_named(kind):
    rng = np.random.default_rng(4400 + DAMAGES.index(kind))
    tables = _sorted(random_tree(rng, 3, max_entries=40))
    everything = (b"", b"\xff" * 80)
    bad_tables = damage(tables, kind, 1, 0)
    if kind == "empty_table" or kind == "ragged_index":
        if kind == "empty_table":
            assert rlo.seek_stop(bad_tables, everything) == (1, rlo.PANIC, 0)
        return
    stop = rlo.seek_stop(bad_tables, everything)
    a, bad = rlo.damaged_merge(bad_tables, everything)
    if stop is None:  # record 0 of table 1 starts its span: it is damaged, and the clean answer is gone
        assert (1, 0) in bad
        assert rlo.clean(bad_tables, everything, 5) is None
        t1 = set(_table_entries(*tables[1]).values())  # A_q holds no record of table 1
        t_other = set(v for j, t in enumerate(tables) if j != 1 for v in _table_entries(*t).values())
        assert all(e in t_other or e not in t1 for e in a)


def test_unsorted_record_is_named():
    rng = np.random.default_rng(4500)
    tables = random_tree(rng, 2, max_entries=40)  # table 1 shuffled, one record listed twice
    everything = (b"", b"\xff" * 80)
    a, bad = rlo.damaged_merge(tables, everything)
    assert [w for (t, _), w in bad.items() if t == 1] == ["unsorted"]


def damage_model(tables, rng_, keep):
    """A_q and the damaged records, restated: per table the records of [seek(start), seek(end)) listed with their keys
    (None when the scan's decode fails), cut at the first None or non-ascending key; then newest table first, the first
    version of every key wins."""
    import seek_oracle
    from scan_cases import _decode
    s, e = rng_
    cut_tables, bad = [], {}
    if not s < e:  # no record is searched or read
        return [], {}
    for t, (d, ix) in enumerate(tables):
        d, ix = bytes(np.asarray(d, np.uint8)), bytes(np.asarray(ix, np.uint8))
        lo, _ = seek_oracle.seek(d, ix, s)
        hi, _ = seek_oracle.seek(d, ix, e)
        recs = []
        for r in range(lo, max(lo, hi)):
            off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
            ok = fs > 0 and off <= len(d) and fs <= len(d) - off
            dec = _decode(d[off:off + fs]) if ok else None
            recs.append((r, dec[0] if dec else None, d[off:off + fs], None if dec else (rlo.ERR if ok else rlo.PANIC)))
        keep_recs = []
        for j, (r, k, ent, why) in enumerate(recs):
            if why is None and j and k <= recs[j - 1][1]:
                why = "unsorted"
            if why is not None:
                bad[(t, r)] = why
                break
            keep_recs.append((k, ent))
        cut_tables.append(keep_recs)
    newest = {}
    for recs in reversed(cut_tables):
        for k, ent in recs:
            newest.setdefault(k, ent)
    out = [newest[k] for k in sorted(newest)
           if keep or struct.unpack_from("<Q", newest[k], 8 + len(k))[0]]
    return out, bad


@pytest.mark.parametrize("kind", [k for k in DAMAGES if k not in ("empty_table", "ragged_index")])
def test_damaged_merge_matches_an_independent_walk(kind):
    for seed in range(4):
        rng = np.random.default_rng(4600 + 10 * DAMAGES.index(kind) + seed)
        tables = _sorted(random_tree(rng, 2 + seed % 3, max_entries=50))
        for rec in (0, 3, 17, 49):
            bad_tables = damage(tables, kind, int(rng.integers(0, len(tables))), rec)
            for rng_ in key_ranges(tables) + _ranges(rng, tables):  # bounds from the undamaged tables
                if rlo.seek_stop(bad_tables, rng_) is not None:
                    continue  # a failed seek: no record is read
                for keep in (False, True):
                    assert rlo.damaged_merge(bad_tables, rng_, keep) == damage_model(bad_tables, rng_, keep)


def test_damaged_merge_matches_an_independent_walk_on_shuffled_tables():
    for seed in range(6):
        rng = np.random.default_rng(4700 + seed)
        tables = random_tree(rng, 2 + seed % 4, max_entries=50)  # table 1 shuffled, a record listed twice
        for rng_ in key_ranges(tables) + _ranges(rng, tables):
            if rlo.seek_stop(tables, rng_) is None:
                assert rlo.damaged_merge(tables, rng_) == damage_model(tables, rng_, False)
