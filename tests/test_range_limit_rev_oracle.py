"""The reverse limited range oracle (tests/range_limit_rev_oracle.py) against an independent model: on sorted trees, the
newest table's version of every key a range takes, in descending key order, cut to the limit; on damaged and shuffled
trees, the damage rule's A'_q and damaged records against a walk of every table's span records from the top down."""
import struct

import numpy as np
import pytest

import range_limit_oracle as rlo
import range_limit_rev_oracle as rro
from scan_cases import DAMAGES, damage, key_ranges, random_tree
from test_range_oracle import _ranges, _sorted, _table_entries


def model(tables, rng_, limit, keep):
    newest = {}
    for d, i in tables:  # later tables are newer: their version replaces the older one
        newest.update(_table_entries(d, i))
    s, e = rng_
    out = [newest[k] for k in sorted(newest, reverse=True)
           if s <= k < e and (keep or struct.unpack_from("<Q", newest[k], 8 + len(k))[0])]
    return out[:limit], len(out) > limit


@pytest.mark.parametrize("seed", range(12))
def test_clean_answer_matches_the_newest_table_model(seed):
    rng = np.random.default_rng(5200 + seed)
    tables = _sorted(random_tree(rng, 1 + seed % 6, max_entries=50))
    for rng_ in key_ranges(tables) + _ranges(rng, tables):
        for limit in (1, 2, 7, 1000):
            for keep in (False, True):
                assert rro.clean(tables, rng_, limit, keep) == model(tables, rng_, limit, keep)


def test_clean_reverse_is_the_forward_answer_reversed():
    rng = np.random.default_rng(5250)
    tables = _sorted(random_tree(rng, 4, max_entries=60))
    for rng_ in key_ranges(tables) + _ranges(rng, tables):
        whole = rlo.clean(tables, rng_, 10 ** 6)
        if whole is None:
            continue
        for limit in (1, 3, 10 ** 6):
            assert rro.clean(tables, rng_, limit) == (whole[0][::-1][:limit], len(whole[0]) > limit)


def damage_model(tables, rng_, keep):
    """A'_q and the damaged records, restated: per table the records of [seek(start), seek(end)) listed with their keys
    (None when the scan's decode fails), walked from the last one down and cut at the first None or at a key not below
    the one after it; then newest table first, the first version of every key wins, listed in ascending key order."""
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
        kept, after = [], None
        for r in range(max(lo, hi) - 1, lo - 1, -1):
            off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
            ok = fs > 0 and off <= len(d) and fs <= len(d) - off
            dec = _decode(d[off:off + fs]) if ok else None
            why = None if dec else (rro.ERR if ok else rro.PANIC)
            if why is None and after is not None and not dec[0] < after:
                why = "unsorted"
            if why is not None:
                bad[(t, r)] = why
                break
            kept.append((dec[0], d[off:off + fs]))
            after = dec[0]
        cut_tables.append(kept)
    newest = {}
    for recs in reversed(cut_tables):
        for k, ent in recs:
            newest.setdefault(k, ent)
    out = [newest[k] for k in sorted(newest)
           if keep or struct.unpack_from("<Q", newest[k], 8 + len(k))[0]]
    return out, bad


@pytest.mark.parametrize("kind", [k for k in DAMAGES if k not in ("empty_table", "ragged_index")])
def test_damaged_merge_matches_an_independent_downward_walk(kind):
    for seed in range(4):
        rng = np.random.default_rng(5600 + 10 * DAMAGES.index(kind) + seed)
        tables = _sorted(random_tree(rng, 2 + seed % 3, max_entries=50))
        for rec in (0, 3, 17, 49, -1):
            t = int(rng.integers(0, len(tables)))
            n = np.asarray(tables[t][1]).size // 16
            if n == 0:
                continue
            bad_tables = damage(tables, kind, t, n - 1 if rec < 0 else min(rec, n - 1))
            for rng_ in key_ranges(tables) + _ranges(rng, tables):  # bounds from the undamaged tables
                if rro.seek_stop(bad_tables, rng_) is not None:
                    continue  # a failed seek: no record is read
                for keep in (False, True):
                    assert rro.damaged_merge(bad_tables, rng_, keep) == damage_model(bad_tables, rng_, keep)


@pytest.mark.parametrize("kind", DAMAGES)
def test_damage_kinds_at_a_span_end_are_named(kind):
    """Damage at the last record of table 1 sits at the top of its span of the whole key space: the downward walk meets
    it first, so the clean answer is gone and the record is named -- or, for the kinds a seek meets, the seek stops."""
    rng = np.random.default_rng(5500 + DAMAGES.index(kind))
    tables = _sorted(random_tree(rng, 3, max_entries=40))
    everything = (b"", b"\xff" * 80)
    n = np.asarray(tables[1][1]).size // 16
    bad_tables = damage(tables, kind, 1, 0 if kind == "empty_table" else n - 1)
    if kind in ("empty_table", "ragged_index"):
        if kind == "empty_table":
            assert rro.seek_stop(bad_tables, everything) == (1, rro.PANIC, 0)
        return
    if rro.seek_stop(bad_tables, everything) is not None:
        return
    a, bad = rro.damaged_merge(bad_tables, everything)
    assert bad.get((1, n - 1)) in (rro.ERR, rro.PANIC)
    assert rro.clean(bad_tables, everything, 5) is None
    assert a == damage_model(bad_tables, everything, False)[0]


def test_unsorted_record_is_named():
    rng = np.random.default_rng(5700)
    tables = random_tree(rng, 2, max_entries=40)  # table 1 shuffled, one record listed twice
    everything = (b"", b"\xff" * 80)
    a, bad = rro.damaged_merge(tables, everything)
    assert [w for (t, _), w in bad.items() if t == 1] == ["unsorted"]


def test_damaged_merge_matches_an_independent_downward_walk_on_shuffled_tables():
    for seed in range(6):
        rng = np.random.default_rng(5800 + seed)
        tables = random_tree(rng, 2 + seed % 4, max_entries=50)  # table 1 shuffled, a record listed twice
        for rng_ in key_ranges(tables) + _ranges(rng, tables):
            if rro.seek_stop(tables, rng_) is None:
                for keep in (False, True):
                    assert rro.damaged_merge(tables, rng_, keep) == damage_model(tables, rng_, keep)


def test_check_row_reverse():
    """check_row accepts the model's rows and refuses the forward order."""
    rng = np.random.default_rng(5900)
    tables = _sorted(random_tree(rng, 3, max_entries=50))
    for rng_ in key_ranges(tables):
        want, more = model(tables, rng_, 5, False)
        if rro.seek_stop(tables, rng_) is not None or not bytes(rng_[0]) < bytes(rng_[1]):
            continue
        row = (0, len(want), rro.MORE if more else 0, (-1, 0, 0))
        rro.check_row(tables, rng_, 5, False, row, want)
        if len(want) > 1:
            with pytest.raises(AssertionError):
                rro.check_row(tables, rng_, 5, False, row, want[::-1])
