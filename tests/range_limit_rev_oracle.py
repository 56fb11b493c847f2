"""A pure-Python restatement of dbeel_reader_get_ranges_reverse (include/dbeel_compact.h), next to the forward one in
tests/range_limit_oracle.py: the clean answer of a query is the LAST entries of G_q (what range_oracle.get_range returns for
its range alone), in descending key order, cut to the limit; a damaged query may instead name a damaged record of its
spans, or return the last entries of A'_q, descending -- the merge of every table's span records, each walked from its top
down and cut just above its first record that does not decode or is not strictly below the record after it."""
from __future__ import annotations

import struct

import numpy as np

import range_oracle
import seek_oracle
from range_limit_oracle import MORE, STOPPED, UNSORTED, _entries, record_damage, seek_stop  # noqa: F401 (re-exported)
from scan_cases import ERR, PANIC, _decode  # noqa: F401 (re-exported)


def clean(tables, rng_, limit: int, keep_tombstones: bool = False):
    """(entries, more) when the query is clean (get_range on its range alone gives no stop and not UNSORTED_RUN); else
    None.  entries: the stored bytes of each returned entry, largest key first."""
    got = range_oracle.get_range(tables, [rng_], keep_tombstones)
    if got == range_oracle.UNSORTED or got[1][0] >= 0:
        return None
    g = _entries(*got[0][0])[::-1]
    return g[:limit], len(g) > limit


def damaged_merge(tables, rng_, keep_tombstones: bool = False):
    """(A'_q as a list of entry bytes in ascending key order, {(table, record): "unsorted" | ERR | PANIC} of the damaged
    records met walking each table's spans from the top down, each table's up to and including its first)."""
    sp, _ = seek_oracle.spans(tables, [rng_])
    last, bad = {}, {}
    for t, s in enumerate(sp):
        d, ix = bytes(np.asarray(tables[t][0], np.uint8)), bytes(np.asarray(tables[t][1], np.uint8))
        after = None  # the key of the record above, already walked
        for lo, hi in reversed(s):
            for rec in range(hi - 1, lo - 1, -1):
                why = record_damage(d, ix, rec)
                key = None
                if why is None:
                    off, _, fs = struct.unpack_from("<QII", ix, 16 * rec)
                    e = d[off:off + fs]
                    key = _decode(e)[0]
                    if after is not None and not key < after:
                        why = "unsorted"
                if why is not None:
                    bad[(t, rec)] = why
                    break
                last[key] = e
                after = key
            else:
                continue
            break
    out = []
    for key in sorted(last):
        e = last[key]
        if keep_tombstones or struct.unpack_from("<Q", e, 8 + len(key))[0]:
            out.append(e)
    return out, bad


def check_row(tables, rng_, limit: int, keep_tombstones, row, entries):
    """Asserts that one reverse row (first, count, flags, (table, reason, record)) and its entries are what the contract
    allows."""
    count, flags, stop = int(row[1]), int(row[2]), tuple(int(x) for x in row[3])
    s = seek_stop(tables, rng_)
    if not bytes(rng_[0]) < bytes(rng_[1]):
        if s is not None:
            assert (flags, count, stop) == (STOPPED, 0, s)
        else:
            assert (flags, count, stop) == (0, 0, (-1, 0, 0))
        return
    if s is not None:
        assert (flags, count, stop) == (STOPPED, 0, s), (row, s)
        return
    want = clean(tables, rng_, limit, keep_tombstones)
    if want is not None:
        assert flags == (MORE if want[1] else 0) and stop == (-1, 0, 0), (row, want[1])
        assert [bytes(e) for e in entries] == want[0]
        return
    a, bad = damaged_merge(tables, rng_, keep_tombstones)
    if flags & (STOPPED | UNSORTED):
        assert count == 0 and not entries
        why = bad.get((stop[0], stop[2]))
        assert why is not None, (row, bad)
        if flags == UNSORTED:
            assert why == "unsorted" and stop[1] == 0
        else:
            assert flags == STOPPED and why == stop[1]
        return
    assert flags == (MORE if len(a) > limit else 0) and stop == (-1, 0, 0)
    assert [bytes(e) for e in entries] == a[::-1][:limit]
