"""A pure-Python restatement of dbeel_reader_get_ranges (include/dbeel_compact.h): the clean answer of a query is G_q (what
range_oracle.get_range returns for its range alone) cut to the limit; a damaged query may instead name a damaged record of
its spans, or return the first entries of A_q -- the merge of every table's span records, each cut just before its first
record that does not decode or is not strictly above its predecessor."""
from __future__ import annotations

import struct

import numpy as np

import range_oracle
import seek_oracle
from scan_cases import ERR, PANIC, _decode

MORE, STOPPED, UNSORTED = 0x1, 0x2, 0x4


def _entries(d, ix):
    return [e for _, e in range_oracle._records(bytes(np.asarray(d, np.uint8)), bytes(np.asarray(ix, np.uint8)))]


def clean(tables, rng_, limit: int, keep_tombstones: bool = False):
    """(entries, more) when the query is clean (get_range on its range alone gives no stop and not UNSORTED_RUN); else
    None.  entries: the stored bytes of each returned entry, in order."""
    got = range_oracle.get_range(tables, [rng_], keep_tombstones)
    if got == range_oracle.UNSORTED or got[1][0] >= 0:
        return None
    g = _entries(*got[0][0])
    return g[:limit], len(g) > limit


def seek_stop(tables, rng_):
    """The stop of the query's bound searches and empty tables (seek_oracle.spans' stop), or None."""
    return seek_oracle.spans(tables, [rng_])[1]


def record_damage(d: bytes, ix: bytes, rec: int):
    """ERR / PANIC as dbeel_scan classifies record rec of a table, or None when it decodes."""
    off, _, fs = struct.unpack_from("<QII", ix, 16 * rec)
    if fs == 0 or off > len(d) or fs > len(d) - off:
        return PANIC
    return None if _decode(d[off:off + fs]) else ERR


def damaged_merge(tables, rng_, keep_tombstones: bool = False):
    """(A_q as a list of entry bytes in key order, {(table, record): "unsorted" | ERR | PANIC} of the damaged records of
    the query's spans, each table's up to and including its first)."""
    sp, _ = seek_oracle.spans(tables, [rng_])
    last, bad = {}, {}
    for t, s in enumerate(sp):
        d, ix = bytes(np.asarray(tables[t][0], np.uint8)), bytes(np.asarray(tables[t][1], np.uint8))
        prev = None
        for lo, hi in s:
            for rec in range(lo, hi):
                why = record_damage(d, ix, rec)
                key = None
                if why is None:
                    off, _, fs = struct.unpack_from("<QII", ix, 16 * rec)
                    e = d[off:off + fs]
                    key = _decode(e)[0]
                    if prev is not None and not key > prev:
                        why = "unsorted"
                if why is not None:
                    bad[(t, rec)] = why
                    break
                last[key] = e
                prev = key
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
    """Asserts that one row (first, count, flags, (table, reason, record)) and its entries are what the contract allows."""
    count, flags, stop = int(row[1]), int(row[2]), tuple(int(x) for x in row[3])
    if not bytes(rng_[0]) < bytes(rng_[1]):
        s = seek_stop(tables, rng_)
        if s is not None:
            assert (flags, count, stop) == (STOPPED, 0, s)
        else:
            assert (flags, count, stop) == (0, 0, (-1, 0, 0))
        return
    s = seek_stop(tables, rng_)
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
    assert [bytes(e) for e in entries] == a[:limit]
