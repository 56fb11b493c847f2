"""A pure-Python restatement of dbeel_reader_scan's key ranges (include/dbeel_compact.h): seek_t, the spans, the scan of
the tables cut down to their spans (scan_oracle.scan) with record numbers mapped back, and the stop of a failed seek."""
from __future__ import annotations

import struct

import numpy as np

import scan_oracle
from scan_cases import ERR, KEY, NONE, PANIC


def _probe(d: bytes, ix: bytes, rec: int, key: bytes):
    """lookup.cuh's probe(): (comparison of record rec's key with `key`, or None when the record is corrupt)."""
    off = struct.unpack_from("<Q", ix, 16 * rec)[0]
    if off > len(d) or len(d) - off < 8:
        return None
    klen = struct.unpack_from("<Q", d, off)[0]
    if klen > len(d) - off - 8:
        return None
    k = d[off + 8:off + 8 + klen]
    return (k > key) - (k < key)


def seek(d: bytes, ix: bytes, key: bytes):
    """seek_t(key): (the first position a with no record before it comparing >= key on the probe path, None), or
    (None, the corrupt record the search probed)."""
    a, b = 0, len(ix) // 16
    while a < b:
        mid = a + (b - a) // 2
        c = _probe(d, ix, mid, key)
        if c is None:
            return None, mid
        if c < 0:
            a = mid + 1
        else:
            b = mid
    return a, None


def _index_panics(d: bytes, ix: bytes, rec: int) -> bool:
    off, _, fs = struct.unpack_from("<QII", ix, 16 * rec)
    return fs == 0 or off > len(d) or fs > len(d) - off


def spans(tables, ranges):
    """Per table, the merged record spans, up to (not including) the first table with no index record or a failed seek;
    and that table's stop, or None."""
    out = []
    for t, tb in enumerate(tables):
        d, ix = bytes(np.asarray(tb[0], np.uint8)), bytes(np.asarray(tb[1], np.uint8))
        if len(ix) < 16:
            return out, (t, PANIC, 0)
        iv, bad = [], []
        for start, end in ranges:
            if not bytes(start) < bytes(end):
                continue
            lo, b0 = seek(d, ix, bytes(start))
            hi, b1 = seek(d, ix, bytes(end))
            bad += [r for r in (b0, b1) if r is not None]
            if lo is not None and hi is not None and lo < hi:
                iv.append((lo, hi))
        if bad:
            r = min(bad)
            return out, (t, PANIC if _index_panics(d, ix, r) else ERR, r)
        merged = []
        for lo, hi in sorted(iv):
            if merged and lo <= merged[-1][1]:
                merged[-1] = (merged[-1][0], max(merged[-1][1], hi))
            else:
                merged.append((lo, hi))
        out.append(merged)
    return out, None


def cut(tables, sp):
    """The tables cut down to their spans: [(data, index)] and, per cut table, (original table, [(cut start, span)])."""
    cut_tables, where = [], []
    for t, s in enumerate(sp):
        if not s:
            continue
        d, ix = np.asarray(tables[t][0], np.uint8), np.asarray(tables[t][1], np.uint8)
        parts, pos = [], []
        c = 0
        for lo, hi in s:
            parts.append(ix[16 * lo:16 * hi])
            pos.append((c, lo, hi))
            c += hi - lo
        cut_tables.append((d, np.concatenate(parts)))
        where.append((t, pos))
    return cut_tables, where


def reader_scan(tables, ranges):
    """dbeel_reader_scan(DBEEL_SCAN_KEY): ([(data, index)] per range, (table, reason, record))."""
    sp, seek_stop = spans(tables, ranges)
    cut_tables, where = cut(tables, sp)
    if cut_tables:
        out, (t, reason, rec) = scan_oracle.scan(cut_tables, ranges, KEY)
    else:
        out = scan_oracle.scan([], ranges, KEY)[0]
        t, reason, rec = -1, NONE, 0
    if t >= 0:
        orig, pos = where[t]
        c, lo, _ = [p for p in pos if p[0] <= rec][-1]
        return out, (orig, reason, lo + rec - c)
    return out, seek_stop or (-1, NONE, 0)
