"""A pure-Python restatement of dbeel_reader_get_range (include/dbeel_compact.h) on top of the seek oracle: S_d is what
seek_oracle.reader_scan returns for destination d; the result keeps the last entry of S_d per key, sorted by key, with
tombstones (dlen == 0) dropped unless asked for.  A stop is the raw scan's stop with empty results; with no stop, a table
whose span records do not strictly ascend by key is DBEEL_ERR_UNSORTED_RUN."""
from __future__ import annotations

import struct

import numpy as np

import seek_oracle
from dbeel_b200 import sstable

UNSORTED = "unsorted"


def _records(d: bytes, ix: bytes):
    """(key, entry bytes) of every index record of one SSTable pair, in record order."""
    out = []
    for r in range(len(ix) // 16):
        off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
        e = d[off:off + fs]
        klen = struct.unpack_from("<Q", e, 0)[0]
        out.append((e[8:8 + klen], e))
    return out


def _pack(entries):
    d, i = bytearray(), bytearray()
    for key, e in entries:
        i += sstable.encode_index_record(len(d), len(key), len(e))
        d += e
    return np.frombuffer(bytes(d), np.uint8).copy(), np.frombuffer(bytes(i), np.uint8).copy()


def merge(d, ix, keep_tombstones: bool = False):
    """One destination's S_d (an SSTable pair) merged: last entry per key, ascending keys, tombstones per the flag."""
    last = {}
    for key, e in _records(bytes(np.asarray(d, np.uint8)), bytes(np.asarray(ix, np.uint8))):
        last[key] = e
    keep = []
    for key in sorted(last):
        e = last[key]
        dlen = struct.unpack_from("<Q", e, 8 + len(key))[0]
        if dlen or keep_tombstones:
            keep.append((key, e))
    return _pack(keep)


def unsorted_tables(tables, ranges):
    """Tables whose span records (the union of their spans, in record order) do not strictly ascend by key."""
    sp, _ = seek_oracle.spans(tables, ranges)
    bad = []
    for t, s in enumerate(sp):
        d, ix = bytes(np.asarray(tables[t][0], np.uint8)), bytes(np.asarray(tables[t][1], np.uint8))
        keys = [k for lo, hi in s for k, _ in _records(d, ix[16 * lo:16 * hi])]
        if any(a >= b for a, b in zip(keys, keys[1:])):
            bad.append(t)
    return bad


def get_range(tables, ranges, keep_tombstones: bool = False):
    """([(data, index)] per range, (table, reason, record)), or UNSORTED for DBEEL_ERR_UNSORTED_RUN."""
    out, stop = seek_oracle.reader_scan(tables, ranges)
    empty = (np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    if stop[0] >= 0:
        return [empty for _ in ranges], stop
    if unsorted_tables(tables, ranges):
        return UNSORTED
    return [merge(d, i, keep_tombstones) for d, i in out], stop
