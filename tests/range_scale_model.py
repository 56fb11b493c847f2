"""A vectorised model of the reader's key-range reads on trees of integer keys, for trees of millions of records.

A tree is a list of tables, oldest first.  Table t holds a set of integers i (a sorted numpy array) and a tombstone flag
per integer.  Integer i has the key ``prefix + be64(i)``: with the default empty prefix every comparison is decided by the
8-byte key prefix the kernels compare first; with SHARED_PREFIX every 8-byte prefix ties and the full key comparison
decides.  A live entry's value is ``le32(t) ++ le32(i)`` (8 bytes), so every output entry names its table and record; a
tombstone has an empty value.  Timestamps are BASE_TS + t.

A key range is a pair of integers (a, b): the keys [key(a), key(b)).  Since every key has the same length, key order is
integer order, so every answer is computed on the integers and turned into bytes only at the end (entries).

The answers restate, in numpy, what tests/range_oracle.py, range_limit_oracle.py, range_limit_rev_oracle.py and
seek_oracle.py say for clean, sorted trees (tests/test_range_scale_model.py checks that they agree):

  reader_scan   per destination d, every span record whose key lies in range d and in no earlier range, in iteration
                order (tables ascending, each in record order)
  get_range     per destination, those records merged: the newest table's version of every key, ascending, tombstones
                dropped unless kept
  get_ranges    per query, get_range of its range alone (G_q) cut to the limit -- its first entries, or with reverse its
                last entries in descending key order -- with MORE when G_q holds more
"""
from __future__ import annotations

import numpy as np

from dbeel_b200 import sstable

BASE_TS = 1_700_000_000_000_000_000
SHARED_PREFIX = b"SHAREDPF"
MORE = 0x1


def keys_of(ids, prefix: bytes = b"") -> np.ndarray:
    """[n, len(prefix) + 8] uint8: prefix + be64(i) per integer."""
    ids = np.asarray(ids, np.uint64)
    out = np.empty((ids.size, len(prefix) + 8), np.uint8)
    if prefix:
        out[:, :len(prefix)] = np.frombuffer(prefix, np.uint8)
    out[:, len(prefix):] = ids.astype(">u8").view(np.uint8).reshape(-1, 8)
    return out


def key(i: int, prefix: bytes = b"") -> bytes:
    return prefix + int(i).to_bytes(8, "big")


def entries(ids, tabs, tomb, prefix: bytes = b""):
    """(data, index) of one SSTable holding the entries (ids[k] of table tabs[k], a tombstone when tomb[k]) in the given
    order -- what sstable.build_run writes for them, built without a per-entry loop."""
    ids = np.asarray(ids, np.uint64)
    n = ids.size
    tabs = np.broadcast_to(np.asarray(tabs, np.int64), (n,))
    tomb = np.broadcast_to(np.asarray(tomb, bool), (n,))
    if n == 0:
        return np.zeros(0, np.uint8), np.zeros(0, np.uint8)
    k = keys_of(ids, prefix)
    klen = k.shape[1]
    full = sstable.ENTRY_OVERHEAD + klen + 8
    dense = np.empty((n, full), np.uint8)
    doc = dense[:, 16 + klen:24 + klen]
    doc[:, 0:4] = tabs.astype("<u4").view(np.uint8).reshape(n, 4)
    doc[:, 4:8] = ids.astype("<u4").view(np.uint8).reshape(n, 4)
    # every row laid out as a live entry; the tombstones then lose their 8 value bytes and get dlen = 0
    data, index = sstable.build_run_dense(dense, k, BASE_TS + tabs, np.zeros(n, bool))
    if not tomb.any():
        return data, index
    dense[tomb, 8 + klen:16 + klen] = 0
    keep = np.ones((n, full), bool)
    keep[tomb, 16 + klen:24 + klen] = False
    sizes = np.where(tomb, full - 8, full).astype(np.uint64)
    offsets = np.zeros(n, np.uint64)
    np.cumsum(sizes[:-1], out=offsets[1:])
    ix = index.view("<u4").reshape(n, 4)
    ix[:, 0:2] = offsets.astype("<u8").view("<u4").reshape(n, 2)
    ix[:, 3] = sizes.astype("<u4")
    return dense[keep], index


class Tree:
    """Tables of integers, oldest first: tables[t] = (ids ascending, tombstone flags)."""

    def __init__(self, tables, prefix: bytes = b""):
        self.tables = [(np.asarray(ids, np.uint64), np.asarray(tomb, bool)) for ids, tomb in tables]
        for ids, tomb in self.tables:
            assert ids.size == tomb.size and (ids.size < 2 or bool(np.all(ids[1:] > ids[:-1])))
        self.prefix = prefix

    def built(self):
        """[(data, index)] of every table."""
        return [entries(ids, t, tomb, self.prefix) for t, (ids, tomb) in enumerate(self.tables)]

    def bounds(self, ranges):
        """The ranges as the key pairs the reader takes."""
        return [(key(a, self.prefix), key(b, self.prefix)) for a, b in ranges]

    def span(self, a: int, b: int):
        """Per table, its records [lo, hi) with keys in [key(a), key(b))."""
        if a >= b:
            return [(0, 0) for _ in self.tables]
        return [(int(np.searchsorted(ids, a)), int(np.searchsorted(ids, b))) for ids, _ in self.tables]

    def count(self, a: int, b: int) -> int:
        """Span records of range (a, b): what one destination's span holds."""
        return sum(hi - lo for lo, hi in self.span(a, b))

    def _gather(self, pick):
        """Concatenated (ids, tables, tombs) of pick(t, ids) -> a mask or slice per table, tables ascending."""
        ids, tabs, tombs = [], [], []
        for t, (x, tb) in enumerate(self.tables):
            s = pick(t, x)
            ids.append(x[s])
            tabs.append(np.full(ids[-1].size, t, np.int64))
            tombs.append(tb[s])
        return np.concatenate(ids), np.concatenate(tabs), np.concatenate(tombs)

    def _dest(self, ranges, x):
        """Per integer of x, the first range holding it (-1: none) -- dbeel_scan's destination rule."""
        d = np.full(x.size, -1, np.int64)
        for j, (a, b) in enumerate(ranges):
            if a < b:
                lo, hi = np.searchsorted(x, a), np.searchsorted(x, b)
                seg = d[lo:hi]
                seg[seg < 0] = j
        return d

    def scan_records(self, ranges):
        """Per destination, (ids, tables, tombs) of its records in iteration order."""
        picks = []  # per table: its records grouped by destination, record order kept, and each group's bounds
        for x, _ in self.tables:
            d = self._dest(ranges, x)
            rec = np.flatnonzero(d >= 0)
            rec = rec[np.argsort(d[rec], kind="stable")]
            picks.append((rec, np.searchsorted(d[rec], np.arange(len(ranges) + 1))))
        return [self._gather(lambda t, x, j=j: picks[t][0][picks[t][1][j]:picks[t][1][j + 1]]) for j in range(len(ranges))]

    def reader_scan(self, ranges):
        """dbeel_reader_scan(DBEEL_SCAN_KEY) per destination: (data, index)."""
        return [entries(i, t, tb, self.prefix) for i, t, tb in self.scan_records(ranges)]

    @staticmethod
    def merge(ids, tabs, tombs, keep_tombstones: bool = False):
        """The newest table's version of every key, ascending, tombstones dropped unless kept: (ids, tables, tombs)."""
        order = np.lexsort((tabs, ids))
        ids, tabs, tombs = ids[order], tabs[order], tombs[order]
        last = np.ones(ids.size, bool)
        last[:-1] = ids[1:] != ids[:-1]
        if not keep_tombstones:
            last &= ~tombs
        return ids[last], tabs[last], tombs[last]

    def get_range(self, ranges, keep_tombstones: bool = False):
        """dbeel_reader_get_range per destination: (data, index)."""
        return [entries(*self.merge(*r, keep_tombstones), self.prefix) for r in self.scan_records(ranges)]

    def group(self, a: int, b: int, keep_tombstones: bool = False):
        """G_q of range (a, b) alone: (ids, tables, tombs) ascending."""
        sp = self.span(a, b)
        return self.merge(*self._gather(lambda t, x: slice(*sp[t])), keep_tombstones)

    def get_ranges(self, ranges, limits, keep_tombstones: bool = False, reverse: bool = False):
        """dbeel_reader_get_ranges / _reverse: (first, count, flags) per query as int64 arrays, and the packed (data,
        index) of every query's entries in query order."""
        lim = np.broadcast_to(np.asarray(limits, np.int64), (len(ranges),))
        first, count, flags, parts = [], [], [], []
        at = 0
        for (a, b), L in zip(ranges, lim.tolist()):
            ids, tabs, tombs = self.group(a, b, keep_tombstones)
            if reverse:
                ids, tabs, tombs = ids[::-1], tabs[::-1], tombs[::-1]
            c = min(ids.size, L)
            first.append(at)
            count.append(c)
            flags.append(MORE if ids.size > L else 0)
            parts.append((ids[:c], tabs[:c], tombs[:c]))
            at += c
        cat = [np.concatenate([p[k] for p in parts]) if parts else np.zeros(0) for k in range(3)]
        return (np.array(first, np.int64), np.array(count, np.int64), np.array(flags, np.int64)), \
            entries(*cat, self.prefix)

    def group_size(self, a: int, b: int, keep_tombstones: bool = False) -> int:
        return int(self.group(a, b, keep_tombstones)[0].size)


def cumulative(tree: Tree, end: int) -> np.ndarray:
    """C[x] = span records of (0, x) for x in [0, end]: the records of all tables with key below key(x)."""
    c = np.zeros(end + 1, np.int64)
    for ids, _ in tree.tables:
        c += np.searchsorted(ids, np.arange(end + 1, dtype=np.uint64)).astype(np.int64)
    return c


def range_with(c: np.ndarray, a: int, n: int):
    """The first (a', b) with a' >= a, c[b] - c[a'] == n and a' < b (a range of exactly n span records), or None."""
    for s in range(a, min(a + 4096, c.size - 1)):
        want = c[s] + n
        b = int(np.searchsorted(c, want))
        if b < c.size and c[b] == want and b > s:
            return s, b
    return None
