"""A table past 2^32 records that exists only as a function of the record number, and a closed-form model of what every
read entry point returns on it (tests/test_gpu_reads_past_4gib.py; the model itself is checked on the CPU by
tests/test_reads_past_4gib_model.py).

T_big has N_BIG = 2^32 + 2^20 + 3 records of 48 bytes each: record r is the entry (key be64(2r + 1), value le64(r),
timestamp BIG_TS) at .data offset 48 r, and its .index record is (48 r, key_size 16, full_size 48).  Keys ascend with r
and the even values be64(2r) fall between records, so a key names its record and every returned entry names its own
record.  .data is 192 GiB and .index 64 GiB; a read callback synthesises any byte range of either on demand.

The model reads a table only through Table.read, the same bytes the engine's callback serves, and restates the
searches of lookup.cuh (both modes), seek_t, dbeel_scan's decode and the range rules of include/dbeel_compact.h.  It
never asks the engine.
"""
from __future__ import annotations

import struct

import numpy as np

from dbeel_b200 import capi
from helpers import BASE_TS
from scan_cases import ERR, NONE, PANIC, _decode

ENT = 48                            # full_size of every T_big entry: u64 8 | 8-byte key | u64 8 | 8-byte value | i128 ts
N_BIG = (1 << 32) + (1 << 20) + 3
TWO32 = 1 << 32
BIG_TS = BASE_TS
BAD_TS = 10 ** 30                   # scan_cases.damage's "timestamp" defect: a timestamp that does not decode
MORE, STOPPED, UNSORTED = 0x1, 0x2, 0x4
BAD_ENTRY, CORRUPT = capi.LOOKUP_BAD_ENTRY, capi.LOOKUP_CORRUPT
_TS16 = np.frombuffer(BIG_TS.to_bytes(16, "little", signed=True), np.uint8)
_BAD16 = np.frombuffer(BAD_TS.to_bytes(16, "little", signed=True), np.uint8)
_LE8 = np.frombuffer((8).to_bytes(8, "little"), np.uint8)
MAX_READ = 256 << 20                # the largest single read the synthetic files serve (a leaf is about 4 MiB)


def key_of(r: int) -> bytes:
    """The key of T_big's record r; key_of(r) with 2r + 1 replaced by 2r is a miss just below it."""
    return (2 * r + 1).to_bytes(8, "big")


def miss_below(r: int) -> bytes:
    return (2 * r).to_bytes(8, "big")


def value_of(r: int) -> bytes:
    return r.to_bytes(8, "little")


def entry_of(r: int, ts: int = BIG_TS) -> bytes:
    return (8).to_bytes(8, "little") + key_of(r) + (8).to_bytes(8, "little") + value_of(r) + ts.to_bytes(16, "little", signed=True)


class SynTable:
    """T_big (or a damaged copy of it: defects = {record: "offset_eof" | "timestamp"}, scan_cases.damage's defects of those
    names) as a read callback over n records."""

    def __init__(self, n: int = N_BIG, defects=None):
        self.n = n
        self.data_len, self.index_len = ENT * n, 16 * n
        self.defects = dict(defects or {})
        for r, kind in self.defects.items():
            assert kind in ("offset_eof", "timestamp") and 0 <= r < n - 1

    def index_records(self, r0: int, r1: int) -> np.ndarray:
        """.index records r0 .. r1 - 1 as a (count, 16) byte array."""
        rec = np.empty((r1 - r0, 2), "<u8")
        rec[:, 0] = np.arange(r0, r1, dtype=np.uint64) * np.uint64(ENT)
        rec[:, 1] = np.uint64(16 | (ENT << 32))
        for r, kind in self.defects.items():
            if kind == "offset_eof" and r0 <= r < r1:
                rec[r - r0, 0] = self.data_len - ENT + 1   # the entry would end one byte past .data
        return rec.view(np.uint8).reshape(-1, 16)

    def entries(self, r0: int, r1: int) -> np.ndarray:
        """.data of records r0 .. r1 - 1 as a (count, 48) byte array."""
        r = np.arange(r0, r1, dtype=np.uint64)
        e = np.empty((r1 - r0, ENT), np.uint8)
        e[:, 0:8] = _LE8
        e[:, 8:16] = (2 * r + 1).astype(">u8").view(np.uint8).reshape(-1, 8)
        e[:, 16:24] = _LE8
        e[:, 24:32] = r.astype("<u8").view(np.uint8).reshape(-1, 8)
        e[:, 32:48] = _TS16
        for d, kind in self.defects.items():
            if kind == "timestamp" and r0 <= d < r1:
                e[d - r0, 32:48] = _BAD16
        return e

    def read(self, kind: int, off: int, size: int):
        """The callback's answer: the bytes [off, off + size) of .data (kind 1) or .index (kind 2), or error 4243 for a
        read outside the file.  Reads may start and end inside a record."""
        flen, unit = (self.data_len, ENT) if kind == 1 else (self.index_len, 16)
        if off < 0 or size < 0 or off + size > flen or size > MAX_READ:
            return 4243
        if size == 0:
            return np.zeros(0, np.uint8)
        r0, r1 = off // unit, (off + size + unit - 1) // unit
        blk = self.entries(r0, r1) if kind == 1 else self.index_records(r0, r1)
        lo = off - unit * r0
        return blk.reshape(-1)[lo:lo + size]

    def callback(self):
        return lambda _t, kind, off, size: self.read(kind, off, size)


class MemTable:
    """A materialised SSTable pair behind the same read interface."""

    def __init__(self, data, index):
        self.data, self.index = np.asarray(data, np.uint8), np.asarray(index, np.uint8)
        self.data_len, self.index_len, self.n = self.data.size, self.index.size, self.index.size // 16

    def read(self, kind: int, off: int, size: int):
        f = self.data if kind == 1 else self.index
        return f[off:off + size] if 0 <= off and off + size <= f.size else 4243


def _bytes(t, kind, off, size) -> bytes:
    got = t.read(kind, off, size)
    assert not isinstance(got, int), (kind, off, size)
    return bytes(np.asarray(got, np.uint8))


def index_record(t, r: int):
    return struct.unpack("<QII", _bytes(t, 2, 16 * r, 16))


def probe(t, r: int, key: bytes):
    """lookup.cuh's probe(): the comparison of record r's key with `key` (<0, 0, >0), or None when it is corrupt."""
    off = index_record(t, r)[0]
    if off > t.data_len or t.data_len - off < 8:
        return None
    klen = struct.unpack("<Q", _bytes(t, 1, off, 8))[0]
    if klen > t.data_len - off - 8:
        return None
    k = _bytes(t, 1, off + 8, klen)
    return (k > key) - (k < key)


def search(t, key: bytes, mode: int):
    """One table's search in lookup_query: (record | None, corrupt).  Mode 0 is the reference's binary_search loop with
    its exit after index 0 (ref_binary_search of test_gpu_get_values_stream.py for any n); mode 1 a lower-bound search."""
    n = t.n
    if n == 0:
        return None, False
    if mode == capi.LOOKUP_REFERENCE:
        half, high, low = n // 2, n - 1, 0
        while True:
            c = probe(t, half, key)
            if c is None:
                return None, True
            if c == 0:
                return half, False
            low = half + 1 if c < 0 else low
            high = max(half, 1) - 1 if c > 0 else high
            if half == 0 or half == n:
                return None, False
            half = (high + low) // 2
            if low > high:
                return None, False
    lo, hi = 0, n
    while lo < hi:
        mid = lo + (hi - lo) // 2
        c = probe(t, mid, key)
        if c is None:
            return None, True
        if c == 0:
            return mid, False
        if c < 0:
            lo = mid + 1
        else:
            hi = mid
    return None, False


def _ts_decodes(ts: int) -> bool:
    secs = ts // 1_000_000_000
    secs = ((secs + (1 << 63)) % (1 << 64)) - (1 << 63)
    return -377705116800 <= secs <= 253402300799


def hit_entry(t, r: int, klen: int):
    """k_lookup_emit's decode of a hit: the entry's bytes, or None when it does not decode (LOOKUP_BAD_ENTRY)."""
    off, ks, fs = index_record(t, r)
    if not (ks == 8 + klen and fs >= ks + 24 and fs <= t.data_len - off):
        return None
    e = _bytes(t, 1, off, fs)
    if struct.unpack_from("<Q", e, ks)[0] != fs - ks - 24:
        return None
    return e if _ts_decodes(int.from_bytes(e[fs - 16:], "little", signed=True)) else None


def lookup_rows(tables, keys, mode: int):
    """get_values' rows alone: (rows as LOOKUP_DTYPE, [(table, record)] of the answered rows in query order).  The hit's
    decode (hit_entry's checks) reads only its index record, its dlen and its timestamp, so entries may be gigabytes."""
    rows = np.zeros(len(keys), capi.LOOKUP_DTYPE)
    answered = []
    for q, key in enumerate(keys):
        table, flags, rec = -1, 0, 0
        for ti in range(len(tables) - 1, -1, -1):
            r, bad = search(tables[ti], key, mode)
            if bad:
                flags |= CORRUPT
                break
            if r is not None:
                table, rec = ti, r
                break
        if table >= 0:
            t = tables[table]
            off, ks, fs = index_record(t, rec)
            ok = ks == 8 + len(key) and ks + 24 <= fs <= t.data_len - off
            ok = ok and struct.unpack("<Q", _bytes(t, 1, off + ks, 8))[0] == fs - ks - 24
            if ok and _ts_decodes(int.from_bytes(_bytes(t, 1, off + fs - 16, 16), "little", signed=True)):
                answered.append((table, rec))
            else:
                flags |= BAD_ENTRY
        rows[q] = (table, flags, rec)
    return rows, answered


def get_values(tables, keys, mode: int):
    """dbeel_get_values on tables (oldest first, no filters): (rows as LOOKUP_DTYPE, data, index), the index records
    running sums of full_size in query order."""
    rows = np.zeros(len(keys), capi.LOOKUP_DTYPE)
    ents = []
    for q, key in enumerate(keys):
        table, flags, rec = -1, 0, 0
        for ti in range(len(tables) - 1, -1, -1):
            r, bad = search(tables[ti], key, mode)
            if bad:
                flags |= CORRUPT
                break
            if r is not None:
                table, rec = ti, r
                break
        if table >= 0:
            e = hit_entry(tables[table], rec, len(key))
            if e is None:
                flags |= BAD_ENTRY
            else:
                ents.append(e)
        rows[q] = (table, flags, rec)
    return (rows,) + pack(ents)


def pack(ents):
    """Entries back to back and their .index: offsets the running sums of full_size, key_size 8 + klen."""
    idx = np.zeros((len(ents), 2), "<u8")
    pos = 0
    for j, e in enumerate(ents):
        klen = struct.unpack_from("<Q", e, 0)[0]
        idx[j] = (pos, (8 + klen) | (len(e) << 32))
        pos += len(e)
    return np.frombuffer(b"".join(ents), np.uint8).copy(), idx.view(np.uint8).reshape(-1)


# ------------------------------------------------------------------------------------------------------------ key ranges


def seek(t, key: bytes):
    """seek_t(key) (seek_oracle.seek over the read interface): (position, None) or (None, the corrupt record probed)."""
    a, b = 0, t.n
    while a < b:
        mid = a + (b - a) // 2
        c = probe(t, mid, key)
        if c is None:
            return None, mid
        if c < 0:
            a = mid + 1
        else:
            b = mid
    return a, None


def record_damage(t, r: int):
    """ERR / PANIC as dbeel_scan classifies record r, or None when it decodes."""
    off, _, fs = index_record(t, r)
    if fs == 0 or off > t.data_len or fs > t.data_len - off:
        return PANIC
    return None if _decode(_bytes(t, 1, off, fs)) else ERR


def span(t, rng_):
    """The records [lo, hi) of one table a key range covers, or a stop (PANIC / ERR, record) of its bound searches."""
    lo, b0 = seek(t, bytes(rng_[0]))
    hi, b1 = seek(t, bytes(rng_[1]))
    bad = [r for r in (b0, b1) if r is not None]
    if bad:
        r = min(bad)
        off, _, fs = index_record(t, r)
        return None, (PANIC if fs == 0 or off > t.data_len or fs > t.data_len - off else ERR, r)
    return (lo, max(lo, hi)), None


def span_entries(t, lo: int, hi: int, reverse: bool = False):
    """Walk records [lo, hi) up (or down): ([(key, entry bytes)] up to the first damaged record, (reason, record) of it or
    None)."""
    out = []
    for r in (range(hi - 1, lo - 1, -1) if reverse else range(lo, hi)):
        why = record_damage(t, r)
        if why is not None:
            return out, (why, r)
        off, _, fs = index_record(t, r)
        e = _bytes(t, 1, off, fs)
        out.append((_decode(e)[0], e))
    return out, None


def reader_scan(t, ranges):
    """dbeel_reader_scan(SCAN_KEY) on a reader of the one table t: ([(data, index)] per range, stop, span records)."""
    spans = []
    for rng_ in ranges:
        if not bytes(rng_[0]) < bytes(rng_[1]):
            continue
        s, stop = span(t, rng_)
        if stop is not None:
            return [pack([]) for _ in ranges], (0, stop[0], stop[1]), 0
        if s[0] < s[1]:
            spans.append(s)
    merged = []
    for lo, hi in sorted(spans):
        if merged and lo <= merged[-1][1]:
            merged[-1] = (merged[-1][0], max(merged[-1][1], hi))
        else:
            merged.append((lo, hi))
    outs = [[] for _ in ranges]
    stop = (-1, NONE, 0)
    for lo, hi in merged:
        got, bad = span_entries(t, lo, hi)
        for key, e in got:
            d = next((j for j, (a, b) in enumerate(ranges) if bytes(a) <= key < bytes(b)), None)
            if d is not None:
                outs[d].append(e)
        if bad is not None:
            stop = (0, bad[0], bad[1])
            break
    return [pack(o) for o in outs], stop, sum(hi - lo for lo, hi in merged)


def _merge(versions, keep_tombstones):
    """versions: [(key, entry)] oldest table first; the last version of every key, ascending, tombstones per the flag."""
    last = {}
    for key, e in versions:
        last[key] = e
    return [last[k] for k in sorted(last) if keep_tombstones or struct.unpack_from("<Q", last[k], 8 + len(k))[0]]


def get_range(tables, rng_, keep_tombstones: bool):
    """G_q of dbeel_reader_get_range for one range on sorted tables: (entries, stop)."""
    versions = []
    if not bytes(rng_[0]) < bytes(rng_[1]):
        return [], (-1, NONE, 0)
    for ti, t in enumerate(tables):
        s, stop = span(t, rng_)
        if stop is not None:
            return [], (ti, stop[0], stop[1])
        got, bad = span_entries(t, *s)
        if bad is not None:
            return [], (ti, bad[0], bad[1])
        versions += got
    return _merge(versions, keep_tombstones), (-1, NONE, 0)


def limited_rule(tables, rng_, limit: int, keep_tombstones: bool, reverse: bool):
    """What a row of dbeel_reader_get_ranges(_reverse) may be: ("clean", entries, flags) or ("damaged", A_q entries in
    output order, more, {(table, record): reason})."""
    g, stop = get_range(tables, rng_, keep_tombstones)
    if stop[0] < 0:
        g = g[::-1] if reverse else g
        return "clean", g[:limit], MORE if len(g) > limit else 0
    versions, bad = [], {}
    for ti, t in enumerate(tables):
        s, sstop = span(t, rng_)
        assert sstop is None, "the damage is on a bound search: not a case the big-table tests make"
        got, why = span_entries(t, *s, reverse=reverse)
        versions += got
        if why is not None:
            bad[(ti, why[1])] = why[0]
    a = _merge(versions, keep_tombstones)
    a = a[::-1] if reverse else a
    return "damaged", a[:limit], MORE if len(a) > limit else 0, bad


def check_limited_row(tables, rng_, limit, keep_tombstones, reverse, row, entries):
    """One row (first, count, flags, table, reason, record) and its entries against limited_rule."""
    flags, count = int(row["flags"]), int(row["count"])
    stop = (int(row["table"]), int(row["reason"]), int(row["record"]))
    want = limited_rule(tables, rng_, limit, keep_tombstones, reverse)
    if want[0] == "clean":
        assert (flags, stop) == (want[2], (-1, NONE, 0)), (rng_, limit, row, want[2])
        assert entries == want[1], f"range {rng_} limit {limit}: entries differ from the model"
        return None
    if flags & STOPPED:
        assert flags == STOPPED and count == 0 and not entries, row
        assert want[3].get((stop[0], stop[2])) == stop[1], f"stop {stop} is not a damaged record {want[3]}"
        return stop
    assert flags == want[2] and stop == (-1, NONE, 0), (row, want[2])
    assert entries == want[1], f"damaged range {rng_} limit {limit}: entries differ from A_q"
    return None


# ------------------------------------------------------------------------------------------------- fences of a reader


NODE_BYTES = 2 * (16 + 8 + 80)   # one probe-tree node of a reader's cached fences, both modes (host/lookup_plan.h)


def lookup_max_depth(n: int) -> int:
    d = 0
    while d < 16 and (2 << d) <= n:
        d += 1
    return d


def reader_depths(ns, data_lens, fence_bytes: int = 0):
    """reader_depths (host/lookup_plan.h) for tables opened together: each next level goes to the table whose leaves are
    largest ((data_len + 16 n) >> D, ties to the lower position) while it fits the budget."""
    left = fence_bytes or capi.DEFAULT_READER_FENCE_BYTES
    d = [0] * len(ns)
    open_ = set(range(len(ns)))
    while open_:
        t = max(open_, key=lambda j: ((data_lens[j] + 16 * ns[j]) >> d[j], -j))
        open_.discard(t)
        step = (NODE_BYTES << (d[t] + 1)) - (NODE_BYTES << d[t] if d[t] else 0)
        if d[t] >= lookup_max_depth(ns[t]) or step > left:
            continue
        left -= step
        d[t] += 1
        open_.add(t)
    return d


# --------------------------------------------------------------------------------------------------- compare helpers


def compare_rows(what, got, want):
    """Rows field by field; a record is reported with its high word, so a truncation to 32 bits names itself."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: {got.shape[0]} rows, model {want.shape[0]}"
    for f in ("table", "bloom_rejects", "record"):
        bad = np.flatnonzero(got[f] != want[f])
        if bad.size:
            q = int(bad[0])
            raise AssertionError(f"{what}: row {q} {f} is {int(got[f][q])} (high word {int(got[f][q]) >> 32}), "
                                 f"model {int(want[f][q])} (high word {int(want[f][q]) >> 32})")


def compare_out(what, got_data, got_index, want_data, want_index):
    """An output SSTable pair against the model: .index record by record (offsets with their high word), then .data."""
    gi, wi = np.asarray(got_index, np.uint8), np.asarray(want_index, np.uint8)
    assert gi.size == wi.size, f"{what}: .index is {gi.size} bytes, model {wi.size}"
    if not np.array_equal(gi, wi):
        b = int(np.flatnonzero(gi != wi)[0])
        field = ("offset low word", "offset high word", "key_size", "full_size")[b % 16 // 4]
        raise AssertionError(f"{what}: .index differs at record {b // 16} ({field})")
    gd, wd = np.asarray(got_data, np.uint8), np.asarray(want_data, np.uint8)
    assert gd.size == wd.size, f"{what}: .data is {gd.size} bytes, model {wd.size}"
    if not np.array_equal(gd, wd):
        b = int(np.flatnonzero(gd != wd)[0])
        raise AssertionError(f"{what}: .data differs at byte {b} (0x{b:x})")


def compare_stop(what, got, want):
    got, want = tuple(int(x) for x in got), tuple(int(x) for x in want)
    assert got == want, f"{what}: stop {got} (record high word {got[2] >> 32}), model {want} (high word {want[2] >> 32})"
