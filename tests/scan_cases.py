"""Trees, ranges and damage for the scan tests, plus an independent pure-Python restatement of the SSTable part of
LSMTree::iter_filter (AsyncIter::read_one, lsm_tree.rs:210-281, with migration.rs's between_cmp :54-60)."""
from __future__ import annotations

import struct

import numpy as np

from dbeel_b200 import sstable
from helpers import BASE_TS, nasty_keys

HASH, KEY = 0, 1
NONE, ERR, PANIC = 0, 1, 2


def py_murmur3_32(data: bytes, seed: int = 0) -> int:
    c1, c2, m = 0xCC9E2D51, 0x1B873593, 0xFFFFFFFF
    h = seed
    n = len(data) // 4
    for b in range(n):
        k = int.from_bytes(data[4 * b:4 * b + 4], "little")
        k = (k * c1) & m
        k = ((k << 15) | (k >> 17)) & m
        k = (k * c2) & m
        h ^= k
        h = ((h << 13) | (h >> 19)) & m
        h = (h * 5 + 0xE6546B64) & m
    tail = data[4 * n:]
    if tail:
        k = int.from_bytes(tail, "little")
        k = (k * c1) & m
        k = ((k << 15) | (k >> 17)) & m
        k = (k * c2) & m
        h ^= k
    h ^= len(data)
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & m
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & m
    h ^= h >> 16
    return h


def py_between_cmp(h: int, start: int, end: int) -> bool:
    if end < start:
        return h < start or h >= end
    return start <= h < end


def _ts_decodes(ts: int) -> bool:
    secs = ts // 1_000_000_000  # floor division, then `as i64` wraps
    secs = ((secs + (1 << 63)) % (1 << 64)) - (1 << 63)
    return -377705116800 <= secs <= 253402300799


def _decode(e: bytes):
    n = len(e)
    if n < 8:
        return None
    klen = int.from_bytes(e[:8], "little")
    if klen > n - 8 or n - 8 - klen < 8:
        return None
    dlen = int.from_bytes(e[8 + klen:16 + klen], "little")
    rest = n - 16 - klen
    if dlen > rest or rest - dlen != 16:
        return None
    ts = int.from_bytes(e[n - 16:], "little", signed=True)
    if not _ts_decodes(ts):
        return None
    return e[8:8 + klen], e[16 + klen:16 + klen + dlen], ts


def py_scan(tables, ranges, kind):
    """Returns ([(data, index)] per range, (table, reason, record))."""
    outs = [[] for _ in ranges]
    stop = (-1, NONE, 0)
    for t, tb in enumerate(tables):
        d, ix = bytes(np.asarray(tb[0], np.uint8)), bytes(np.asarray(tb[1], np.uint8))
        size = len(ix) // 16
        rec = 0
        while True:
            if 16 * rec + 16 > len(ix):
                stop = (t, PANIC, rec)
                break
            off, _key_size, fs = struct.unpack_from("<QII", ix, 16 * rec)
            if fs == 0 or off + fs > len(d):
                stop = (t, PANIC, rec)
                break
            ent = _decode(d[off:off + fs])
            if ent is None:
                stop = (t, ERR, rec)
                break
            k = ent[0]
            for j, (a, b) in enumerate(ranges):
                if (py_between_cmp(py_murmur3_32(k), a, b) if kind == HASH else a <= k < b):
                    outs[j].append(ent)
                    break
            rec += 1
            if rec >= size:
                break
        if stop[0] >= 0:
            break
    return [sstable.build_run(o) for o in outs], stop


# ----------------------------------------------------------------------------- inputs

def random_tree(rng: np.random.Generator, n_tables: int, max_entries: int = 60, big: bool = False):
    """Tables of ragged sizes (some empty of entries but never of records unless asked), adversarial keys, duplicates
    across tables, tombstones; one table's index records shuffled and one record repeated (offsets need not run)."""
    pool = nasty_keys(rng, max(8, 3 * max_entries))
    tables = []
    for t in range(n_tables):
        n = int(rng.integers(1, max_entries + 1))
        idx = rng.choice(len(pool), size=min(n, len(pool)), replace=False)
        ents = []
        for k in sorted(pool[i] for i in idx):
            v = b"" if rng.random() < 0.15 else bytes(rng.integers(0, 256, int(rng.integers(1, 80)), dtype=np.uint8))
            ents.append((k, v, BASE_TS + int(rng.integers(-50, 50))))
        if big and t == 0:
            ents[0] = (ents[0][0], bytes(rng.integers(0, 256, 3_000_000 + int(rng.integers(0, 100)), dtype=np.uint8)), BASE_TS)
        d, i = sstable.build_run(ents)
        tables.append((np.asarray(d, np.uint8).copy(), np.asarray(i, np.uint8).copy()))
    if n_tables >= 2:  # read order != .data order, and one entry listed twice
        d, i = tables[1]
        recs = i.reshape(-1, 16).copy()
        rng.shuffle(recs)
        recs = np.concatenate([recs, recs[:1]])
        tables[1] = (d, recs.reshape(-1).copy())
    return tables


def hash_ranges(rng: np.random.Generator, n: int):
    """n ranges: some ordinary, some wrapped (end < start: every hash), some empty (start == end), overlapping."""
    out = []
    for j in range(n):
        a, b = (int(x) for x in rng.integers(0, 1 << 32, 2, dtype=np.uint64))
        style = j % 7
        if style == 0:
            out.append((a, a))
        elif style == 1 and n > 1 and j > n // 2:
            out.append((max(a, b), min(a, b)))  # wrapped
        else:
            out.append((min(a, b), max(a, b)))
    return out


def eighths():
    step = 1 << 29
    return [(k * step, (k + 1) * step if k < 7 else 0xFFFFFFFF) for k in range(8)]


def key_ranges(tables):
    keys = sorted({k for d, i in tables for k, _, _ in _entries(d, i)})
    mid = keys[len(keys) // 2] if keys else b"m"
    return [(b"", b"\x00"), (b"ab", b"ab\x00\x00"), (mid, b"\xff\xff\xff\xff"), (b"", b"\xff" * 64), (b"\x00", mid)]


def _entries(d, ix):
    out = []
    ix = bytes(np.asarray(ix, np.uint8))
    d = bytes(np.asarray(d, np.uint8))
    for r in range(len(ix) // 16):
        off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
        e = _decode(d[off:off + fs]) if fs and off + fs <= len(d) else None
        if e:
            out.append(e)
    return out


DAMAGES = ["full_size", "klen", "timestamp", "offset_eof", "full_size_zero", "empty_table", "ragged_index"]


def damage(tables, kind: str, t: int, rec: int):
    """A copy of `tables` with one defect at (table t, record rec)."""
    tables = [(d.copy(), i.copy()) for d, i in tables]
    d, i = tables[t]
    if kind == "empty_table":
        tables[t] = (d, i[:int(rec) % 16])
        return tables
    if kind == "ragged_index":
        tables[t] = (d, np.concatenate([i, np.full(1 + rec % 15, 7, np.uint8)]))
        return tables
    rec = rec % (i.size // 16)
    r = i[16 * rec:16 * rec + 16]
    off = int(r[:8].view("<u8")[0])
    fs = int(r[12:16].view("<u4")[0])
    if kind == "full_size":
        r[12:16] = np.array([fs - 1 if fs + off >= d.size else fs + 1], "<u4").view(np.uint8)
    elif kind == "klen":
        klen = int(d[off:off + 8].view("<u8")[0])
        d[off:off + 8] = np.array([klen + 1], "<u8").view(np.uint8)
    elif kind == "timestamp":
        d[off + fs - 16:off + fs] = np.frombuffer((10 ** 30).to_bytes(16, "little", signed=True), np.uint8)
    elif kind == "offset_eof":
        r[:8] = np.array([d.size - fs + 1], "<u8").view(np.uint8)
    elif kind == "full_size_zero":
        r[12:16] = 0
    return tables
