"""The get_values oracle (tests/get_values_oracle.c: get_entry's SSTable loop with the entry binary_search decodes,
lsm_tree.rs:605-670, 686-723) against a short, independent Python model, on hand-built tables with every rule of the
bad-entry flag, tombstones, duplicate queries and empty keys."""
import numpy as np

import get_values_oracle as gvo
from dbeel_b200 import sstable
from helpers import BASE_TS

TS_MAX = 253402300799 * 10**9 + 999_999_999  # 9999-12-31T23:59:59.999999999Z (utils/timestamp_nanos.rs:15-24)
TS_MIN = -377705116800 * 10**9                # -9999-01-01T00:00:00Z


def _rec(index, r):
    b = bytes(index[16 * r:16 * r + 16])
    return int.from_bytes(b[:8], "little"), int.from_bytes(b[8:12], "little"), int.from_bytes(b[12:], "little")


def _key_at(data, off):
    klen = int.from_bytes(bytes(data[off:off + 8]), "little")
    return bytes(data[off + 8:off + 8 + klen])


def _search(data, index, key):
    """binary_search (lsm_tree.rs:605-670) as the reference loops: the record number of the key, or None."""
    n = len(index) // 16
    if n == 0:
        return None
    half, high, low = n // 2, n - 1, 0
    while True:
        cur = _key_at(data, _rec(index, half)[0])
        if cur == key:
            return half
        if cur < key:
            low = half + 1
        else:
            high = max(half, 1) - 1
        if half == 0 or half == n:
            return None
        half = (high + low) // 2
        if low > high:
            return None


def _decode(data, index, r, key):
    """(value, timestamp) of the hit, or None when read_at(..) does not deserialize the way binary_search needs."""
    off, ks, fs = _rec(index, r)
    if ks != 8 + len(key) or fs < ks or off + fs > len(data):
        return None
    v = bytes(data[off + ks:off + fs])
    if len(v) < 8:
        return None
    dlen = int.from_bytes(v[:8], "little")
    if 8 + dlen + 16 != len(v):
        return None
    ts = int.from_bytes(v[8 + dlen:], "little", signed=True)
    if not TS_MIN <= ts <= TS_MAX:
        return None
    return v[8:8 + dlen], ts


def model(tables, keys):
    """Rows (table, bad) per key and the answered entries, newest table first, no filters."""
    rows, ents = [], []
    for k in keys:
        row = (-1, False)
        for t in range(len(tables) - 1, -1, -1):
            r = _search(tables[t][0], tables[t][1], k)
            if r is None:
                continue
            got = _decode(tables[t][0], tables[t][1], r, k)
            row = (t, got is None)
            if got is not None:
                ents.append((k, got[0], got[1]))
            break
        rows.append(row)
    return rows, sstable.build_run(ents) if ents else (np.zeros(0, np.uint8), np.zeros(0, np.uint8))


def check(tables, keys):
    blob = np.frombuffer(b"".join(keys), np.uint8) if keys else np.zeros(0, np.uint8)
    off = np.zeros(len(keys) + 1, np.uint64)
    off[1:] = np.cumsum([len(k) for k in keys]) if keys else []
    t, r, j, d, i = gvo.get_values([(td, ti, None) for td, ti in tables], blob, off)
    rows, (ed, ei) = model(tables, keys)
    assert [(int(a), bool(b & gvo.BAD_ENTRY)) for a, b in zip(t, j)] == rows
    assert bytes(d) == bytes(ed) and bytes(i) == bytes(ei)
    return t, j


def _set_u32(index, r, field, v):
    index[16 * r + field:16 * r + field + 4] = np.frombuffer(int(v).to_bytes(4, "little"), np.uint8)


def test_the_bad_entry_flag_rule_by_rule():
    ents = [(b"k%02d" % n, b"value-%d" % n, BASE_TS + n) for n in range(16)]
    keys = [k for k, _, _ in ents]
    d, i = sstable.build_run(ents)
    t, j = check([(d, i)], keys)
    assert (t >= 0).sum() >= 12 and not (j & gvo.BAD_ENTRY).any()
    for name, r, field, delta in (("key_size + 1", 5, 8, 1), ("key_size - 1", 5, 8, -1),
                                  ("value frame one byte short", 6, 12, -1), ("value frame one byte long", 6, 12, 1)):
        bad = i.copy()
        _set_u32(bad, r, field, _rec(i, r)[1 if field == 8 else 2] + delta)
        t, j = check([(d, bad)], keys)
        assert t[r] == 0 and j[r] & gvo.BAD_ENTRY, name
        assert np.count_nonzero(j & gvo.BAD_ENTRY) == 1, name
    bad = i.copy()  # full_size < key_size
    _set_u32(bad, 7, 12, _rec(i, 7)[1] - 1)
    t, j = check([(d, bad)], keys)
    assert j[7] & gvo.BAD_ENTRY
    # a value running past the end of .data: the last entry's frame loses its last byte
    t, j = check([(d[:-1].copy(), i)], keys)
    assert np.count_nonzero(j & gvo.BAD_ENTRY) == (1 if t[15] == 0 else 0)
    assert t[15] == 0 or _search(d, i, keys[15]) is None


def test_timestamps_one_nanosecond_outside_the_range():
    for ts, ok in ((TS_MAX, True), (TS_MAX + 1, False), (TS_MIN, True), (TS_MIN - 1, False)):
        d, i = sstable.build_run([(b"a", b"x", BASE_TS), (b"b", b"yy", ts), (b"c", b"zzz", BASE_TS)])
        t, j = check([(d, i)], [b"a", b"b", b"c"])
        assert bool(j[1] & gvo.BAD_ENTRY) == (not ok) and (t[1] == 0 or _search(d, i, b"b") is None), ts


def test_tombstones_duplicates_empty_keys_and_older_tables():
    old = sstable.build_run([(b"", b"old-empty", BASE_TS), (b"a", b"old-a", BASE_TS), (b"m", b"old-m", BASE_TS)])
    new = sstable.build_run([(b"", b"", BASE_TS + 1), (b"a", b"new-a", BASE_TS + 1), (b"z", b"", BASE_TS + 1)])
    keys = [b"", b"a", b"a", b"m", b"z", b"q", b"", b"m"]
    t, j = check([old, new], keys)
    assert list(t[:5]) == [1, 1, 1, 0, 1] and t[5] == -1
    # a bad entry in the newest table hides the older one: no entry, no fall-through (`?` returns Err)
    nd, ni = new[0], new[1].copy()
    _set_u32(ni, 1, 8, _rec(ni, 1)[1] + 1)
    t, j = check([old, (nd, ni)], [b"a", b"m"])
    assert t[0] == 1 and j[0] & gvo.BAD_ENTRY and t[1] == 0


def test_random_tables_against_the_model():
    rng = np.random.default_rng(5)
    for trial in range(20):
        tables = []
        for _ in range(int(rng.integers(1, 4))):
            ks = sorted({bytes(rng.integers(97, 100, int(rng.integers(0, 4)), dtype=np.uint8)) for _ in range(12)})
            ents = [(k, bytes(rng.integers(0, 256, int(rng.integers(0, 9)), dtype=np.uint8)), BASE_TS + int(rng.integers(9)))
                    for k in ks]
            d, i = sstable.build_run(ents)
            for r in rng.choice(len(ents), min(2, len(ents)), replace=False):
                if rng.random() < 0.5:
                    _set_u32(i, int(r), 8 + 4 * int(rng.integers(2)), _rec(i, int(r))[1 + int(rng.integers(2))] + int(rng.integers(-1, 2)))
            tables.append((d, i))
        keys = [bytes(rng.integers(97, 100, int(rng.integers(0, 4)), dtype=np.uint8)) for _ in range(40)]
        check(tables, keys)
