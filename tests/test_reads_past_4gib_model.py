"""The closed-form model of tests/test_gpu_reads_past_4gib.py, checked on the CPU: the synthetic table's bytes are what
sstable.build_run writes for the same entries (at record numbers and offsets near 2^32 and 2^33 too), the model's searches
and decode are the get_values and scan oracles' on materialised tables, the damaged records give the stop reasons and row
flags the GPU tests expect, and the compare helpers report a lost high word."""
import numpy as np
import pytest

import get_values_oracle as gvo
import reads_model as M
import scan_oracle
from dbeel_b200 import capi, sstable
from scan_cases import ERR, PANIC, damage

D1, D2 = M.TWO32 + 12345, M.TWO32 + (1 << 19) + 7   # the records test_gpu_reads_past_4gib.py damages in T_bad


def built(r0, r1):
    """sstable.build_run of T_big's records r0 .. r1 - 1 (offsets from 0)."""
    return sstable.build_run([(M.key_of(r), M.value_of(r), M.BIG_TS) for r in range(r0, r1)])


def shifted_index(index, by):
    recs = np.asarray(index, np.uint8).reshape(-1, 16).copy()
    off = recs[:, :8].copy().view("<u8") + np.uint64(by)
    recs[:, :8] = off.view(np.uint8)
    return recs.reshape(-1)


def test_entry_layout():
    assert len(M.entry_of(7)) == M.ENT == sstable.ENTRY_OVERHEAD + 16
    assert M.key_of(M.TWO32) == b"\x00\x00\x00\x02\x00\x00\x00\x01" and M.miss_below(M.TWO32) < M.key_of(M.TWO32)
    assert M.key_of(M.TWO32 - 1) < M.miss_below(M.TWO32) and M.key_of(M.N_BIG - 1) < b"\xff"
    assert M.ENT * M.N_BIG > 192 << 30 and 16 * M.N_BIG > 64 << 30


def test_generator_equals_build_run_for_a_small_table():
    n = 50
    t = M.SynTable(n)
    d, i = built(0, n)
    assert t.data_len == d.size and t.index_len == i.size
    assert np.array_equal(t.read(1, 0, d.size), d) and np.array_equal(t.read(2, 0, i.size), i)
    rng = np.random.default_rng(1)
    for _ in range(300):   # reads that start and end inside records
        kind = int(rng.integers(1, 3))
        f = d if kind == 1 else i
        off = int(rng.integers(0, f.size))
        size = int(rng.integers(0, f.size - off + 1))
        assert np.array_equal(t.read(kind, off, size), f[off:off + size]), (kind, off, size)
    assert t.read(1, d.size - 3, 4) == 4243 and t.read(2, i.size, 1) == 4243


@pytest.mark.parametrize("r0", [M.TWO32 - 40, (1 << 33) // M.ENT - 20, (1 << 32) // M.ENT - 20, (1 << 28) - 20,
                                M.TWO32 + (1 << 19) - 20, M.N_BIG - 40])
def test_generator_equals_build_run_near_the_boundaries(r0):
    """Windows at record numbers near 2^32 and the end, at .data offsets crossing 2^32 and 2^33 (records 89478485 and
    178956970 straddle them) and at the .index record that starts at 2^32 (record 2^28)."""
    r1 = min(M.N_BIG, r0 + 40)
    t = M.SynTable()
    d, i = built(r0, r1)
    base = M.ENT * r0
    assert np.array_equal(t.read(1, base, d.size), d)
    assert np.array_equal(t.read(2, 16 * r0, i.size), shifted_index(i, base))
    for a, b in ((5, 77), (47, 49), (0, d.size), (d.size - 9, d.size)):
        assert np.array_equal(t.read(1, base + a, b - a), d[a:b])
    offs = t.read(2, 16 * r0, i.size).reshape(-1, 16)[:, :8].copy().view("<u8").ravel()
    assert np.array_equal(offs, np.arange(r0, r1, dtype=np.uint64) * np.uint64(M.ENT))
    if r0 >= M.TWO32:
        assert all(int(x) >> 32 for x in offs)


def test_damaged_generator_equals_scan_cases_damage():
    """SynTable's defects are scan_cases.damage's "offset_eof" and "timestamp" on the materialised table."""
    n = 64
    d, i = built(0, n)
    want = damage(damage([(d, i)], "offset_eof", 0, 20), "timestamp", 0, 41)[0]
    t = M.SynTable(n, {20: "offset_eof", 41: "timestamp"})
    assert np.array_equal(t.read(1, 0, t.data_len), want[0]) and np.array_equal(t.read(2, 0, t.index_len), want[1])


def _keys_for(n, rng):
    present = [M.key_of(r) for r in range(n)]
    misses = [M.miss_below(r) for r in range(n + 1)]
    keys = present + misses + [b"", b"\xff" * 9, M.key_of(0)[:7], M.key_of(n // 2) + b"\x00"]
    rng.shuffle(keys)
    return keys


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 100, 1023, 1024, 1025, 3001])
def test_reference_search_equals_the_get_values_oracle(n):
    """The model's reference-mode loop, with its early exit, and its decode equal get_values_oracle on tables of n
    records; the exact mode finds every present key."""
    rng = np.random.default_rng(n)
    d, i = built(0, n)
    t = M.MemTable(d, i)
    keys = _keys_for(n, rng)
    blob, off = capi.pack_keys(keys)
    ot, orr, oj, od, oi = gvo.get_values([(d, i, None)], blob, off)
    rows, md, mi = M.get_values([t], keys, capi.LOOKUP_REFERENCE)
    assert np.array_equal(rows["table"], ot) and np.array_equal(rows["bloom_rejects"], oj)
    assert np.array_equal(np.where(ot >= 0, rows["record"], 0), np.where(ot >= 0, orr, 0))
    M.compare_out(f"n={n}", md, mi, od, oi)
    if n > 3:
        assert (rows["table"] < 0).sum() > n + 1, "the reference mode misses no present key"
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):   # the rows-only form run A's point reads use
        lr, answered = M.lookup_rows([t], keys, mode)
        assert np.array_equal(lr, M.get_values([t], keys, mode)[0])
        assert answered == [(0, int(x["record"])) for x in lr if x["table"] == 0]
    rows, md, mi = M.get_values([t], keys, capi.LOOKUP_EXACT)
    for q, k in enumerate(keys):
        r = int.from_bytes(k, "big")
        hit = len(k) == 8 and r % 2 == 1 and r // 2 < n
        assert (int(rows["table"][q]), int(rows["record"][q])) == ((0, r // 2) if hit else (-1, 0)), k
    assert np.array_equal(md.reshape(-1, M.ENT)[:, 24:32].copy().view("<u8").ravel(),
                          np.array([int(rows["record"][q]) for q in range(len(keys)) if rows["table"][q] == 0], np.uint64))


def test_reference_search_on_a_synthetic_table_matches_the_materialised_one():
    """The same loop through SynTable (the bytes the engine's callback serves) and through build_run's bytes."""
    n = 3001
    d, i = built(0, n)
    keys = _keys_for(n, np.random.default_rng(5))[:400]
    for mode in (capi.LOOKUP_REFERENCE, capi.LOOKUP_EXACT):
        a = M.get_values([M.SynTable(n)], keys, mode)
        b = M.get_values([M.MemTable(d, i)], keys, mode)
        M.compare_rows(f"mode {mode}", a[0], b[0])
        M.compare_out(f"mode {mode}", a[1], a[2], b[1], b[2])


def test_damage_expectations():
    """T_bad's two defects on a materialised slice: the scan oracle stops with PANIC at the offset_eof record and with ERR
    at the timestamp record; the get_values oracle answers the timestamp record's key with LOOKUP_BAD_ENTRY and no entry,
    and the offset_eof record's key (its probe reads the length prefix of the last entry's tail: an empty key) as a miss.
    The model says the same on the slice and on the synthetic table."""
    n, a, b = 96, 30, 71
    d, i = built(0, n)
    bad = damage(damage([(d, i)], "offset_eof", 0, a), "timestamp", 0, b)[0]
    syn = M.SynTable(n, {a: "offset_eof", b: "timestamp"})
    mem = M.MemTable(*bad)
    _, stop = scan_oracle.scan([bad], [(b"", b"\xff")], scan_oracle.SCAN_KEY)
    assert stop == (0, PANIC, a)
    only_b = damage([(d, i)], "timestamp", 0, b)[0]
    _, stop = scan_oracle.scan([only_b], [(b"", b"\xff")], scan_oracle.SCAN_KEY)
    assert stop == (0, ERR, b)
    assert M.record_damage(syn, a) == PANIC and M.record_damage(syn, b) == ERR
    # a seek that probes the offset_eof record reads an empty key there and moves past it, so a range covers it only
    # when neither bound's search probes it: the model's seek is seek_oracle's
    import seek_oracle
    stops = set()
    for lo, hi in ((a - 3, a + 3), (a - 20, a + 1), (0, n - 1), (a - 1, b + 2), (b - 3, b + 3), (a + 1, b + 1)):
        rg = [(M.key_of(lo), M.key_of(hi))]
        for t in (syn, mem):
            out, stop, _ = M.reader_scan(t, rg)
            want, wstop = seek_oracle.reader_scan([bad], rg)
            assert stop == wstop, (lo, hi)
            M.compare_out(f"scan [{lo}, {hi})", out[0][0], out[0][1], want[0][0], want[0][1])
            stops.add(stop)
    assert {(0, PANIC, a), (0, ERR, b)} <= stops
    keys = [M.key_of(r) for r in range(n)]
    blob, off = capi.pack_keys(keys)
    ot, orr, oj, od, oi = gvo.get_values([(bad[0], bad[1], None)], blob, off)
    assert ot[b] == 0 and orr[b] == b and oj[b] == gvo.BAD_ENTRY
    assert ot[a] == -1 and oj[a] == 0
    for t in (syn, mem):
        rows, md, mi = M.get_values([t], keys, capi.LOOKUP_REFERENCE)
        assert np.array_equal(rows["table"], ot) and np.array_equal(rows["bloom_rejects"], oj)
        M.compare_out("damaged slice", md, mi, od, oi)
        rows = M.get_values([t], keys, capi.LOOKUP_EXACT)[0]
        lr, answered = M.lookup_rows([t], keys, capi.LOOKUP_EXACT)
        assert np.array_equal(lr, rows) and (0, b) not in answered
        assert (int(rows["table"][b]), int(rows["bloom_rejects"][b]), int(rows["record"][b])) == (0, M.BAD_ENTRY, b)
        assert int(rows["table"][a]) == -1


def test_scan_and_range_models_equal_the_oracles_on_a_materialised_table():
    """reader_scan / get_range / the limited rule of the model against seek_oracle, range_oracle and the limited range
    oracles, on a slice with a newer table over some of its keys."""
    import range_limit_oracle as rlo
    import range_limit_rev_oracle as rlro
    import range_oracle
    import seek_oracle
    n = 600
    d, i = built(0, n)
    newer = sstable.build_run(sorted([(M.key_of(r), b"" if r % 3 == 0 else b"new%d" % r, M.BIG_TS + 5) for r in range(290, 310)]
                                     + [(M.miss_below(r), b"between", M.BIG_TS + 5) for r in (295, 305)]))
    tables = [(d, i), newer]
    mt = [M.MemTable(*t) for t in tables]
    ranges = [(M.key_of(280), M.key_of(320)), (M.miss_below(300), M.miss_below(302)), (M.key_of(590), b"\xff"),
              (M.key_of(10), M.key_of(5))]
    out, stop, _ = M.reader_scan(mt[0], ranges)
    want, wstop = seek_oracle.reader_scan(tables[:1], ranges)
    assert stop == wstop
    for g, w in zip(out, want):
        M.compare_out("scan", g[0], g[1], w[0], w[1])
    for keep in (False, True):
        for rg in ranges:
            g, stop = M.get_range(mt, rg, keep)
            w, wstop = range_oracle.get_range(tables, [rg], keep)
            assert stop == wstop
            M.compare_out("get_range", *M.pack(g), *w[0])
            for limit in (1, 7, 1000):
                for rev, oracle_ in ((False, rlo), (True, rlro)):
                    c = oracle_.clean(tables, rg, limit, keep)
                    rule = M.limited_rule(mt, rg, limit, keep, rev)
                    assert rule[0] == "clean" and rule[1] == c[0] and rule[2] == (M.MORE if c[1] else 0)
    bad = damage([(d, i)], "timestamp", 0, 300)
    mb = [M.MemTable(*bad[0])]
    for limit in (1, 7, 1000):
        for rev, oracle_ in ((False, rlo), (True, rlro)):
            rule = M.limited_rule(mb, ranges[0], limit, False, rev)
            a, bad_recs = oracle_.damaged_merge(bad, ranges[0])
            assert rule[0] == "damaged" and rule[3] == bad_recs == {(0, 300): ERR}
            assert rule[1] == (a[::-1] if rev else a)[:limit]


def test_reader_depths_restatement():
    """T_big alone, and with a small table next to it, reaches depth 16 within the default fence budget."""
    assert M.reader_depths([M.N_BIG], [M.ENT * M.N_BIG]) == [16]
    d = M.reader_depths([M.N_BIG, 700], [M.ENT * M.N_BIG, 700 * 60])
    assert d[0] == 16 and d[1] == M.lookup_max_depth(700)
    assert M.reader_depths([20000], [20000 * 40], 4 * M.NODE_BYTES) == [2]


# ------------------------------------------------------------------------------------ the compare helpers see a lost high word


def _rows_past_2_32():
    rows = np.zeros(4, capi.LOOKUP_DTYPE)
    rows["table"] = [0, -1, 0, 1]
    rows["record"] = [M.TWO32 + 5, 0, M.TWO32 - 1, M.N_BIG - 1]
    return rows


def test_compare_rows_reports_a_record_with_its_high_word_cleared():
    want = _rows_past_2_32()
    M.compare_rows("untouched", want.copy(), want)
    got = want.copy()
    got["record"][3] &= np.uint64(0xFFFFFFFF)
    with pytest.raises(AssertionError, match=r"row 3 record is 1048578 \(high word 0\), model 4296015874 \(high word 1\)"):
        M.compare_rows("cleared", got, want)


def test_compare_out_reports_an_index_offset_with_its_high_word_cleared():
    ents = [M.entry_of(r) for r in range(4)]
    d, i = M.pack(ents)
    recs = i.reshape(-1, 16).copy()
    recs[2, :8] = np.array([M.TWO32 + 96], "<u8").view(np.uint8)   # an output offset past 4 GiB
    want = recs.reshape(-1)
    M.compare_out("untouched", d, want.copy(), d, want)
    got = want.copy()
    got[2 * 16 + 4:2 * 16 + 8] = 0
    with pytest.raises(AssertionError, match=r"record 2 \(offset high word\)"):
        M.compare_out("cleared", d, got, d, want)


def test_compare_stop_reports_a_record_off_by_2_32():
    want = (0, PANIC, M.TWO32 + 12345)
    M.compare_stop("same", want, want)
    with pytest.raises(AssertionError, match=r"stop \(0, 2, 12345\) \(record high word 0\)"):
        M.compare_stop("off by 2^32", (0, PANIC, 12345), want)


def test_compare_out_reports_two_words_swapped_across_2_32():
    """Two 8-byte words on either side of .data offset 2^32 of T_big swapped: the bytes at the first differ."""
    t = M.SynTable()
    lo = M.TWO32 - 8 - 48 * 2
    want = np.asarray(t.read(1, lo, 8 * 26), np.uint8).copy()
    at = M.TWO32 - 8 - lo
    assert not np.array_equal(want[at:at + 8], want[at + 8:at + 16])
    got = want.copy()
    got[at:at + 8], got[at + 8:at + 16] = want[at + 8:at + 16], want[at:at + 8]
    idx = np.zeros(0, np.uint8)
    M.compare_out("untouched", want.copy(), idx, want, idx)
    with pytest.raises(AssertionError, match=f"differs at byte {at} "):
        M.compare_out("swapped", got, idx, want, idx)
