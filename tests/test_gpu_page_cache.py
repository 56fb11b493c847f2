"""The readers' device page cache (dbeel_page_cache_*): a reader with a cache attached returns exactly what it returns
without one, for caches that hold everything, that evict heavily and that are smaller than one leaf; pages it holds are
never read again, across batches, readers and tree snapshots; what it reads is page-aligned and inside its file."""
import os
from collections import Counter

import numpy as np
import pytest

from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from helpers import BASE_TS, assert_run_equal
from test_gpu_get_values import _rec, _set_u32
from test_gpu_get_values_stream import all_cases, case_compacted_with_filter, case_four_overlapping
from test_gpu_reader import MODES, same, table_20000
from test_gpu_reader_scan import _table_20000
from test_gpu_reader_scan import check as scan_check

pytestmark = pytest.mark.gpu

PAGE = 4096
SIZES = {"all": 256 << 20, "few": 6 * PAGE, "one": PAGE}  # everything fits / heavy eviction / smaller than a leaf


@pytest.fixture
def tiny_engine(monkeypatch):
    """An engine whose leaf groups are 4 KB."""
    monkeypatch.setenv("DBEEL_PARTITION_KB", "4")
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    e = capi.Engine(0)
    yield e
    e.close()


def pages_of(reads):
    """(table, kind, page) of every page the reads cover; each read must be page-aligned."""
    out = []
    for t, kind, off, size in reads:
        assert off % PAGE == 0, (t, kind, off, size)
        out += [(t, kind, p) for p in range(off // PAGE, (off + size - 1) // PAGE + 1)]
    return out


def check_page_reads(tables, reads):
    """Leaf, window and entry reads through a cache: page-aligned, inside the file, ending on a page boundary or at EOF."""
    for t, kind, off, size in reads:
        n = len(tables[t][0] if kind == 1 else tables[t][1])
        assert off % PAGE == 0 and off + size <= n and ((off + size) % PAGE == 0 or off + size == n), (t, kind, off, size, n)


def cached_same(e, r, tables, keys, mode, cache, ref_engine=None):
    """same() on a cached reader, plus: the cache's counters move by what the batch planned, and never past capacity."""
    before = cache.stats()
    out = same(e, r, tables, keys, mode, ref_engine=ref_engine)
    after = cache.stats()
    assert after["resident_pages"] <= after["capacity_pages"]
    assert after["hits"] >= before["hits"] and after["misses"] >= before["misses"]
    return out


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("budget", ["default", "tiny"])
def test_parity_on_every_case(engine, tiny_engine, budget, size):
    """Three batches per mode on one cached reader, on every table set of the stream's tests, damage cases included."""
    e = engine if budget == "default" else tiny_engine
    rng = np.random.default_rng(51)
    with e.open_page_cache(SIZES[size]) as cache:
        for tables, keys in all_cases(engine):
            with e.open_reader(tables) as r:
                r.attach_page_cache(cache)
                for mode in MODES:
                    half = [keys[j] for j in rng.permutation(len(keys))[:len(keys) // 2]]
                    for batch in (keys, half, keys[:7]):
                        cached_same(e, r, tables, batch, mode, cache, ref_engine=engine)


def test_damage_at_fences_and_inside_leaves(engine):
    ents = [(b"key-%06d" % n, b"v%d" % n, BASE_TS + n) for n in range(2000)]
    d, i = sstable.build_run(ents)
    keys = [k for k, _, _ in ents[::7]] + [b"key-%06dx" % n for n in range(0, 2000, 13)]
    rng = np.random.default_rng(52)
    with engine.open_page_cache(1 << 20) as cache:
        for r in list(rng.choice(2000, 6, replace=False)) + [0, 1, 1000, 1999]:
            off, ks, fs = _rec(i, int(r))
            for kind in range(4):
                bi, bd = i.copy(), d
                if kind == 0:
                    bi[16 * r:16 * r + 8] = np.frombuffer((d.size - 4).to_bytes(8, "little"), np.uint8)
                elif kind == 1:
                    bd = d.copy()
                    bd[off:off + 8] = np.frombuffer((1 << 50).to_bytes(8, "little"), np.uint8)
                elif kind == 2:
                    _set_u32(bi, int(r), 8, ks + 3)
                else:
                    bi[16 * r:16 * r + 8] = np.frombuffer((off + 5).to_bytes(8, "little"), np.uint8)
                tables = [(bd, bi, None)]
                with engine.open_reader(tables) as rd:
                    rd.attach_page_cache(cache)
                    for mode in MODES:
                        for _ in range(2):
                            cached_same(engine, rd, tables, keys + [ents[int(r)][0]], mode, cache)


def test_a_repeated_batch_reads_nothing(engine):
    tables, keys = case_four_overlapping(engine)
    t2, k2 = case_compacted_with_filter(engine)
    tables, keys = tables + t2, keys + k2
    rng = np.random.default_rng(53)
    with engine.open_page_cache(512 << 20) as cache:
        for mode in MODES:
            with engine.open_reader(tables) as r:
                same(engine, r, tables, keys, mode)  # loads the fences, uncached
                r.attach_page_cache(cache)
                seen = Counter()
                _, _, _, reads, _, _, _ = cached_same(engine, r, tables, keys, mode, cache)
                check_page_reads(tables, reads)
                seen.update(pages_of(reads))
                s0 = cache.stats()
                _, _, _, reads, st, _, _ = cached_same(engine, r, tables, keys, mode, cache)
                assert reads == [] and st["input_bytes"] == 0
                s1 = cache.stats()
                assert s1["misses"] == s0["misses"] and s1["hits"] > s0["hits"] and s1["evictions"] == 0
                for _ in range(6):  # many batches: no page is read twice
                    batch = [keys[j] for j in rng.choice(len(keys), 700, replace=False)]
                    reads = same(engine, r, tables, batch, mode)[3]
                    check_page_reads(tables, reads)
                    seen.update(pages_of(reads))
                assert max(seen.values()) == 1
            cache_stats = cache.stats()
            assert cache_stats["resident_pages"] <= cache_stats["capacity_pages"]


def test_short_files_and_an_entry_at_eof(engine):
    """A .data shorter than one page, and a hit whose entry ends at EOF: the last page is read up to the file's length."""
    small = sstable.build_run([(b"a%02d" % n, b"x" * n, BASE_TS + n) for n in range(30)])
    big_tail = sstable.build_run([(b"b%05d" % n, b"y" * (n % 50), BASE_TS + n) for n in range(3000)])
    tables = [(small[0], small[1], None), (big_tail[0], big_tail[1], None)]
    assert small[0].size < PAGE and big_tail[0].size % PAGE
    keys = [b"a%02d" % n for n in range(0, 30, 3)] + [b"b%05d" % 2999, b"b%05d" % 0, b"a29"]
    with engine.open_page_cache(1 << 20) as cache:
        for mode in MODES:
            with engine.open_reader(tables) as r:
                same(engine, r, tables, keys, mode)
                r.attach_page_cache(cache)
                reads = cached_same(engine, r, tables, keys, mode, cache)[3]
                check_page_reads(tables, reads)
                assert any(t == 0 and k == 1 and off == 0 and size == small[0].size for t, k, off, size in reads), reads
                assert cached_same(engine, r, tables, keys, mode, cache)[3] == []


def test_stats_add_up_and_device_memory_is_the_capacity(engine):
    import torch
    tables, keys = case_four_overlapping(engine)
    cap = 64 << 20
    for mode in MODES:  # the engine's own workspaces grow to this batch first, with and without a cache
        engine.get_values_stream(tables, keys, mode)
        with engine.open_page_cache(cap) as c, engine.open_reader(tables) as r:
            r.attach_page_cache(c)
            r.get_values(keys, mode)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    cache = engine.open_page_cache(cap + 123)
    torch.cuda.synchronize()
    taken = free0 - torch.cuda.mem_get_info()[0]
    assert cap <= taken <= cap + (2 << 20), taken
    assert cache.stats() == {"capacity_pages": cap // PAGE, "resident_pages": 0, "hits": 0, "misses": 0, "evictions": 0}
    with engine.open_reader(tables) as r:
        for mode in MODES:
            same(engine, r, tables, keys, mode)
        r.attach_page_cache(cache)
        for mode in MODES:
            for _ in range(2):
                s0 = cache.stats()
                reads = same(engine, r, tables, keys, mode)[3]
                s1 = cache.stats()
                # every page read is a miss; hits + misses are the pages requested, which a repeat requests again
                assert s1["misses"] - s0["misses"] == len(set(pages_of(reads))) == len(pages_of(reads))
                assert s1["resident_pages"] == s0["resident_pages"] + (s1["misses"] - s0["misses"]) - (s1["evictions"] - s0["evictions"])
            assert s1["misses"] == s0["misses"] and s1["hits"] - s0["hits"] > 0
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
    cache.close()
    torch.cuda.synchronize()
    # the cache holds what it took at create and nothing more (the engine's own workspaces may have grown by then)
    assert cap <= used - (free0 - torch.cuda.mem_get_info()[0]) <= cap + (2 << 20)


def test_tree_readers_share_pages_across_flushes_and_compactions(engine, tmp_path):
    d = str(tmp_path)
    tree = se.LSMTree.open_or_create(d, engine, sstable_bloom_min_size=1)
    rng = np.random.default_rng(54)
    writes = [(b"t%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), BASE_TS + n)
              for n in range(3000)]
    for lo, hi in ((0, 1000), (700, 2000), (1500, 3000)):
        tree.flush(sstable.build_run(sorted(writes[lo:hi])))
    keys = [b"t%05d" % n for n in range(0, 3100, 7)] + [b"t00001", b"t00001"]
    snap = tree.sstable_indices_and_sizes()
    cache = engine.open_page_cache(64 << 20)
    a = tree.open_reader(page_cache=cache)
    assert a.last_stream_reads is None
    before = {}
    for mode in MODES:
        a.get_values(keys, mode)  # loads the fences, fills the cache
        before[mode] = a.get_values(keys, mode)
        assert engine.stats()["input_bytes"] == 0
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert np.array_equal(before[mode][0], sr)
        assert_run_equal(before[mode][1:], (sd, si), "tree reader A")
    # B opened after a flush shares A's three tables: its batch on their keys reads nothing of them and misses none of
    # their pages (the new one-record table, which a filter false positive may reach, is one page of each file)
    new = sstable.build_run([(b"u", b"x", BASE_TS)])
    tree.flush(new)
    b = tree.open_reader(page_cache=cache)
    for mode in MODES:
        m0 = cache.stats()["misses"]
        rb, db, ib = b.get_values(keys, mode)
        assert engine.stats()["input_bytes"] <= new[0].size + new[1].size and cache.stats()["misses"] <= m0 + 2
        m0 = cache.stats()["misses"]
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert np.array_equal(rb, sr)
        assert_run_equal((db, ib), (sd, si), "tree reader B")
        # two live readers share pages: A's batch hits what B's just hit
        h0 = cache.stats()["hits"]
        a.get_values(keys, mode)
        assert cache.stats()["hits"] > h0 and cache.stats()["misses"] == m0
    tree.compact([idx for idx, _ in tree.sstable_indices_and_sizes()], 7, True)
    assert not any(os.path.exists(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT))) for idx, _ in snap)
    c = tree.open_reader(page_cache=cache)
    for mode in MODES:
        ra, da, ia = a.get_values(keys, mode)  # A answers from its snapshot, its files unlinked
        assert np.array_equal(ra, before[mode][0])
        assert_run_equal((da, ia), before[mode][1:], "A after the compaction")
        rc_, dc_, ic_ = c.get_values(keys, mode)
        sr, sd, si = tree.get_values_stream(keys, mode)
        assert np.array_equal(rc_, sr)
        assert_run_equal((dc_, ic_), (sd, si), "reader C")
    for r in (a, b, c):
        r.close()
    cache.close()
    tree.close()


def test_scans(engine):
    d, i = _table_20000()
    tables = [(d, i)]
    narrow = [(b"key-%06d" % 7000, b"key-%06d" % 7020)]
    with engine.open_reader([(d, i, None)]) as plain:
        scan_check(engine, plain, tables, narrow, sorted_clean=True)
        want_out, want_stop, plain_reads, _ = scan_check(engine, plain, tables, narrow, sorted_clean=True)
    with engine.open_page_cache(16 << 20) as cache, engine.open_reader([(d, i, None)]) as r:
        scan_check(engine, r, tables, narrow, sorted_clean=True)  # loads the fences
        r.attach_page_cache(cache)
        first = scan_check(engine, r, tables, narrow, sorted_clean=True)
        out, stop, second, _ = scan_check(engine, r, tables, narrow, sorted_clean=True)
        assert stop == want_stop
        for g, w in zip(out, want_out):
            assert_run_equal(g, w, "cached scan")
        # the second call reads no seek leaf: only the span partitions, which the uncached reader reads too
        assert second and set(second) <= set(plain_reads) and len(second) < len(plain_reads), (second, plain_reads)
        assert len(second) < len(first[2])
        # hash scans: what the uncached reader reads, and the cache untouched
        hr = [(0, 1 << 31), (1 << 31, (1 << 32) - 1)]
        s0 = cache.stats()
        out_h, stop_h = r.scan(hr, capi.SCAN_HASH)
        reads_h = r.last_stream_reads
        with engine.open_reader([(d, i, None)]) as p2:
            ref_h, rstop = p2.scan(hr, capi.SCAN_HASH)
            assert sorted(p2.last_stream_reads) == sorted(reads_h)
        assert stop_h == rstop and cache.stats() == s0
        for g, w in zip(out_h, ref_h):
            assert_run_equal(g, w, "hash scan")


def test_failures_leave_reader_and_cache_usable(engine):
    tables, keys = case_four_overlapping(engine)
    mode = capi.LOOKUP_EXACT
    with engine.open_page_cache(8 << 20) as cache, engine.open_reader(tables) as r:
        same(engine, r, tables, keys, mode)
        r.attach_page_cache(cache)
        for at in (0, 3, 10):  # a cold cache each time, so that the batch reads
            with engine.open_page_cache(8 << 20) as cold:
                r.attach_page_cache(cold)
                with pytest.raises(capi.DbeelError) as ei:
                    r.get_values(keys[:600], mode, fail_read_at=at)
                assert ei.value.code == 4242
                st = cold.stats()
                assert st["resident_pages"] <= st["misses"] and st["resident_pages"] <= st["capacity_pages"]
                cached_same(engine, r, tables, keys[:600], mode, cold)
                assert cached_same(engine, r, tables, keys[:600], mode, cold)[3] == []
        r.attach_page_cache(cache)
        rows, d, i, _, _, _, _ = cached_same(engine, r, tables, keys, mode, cache)
        for caps in ((d.size - 1, i.size), (d.size, i.size - 1)):
            with pytest.raises(capi.DbeelError) as ei:
                r.get_values(keys, mode, caps=caps)
            assert ei.value.code == capi.ERR_CAPACITY and ei.value.needed == (d.size, i.size)
            r2, d2, i2 = r.get_values(keys, mode)
            assert np.array_equal(r2, rows) and np.array_equal(d2, d) and np.array_equal(i2, i)
    # destroying an attached cache: its readers go on, uncached
    with engine.open_reader(tables) as r1, engine.open_reader(tables) as r2, engine.open_reader(tables) as r3:
        same(engine, r3, tables, keys, mode)
        plain = same(engine, r3, tables, keys, mode)[3]  # an uncached reader's reads once its fences are loaded
        cache = engine.open_page_cache(8 << 20)
        r1.attach_page_cache(cache)
        r2.attach_page_cache(cache)
        same(engine, r1, tables, keys, mode)
        same(engine, r2, tables, keys, mode)
        cache.close()
        for rr in (r1, r2):
            assert sorted(same(engine, rr, tables, keys, mode)[3]) == sorted(plain)
        cache.close()  # a second close is a no-op
    # errors
    with pytest.raises(capi.DbeelError) as ei:
        engine.open_page_cache(0)
    assert ei.value.code == capi.ERR_INVALID_ARG
    with pytest.raises(capi.DbeelError) as ei:
        engine.open_page_cache(PAGE - 1)
    assert ei.value.code == capi.ERR_INVALID_ARG
    other = capi.Engine(0)
    try:
        foreign = other.open_page_cache(PAGE)
        with engine.open_reader(tables) as r:
            with pytest.raises(capi.DbeelError) as ei:
                r.attach_page_cache(foreign)
            assert ei.value.code == capi.ERR_INVALID_ARG
            r.attach_page_cache(None)
            same(engine, r, tables, keys[:50], mode)
    finally:
        other.close()


def test_engine_destroy_with_caches_open():
    tables, keys = [table_20000()[0]], [b"key-000001", b"key-019999"]
    e = capi.Engine(0)
    cache = e.open_page_cache(1 << 20)
    e.open_page_cache(2 << 20)
    r = e.open_reader(tables)
    r.attach_page_cache(cache)
    rows, _, _ = r.get_values(keys, capi.LOOKUP_EXACT)
    assert list(rows["table"]) == [0, 0]
    e.close()
    cache.close()  # the engine destroyed it already
    r.close()
