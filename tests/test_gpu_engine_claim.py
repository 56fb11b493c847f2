"""Taking the engine: every call goes through one claim.  While a submitted compaction is unreaped, every call that takes
the engine is refused with ERR_BUSY and leaves the job's error text and stats alone; after the job is reaped they all
work again.  A call that takes the engine starts from zeroed stats."""
import time

import numpy as np
import pytest
import torch

import oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import storage_engine as se
from dbeel_b200 import workloads as W
from helpers import BASE_TS, assert_run_equal

pytestmark = pytest.mark.gpu

SEED = bytes(range(32))
TIMES = ("ms_total", "ms_h2d", "ms_d2h", "ms_extract", "ms_merge", "ms_resolve", "ms_gather")


@pytest.fixture
def eng():
    """An engine of this file's own: a job left unreaped cannot reach another test."""
    e = capi.Engine(0)
    yield e
    e.close()


def _dev(a):
    return torch.from_numpy(np.array(a)).to("cuda:0")  # a writable copy, dtype kept


class Buf:
    """A zeroed device buffer of n bytes (16-byte aligned, as torch allocates)."""

    def __init__(self, n):
        self.t = torch.zeros(max(16, n), dtype=torch.uint8, device="cuda:0")
        self.n, self.ptr = n, self.t.data_ptr()


def _calls(eng, tree):
    """Every call that takes the engine, each with valid arguments, by name; and what they need kept alive (a reader and
    a page cache among them, opened now)."""
    rng = np.random.default_rng(5)
    writes = [(b"c%05d" % n, bytes(rng.integers(0, 256, int(rng.integers(0, 200)), dtype=np.uint8)), BASE_TS + n)
              for n in range(600)]
    batch = sstable.build_run(writes)
    run2 = sstable.build_run(writes[::3])
    runs = [batch, run2]
    tables = [(batch[0], batch[1], None)]
    keys = [b"c%05d" % n for n in range(0, 700, 11)]
    wal = sstable.build_wal(writes[:200])
    d, i, dw = _dev(batch[0]), _dev(batch[1]), _dev(wal)
    dk, dko = _dev(np.frombuffer(b"".join(keys), np.uint8)), _dev(capi.pack_keys(keys)[1])
    drun = (d.data_ptr(), batch[0].size, i.data_ptr(), batch[1].size)
    dtab = drun + (0, 0)
    od, oi, ob = Buf(4 * batch[0].size), Buf(4 * batch[1].size + 4096 * 16), Buf(1 << 16)
    res, h64 = Buf(16 * len(keys)), Buf(8 * (batch[1].size // 16))
    ring = np.array([0, 1 << 31], np.uint32)
    out6, out4 = (od.ptr, od.n, oi.ptr, oi.n, ob.ptr, ob.n), (od.ptr, od.n, oi.ptr, oi.n)
    hashes, key_ranges = [(0, (1 << 32) - 1)], [(b"c00010", b"c00300")]
    reader, cache = eng.open_reader(tables), eng.open_page_cache(1 << 20)
    torch.cuda.synchronize()
    keep = [d, i, dw, dk, dko, od, oi, ob, res, h64, reader, cache]
    return keep, {
        "compact": lambda: eng.compact(runs, seed=SEED),
        "compact_stream": lambda: eng.compact_stream(runs, seed=SEED),
        "compact_async": lambda: eng.compact_async(runs, seed=SEED)(True),
        "compact_device": lambda: eng.compact_device([drun], out6, capi.make_opts(seed=SEED)),
        "flush": lambda: eng.flush(batch),
        "flush_device": lambda: eng.flush_device(drun, out4),
        "flush_many": lambda: eng.flush_many(runs),
        "flush_many_device": lambda: eng.flush_many_device([drun], out4),
        "flush_many_sparse_device": lambda: eng.flush_many_sparse_device([drun], batch[0].size, out4),
        "memtable_cuts_device": lambda: eng.memtable_cuts_device(h64.ptr, [0, batch[1].size // 16], 100),
        "route_device": lambda: eng.route_device(drun, ring, oi.ptr, oi.n, 0, h64.ptr),
        "compact_many": lambda: eng.compact_many([(runs, False), ([run2], True)]),
        "compact_many_device": lambda: eng.compact_many_device([([drun], False)], out6, seeds=[SEED]),
        "wal_flush": lambda: eng.wal_flush(wal),
        "wal_flush_device": lambda: eng.wal_flush_device(dw.data_ptr(), wal.size, out4),
        "get_many": lambda: eng.get_many(tables, keys),
        "get_many_device": lambda: eng.get_many_device([dtab], dk.data_ptr(), dko.data_ptr(), len(keys), res.ptr),
        "get_values": lambda: eng.get_values(tables, keys),
        "get_values_device": lambda: eng.get_values_device([dtab], dk.data_ptr(), dko.data_ptr(), len(keys), res.ptr, out4),
        "get_values_stream": lambda: eng.get_values_stream(tables, keys),
        "scan": lambda: eng.scan(tables, hashes),
        "scan_device": lambda: eng.scan_device([drun], hashes, out4),
        "scan_stream": lambda: eng.scan_stream(tables, hashes),
        "open_reader": lambda: eng.open_reader(tables).close(),
        "open_page_cache": lambda: eng.open_page_cache(1 << 20).close(),
        "readers_get_values": lambda: eng.readers_get_values([(reader, keys, capi.LOOKUP_REFERENCE)]),
        "readers_get_ranges": lambda: eng.readers_get_ranges([(reader, key_ranges, 5, False, False)]),
        "reader.get_values": lambda: reader.get_values(keys),
        "reader.scan": lambda: reader.scan(key_ranges),
        "reader.get_range": lambda: reader.get_range(key_ranges),
        "reader.get_ranges": lambda: reader.get_ranges(key_ranges, 5),
        "reader.get_ranges_reverse": lambda: reader.get_ranges(key_ranges, 5, reverse=True),
        "reader.attach_page_cache": lambda: reader.attach_page_cache(cache),
        "page_cache.stats": lambda: cache.stats(),
        "tree.open_reader": lambda: tree.open_reader().close(),
        "tree.scan_stream": lambda: tree.scan_stream(hashes),
    }


def test_unreaped_job_refuses_every_call(eng, tmp_path):
    job = W.make_merge_runs(W.scaled(W.CFG2, 20_000))
    tree = se.LSMTree.open_or_create(str(tmp_path), eng, sstable_bloom_min_size=1)
    try:
        tree.flush(sstable.build_run([(b"t%04d" % n, b"v" * (n % 50), BASE_TS + n) for n in range(500)]))
        keep, calls = _calls(eng, tree)
        for call in calls.values():  # every call works before the job
            call()
        eng.compact(job, seed=SEED)  # the job run alone
        solo = eng.stats()
        with pytest.raises(capi.DbeelError):  # an error text of its own, which the job's replaces
            eng.get_many([(job[0][0], job[0][1], None)], [b"k"], mode=9)
        assert capi.lib().dbeel_last_error(eng._h).decode() == "unknown lookup mode"
        reap = eng.compact_async(job, seed=SEED)
        for name, call in calls.items():
            with pytest.raises(capi.DbeelError) as ei:
                call()
            assert ei.value.code == capi.ERR_BUSY, name
        time.sleep(1)  # most likely finished by now; finished or not, the job is unreaped
        for name in ("scan_stream", "tree.scan_stream", "tree.open_reader", "compact_stream", "compact"):
            with pytest.raises(capi.DbeelError) as ei:
                calls[name]()
            assert ei.value.code == capi.ERR_BUSY, name
        got = reap(True)
        assert capi.lib().dbeel_last_error(eng._h).decode() == ""
        st = eng.stats()
        assert {k: v for k, v in st.items() if k not in TIMES} == {k: v for k, v in solo.items() if k not in TIMES}
        od, oi, ob, on = oracle.compact(job, keep_tombstones=False, seed=SEED)
        assert got[3] == on
        assert_run_equal((got[0], got[1]), (od, oi), "reaped job")
        assert np.array_equal(got[2], ob)
        for call in calls.values():  # and every call works again
            call()
        del keep
    finally:
        tree.close()


def test_calls_start_from_zeroed_stats(eng):
    runs = W.make_merge_runs(W.scaled(W.CFG2, 2_000))
    eng.compact(runs, seed=SEED)
    assert eng.stats()["ms_h2d"] > 0
    batch = sstable.build_run([(b"f%05d" % n, b"v" * (n % 40), BASE_TS + n) for n in range(3000)])
    d, i = _dev(batch[0]), _dev(batch[1])
    od, oi = Buf(batch[0].size), Buf(batch[1].size)
    torch.cuda.synchronize()
    eng.flush_many_device([(d.data_ptr(), batch[0].size, i.data_ptr(), batch[1].size)], (od.ptr, od.n, oi.ptr, oi.n))
    st = eng.stats()
    assert st["ms_h2d"] == 0 and st["ms_d2h"] == 0 and st["entries_in"] == 3000
    # the host forms of the many-job calls report their copies
    eng.flush_many([batch])
    assert eng.stats()["ms_h2d"] > 0 and eng.stats()["ms_d2h"] > 0
    eng.compact_many([(runs, False)])
    assert eng.stats()["ms_h2d"] > 0 and eng.stats()["ms_d2h"] > 0
