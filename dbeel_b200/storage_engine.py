"""Python face of the host-side mirror (include/dbeel_tree.h, csrc/host/lsm_tree_host.cc).

Names and argument meaning follow the reference's storage engine so the tests read like its own
(src/storage_engine/lsm_tree.rs): ``LSMTree.open_or_create``, ``.compact(indices_to_compact,
output_index, keep_tombstones)``, ``.flush``, ``.sstable_indices_and_sizes``; the size-tiered
picker of src/tasks/compaction.rs:35-102 is ``plan_compactions`` / ``compact_tree``.
All the work happens in the C++/CUDA library; this file only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import capi

ERR_IO = 20
ERR_NO_SSTABLE = 21
DEFAULT_TREE_CAPACITY = 8192  # mod.rs:18
DEFAULT_SSTABLE_BLOOM_MIN_SIZE = 1_048_576  # mod.rs:19

FILE_DATA, FILE_INDEX = 1, 2  # FileTypeKind::{Data, Index} (mod.rs:36-42)
PAGE_SIZE = 4096  # page_cache.rs:10
PAGE_SINK = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint8))

_bound = False


def _lib():
    global _bound
    L = capi.lib()
    if not _bound:
        L.dbeel_tree_open.restype = C.c_int
        L.dbeel_tree_open.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
        L.dbeel_tree_close.restype = None
        L.dbeel_tree_close.argtypes = [C.c_void_p]
        L.dbeel_tree_sstables.restype = C.c_uint32
        L.dbeel_tree_sstables.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_uint32]
        L.dbeel_tree_write_sstable_index.restype = C.c_uint64
        L.dbeel_tree_write_sstable_index.argtypes = [C.c_void_p]
        L.dbeel_tree_compact.restype = C.c_int
        L.dbeel_tree_compact.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint32, C.c_uint64, C.c_int, C.c_char_p]
        L.dbeel_tree_flush.restype = C.c_int
        L.dbeel_tree_flush.argtypes = [C.c_void_p, C.POINTER(capi.Run), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.dbeel_tree_compact_many.restype = C.c_int
        L.dbeel_tree_compact_many.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_uint32,
                                              C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.c_char_p]
        L.dbeel_tree_get_many.restype = C.c_int
        L.dbeel_tree_get_many.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
        L.dbeel_tree_get_values.restype = C.c_int
        L.dbeel_tree_get_values.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(capi.Out),
                                            C.c_void_p]
        L.dbeel_tree_get_values_stream.restype = C.c_int
        L.dbeel_tree_get_values_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                                   C.POINTER(capi.Out), C.c_void_p]
        L.dbeel_tree_reader_open.restype = C.c_int
        L.dbeel_tree_reader_open.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
        L.dbeel_tree_scan.restype = C.c_int
        L.dbeel_tree_scan.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(capi.Out),
                                      C.POINTER(capi.JobResult), C.POINTER(capi.ScanStop)]
        L.dbeel_tree_scan_stream.restype = C.c_int
        L.dbeel_tree_scan_stream.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, capi.SCAN_WRITE_FN, C.c_void_p,
                                             C.POINTER(capi.JobResult), C.POINTER(capi.ScanStop)]
        L.dbeel_tree_recover_wal.restype = C.c_int
        L.dbeel_tree_recover_wal.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.dbeel_tree_last_error.restype = C.c_char_p
        L.dbeel_tree_last_error.argtypes = [C.c_void_p]
        L.dbeel_memtable_cut.restype = C.c_uint64
        L.dbeel_memtable_cut.argtypes = [C.POINTER(capi.Run), C.c_uint64, C.c_uint32]
        L.dbeel_plan_compactions.restype = C.c_uint32
        L.dbeel_plan_compactions.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_uint32, C.c_uint32,
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64),
                                             C.POINTER(C.c_int32)]
        L.dbeel_out_pages.restype = C.c_int
        L.dbeel_out_pages.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64, PAGE_SINK, C.c_void_p]
        L.dbeel_tree_set_page_sink.restype = None
        L.dbeel_tree_set_page_sink.argtypes = [C.c_void_p, PAGE_SINK, C.c_void_p]
        _bound = True
    return L


TREE_EXPORTS = ["dbeel_tree_open", "dbeel_tree_close", "dbeel_tree_sstables", "dbeel_tree_write_sstable_index",
                "dbeel_tree_compact", "dbeel_tree_compact_many", "dbeel_tree_flush", "dbeel_tree_recover_wal", "dbeel_tree_get_many", "dbeel_tree_get_values", "dbeel_tree_get_values_stream", "dbeel_tree_reader_open", "dbeel_tree_scan", "dbeel_tree_scan_stream", "dbeel_tree_last_error", "dbeel_memtable_cut",
                "dbeel_plan_compactions", "dbeel_out_pages", "dbeel_tree_set_page_sink"]


def _run_struct(batch) -> Tuple[capi.Run, tuple]:
    d, i = capi._u8(batch[0]), capi._u8(batch[1])
    return capi.Run(d.ctypes.data, d.size, i.ctypes.data, i.size), (d, i)


def memtable_cut(batch, first_record: int = 0, capacity: int = DEFAULT_TREE_CAPACITY) -> int:
    """Arrivals from `first_record` on that one memtable of `capacity` distinct keys absorbs."""
    run, _keep = _run_struct(batch)
    return int(_lib().dbeel_memtable_cut(C.byref(run), first_record, capacity))


def plan_compactions(indices_and_sizes: Sequence[Tuple[int, int]], compaction_factor: int = 2):
    """compact_tree's picker, deterministic: [(indices_to_compact, output_index, keep_tombstones)]."""
    n = len(indices_and_sizes)
    if n == 0:
        return []
    idx = (C.c_uint64 * n)(*[i for i, _ in indices_and_sizes])
    siz = (C.c_uint64 * n)(*[s for _, s in indices_and_sizes])
    members = (C.c_uint64 * n)()
    start = (C.c_uint32 * (n + 1))()
    outs = (C.c_uint64 * n)()
    keeps = (C.c_int32 * n)()
    g = _lib().dbeel_plan_compactions(idx, siz, n, compaction_factor, members, start, outs, keeps)
    return [([int(members[k]) for k in range(start[j], start[j + 1])], int(outs[j]), bool(keeps[j])) for j in range(g)]


class LSMTree:
    """The compaction-facing part of dbeel's LSMTree over a directory of SSTable files."""

    def __init__(self, directory: str, engine, sstable_bloom_min_size: int = DEFAULT_SSTABLE_BLOOM_MIN_SIZE):
        self._h = C.c_void_p()
        self._engine = engine
        eh = engine._h if hasattr(engine, "_h") else engine
        rc = _lib().dbeel_tree_open(directory.encode(), eh, sstable_bloom_min_size, C.byref(self._h))
        if rc:
            raise capi.DbeelError(rc, f"dbeel_tree_open({directory})")
        self.dir = directory

    open_or_create = classmethod(lambda cls, *a, **k: cls(*a, **k))

    def close(self):
        if self._h:
            _lib().dbeel_tree_close(self._h)
            self._h = C.c_void_p()

    def set_page_cache(self, cache: Optional[dict]):
        """Mirror EntryWriter's write-through: every SSTable this tree writes from now on is also `set` page by page into
        `cache` under the reference's key ((FileTypeKind, files_index), address) (entry_writer.rs:100-156).  None = off.
        This is a host-side mirror of the reference's cache; the device page cache that readers read through is
        capi.PageCache (open_reader(page_cache=...)), which this does not fill."""
        if cache is None:
            self._sink = PAGE_SINK(0)
        else:
            def sink(_ctx, kind, files_index, address, page):
                cache[((int(kind), int(files_index)), int(address))] = bytes(page[:PAGE_SIZE])
            self._sink = PAGE_SINK(sink)
        _lib().dbeel_tree_set_page_sink(self._h, self._sink, None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc:
            raise capi.DbeelError(rc, f"{what}: {_lib().dbeel_tree_last_error(self._h).decode()}")

    def sstable_indices_and_sizes(self) -> List[Tuple[int, int]]:
        n = _lib().dbeel_tree_sstables(self._h, None, None, 0)
        idx, siz = (C.c_uint64 * max(1, n))(), (C.c_uint64 * max(1, n))()
        _lib().dbeel_tree_sstables(self._h, idx, siz, n)
        return [(int(idx[k]), int(siz[k])) for k in range(n)]

    @property
    def write_sstable_index(self) -> int:
        return int(_lib().dbeel_tree_write_sstable_index(self._h))

    def compact(self, indices_to_compact: Sequence[int], output_index: int, keep_tombstones: bool,
                bloom_seed: Optional[bytes] = None) -> None:
        arr = (C.c_uint64 * max(1, len(indices_to_compact)))(*indices_to_compact)
        self._check(_lib().dbeel_tree_compact(self._h, arr, len(indices_to_compact), output_index,
                                              int(keep_tombstones), bloom_seed), "LSMTree.compact")

    def flush(self, batch) -> Tuple[int, int]:
        """One memtable's arrivals -> the next even-indexed SSTable.  Returns (index, items)."""
        run, _keep = _run_struct(batch)
        wi, n = C.c_uint64(), C.c_uint64()
        self._check(_lib().dbeel_tree_flush(self._h, C.byref(run), C.byref(wi), C.byref(n)), "LSMTree.flush")
        return int(wi.value), int(n.value)

    def get_many(self, keys: Sequence[bytes], mode: int = capi.LOOKUP_REFERENCE):
        """get_entry's SSTable loop for a batch of keys: a list of `data` bytes (b"" = tombstone) or None per key,
        like LSMTree::get (lsm_tree.rs:722-724) after the memtables missed."""
        import numpy as np
        from . import sstable
        blob, off = capi.pack_keys(keys)
        res = np.zeros(len(keys), dtype=capi.LOOKUP_DTYPE)
        self._check(_lib().dbeel_tree_get_many(self._h, blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys), mode,
                                               res.ctypes.data), "LSMTree.get_many")
        tables = self.sstable_indices_and_sizes()
        files = {}
        out = []
        for row in res:
            if row["table"] < 0:
                out.append(None)
                continue
            idx = tables[int(row["table"])][0]
            if idx not in files:
                files[idx] = sstable.read_run_files(self.dir, idx)
            d, i = files[idx]
            rec = bytes(i[16 * int(row["record"]):16 * int(row["record"]) + 16])
            o, ks, fs = int.from_bytes(rec[:8], "little"), int.from_bytes(rec[8:12], "little"), int.from_bytes(rec[12:], "little")
            out.append(bytes(d[o + ks + 8:o + fs - 16]))  # EntryValue.data (entry = key | dlen | data | ts)
        return out

    def get_values(self, keys: Sequence[bytes], mode: int = capi.LOOKUP_REFERENCE):
        """dbeel_tree_get_values: get_entry's SSTable loop with the entries, one call.  Returns (rows, data, index) like
        Engine.get_values: rows as in get_many's dbeel_tree_get_many, and the answered rows' entries in query order as an
        arrival batch (row i's entry is entry number (answered rows before i); a row with LOOKUP_BAD_ENTRY has none, as
        the reference's get returns Err for it)."""
        from . import sstable
        blob, off = capi.pack_keys(keys)
        res = np.zeros(len(keys), dtype=capi.LOOKUP_DTYPE)
        dc = sum(os.path.getsize(os.path.join(self.dir, sstable.file_name(idx, sstable.DATA_FILE_EXT)))
                 for idx, _ in self.sstable_indices_and_sizes())
        ic = 16 * len(keys)
        for attempt in range(2):  # one more call with the reported sizes when duplicate keys need more than the files hold
            od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
            out = capi.Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
            rc = _lib().dbeel_tree_get_values(self._h, blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys), mode,
                                              C.byref(out), res.ctypes.data)
            if rc == capi.ERR_CAPACITY and not attempt:
                dc, ic = int(out.data_len), int(out.index_len)
                continue
            self._check(rc, "LSMTree.get_values")
            return res, od[:out.data_len], oi[:out.index_len]

    def get_values_stream(self, keys: Sequence[bytes], mode: int = capi.LOOKUP_REFERENCE):
        """dbeel_tree_get_values_stream: what get_values returns, with .data and .index read from the files only where the
        searches reach (each .bloom is read whole), so trees larger than device or host memory answer too."""
        from . import sstable
        blob, off = capi.pack_keys(keys)
        res = np.zeros(len(keys), dtype=capi.LOOKUP_DTYPE)
        dc = min(64 << 20, sum(os.path.getsize(os.path.join(self.dir, sstable.file_name(idx, sstable.DATA_FILE_EXT)))
                               for idx, _ in self.sstable_indices_and_sizes()))
        ic = 16 * len(keys)
        for attempt in range(2):  # one more call with the reported sizes when the first caps are short
            od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
            out = capi.Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
            rc = _lib().dbeel_tree_get_values_stream(self._h, blob.ctypes.data if blob.size else None, off.ctypes.data,
                                                     len(keys), mode, C.byref(out), res.ctypes.data)
            if rc == capi.ERR_CAPACITY and not attempt:
                dc, ic = int(out.data_len), int(out.index_len)
                continue
            self._check(rc, "LSMTree.get_values_stream")
            return res, od[:out.data_len], oi[:out.index_len]

    def open_reader(self, fence_bytes: int = 0, page_cache: Optional[capi.PageCache] = None) -> capi.Reader:
        """dbeel_tree_reader_open: a capi.Reader over a snapshot of the tree's SSTables (get_values answers what
        get_values_stream answered at open, scan what scan_stream returned at open, table = a position in the snapshot),
        unaffected by later flushes and compactions.  Readers share the tables they have in common: one opened after a
        flush loads only the new ones.  page_cache: a capi.PageCache (Engine.open_page_cache) the reader reads its leaves
        and entries through; pages of the tables it shares with earlier readers of the same cache are hits.  (Not
        set_page_cache, the host-side mirror of the reference's write-through.)"""
        from . import sstable
        h = C.c_void_p()
        self._check(_lib().dbeel_tree_reader_open(self._h, fence_bytes, C.byref(h)), "LSMTree.open_reader")
        dc = sum(os.path.getsize(os.path.join(self.dir, sstable.file_name(idx, sstable.DATA_FILE_EXT)))
                 for idx, _ in self.sstable_indices_and_sizes())
        r = capi.Reader(h, self._engine, data_cap=dc)
        if page_cache is not None:
            r.attach_page_cache(page_cache)
        return r

    def scan(self, ranges, kind: int = capi.SCAN_HASH):
        """The SSTable part of iter_filter (lsm_tree.rs:133-282) over the tree's files, oldest table first: every entry
        goes to the first of `ranges` that accepts it ((start, end) u32 hash ranges with between_cmp, or byte-string key
        ranges).  Returns ([(data, index)] per range, (table, reason, record) of the first record the reference's iterator
        fails on, table = position in sstable_indices_and_sizes() order).  The memtables are the caller's."""
        from . import sstable
        dc = ic = 0
        for idx, _ in self.sstable_indices_and_sizes():
            dc += os.path.getsize(os.path.join(self.dir, sstable.file_name(idx, sstable.DATA_FILE_EXT)))
            ic += os.path.getsize(os.path.join(self.dir, sstable.file_name(idx, sstable.INDEX_FILE_EXT)))
        od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(16, ic), np.uint8)
        out = capi.Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
        rptr, _keep = capi.pack_ranges(kind, ranges)
        n = len(ranges)
        res = (capi.JobResult * max(1, n))()
        stop = capi.ScanStop()
        self._check(_lib().dbeel_tree_scan(self._h, kind, rptr, n, C.byref(out), res, C.byref(stop)), "LSMTree.scan")
        return ([(od[r.data_off:r.data_off + r.data_len].copy(), oi[r.index_off:r.index_off + r.index_len].copy())
                 for r in res[:n]], stop.as_tuple())

    def scan_stream(self, ranges, kind: int = capi.SCAN_HASH, write=None):
        """scan() with the files streamed through the engine (dbeel_tree_scan_stream): nothing is read whole, so trees
        larger than memory scan too.  write(dest, kind, offset, src_address, length) -> 0 or an error code receives every
        piece of every destination's .data (kind 1) / .index (kind 2), from several threads (src_address: host memory
        valid during the call); without one the pieces are collected in memory.  Returns ([(data_len, index_len, items)]
        per range when `write` is given, else [(data, index)] per range like scan(), and the stop as scan() does."""
        import threading
        n = len(ranges)
        files = [{1: bytearray(), 2: bytearray()} for _ in range(n)]
        mu = threading.Lock()

        def collect(dest, kind_, off, src, size):
            with mu:
                f = files[dest][kind_]
                if len(f) < off + size:
                    f.extend(bytes(off + size - len(f)))
                f[off:off + size] = C.string_at(src, size)
            return 0

        cb = capi.SCAN_WRITE_FN(lambda _ctx, dest, kind_, off, src, size: (write or collect)(dest, kind_, off, src, size))
        rptr, _keep = capi.pack_ranges(kind, ranges)
        res = (capi.JobResult * max(1, n))()
        stop = capi.ScanStop()
        self._check(_lib().dbeel_tree_scan_stream(self._h, kind, rptr, n, cb, None, res, C.byref(stop)), "LSMTree.scan_stream")
        if write is not None:
            return [(int(r.data_len), int(r.index_len), int(r.items_written)) for r in res[:n]], stop.as_tuple()
        return ([(np.frombuffer(bytes(f[1]), np.uint8).copy(), np.frombuffer(bytes(f[2]), np.uint8).copy()) for f in files],
                stop.as_tuple())

    def recover_wal(self, tree_capacity: int = capi.DEFAULT_TREE_CAPACITY) -> Tuple[int, int]:
        """open_or_create_ex's WAL step (lsm_tree.rs:466-513): with two `.memtable` files the older one is replayed and
        flushed.  Returns (index of the log that stays active, entries of the recovered SSTable)."""
        wi, n = C.c_uint64(), C.c_uint64()
        self._check(_lib().dbeel_tree_recover_wal(self._h, tree_capacity, C.byref(wi), C.byref(n)), "LSMTree.recover_wal")
        return int(wi.value), int(n.value)

    def compact_many(self, plan, bloom_seeds: Optional[Sequence[bytes]] = None) -> None:
        """All groups of a plan_compactions() result through ONE dbeel_compact_many, committed group by group."""
        members = [i for indices, _, _ in plan for i in indices]
        starts = [0]
        for indices, _, _ in plan:
            starts.append(starts[-1] + len(indices))
        n = len(plan)
        m = (C.c_uint64 * max(1, len(members)))(*members)
        gs = (C.c_uint32 * (n + 1))(*starts)
        oi = (C.c_uint64 * max(1, n))(*[o for _, o, _ in plan])
        kt = (C.c_int32 * max(1, n))(*[int(k) for _, _, k in plan])
        seeds = b"".join(bloom_seeds) if bloom_seeds is not None else None
        self._check(_lib().dbeel_tree_compact_many(self._h, m, gs, n, oi, kt, seeds), "LSMTree.compact_many")

    def compact_tree(self, compaction_factor: int = 2, bloom_seed: Optional[bytes] = None, batched: bool = False):
        """tasks/compaction.rs compact_tree: plan with the picker, run every group (batched: in one launch sequence)."""
        plan = plan_compactions(self.sstable_indices_and_sizes(), compaction_factor)
        if batched and plan:
            self.compact_many(plan, [bloom_seed] * len(plan) if bloom_seed is not None else None)
            return plan
        for indices, out, keep in plan:
            self.compact(indices, out, keep, bloom_seed)
        return plan


def out_pages(data, index, files_index: int):
    """dbeel_out_pages: the (file kind, files_index, address, page bytes) sequence EntryWriter would `set` for this SSTable."""
    d, i = capi._u8(data), capi._u8(index)
    seq = []

    def sink(_ctx, kind, fi, address, page):
        seq.append((int(kind), int(fi), int(address), bytes(page[:PAGE_SIZE])))
    cb = PAGE_SINK(sink)
    rc = _lib().dbeel_out_pages(d.ctypes.data if d.size else None, d.size, i.ctypes.data if i.size else None, i.size, files_index, cb, None)
    if rc:
        raise capi.DbeelError(rc, "dbeel_out_pages")
    return seq
