"""ctypes binding of include/dbeel_compact.h -- the same C ABI a Rust `extern "C"` block
would bind (INTEGRATION.md).  There is no CPU fallback: if libdbeel_compact.so is missing or
no sm_90 device is present, this module raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DBEEL_LIB") or os.path.join(_HERE, "libdbeel_compact.so")  # DBEEL_LIB: A/B builds only

DBEEL_OK = 0
ERR_NAMES = {1: "INVALID_ARG", 2: "CAPACITY", 3: "ITEM_TOO_LARGE", 4: "CUDA", 5: "NOMEM", 6: "TOO_MANY_RUNS",
             7: "TOO_MANY_ENTRIES", 8: "UNSORTED_RUN", 9: "NO_DEVICE", 10: "BUSY", 11: "BAD_BLOOM", 12: "TREE_FULL"}
ERR_BAD_BLOOM = 11
ERR_TREE_FULL = 12
ERR_ITEM_TOO_LARGE = 3
DEFAULT_TREE_CAPACITY = 8192  # mod.rs:18
LOOKUP_REFERENCE = 0  # the reference's binary_search loop, step for step (lsm_tree.rs:605-670)
LOOKUP_EXACT = 1      # lower-bound search: every present key is found
LOOKUP_CORRUPT = 0x80000000
LOOKUP_BAD_ENTRY = 0x40000000  # get_values: the hit's entry does not decode (the reference's get returns Err)
SCAN_HASH = 0  # ranges: (start, end) u32 pairs, murmur3_32(key) tested with migration.rs's between_cmp
SCAN_KEY = 1   # ranges: (start, end) byte strings, start <= key < end
SCAN_STOP_NONE, SCAN_STOP_ERR, SCAN_STOP_PANIC = 0, 1, 2
RANGE_KEEP_TOMBSTONES = 0x1  # dbeel_reader_get_range: keep entries with dlen == 0
RANGE_LIMIT_MAX = 65536  # dbeel_reader_get_ranges: the largest limit of one query
RANGE_MORE, RANGE_STOPPED, RANGE_UNSORTED = 0x1, 0x2, 0x4  # dbeel_range_row.flags
ERR_UNSORTED_RUN = 8
ERR_CAPACITY = 2
ERR_INVALID_ARG = 1
ERR_NO_DEVICE = 9
ERR_BUSY = 10
FLAG_VERIFY_SORTED = 0x1
FLAG_REFERENCE_READER = 0x2  # decode runs like read_next_entry (lsm_tree.rs:1158-1170): offset / key_size ignored, timestamps range-checked
DEFAULT_BLOOM_MIN_SIZE = 1_048_576
DEFAULT_BLOOM_FP = 0.01

EXPORTS = ["dbeel_abi_version", "dbeel_engine_create", "dbeel_engine_destroy", "dbeel_compact_bound",
           "dbeel_compact", "dbeel_compact_stream", "dbeel_compact_device", "dbeel_compact_submit", "dbeel_poll", "dbeel_wait",
           "dbeel_flush", "dbeel_flush_device", "dbeel_flush_many", "dbeel_flush_many_device",
           "dbeel_get_many", "dbeel_get_many_device", "dbeel_wal_flush", "dbeel_wal_flush_device",
           "dbeel_compact_many_bound", "dbeel_compact_many", "dbeel_compact_many_device",
           "dbeel_bloom_bitmap_bytes", "dbeel_bloom_k_num", "dbeel_bloom_file_size", "dbeel_host_alloc",
           "dbeel_host_free", "dbeel_last_stats", "dbeel_last_error", "dbeel_strerror",
           "dbeel_murmur3_32", "dbeel_ring_owner", "dbeel_shard_ring", "dbeel_route_device", "dbeel_flush_many_sparse_device",
           "dbeel_gpu_numa_node", "dbeel_bind_to_gpu", "dbeel_memtable_cuts_device", "dbeel_engine_stream",
           "dbeel_scan_bound", "dbeel_scan", "dbeel_scan_device", "dbeel_scan_stream", "dbeel_get_values",
           "dbeel_get_values_device", "dbeel_get_values_stream", "dbeel_reader_open", "dbeel_reader_get_values",
           "dbeel_readers_get_values",
           "dbeel_reader_scan", "dbeel_reader_get_range", "dbeel_reader_get_ranges",
           "dbeel_reader_get_ranges_reverse", "dbeel_readers_get_ranges", "dbeel_reader_close", "dbeel_page_cache_create", "dbeel_page_cache_destroy",
           "dbeel_reader_attach_page_cache", "dbeel_page_cache_stats"]


class Run(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_len", C.c_uint64), ("index", C.c_void_p), ("index_len", C.c_uint64)]


STREAM_READ_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p)
STREAM_WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64)


class StreamIO(C.Structure):
    _fields_ = [("read", STREAM_READ_FN), ("write", STREAM_WRITE_FN), ("ctx", C.c_void_p)]


SCAN_WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64)


class ScanIO(C.Structure):
    _fields_ = [("read", STREAM_READ_FN), ("write", SCAN_WRITE_FN), ("ctx", C.c_void_p)]


class Out(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_cap", C.c_uint64), ("data_len", C.c_uint64),
                ("index", C.c_void_p), ("index_cap", C.c_uint64), ("index_len", C.c_uint64),
                ("bloom", C.c_void_p), ("bloom_cap", C.c_uint64), ("bloom_len", C.c_uint64),
                ("items_written", C.c_uint64)]


class FlushTable(C.Structure):
    _fields_ = [("data_off", C.c_uint64), ("data_len", C.c_uint64), ("index_off", C.c_uint64),
                ("index_len", C.c_uint64), ("items", C.c_uint64)]


class Job(C.Structure):
    _fields_ = [("runs", C.POINTER(Run)), ("n_runs", C.c_uint32), ("keep_tombstones", C.c_int32), ("bloom_seed", C.c_char_p)]


class JobResult(C.Structure):
    _fields_ = [("data_off", C.c_uint64), ("data_len", C.c_uint64), ("index_off", C.c_uint64), ("index_len", C.c_uint64),
                ("bloom_off", C.c_uint64), ("bloom_len", C.c_uint64), ("items_written", C.c_uint64)]


class Table(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_len", C.c_uint64), ("index", C.c_void_p), ("index_len", C.c_uint64),
                ("bloom", C.c_void_p), ("bloom_len", C.c_uint64)]


class KeyRanges(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("key_offsets", C.c_void_p)]


class ScanStop(C.Structure):
    _fields_ = [("table", C.c_int32), ("reason", C.c_uint32), ("record", C.c_uint64)]

    def as_tuple(self):
        """(table, reason, record); (-1, SCAN_STOP_NONE, 0) when every record was read."""
        return int(self.table), int(self.reason), int(self.record)


# dbeel_range_row: the query's first entry number in out, its entry count, DBEEL_RANGE_* flags and its stop
RANGE_ROW_DTYPE = np.dtype([("first", "<u8"), ("count", "<u4"), ("flags", "<u4"), ("table", "<i4"), ("reason", "<u4"),
                            ("record", "<u8")])


def pack_ranges(kind: int, ranges):
    """The `ranges` argument of dbeel_scan: hash ranges as a u32 array, key ranges as a KeyRanges over a packed blob.
    Returns (pointer-bearing object, things to keep alive)."""
    if kind == SCAN_HASH:
        arr = np.ascontiguousarray(np.array([[int(a), int(b)] for a, b in ranges], dtype=np.uint32).reshape(-1))
        return arr.ctypes.data, (arr,)
    blob, off = pack_keys([bytes(k) for pair in ranges for k in pair])
    kr = KeyRanges(blob.ctypes.data if blob.size else None, off.ctypes.data)
    return C.addressof(kr), (kr, blob, off)


class LookupResult(C.Structure):
    _fields_ = [("table", C.c_int32), ("bloom_rejects", C.c_uint32), ("record", C.c_uint64)]


LOOKUP_DTYPE = np.dtype([("table", "<i4"), ("bloom_rejects", "<u4"), ("record", "<u8")])
MAX_READER_BATCHES = 1024  # DBEEL_MAX_READER_BATCHES


class ReaderBatch(C.Structure):
    _fields_ = [("reader", C.c_void_p), ("keys", C.c_void_p), ("key_offsets", C.c_void_p), ("n_keys", C.c_uint64),
                ("mode", C.c_uint32), ("reserved", C.c_uint32)]


class RangeBatch(C.Structure):
    """dbeel_range_batch: one reader's limited range reads in dbeel_readers_get_ranges."""
    _fields_ = [("reader", C.c_void_p), ("ranges", KeyRanges), ("limits", C.c_void_p), ("n_ranges", C.c_uint32),
                ("flags", C.c_uint32), ("reverse", C.c_uint32), ("reserved", C.c_uint32)]


DbeelRangeBatch = RangeBatch


def pack_keys(keys: Sequence[bytes]) -> Tuple[np.ndarray, np.ndarray]:
    """Query keys in the layout dbeel_get_many takes: (bytes back to back, n + 1 offsets)."""
    off = np.zeros(len(keys) + 1, dtype=np.uint64)
    if keys:
        off[1:] = np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=len(keys)))
    blob = np.frombuffer(b"".join(keys), dtype=np.uint8) if keys else np.zeros(0, np.uint8)
    return blob, off


class Opts(C.Structure):
    _fields_ = [("keep_tombstones", C.c_int32), ("flags", C.c_uint32), ("bloom_min_size", C.c_uint64),
                ("bloom_fp", C.c_double), ("bloom_seed", C.c_char_p)]


class Stats(C.Structure):
    _fields_ = [("input_bytes", C.c_uint64), ("output_bytes", C.c_uint64), ("entries_in", C.c_uint64),
                ("entries_valid", C.c_uint64), ("entries_out", C.c_uint64), ("runs_truncated", C.c_uint32),
                ("key_prefix_len", C.c_uint32), ("merge_passes", C.c_uint32), ("kernel_launches", C.c_uint32),
                ("ms_total", C.c_float), ("ms_extract", C.c_float), ("ms_merge", C.c_float),
                ("ms_resolve", C.c_float), ("ms_gather", C.c_float), ("ms_h2d", C.c_float), ("ms_d2h", C.c_float),
                ("gather_bytes", C.c_uint64), ("partitions", C.c_uint32), ("index_repaired", C.c_uint32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class DbeelError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"dbeel error {code} ({ERR_NAMES.get(code, '?')}): {msg}")
        self.code = code
        self.needed = None  # get_values*: (data_len, index_len) the output needs, on ERR_CAPACITY


_lib = None


def lib():
    """The loaded library.  Fails loudly when it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH) and "DBEEL_LIB" not in os.environ:
            try:  # a fresh checkout: the .so is git-ignored; build it in-tree if the toolkit is here
                from . import _build
                _build.build()
            except Exception as ex:
                raise RuntimeError(f"{LIB_PATH} is missing and could not be built ({ex}): run "
                                   "`python -m dbeel_b200._build` where nvcc is. There is no CPU fallback "
                                   "for the compaction path.") from ex
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing. There is no CPU fallback for the compaction path.")
        L = C.CDLL(LIB_PATH)
        L.dbeel_abi_version.restype = C.c_int
        L.dbeel_engine_create.restype = C.c_int
        L.dbeel_engine_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.dbeel_engine_stream.restype = C.c_void_p
        L.dbeel_engine_stream.argtypes = [C.c_void_p]
        L.dbeel_engine_destroy.restype = None
        L.dbeel_engine_destroy.argtypes = [C.c_void_p]
        L.dbeel_compact_bound.restype = C.c_int
        L.dbeel_compact_bound.argtypes = [C.POINTER(Run), C.c_uint32, C.POINTER(Opts)] + [C.POINTER(C.c_uint64)] * 3
        for name in ("dbeel_compact", "dbeel_compact_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Run), C.c_uint32, C.POINTER(Opts), C.POINTER(Out)]
        L.dbeel_compact_stream.restype = C.c_int
        L.dbeel_compact_stream.argtypes = [C.c_void_p, C.POINTER(Run), C.c_uint32, C.POINTER(Opts), C.POINTER(StreamIO), C.POINTER(Out)]
        L.dbeel_compact_submit.restype = C.c_int
        L.dbeel_compact_submit.argtypes = [C.c_void_p, C.POINTER(Run), C.c_uint32, C.POINTER(Opts), C.POINTER(Out)]
        L.dbeel_poll.restype = C.c_int
        L.dbeel_poll.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        L.dbeel_wait.restype = C.c_int
        L.dbeel_wait.argtypes = [C.c_void_p]
        for name in ("dbeel_flush", "dbeel_flush_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Run), C.POINTER(Out)]
        for name in ("dbeel_flush_many", "dbeel_flush_many_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Run), C.c_uint32, C.POINTER(Out), C.POINTER(FlushTable)]
        for name in ("dbeel_get_many", "dbeel_get_many_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                          C.c_void_p]
        for name in ("dbeel_get_values", "dbeel_get_values_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                          C.POINTER(Out), C.c_void_p]
        L.dbeel_get_values_stream.restype = C.c_int
        L.dbeel_get_values_stream.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64,
                                              C.c_uint32, C.POINTER(ScanIO), C.POINTER(Out), C.c_void_p]
        L.dbeel_reader_open.restype = C.c_int
        L.dbeel_reader_open.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.POINTER(ScanIO), C.c_uint64,
                                        C.POINTER(C.c_void_p)]
        L.dbeel_reader_get_values.restype = C.c_int
        L.dbeel_reader_get_values.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(Out),
                                              C.c_void_p]
        L.dbeel_readers_get_values.restype = C.c_int
        L.dbeel_readers_get_values.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(Out), C.c_void_p]
        L.dbeel_reader_scan.restype = C.c_int
        L.dbeel_reader_scan.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, SCAN_WRITE_FN, C.c_void_p,
                                        C.POINTER(JobResult), C.POINTER(ScanStop)]
        L.dbeel_reader_get_range.restype = C.c_int
        L.dbeel_reader_get_range.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, SCAN_WRITE_FN, C.c_void_p,
                                             C.POINTER(JobResult), C.POINTER(ScanStop)]
        L.dbeel_reader_get_ranges.restype = C.c_int
        L.dbeel_reader_get_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(Out),
                                              C.c_void_p]
        L.dbeel_reader_get_ranges_reverse.restype = C.c_int
        L.dbeel_reader_get_ranges_reverse.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                                      C.POINTER(Out), C.c_void_p]
        L.dbeel_readers_get_ranges.restype = C.c_int
        L.dbeel_readers_get_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(Out), C.c_void_p]
        L.dbeel_reader_close.restype = None
        L.dbeel_reader_close.argtypes = [C.c_void_p]
        L.dbeel_page_cache_create.restype = C.c_int
        L.dbeel_page_cache_create.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
        L.dbeel_page_cache_destroy.restype = None
        L.dbeel_page_cache_destroy.argtypes = [C.c_void_p]
        L.dbeel_reader_attach_page_cache.restype = C.c_int
        L.dbeel_reader_attach_page_cache.argtypes = [C.c_void_p, C.c_void_p]
        L.dbeel_page_cache_stats.restype = C.c_int
        L.dbeel_page_cache_stats.argtypes = [C.c_void_p, C.POINTER(PageCacheStats)]
        L.dbeel_scan_bound.restype = C.c_int
        L.dbeel_scan_bound.argtypes = [C.POINTER(Table), C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        for name in ("dbeel_scan", "dbeel_scan_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(Out),
                          C.POINTER(JobResult), C.POINTER(ScanStop)]
        L.dbeel_scan_stream.restype = C.c_int
        L.dbeel_scan_stream.argtypes = [C.c_void_p, C.POINTER(Table), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                        C.POINTER(ScanIO), C.POINTER(JobResult), C.POINTER(ScanStop)]
        L.dbeel_compact_many_bound.restype = C.c_int
        L.dbeel_compact_many_bound.argtypes = [C.POINTER(Job), C.c_uint32, C.c_uint64, C.c_double] + [C.POINTER(C.c_uint64)] * 3
        for name in ("dbeel_compact_many", "dbeel_compact_many_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.POINTER(Job), C.c_uint32, C.c_uint64, C.c_double, C.POINTER(Out), C.POINTER(JobResult)]
        for name in ("dbeel_wal_flush", "dbeel_wal_flush_device"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(Out)]
        L.dbeel_bloom_bitmap_bytes.restype = C.c_uint64
        L.dbeel_bloom_bitmap_bytes.argtypes = [C.c_uint64, C.c_double]
        L.dbeel_bloom_k_num.restype = C.c_uint32
        L.dbeel_bloom_k_num.argtypes = [C.c_uint64, C.c_uint64]
        L.dbeel_bloom_file_size.restype = C.c_uint64
        L.dbeel_bloom_file_size.argtypes = [C.c_uint64, C.c_double]
        L.dbeel_host_alloc.restype = C.c_void_p
        L.dbeel_host_alloc.argtypes = [C.c_uint64]
        L.dbeel_host_free.restype = None
        L.dbeel_host_free.argtypes = [C.c_void_p]
        L.dbeel_last_stats.restype = C.c_int
        L.dbeel_last_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        L.dbeel_last_error.restype = C.c_char_p
        L.dbeel_last_error.argtypes = [C.c_void_p]
        L.dbeel_strerror.restype = C.c_char_p
        L.dbeel_strerror.argtypes = [C.c_int]
        L.dbeel_gpu_numa_node.restype = C.c_int
        L.dbeel_gpu_numa_node.argtypes = [C.c_int]
        L.dbeel_bind_to_gpu.restype = C.c_int
        L.dbeel_bind_to_gpu.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.dbeel_murmur3_32.restype = C.c_uint32
        L.dbeel_murmur3_32.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32]
        L.dbeel_ring_owner.restype = C.c_uint32
        L.dbeel_ring_owner.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.dbeel_shard_ring.restype = C.c_int
        L.dbeel_shard_ring.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.dbeel_route_device.restype = C.c_int
        L.dbeel_route_device.argtypes = [C.c_void_p, C.POINTER(Run), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
        L.dbeel_memtable_cuts_device.restype = C.c_int
        L.dbeel_memtable_cuts_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                 C.c_uint32]
        L.dbeel_flush_many_sparse_device.restype = C.c_int
        L.dbeel_flush_many_sparse_device.argtypes = [C.c_void_p, C.POINTER(Run), C.c_uint32, C.c_uint64, C.POINTER(Out),
                                                     C.POINTER(FlushTable)]
        _lib = L
    return _lib


def _u8(a) -> np.ndarray:
    if isinstance(a, np.ndarray):
        if a.dtype != np.uint8 or not a.flags.c_contiguous:
            a = np.ascontiguousarray(a, dtype=np.uint8)
        return a
    return np.frombuffer(bytes(a), dtype=np.uint8)


def make_opts(keep_tombstones: bool = False, bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE,
              bloom_fp: float = DEFAULT_BLOOM_FP, seed: Optional[bytes] = None, flags: int = 0) -> Opts:
    if seed is not None and len(seed) != 32:
        raise ValueError("bloom seed must be 32 bytes")
    return Opts(int(keep_tombstones), flags, bloom_min_size, bloom_fp, seed)


def compact_bound(runs: Sequence[Tuple[int, int]], opts: Opts) -> Tuple[int, int, int]:
    """runs: (data_len, index_len) pairs -> (data_cap, index_cap, bloom_cap)."""
    arr = (Run * max(1, len(runs)))()
    for j, (dl, il) in enumerate(runs):
        arr[j] = Run(None, dl, None, il)
    d, i, b = C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = lib().dbeel_compact_bound(arr, len(runs), C.byref(opts), C.byref(d), C.byref(i), C.byref(b))
    if rc:
        raise DbeelError(rc, "dbeel_compact_bound")
    return d.value, i.value, b.value


class PinnedBuffer:
    """dbeel_host_alloc'ed memory exposed as a numpy uint8 array."""

    def __init__(self, nbytes: int):
        self.nbytes = int(nbytes)
        self.ptr = lib().dbeel_host_alloc(self.nbytes)
        if not self.ptr:
            raise MemoryError(f"dbeel_host_alloc({nbytes})")
        self.array = np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_uint8)), shape=(max(1, self.nbytes),))[:self.nbytes]

    def free(self):
        if self.ptr:
            self.array = None
            lib().dbeel_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


READER_FRAME_CAP = 64                  # DBEEL_READER_FRAME_CAP: longest key a reader's cached fences serve
DEFAULT_READER_FENCE_BYTES = 64 << 20  # DBEEL_READER_FENCE_BYTES_DEFAULT


class _StreamTables:
    """The tables and the read callback of a streamed read: (data, index, bloom | None) oldest first.  Without `read` the
    callback serves data / index from memory; with it, data / index may be sizes, and read(table, kind, offset, size)
    returns the bytes (kind 1 = .data, 2 = .index; called from several engine threads) or a nonzero int error code.
    Every read is logged as (table, kind, offset, size); fail_read_at = n makes the n-th read of a call return 4242."""

    def __init__(self, tables, read=None):
        import threading

        def size_of(x):
            return int(x) if isinstance(x, (int, np.integer)) else _u8(x).size
        self.keep = [(None if read else _u8(d), None if read else _u8(i), _u8(b) if b is not None and len(b) else None)
                     for d, i, b in tables]
        self.sizes = [(size_of(d), size_of(i)) for d, i, _ in tables]
        self.arr = (Table * max(1, len(self.keep)))()
        for j, ((_, _, b), (ds, isz)) in enumerate(zip(self.keep, self.sizes)):
            self.arr[j] = Table(None, ds, None, isz, b.ctypes.data if b is not None else None, b.size if b is not None else 0)
        self.fail_read_at = -1
        self.log = []
        self.last_reads = []
        mu = threading.Lock()
        keep = self.keep

        def rd(_ctx, table, kind_, offset, size, dst):
            with mu:
                k = len(self.log)
                self.log.append((int(table), int(kind_), int(offset), int(size)))
            if k == self.fail_read_at:
                return 4242
            if read is None:
                src = keep[table][0] if kind_ == 1 else keep[table][1]
                if offset + size > src.size:
                    return 4243
                C.memmove(dst, src.ctypes.data + offset, size)
                return 0
            got = read(int(table), int(kind_), int(offset), int(size))
            if isinstance(got, (int, np.integer)):
                return int(got)
            b = np.ascontiguousarray(np.frombuffer(got, np.uint8) if isinstance(got, (bytes, bytearray)) else _u8(got))
            if b.size != size:
                return 4243
            C.memmove(dst, b.ctypes.data, size)
            return 0

        self.io = ScanIO(STREAM_READ_FN(rd), C.cast(None, SCAN_WRITE_FN), None)


def _stream_values(call, name: str, h, n_keys: int, st: Optional[_StreamTables], caps, data_cap: int = 0):
    """One streamed get_values: call(out, rows) -> rc, with caps (data_cap, index_cap) or by default at most 64 MiB of
    .data (the tables' sizes when known, else data_cap) and 16 bytes per key, retried once with the sizes the engine
    reports.  Returns (rows, data, index); st.last_reads = the reads of the last call."""
    res = np.zeros(n_keys, dtype=LOOKUP_DTYPE)
    dc0 = sum(d for d, _ in st.sizes) if st is not None else data_cap
    dc, ic = caps if caps is not None else (min(dc0, 64 << 20), 16 * n_keys)
    for attempt in range(2):
        od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
        out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
        if st is not None:
            st.log.clear()
        rc = call(out, res)
        if st is not None:
            st.last_reads = list(st.log)
        if rc == 0:
            return res, od[:out.data_len], oi[:out.index_len]
        err = DbeelError(rc, f"{name}: {lib().dbeel_last_error(h).decode()}")
        if rc == ERR_CAPACITY:
            err.needed = (int(out.data_len), int(out.index_len))
        if caps is not None or attempt or rc != ERR_CAPACITY:
            raise err
        dc, ic = err.needed


class PageCacheStats(C.Structure):
    _fields_ = [("capacity_pages", C.c_uint64), ("resident_pages", C.c_uint64), ("hits", C.c_uint64), ("misses", C.c_uint64),
                ("evictions", C.c_uint64)]


class PageCache:
    """dbeel_page_cache_*: 4096-byte pages of readers' .data / .index files kept on the device across batches and across
    the readers attached to it (Reader.attach_page_cache, LSMTree.open_reader(page_cache=...)), made by
    Engine.open_page_cache.  Not LSMTree.set_page_cache, which mirrors the reference's write-through into a Python dict.
    Use it as a context manager or close() it; closing detaches it from its readers, which go on uncached, and the engine
    destroys caches still open when it is destroyed."""

    def __init__(self, handle: C.c_void_p, engine: "Engine"):
        self._h = handle
        self._engine = engine

    def stats(self) -> dict:
        """capacity_pages, resident_pages; hits, misses and evictions in pages since the cache was made."""
        if not self._h:
            raise ValueError("page cache is closed")
        st = PageCacheStats()
        rc = lib().dbeel_page_cache_stats(self._h, C.byref(st))
        if rc:
            raise DbeelError(rc, "dbeel_page_cache_stats")
        return {name: int(getattr(st, name)) for name, _ in PageCacheStats._fields_}

    def close(self):
        if self._h and self._engine._h:  # an engine already destroyed has destroyed its caches
            lib().dbeel_page_cache_destroy(self._h)
        self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class Reader:
    """dbeel_reader_*: get_values_stream's batches and scan_stream's range scans on a fixed set of tables, with the
    filters and fences kept on the device between calls (Engine.open_reader, storage_engine.LSMTree.open_reader).  Use it as a context manager or
    close() it; the engine closes readers still open when it is destroyed."""

    def __init__(self, handle: C.c_void_p, engine: "Engine", st: Optional[_StreamTables] = None, data_cap: int = 0):
        self._h = handle
        self._engine = engine
        self._st = st
        self._data_cap = data_cap
        self.last_stream_reads = None if st is None else []
        self._cache = None

    def attach_page_cache(self, cache: Optional[PageCache]):
        """dbeel_reader_attach_page_cache: read leaf slices, windows and entries through `cache` from the next call on
        (None detaches).  Results stay exactly what they are uncached; only the reads through the callback change."""
        if not self._h:
            raise ValueError("reader is closed")
        h = cache._h if cache is not None else None
        if cache is not None and not h:
            raise ValueError("page cache is closed")
        rc = lib().dbeel_reader_attach_page_cache(self._h, h)
        if rc:
            raise DbeelError(rc, f"dbeel_reader_attach_page_cache: {lib().dbeel_last_error(self._engine._h).decode()}")
        self._cache = cache

    def get_values(self, keys: Sequence[bytes], mode: int = LOOKUP_REFERENCE, caps: Optional[Tuple[int, int]] = None,
                   fail_read_at: int = -1):
        """What get_values_stream returns for the same tables, keys and mode: (rows, data, index).  last_stream_reads lists
        this call's reads (readers of an engine's tables; None for a tree's); fail_read_at as in get_values_stream."""
        if not self._h:
            raise ValueError("reader is closed")
        blob, off = pack_keys(keys)
        if self._st is not None:
            self._st.fail_read_at = fail_read_at

        def call(out, res):
            return lib().dbeel_reader_get_values(self._h, blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys),
                                                 mode, C.byref(out), res.ctypes.data)
        try:
            return _stream_values(call, "dbeel_reader_get_values", self._engine._h, len(keys), self._st, caps, self._data_cap)
        finally:
            if self._st is not None:
                self.last_stream_reads = self._st.last_reads

    def scan(self, ranges, kind: int = SCAN_KEY, write=None, fail_read_at: int = -1):
        """dbeel_reader_scan: what LSMTree.scan_stream returns, on the reader's tables -- ([(data, index)] per range
        collected in memory, or [(data_len, index_len, items)] per range when write(dest, kind, offset, src_address,
        length) -> 0 or an error code receives the pieces), and (table, reason, record) of the stop, table = a position
        in the reader's tables.  Key ranges read only the records from each bound's seek on; hash ranges read every
        table.  last_stream_reads and fail_read_at as in get_values."""
        rptr, _keep = pack_ranges(kind, ranges)
        return self._ranges_call("dbeel_reader_scan", lambda cb, res, stop: lib().dbeel_reader_scan(
            self._h, kind, rptr, len(ranges), cb, None, res, stop), len(ranges), write, fail_read_at)

    def get_range(self, ranges, keep_tombstones: bool = False, write=None, fail_read_at: int = -1):
        """dbeel_reader_get_range: per key range, the newest version of every key in it (get_entry's answer), in key
        order, tombstones dropped unless keep_tombstones -- one SSTable (data, index) per range, or (data_len, index_len,
        items) per range when write(dest, kind, offset, src_address, length) receives the pieces; and the stop, which is
        Reader.scan's for the same ranges (results are then empty).  last_stream_reads and fail_read_at as in get_values."""
        rptr, _keep = pack_ranges(SCAN_KEY, ranges)
        flags = RANGE_KEEP_TOMBSTONES if keep_tombstones else 0
        return self._ranges_call("dbeel_reader_get_range", lambda cb, res, stop: lib().dbeel_reader_get_range(
            self._h, rptr, len(ranges), flags, cb, None, res, stop), len(ranges), write, fail_read_at, void_on_stop=True)

    def get_ranges(self, ranges, limits, keep_tombstones: bool = False, caps: Optional[Tuple[int, int]] = None,
                   fail_read_at: int = -1, reverse: bool = False):
        """dbeel_reader_get_ranges: per key range, its first `limit` entries as get_range returns them, for many ranges in
        one call; with reverse, dbeel_reader_get_ranges_reverse: its last `limit` entries, in descending key order.
        limits is an int (every range) or one per range.  Returns (rows, data, index): rows a RANGE_ROW_DTYPE array
        (first, count, flags, table, reason, record), the entries of every range packed in range order.  Capacity is
        retried once with the sizes the engine reports unless caps is given; last_stream_reads and fail_read_at as in
        get_values."""
        if not self._h:
            raise ValueError("reader is closed")
        n = len(ranges)
        lim = np.ascontiguousarray(np.full(n, limits, np.uint32) if isinstance(limits, (int, np.integer))
                                   else np.array([int(x) for x in limits], np.uint32))
        if lim.size != n:
            raise ValueError("one limit per range")
        rptr, _keep = pack_ranges(SCAN_KEY, ranges)
        flags = RANGE_KEEP_TOMBSTONES if keep_tombstones else 0
        if self._st is not None:
            self._st.fail_read_at = fail_read_at
        rows = np.zeros(max(1, n), RANGE_ROW_DTYPE)
        name = "dbeel_reader_get_ranges_reverse" if reverse else "dbeel_reader_get_ranges"
        fn = getattr(lib(), name)
        dc0 = sum(d for d, _ in self._st.sizes) if self._st is not None else self._data_cap
        dc, ic = caps if caps is not None else (min(dc0, 64 << 20), min(16 * int(lim.sum()), 16 << 20))
        try:
            for attempt in range(2):
                od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
                out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
                if self._st is not None:
                    self._st.log.clear()
                rc = fn(self._h, rptr, n, lim.ctypes.data, flags, C.byref(out), rows.ctypes.data)
                if self._st is not None:
                    self._st.last_reads = list(self._st.log)
                if rc == 0:
                    return rows[:n], od[:out.data_len], oi[:out.index_len]
                err = DbeelError(rc, f"{name}: {lib().dbeel_last_error(self._engine._h).decode()}")
                if rc == ERR_CAPACITY:
                    err.needed = (int(out.data_len), int(out.index_len))
                    err.rows = rows[:n].copy()
                if caps is not None or attempt or rc != ERR_CAPACITY:
                    raise err
                dc, ic = err.needed
        finally:
            if self._st is not None:
                self._st.fail_read_at = -1
                self.last_stream_reads = self._st.last_reads

    def _ranges_call(self, name: str, call, n: int, write, fail_read_at: int, void_on_stop: bool = False):
        import threading
        if not self._h:
            raise ValueError("reader is closed")
        files = [{1: bytearray(), 2: bytearray()} for _ in range(n)]
        mu = threading.Lock()

        def collect(dest, kind_, off, src, size):
            with mu:
                f = files[dest][kind_]
                if len(f) < off + size:
                    f.extend(bytes(off + size - len(f)))
                f[off:off + size] = C.string_at(src, size)
            return 0

        cb = SCAN_WRITE_FN(lambda _ctx, dest, kind_, off, src, size: (write or collect)(dest, kind_, off, src, size))
        res = (JobResult * max(1, n))()
        stop = ScanStop()
        if self._st is not None:
            self._st.fail_read_at = fail_read_at
            self._st.log.clear()
        try:
            rc = call(cb, res, C.byref(stop))
        finally:
            if self._st is not None:
                self._st.last_reads = list(self._st.log)
                self.last_stream_reads = self._st.last_reads
                self._st.fail_read_at = -1
        if rc:
            raise DbeelError(rc, f"{name}: {lib().dbeel_last_error(self._engine._h).decode()}")
        if write is not None:
            return [(int(r.data_len), int(r.index_len), int(r.items_written)) for r in res[:n]], stop.as_tuple()
        if void_on_stop and stop.table >= 0:  # the bytes written before the stop are void
            files = [{1: b"", 2: b""} for _ in range(n)]
        return ([(np.frombuffer(bytes(f[1]), np.uint8).copy(), np.frombuffer(bytes(f[2]), np.uint8).copy()) for f in files],
                stop.as_tuple())

    def close(self):
        if self._h and self._engine._h:  # an engine already destroyed has closed its readers
            lib().dbeel_reader_close(self._h)
        self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One compaction engine bound to one GPU (dbeel_engine_create)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        rc = lib().dbeel_engine_create(device, C.byref(self._h))
        if rc:
            raise DbeelError(rc, f"dbeel_engine_create({device}): {lib().dbeel_strerror(rc).decode()}")
        self.device = device

    def close(self):
        if self._h:
            lib().dbeel_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc:
            raise DbeelError(rc, f"{what}: {lib().dbeel_last_error(self._h).decode()}")

    def stream_ptr(self) -> int:
        """The engine's cudaStream_t as an integer (torch.cuda.ExternalStream(ptr) wraps it)."""
        return int(lib().dbeel_engine_stream(self._h) or 0)

    def stats(self) -> dict:
        s = Stats()
        lib().dbeel_last_stats(self._h, C.byref(s))
        return s.as_dict()

    # ---- host buffers (numpy) -------------------------------------------------------
    def compact(self, runs: Sequence[Tuple[object, object]], keep_tombstones: bool = False,
                bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE, seed: Optional[bytes] = None,
                bloom_fp: float = DEFAULT_BLOOM_FP, flags: int = 0, out_buffers=None):
        """dbeel_compact: returns (data, index, bloom|None, items_written) as numpy uint8 arrays."""
        keep = [(_u8(d), _u8(i)) for d, i in runs]
        arr = (Run * max(1, len(keep)))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Run(d.ctypes.data, d.size, i.ctypes.data, i.size)
        opts = make_opts(keep_tombstones, bloom_min_size, bloom_fp, seed, flags)
        dc, ic, bc = compact_bound([(d.size, i.size) for d, i in keep], opts)
        if out_buffers is None:
            od, oi, ob = (np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8), np.empty(max(1, bc), np.uint8))
        else:
            od, oi, ob = out_buffers
        out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, ob.ctypes.data if bc else None, bc, 0, 0)
        self._check(lib().dbeel_compact(self._h, arr, len(keep), C.byref(opts), C.byref(out)), "dbeel_compact")
        bloom = ob[:out.bloom_len] if out.bloom_len else None
        return od[:out.data_len], oi[:out.index_len], bloom, int(out.items_written)

    def compact_stream(self, runs: Sequence[Tuple[object, object]], keep_tombstones: bool = False,
                       bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE, seed: Optional[bytes] = None, flags: int = 0,
                       fail_read_at: int = -1, fail_write_at: int = -1):
        """dbeel_compact_stream with in-memory "files": the engine pulls the runs through a read callback and pushes the
        output through a write callback (both called from several engine threads).  Returns (data, index, bloom|None,
        items_written) like compact(); fail_*_at = n makes the n-th callback call return error code 4242 (tests)."""
        keep = [(_u8(d), _u8(i)) for d, i in runs]
        arr = (Run * max(1, len(keep)))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Run(None, d.size, None, i.size)
        opts = make_opts(keep_tombstones, bloom_min_size, DEFAULT_BLOOM_FP, seed, flags)
        dc, ic, bc = compact_bound([(d.size, i.size) for d, i in keep], opts)
        outs = {1: np.zeros(max(1, dc), np.uint8), 2: np.zeros(max(1, ic), np.uint8), 3: np.zeros(max(1, bc), np.uint8)}
        calls = {"r": 0, "w": 0}
        import threading
        mu = threading.Lock()

        def rd(_ctx, run, kind, off, n, dst):
            with mu:
                k = calls["r"]
                calls["r"] += 1
            if k == fail_read_at:
                return 4242
            src = keep[run][0] if kind == 1 else keep[run][1]
            if off + n > src.size:
                return 4243
            C.memmove(dst, src.ctypes.data + off, n)
            return 0

        def wr(_ctx, kind, off, src, n):
            with mu:
                k = calls["w"]
                calls["w"] += 1
            if k == fail_write_at:
                return 4242
            dst = outs.get(kind)
            if dst is None or off + n > dst.size:
                return 4244
            C.memmove(dst.ctypes.data + off, src, n)
            return 0

        io = StreamIO(STREAM_READ_FN(rd), STREAM_WRITE_FN(wr), None)
        out = Out(None, 0, 0, None, 0, 0, None, 0, 0, 0)
        self._check(lib().dbeel_compact_stream(self._h, arr, len(keep), C.byref(opts), C.byref(io), C.byref(out)), "dbeel_compact_stream")
        bloom = outs[3][:out.bloom_len] if out.bloom_len else None
        return outs[1][:out.data_len], outs[2][:out.index_len], bloom, int(out.items_written)

    def compact_async(self, runs: Sequence[Tuple[object, object]], keep_tombstones: bool = False,
                      bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE, seed: Optional[bytes] = None):
        """dbeel_compact_submit: returns a callable `reap(block)` -> None while running, else the result tuple."""
        keep = [(_u8(d), _u8(i)) for d, i in runs]
        arr = (Run * max(1, len(keep)))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Run(d.ctypes.data, d.size, i.ctypes.data, i.size)
        opts = make_opts(keep_tombstones, bloom_min_size, DEFAULT_BLOOM_FP, seed, 0)
        dc, ic, bc = compact_bound([(d.size, i.size) for d, i in keep], opts)
        od, oi, ob = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8), np.empty(max(1, bc), np.uint8)
        out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, ob.ctypes.data if bc else None, bc, 0, 0)
        self._check(lib().dbeel_compact_submit(self._h, arr, len(keep), C.byref(opts), C.byref(out)), "dbeel_compact_submit")
        alive = (keep, arr, opts, out, od, oi, ob)  # everything the job points at stays referenced by the closure

        def reap(block: bool = False):
            if block:
                rc = lib().dbeel_wait(self._h)
            else:
                st = C.c_int(0)
                if not lib().dbeel_poll(self._h, C.byref(st)):
                    return None
                rc = st.value
            self._check(rc, "dbeel_compact (async)")
            o = alive[3]
            bloom = ob[:o.bloom_len] if o.bloom_len else None
            return od[:o.data_len], oi[:o.index_len], bloom, int(o.items_written)

        return reap

    def flush(self, batch: Tuple[object, object]):
        """dbeel_flush: returns (data, index, items_written)."""
        d, i = _u8(batch[0]), _u8(batch[1])
        run = Run(d.ctypes.data, d.size, i.ctypes.data, i.size)
        od, oi = np.empty(max(1, d.size), np.uint8), np.empty(max(1, i.size), np.uint8)
        out = Out(od.ctypes.data, d.size, 0, oi.ctypes.data, i.size // 16 * 16, 0, None, 0, 0, 0)
        self._check(lib().dbeel_flush(self._h, C.byref(run), C.byref(out)), "dbeel_flush")
        return od[:out.data_len], oi[:out.index_len], int(out.items_written)

    def flush_many(self, batches: Sequence[Tuple[object, object]]):
        """dbeel_flush_many: one launch sequence for all memtables; returns [(data, index, items)] per batch."""
        keep = [(_u8(d), _u8(i)) for d, i in batches]
        n = len(keep)
        arr = (Run * max(1, n))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Run(d.ctypes.data, d.size, i.ctypes.data, i.size)
        dc = sum(d.size for d, _ in keep)
        ic = sum(i.size // 16 * 16 for _, i in keep)
        od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
        out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
        table = (FlushTable * max(1, n))()
        self._check(lib().dbeel_flush_many(self._h, arr, n, C.byref(out), table), "dbeel_flush_many")
        return [(od[t.data_off:t.data_off + t.data_len], oi[t.index_off:t.index_off + t.index_len], int(t.items))
                for t in table[:n]]

    def flush_many_device(self, batches: Sequence[Tuple[int, int, int, int]], out_ptrs: Tuple[int, int, int, int]):
        """batches: (data_ptr, data_len, index_ptr, index_len) device pointers; out_ptrs: (data_ptr, data_cap,
        index_ptr, index_cap).  Returns (data_len, index_len, items, table rows as dicts)."""
        n = len(batches)
        arr = (Run * max(1, n))()
        for j, b in enumerate(batches):
            arr[j] = Run(*b)
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        table = (FlushTable * max(1, n))()
        self._check(lib().dbeel_flush_many_device(self._h, arr, n, C.byref(out), table), "dbeel_flush_many_device")
        rows = [{k: int(getattr(t, k)) for k, _ in FlushTable._fields_} for t in table[:n]]
        return int(out.data_len), int(out.index_len), int(out.items_written), rows

    def flush_many_sparse_device(self, batches: Sequence[Tuple[int, int, int, int]], payload_bound: int,
                                 out_ptrs: Tuple[int, int, int, int]):
        """dbeel_flush_many_sparse_device: like flush_many_device, for slices of a routed stream (shared .data)."""
        n = len(batches)
        arr = (Run * max(1, n))()
        for j, b in enumerate(batches):
            arr[j] = Run(*b)
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        table = (FlushTable * max(1, n))()
        self._check(lib().dbeel_flush_many_sparse_device(self._h, arr, n, payload_bound, C.byref(out), table),
                    "dbeel_flush_many_sparse_device")
        rows = [{k: int(getattr(t, k)) for k, _ in FlushTable._fields_} for t in table[:n]]
        return int(out.data_len), int(out.index_len), int(out.items_written), rows

    def memtable_cuts_device(self, key_hash64_ptr: int, stream_starts, capacity: int = DEFAULT_TREE_CAPACITY):
        """dbeel_memtable_cuts_device: per stream the list of cumulative arrival counts at which a full memtable ends."""
        starts = np.ascontiguousarray(stream_starts, np.uint64)
        n = starts.size - 1
        cap = int((starts[-1] - starts[0]) // max(1, capacity)) + n + 1
        cuts = np.zeros(cap, np.uint32)
        cs = np.zeros(n + 1, np.uint32)
        self._check(lib().dbeel_memtable_cuts_device(self._h, key_hash64_ptr or None, starts.ctypes.data, n, capacity, cuts.ctypes.data,
                                                     cs.ctypes.data, cap), "dbeel_memtable_cuts_device")
        return [cuts[cs[s]:cs[s + 1]].astype(np.int64) for s in range(n)]

    def route_device(self, batch: Tuple[int, int, int, int], ring: np.ndarray, out_index_ptr: int, out_index_cap: int,
                     shard_of_ptr: int = 0, out_hash64_ptr: int = 0):
        """dbeel_route_device: batch = (data_ptr, data_len, index_ptr, index_len) device pointers.  Returns (counts,
        payload bytes) per ring position as numpy u64 arrays."""
        ring = np.ascontiguousarray(ring, np.uint32)
        run = Run(*batch)
        counts = np.zeros(ring.size, np.uint64)
        nbytes = np.zeros(ring.size, np.uint64)
        self._check(lib().dbeel_route_device(self._h, C.byref(run), ring.ctypes.data, ring.size, out_index_ptr, out_index_cap,
                                             shard_of_ptr or None, out_hash64_ptr or None, counts.ctypes.data, nbytes.ctypes.data),
                    "dbeel_route_device")
        return counts, nbytes

    # ---- N1: many compactions per launch sequence -------------------------------------------
    @staticmethod
    def _jobs_array(jobs_ptrs, seeds):
        """jobs_ptrs: per job (list of (data_ptr, data_len, index_ptr, index_len), keep_tombstones)."""
        n = len(jobs_ptrs)
        arr = (Job * max(1, n))()
        keep = []
        for j, (runs, keep_t) in enumerate(jobs_ptrs):
            ra = (Run * max(1, len(runs)))()
            for k, r in enumerate(runs):
                ra[k] = Run(*r)
            keep.append(ra)
            arr[j] = Job(ra, len(runs), int(keep_t), seeds[j] if seeds is not None else None)
        return arr, keep

    def compact_many(self, jobs: Sequence[Tuple[Sequence[Tuple[object, object]], bool]],
                     bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE, seeds: Optional[Sequence[Optional[bytes]]] = None,
                     fp: float = DEFAULT_BLOOM_FP):
        """dbeel_compact_many over host buffers.  jobs: (runs, keep_tombstones) per compaction.  Returns one
        (data, index, bloom | None, items_written) per job, each what dbeel_compact would return for it."""
        hold = [[(_u8(d), _u8(i)) for d, i in runs] for runs, _ in jobs]
        ptrs = [([(d.ctypes.data, d.size, i.ctypes.data, i.size) for d, i in h], k) for h, (_, k) in zip(hold, jobs)]
        arr, keep = self._jobs_array(ptrs, seeds)
        n = len(jobs)
        dc, ic, bc = C.c_uint64(), C.c_uint64(), C.c_uint64()
        rc = lib().dbeel_compact_many_bound(arr, n, bloom_min_size, fp, C.byref(dc), C.byref(ic), C.byref(bc))
        if rc:
            raise DbeelError(rc, "dbeel_compact_many_bound")
        od, oi, ob = (np.empty(max(1, c.value), np.uint8) for c in (dc, ic, bc))
        out = Out(od.ctypes.data, dc.value, 0, oi.ctypes.data, ic.value, 0, ob.ctypes.data, bc.value, 0, 0)
        res = (JobResult * max(1, n))()
        self._check(lib().dbeel_compact_many(self._h, arr, n, bloom_min_size, fp, C.byref(out), res), "dbeel_compact_many")
        return [(od[r.data_off:r.data_off + r.data_len], oi[r.index_off:r.index_off + r.index_len],
                 ob[r.bloom_off:r.bloom_off + r.bloom_len] if r.bloom_len else None, int(r.items_written)) for r in res[:n]]

    def compact_many_device(self, jobs_ptrs, out_ptrs: Tuple[int, int, int, int, int, int],
                            bloom_min_size: int = DEFAULT_BLOOM_MIN_SIZE, seeds=None, fp: float = DEFAULT_BLOOM_FP):
        """Device pointers everywhere.  Returns the JobResult rows as dicts."""
        arr, keep = self._jobs_array(jobs_ptrs, seeds)
        n = len(jobs_ptrs)
        dp, dc, ip, ic, bp, bc = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, bp if bc else None, bc, 0, 0)
        res = (JobResult * max(1, n))()
        self._check(lib().dbeel_compact_many_device(self._h, arr, n, bloom_min_size, fp, C.byref(out), res),
                    "dbeel_compact_many_device")
        return [{k: int(getattr(r, k)) for k, _ in JobResult._fields_} for r in res[:n]]

    # ---- N4: write-ahead-log replay + flush ------------------------------------------------
    def wal_flush(self, wal, capacity: int = DEFAULT_TREE_CAPACITY):
        """dbeel_wal_flush over a host buffer holding a `.memtable` file: returns (data, index, items_written)."""
        w = _u8(wal)
        od = np.empty(max(1, w.size), np.uint8)
        oi = np.empty(max(16, (w.size + 4095) // 4096 * 16), np.uint8)
        out = Out(od.ctypes.data, od.size, 0, oi.ctypes.data, oi.size, 0, None, 0, 0, 0)
        self._check(lib().dbeel_wal_flush(self._h, w.ctypes.data if w.size else None, w.size, capacity, C.byref(out)),
                    "dbeel_wal_flush")
        return od[:out.data_len], oi[:out.index_len], int(out.items_written)

    def wal_flush_device(self, wal_ptr: int, wal_len: int, out_ptrs: Tuple[int, int, int, int],
                         capacity: int = DEFAULT_TREE_CAPACITY):
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        self._check(lib().dbeel_wal_flush_device(self._h, wal_ptr, wal_len, capacity, C.byref(out)), "dbeel_wal_flush_device")
        return int(out.data_len), int(out.index_len), int(out.items_written)

    # ---- N2: batched point lookups -------------------------------------------------------
    def get_many(self, tables: Sequence[Tuple[object, object, object]], keys: Sequence[bytes],
                 mode: int = LOOKUP_REFERENCE) -> np.ndarray:
        """dbeel_get_many over host buffers.  tables: (data, index, bloom | None) oldest first, like
        LSMTree.sstables.  Returns a structured array (table, bloom_rejects, record), one row per key."""
        keep = [(_u8(d), _u8(i), _u8(b) if b is not None and len(b) else None) for d, i, b in tables]
        arr = (Table * max(1, len(keep)))()
        for j, (d, i, b) in enumerate(keep):
            arr[j] = Table(d.ctypes.data, d.size, i.ctypes.data, i.size, b.ctypes.data if b is not None else None,
                           b.size if b is not None else 0)
        blob, off = pack_keys(keys)
        res = np.zeros(len(keys), dtype=LOOKUP_DTYPE)
        self._check(lib().dbeel_get_many(self._h, arr, len(keep), blob.ctypes.data if blob.size else None,
                                         off.ctypes.data, len(keys), mode, res.ctypes.data), "dbeel_get_many")
        return res

    def get_many_device(self, tables: Sequence[Tuple[int, int, int, int, int, int]], keys_ptr: int, offsets_ptr: int,
                        n_keys: int, results_ptr: int, mode: int = LOOKUP_REFERENCE) -> None:
        """All pointers are device pointers; tables: (data_ptr, data_len, index_ptr, index_len, bloom_ptr, bloom_len)."""
        arr = (Table * max(1, len(tables)))()
        for j, t in enumerate(tables):
            arr[j] = Table(t[0], t[1], t[2], t[3], t[4] if t[5] else None, t[5])
        self._check(lib().dbeel_get_many_device(self._h, arr, len(tables), keys_ptr, offsets_ptr, n_keys, mode,
                                                results_ptr), "dbeel_get_many_device")

    def _get_values_call(self, fn, name: str, arr, n_tables: int, keys_ptr, offsets_ptr, n_keys: int, mode: int, out: Out,
                         results_ptr):
        rc = fn(self._h, arr, n_tables, keys_ptr, offsets_ptr, n_keys, mode, C.byref(out), results_ptr)
        if rc:
            err = DbeelError(rc, f"{name}: {lib().dbeel_last_error(self._h).decode()}")
            if rc == ERR_CAPACITY:
                err.needed = (int(out.data_len), int(out.index_len))
            raise err

    def get_values(self, tables: Sequence[Tuple[object, object, object]], keys: Sequence[bytes], mode: int = LOOKUP_REFERENCE,
                   caps: Optional[Tuple[int, int]] = None):
        """dbeel_get_values over host buffers: get_many's rows plus the entry of every answered row (table >= 0, no
        LOOKUP_BAD_ENTRY), in query order, as an arrival batch.  Returns (rows, data, index); row i's entry is entry number
        (answered rows before i).  caps = (data_cap, index_cap); by default the tables' .data sizes and 16 bytes per key,
        and one more call with the sizes the engine reports when duplicate or overlapping hits need more."""
        keep = [(_u8(d), _u8(i), _u8(b) if b is not None and len(b) else None) for d, i, b in tables]
        arr = (Table * max(1, len(keep)))()
        for j, (d, i, b) in enumerate(keep):
            arr[j] = Table(d.ctypes.data, d.size, i.ctypes.data, i.size, b.ctypes.data if b is not None else None,
                           b.size if b is not None else 0)
        blob, off = pack_keys(keys)
        res = np.zeros(len(keys), dtype=LOOKUP_DTYPE)
        dc, ic = caps if caps is not None else (sum(d.size for d, _, _ in keep), 16 * len(keys))
        for attempt in range(2):
            od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
            out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
            try:
                self._get_values_call(lib().dbeel_get_values, "dbeel_get_values", arr, len(keep),
                                      blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys), mode, out, res.ctypes.data)
                return res, od[:out.data_len], oi[:out.index_len]
            except DbeelError as ex:
                if caps is not None or attempt or ex.code != ERR_CAPACITY:
                    raise
                dc, ic = ex.needed

    def get_values_stream(self, tables: Sequence[Tuple[object, object, object]], keys: Sequence[bytes],
                          mode: int = LOOKUP_REFERENCE, read=None, fail_read_at: int = -1,
                          caps: Optional[Tuple[int, int]] = None):
        """dbeel_get_values_stream: get_values' result for tables the engine reads through a callback, only where the
        searches reach.  tables: (data, index, bloom | None) oldest first.  Without `read` the callback serves data / index
        from memory; with it, data / index may be sizes, and read(table, kind, offset, size) returns the bytes (kind 1 =
        .data, 2 = .index; called from several engine threads) or a nonzero int error code.  fail_read_at = n makes the n-th
        read return 4242 (tests).  last_stream_reads lists every (table, kind, offset, size) read.  Returns (rows, data,
        index); caps as in get_values (by default at most 64 MiB of .data, retried once with the sizes needed)."""
        st = _StreamTables(tables, read)
        st.fail_read_at = fail_read_at
        blob, off = pack_keys(keys)

        def call(out, res):
            return lib().dbeel_get_values_stream(self._h, st.arr, len(st.keep), blob.ctypes.data if blob.size else None,
                                                 off.ctypes.data, len(keys), mode, C.byref(st.io), C.byref(out), res.ctypes.data)
        try:
            return _stream_values(call, "dbeel_get_values_stream", self._h, len(keys), st, caps)
        finally:
            self.last_stream_reads = st.last_reads

    def open_reader(self, tables: Sequence[Tuple[object, object, object]], read=None, fence_bytes: int = 0) -> "Reader":
        """dbeel_reader_open: a Reader that answers get_values_stream's batches on these tables, with every .bloom on the
        device from now on and each table's fences kept there after the first batch in a mode reaches it.  tables / read
        as in get_values_stream; fence_bytes = device bytes for fences (0 = DEFAULT_READER_FENCE_BYTES)."""
        st = _StreamTables(tables, read)
        h = C.c_void_p()
        self._check(lib().dbeel_reader_open(self._h, st.arr, len(st.keep), C.byref(st.io), fence_bytes, C.byref(h)),
                    "dbeel_reader_open")
        return Reader(h, self, st)

    def readers_get_values(self, batches, caps: Optional[Tuple[int, int]] = None, fail_read_at=None):
        """dbeel_readers_get_values: the batches [(reader, keys, mode), ...] of many readers in one call.  Returns
        [(rows, data, index)] per batch, each what reader.get_values(keys, mode) returns alone (index offsets into its own
        data).  caps = (data_cap, index_cap) for the whole call, by default retried once with the sizes needed as
        Reader.get_values does.  Each reader's last_stream_reads = its reads in this call; fail_read_at = {reader: n} makes
        the n-th read of that reader's callback in the call return 4242."""
        fail_read_at = fail_read_at or {}
        arr = (ReaderBatch * max(1, len(batches)))()
        keep, counts, readers = [], [], []
        for j, (r, keys, mode) in enumerate(batches):
            if not r._h:
                raise ValueError("reader is closed")
            blob, off = pack_keys(list(keys))
            keep.append((blob, off))
            counts.append(len(keys))
            arr[j] = ReaderBatch(r._h, blob.ctypes.data if blob.size else None, off.ctypes.data, len(keys), mode, 0)
            if all(r is not x for x in readers):
                readers.append(r)
        sts = [r._st for r in readers if r._st is not None]
        for r in readers:
            if r._st is not None:
                r._st.fail_read_at = fail_read_at.get(r, -1)
        n = sum(counts)
        rows = np.zeros(max(1, n), dtype=LOOKUP_DTYPE)
        dc0 = sum(sum(d for d, _ in r._st.sizes) if r._st is not None else r._data_cap for r in readers)
        dc, ic = caps if caps is not None else (min(dc0, 64 << 20), 16 * n)
        try:
            for attempt in range(2):
                od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
                out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
                for st in sts:
                    st.log.clear()
                rc = lib().dbeel_readers_get_values(self._h, arr, len(batches), C.byref(out), rows.ctypes.data)
                for st in sts:
                    st.last_reads = list(st.log)
                if rc == 0:
                    break
                err = DbeelError(rc, f"dbeel_readers_get_values: {lib().dbeel_last_error(self._h).decode()}")
                if rc == ERR_CAPACITY:
                    err.needed = (int(out.data_len), int(out.index_len))
                    err.rows = rows[:n].copy()
                if caps is not None or attempt or rc != ERR_CAPACITY:
                    raise err
                dc, ic = err.needed
        finally:
            for r in readers:
                if r._st is not None:
                    r._st.fail_read_at = -1
                    r.last_stream_reads = r._st.last_reads
        # split the packed output: batch b's answered rows are its entries, in row order
        data, index = od[:out.data_len], oi[:out.index_len]
        rows = rows[:n]
        answered = (rows["table"] >= 0) & ((rows["bloom_rejects"] & LOOKUP_BAD_ENTRY) == 0)
        res, q0, item0 = [], 0, 0
        for c in counts:
            items = int(answered[q0:q0 + c].sum())
            ix = index[16 * item0:16 * (item0 + items)].copy()
            offs = ix.view("<u8")[0::2] if items else np.zeros(0, np.uint64)
            d0 = int(offs[0]) if items else 0
            d1 = int(offs[-1] + ix.view("<u4")[-1]) if items else 0
            if items:
                offs -= np.uint64(d0)
            res.append((rows[q0:q0 + c].copy(), data[d0:d1].copy(), ix))
            q0, item0 = q0 + c, item0 + items
        return res

    def readers_get_ranges(self, batches, caps: Optional[Tuple[int, int]] = None, fail_read_at=None):
        """dbeel_readers_get_ranges: the limited range reads [(reader, ranges, limits, reverse, keep_tombstones), ...] of
        many readers in one call; limits is an int (every range) or one per range.  Returns [(rows, data, index)] per batch,
        each what reader.get_ranges(ranges, limits, keep_tombstones, reverse=reverse) returns alone (first and the index
        offsets rebased to the batch's own output).  caps = (data_cap, index_cap) for the whole call, by default retried
        once with the sizes needed.  Each reader's last_stream_reads = its reads in this call; fail_read_at = {reader: n}
        makes the n-th read of that reader's callback in the call return 4242."""
        fail_read_at = fail_read_at or {}
        arr = (RangeBatch * max(1, len(batches)))()
        keep, counts, readers, total = [], [], [], 0
        for j, (r, ranges, limits, reverse, keep_tombstones) in enumerate(batches):
            if not r._h:
                raise ValueError("reader is closed")
            n = len(ranges)
            lim = np.ascontiguousarray(np.full(n, limits, np.uint32) if isinstance(limits, (int, np.integer))
                                       else np.array([int(x) for x in limits], np.uint32))
            if lim.size != n:
                raise ValueError("one limit per range")
            blob, off = pack_keys([bytes(k) for pair in ranges for k in pair])
            keep.append((blob, off, lim))
            counts.append(n)
            total += int(lim.sum())
            arr[j] = RangeBatch(r._h, KeyRanges(blob.ctypes.data if blob.size else None, off.ctypes.data),
                                lim.ctypes.data if n else None, n, RANGE_KEEP_TOMBSTONES if keep_tombstones else 0,
                                1 if reverse else 0, 0)
            if all(r is not x for x in readers):
                readers.append(r)
        sts = [r._st for r in readers if r._st is not None]
        for r in readers:
            if r._st is not None:
                r._st.fail_read_at = fail_read_at.get(r, -1)
        n = sum(counts)
        rows = np.zeros(max(1, n), RANGE_ROW_DTYPE)
        dc0 = sum(sum(d for d, _ in r._st.sizes) if r._st is not None else r._data_cap for r in readers)
        dc, ic = caps if caps is not None else (min(dc0, 64 << 20), min(16 * total, 16 << 20))
        try:
            for attempt in range(2):
                od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(1, ic), np.uint8)
                out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
                for st in sts:
                    st.log.clear()
                rc = lib().dbeel_readers_get_ranges(self._h, arr, len(batches), C.byref(out), rows.ctypes.data)
                for st in sts:
                    st.last_reads = list(st.log)
                if rc == 0:
                    break
                err = DbeelError(rc, f"dbeel_readers_get_ranges: {lib().dbeel_last_error(self._h).decode()}")
                if rc == ERR_CAPACITY:
                    err.needed = (int(out.data_len), int(out.index_len))
                    err.rows = rows[:n].copy()
                if caps is not None or attempt or rc != ERR_CAPACITY:
                    raise err
                dc, ic = err.needed
        finally:
            for r in readers:
                if r._st is not None:
                    r._st.fail_read_at = -1
                    r.last_stream_reads = r._st.last_reads
        # split the packed output: batch b's rows hold its entries [first, first + count), in row order
        data, index = od[:out.data_len], oi[:out.index_len]
        rows = rows[:n]
        res, q0, item0 = [], 0, 0
        for c in counts:
            rb = rows[q0:q0 + c].copy()
            items = int(rb["count"].sum())
            rb["first"] -= np.uint64(item0)
            ix = index[16 * item0:16 * (item0 + items)].copy()
            offs = ix.view("<u8")[0::2] if items else np.zeros(0, np.uint64)
            d0 = int(offs[0]) if items else 0
            d1 = int(offs[-1] + ix.view("<u4")[-1]) if items else 0
            if items:
                offs -= np.uint64(d0)
            res.append((rb, data[d0:d1].copy(), ix))
            q0, item0 = q0 + c, item0 + items
        return res

    def open_page_cache(self, nbytes: int) -> PageCache:
        """dbeel_page_cache_create: a PageCache of nbytes // 4096 page slots in one device allocation made now."""
        h = C.c_void_p()
        self._check(lib().dbeel_page_cache_create(self._h, nbytes, C.byref(h)), "dbeel_page_cache_create")
        return PageCache(h, self)

    def get_values_device(self, tables: Sequence[Tuple[int, int, int, int, int, int]], keys_ptr: int, offsets_ptr: int,
                          n_keys: int, results_ptr: int, out_ptrs: Tuple[int, int, int, int],
                          mode: int = LOOKUP_REFERENCE) -> Tuple[int, int, int]:
        """dbeel_get_values_device: every pointer is a device pointer; tables as in get_many_device, out_ptrs = (data_ptr,
        data_cap, index_ptr, index_cap), 16-byte aligned.  Returns (data_len, index_len, items); on ERR_CAPACITY the
        DbeelError carries .needed = (data_len, index_len)."""
        arr = (Table * max(1, len(tables)))()
        for j, t in enumerate(tables):
            arr[j] = Table(t[0], t[1], t[2], t[3], t[4] if t[5] else None, t[5])
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        self._get_values_call(lib().dbeel_get_values_device, "dbeel_get_values_device", arr, len(tables), keys_ptr, offsets_ptr,
                              n_keys, mode, out, results_ptr)
        return int(out.data_len), int(out.index_len), int(out.items_written)

    # ---- N5: scans (LSMTree::iter_filter) ---------------------------------------------------
    def scan(self, tables: Sequence[Tuple[object, ...]], ranges, kind: int = SCAN_HASH):
        """dbeel_scan over host buffers.  tables: (data, index[, bloom]) oldest first; ranges: (start, end) u32 pairs
        (SCAN_HASH) or byte strings (SCAN_KEY).  Returns ([(data, index)] per range, (table, reason, record) of the stop)."""
        keep = [(_u8(t[0]), _u8(t[1])) for t in tables]
        arr = (Table * max(1, len(keep)))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Table(d.ctypes.data, d.size, i.ctypes.data, i.size, None, 0)
        rptr, _rkeep = pack_ranges(kind, ranges)
        # dbeel_scan_bound (the files' sizes), or more when index records share .data bytes: each record is delivered at most once
        dc = sum(max(d.size, int(i[:i.size // 16 * 16].reshape(-1, 16)[:, 12:16].copy().view("<u4").astype(np.uint64).sum()))
                 for d, i in keep)
        ic = sum(i.size for _, i in keep)
        od, oi = np.empty(max(1, dc), np.uint8), np.empty(max(16, ic), np.uint8)
        out = Out(od.ctypes.data, dc, 0, oi.ctypes.data, ic, 0, None, 0, 0, 0)
        n = len(ranges)
        res = (JobResult * max(1, n))()
        stop = ScanStop()
        self._check(lib().dbeel_scan(self._h, arr, len(keep), kind, rptr, n, C.byref(out), res, C.byref(stop)), "dbeel_scan")
        return ([(od[r.data_off:r.data_off + r.data_len], oi[r.index_off:r.index_off + r.index_len]) for r in res[:n]],
                stop.as_tuple())

    def scan_stream(self, tables: Sequence[Tuple[object, ...]], ranges, kind: int = SCAN_HASH, fail_read_at: int = -1,
                    fail_write_at: int = -1):
        """dbeel_scan_stream with in-memory "files": the engine pulls the tables through a read callback and pushes every
        destination's .data / .index through a write callback (both called from several engine threads).  Returns what
        scan() returns; fail_*_at = n makes the n-th callback call return error code 4242 (tests), and
        last_stream_calls holds the (read, write) callback calls of the call."""
        keep = [(_u8(t[0]), _u8(t[1])) for t in tables]
        arr = (Table * max(1, len(keep)))()
        for j, (d, i) in enumerate(keep):
            arr[j] = Table(None, d.size, None, i.size, None, 0)
        rptr, _rkeep = pack_ranges(kind, ranges)
        n = len(ranges)
        outs = [{1: bytearray(), 2: bytearray()} for _ in range(n)]
        calls = {"r": 0, "w": 0}
        import threading
        mu = threading.Lock()

        def rd(_ctx, table, kind_, off, size, dst):
            with mu:
                k = calls["r"]
                calls["r"] += 1
            if k == fail_read_at:
                return 4242
            src = keep[table][0] if kind_ == 1 else keep[table][1]
            if off + size > src.size:
                return 4243
            C.memmove(dst, src.ctypes.data + off, size)
            return 0

        def wr(_ctx, dest, kind_, off, src, size):
            with mu:
                k = calls["w"]
                calls["w"] += 1
                if k == fail_write_at:
                    return 4242
                if dest >= n or kind_ not in (1, 2):
                    return 4244
                f = outs[dest][kind_]
                if len(f) < off + size:
                    f.extend(bytes(off + size - len(f)))
                f[off:off + size] = C.string_at(src, size)
            return 0

        io = ScanIO(STREAM_READ_FN(rd), SCAN_WRITE_FN(wr), None)
        res = (JobResult * max(1, n))()
        stop = ScanStop()
        rc = lib().dbeel_scan_stream(self._h, arr, len(keep), kind, rptr, n, C.byref(io), res, C.byref(stop))
        self.last_stream_calls = (calls["r"], calls["w"])
        self._check(rc, "dbeel_scan_stream")
        out = []
        for d, (r, f) in enumerate(zip(res[:n], outs)):
            if (r.data_off, r.index_off, r.bloom_len, len(f[1]), len(f[2])) != (0, 0, 0, r.data_len, r.index_len):
                raise RuntimeError(f"dbeel_scan_stream: destination {d}'s files do not match its result row")
            out.append((np.frombuffer(bytes(f[1]), np.uint8), np.frombuffer(bytes(f[2]), np.uint8)))
        return out, stop.as_tuple()

    def scan_device(self, tables: Sequence[Tuple[int, int, int, int]], ranges, out_ptrs: Tuple[int, int, int, int],
                    kind: int = SCAN_HASH):
        """dbeel_scan_device: tables (data_ptr, data_len, index_ptr, index_len) and out_ptrs (data_ptr, data_cap, index_ptr,
        index_cap) in device memory.  Returns (JobResult rows as dicts, (table, reason, record) of the stop)."""
        arr = (Table * max(1, len(tables)))()
        for j, t in enumerate(tables):
            arr[j] = Table(t[0], t[1], t[2], t[3], None, 0)
        rptr, _rkeep = pack_ranges(kind, ranges)
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        n = len(ranges)
        res = (JobResult * max(1, n))()
        stop = ScanStop()
        self._check(lib().dbeel_scan_device(self._h, arr, len(tables), kind, rptr, n, C.byref(out), res, C.byref(stop)),
                    "dbeel_scan_device")
        return [{k: int(getattr(r, k)) for k, _ in JobResult._fields_} for r in res[:n]], stop.as_tuple()

    # ---- device buffers (raw pointers; torch tensors own the memory) -------------------
    def compact_device(self, runs: Sequence[Tuple[int, int, int, int]], out_ptrs: Tuple[int, int, int, int, int, int],
                       opts: Opts) -> Tuple[int, int, int, int]:
        """runs: (data_ptr, data_len, index_ptr, index_len); out_ptrs: (data_ptr, data_cap,
        index_ptr, index_cap, bloom_ptr, bloom_cap).  Returns (data_len, index_len, bloom_len, items)."""
        arr = (Run * max(1, len(runs)))()
        for j, (dp, dl, ip, il) in enumerate(runs):
            arr[j] = Run(dp, dl, ip, il)
        dp, dc, ip, ic, bp, bc = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, bp if bc else None, bc, 0, 0)
        self._check(lib().dbeel_compact_device(self._h, arr, len(runs), C.byref(opts), C.byref(out)),
                    "dbeel_compact_device")
        return int(out.data_len), int(out.index_len), int(out.bloom_len), int(out.items_written)

    def flush_device(self, batch: Tuple[int, int, int, int], out_ptrs: Tuple[int, int, int, int]):
        run = Run(*batch)
        dp, dc, ip, ic = out_ptrs
        out = Out(dp, dc, 0, ip, ic, 0, None, 0, 0, 0)
        self._check(lib().dbeel_flush_device(self._h, C.byref(run), C.byref(out)), "dbeel_flush_device")
        return int(out.data_len), int(out.index_len), int(out.items_written)


def murmur3_32(data: bytes, seed: int = 0) -> int:
    return int(lib().dbeel_murmur3_32(bytes(data), len(data), seed))


def shard_ring(n_shards: int, node: Optional[str] = None):
    """(ascending ring hashes, cpu id at each ring position) of a node's shards (shards.rs:213-214,657-670)."""
    h = np.zeros(n_shards, np.uint32)
    ids = np.zeros(n_shards, np.uint32)
    rc = lib().dbeel_shard_ring(node.encode() if node else None, n_shards, h.ctypes.data, ids.ctypes.data)
    if rc:
        raise DbeelError(rc, "dbeel_shard_ring")
    return h, ids


def ring_owner(ring: np.ndarray, key_hash: int) -> int:
    ring = np.ascontiguousarray(ring, np.uint32)
    return int(lib().dbeel_ring_owner(ring.ctypes.data, ring.size, key_hash))


def bind_to_gpu(device: int):
    """dbeel_bind_to_gpu: (numa node, cpus) the calling thread was bound to, (-1, 0) when there is no NUMA topology."""
    node, cpus = C.c_int(-1), C.c_int(0)
    rc = lib().dbeel_bind_to_gpu(device, C.byref(node), C.byref(cpus))
    if rc:
        raise DbeelError(rc, "dbeel_bind_to_gpu")
    return node.value, cpus.value
