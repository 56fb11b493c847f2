"""ctypes front-end of tests/get_values_oracle.c: the CPU restatement of get_entry's SSTable loop with the entries it
returns (test infrastructure, like oracle/).  Built like tests/scan_oracle.py: with the oracle's own flags, on first use,
into a per-user temporary directory keyed by the sources' contents, so the tree itself is never written."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle
from scan_oracle import _oracle_cflags

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "get_values_oracle.c")
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_DEPS = [_SRC, os.path.join(_ORACLE, "dbeel_oracle.c"), os.path.join(_ORACLE, "Makefile")]

BAD_ENTRY = 0x40000000

_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"dbeel_get_values_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, f"libget_values_oracle_{h}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", *_oracle_cflags(), "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_get_values.restype = C.c_int
        L.orc_get_values.argtypes = [C.POINTER(oracle._Run), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.c_uint32,
                                     C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.POINTER(oracle._Out)]
        _lib = L
    return _lib


def get_values(tables, keys_blob: np.ndarray, key_off: np.ndarray):
    """tables = [(data, index, bloom | None)] oldest first, keys packed as (bytes, n + 1 offsets).  Returns (table int32[n],
    record uint64[n], bloom_rejects uint32[n], data, index): the rows of oracle.get_many with BAD_ENTRY on hits that do
    not decode, and the answered entries in query order as EntryWriter writes them."""
    arr, keep = oracle._mk_runs([(d, i) for d, i, _ in tables])
    nt = len(tables)
    blooms = [(oracle._u8(b) if b is not None and len(b) else None) for _, _, b in tables]
    bp = (C.c_void_p * max(1, nt))(*[(b.ctypes.data if b is not None else None) for b in blooms])
    bl = (C.c_uint64 * max(1, nt))(*[(b.size if b is not None else 0) for b in blooms])
    n = key_off.size - 1
    blob = np.ascontiguousarray(keys_blob, dtype=np.uint8)
    off = np.ascontiguousarray(key_off, dtype=np.uint64)
    # an answered entry is re-encoded from what decoded, so it is as long as the key + value frames it came from
    t0, r0, _ = oracle.get_many(tables, blob, off)
    dc = 0
    for t, r in zip(t0, r0):
        if t >= 0:
            rec = keep[t][1][16 * int(r):16 * int(r) + 16]
            dc += int(rec[12:16].view("<u4")[0])
    out, (od, oi, _) = oracle._mk_out(dc, 16 * n, 0)
    t, r, j = np.empty(n, np.int32), np.empty(n, np.uint64), np.empty(n, np.uint32)
    rc = lib().orc_get_values(arr, bp, bl, nt, blob.ctypes.data if blob.size else None, off.ctypes.data, n, t.ctypes.data,
                              r.ctypes.data, j.ctypes.data, C.byref(out))
    if rc:
        raise oracle.OracleError(f"orc_get_values rc={rc}")
    return t, r, j, od[:out.data_len].copy(), oi[:out.index_len].copy()
