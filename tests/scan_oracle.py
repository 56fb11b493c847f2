"""ctypes front-end of tests/scan_oracle.c: the CPU restatement of LSMTree::iter_filter's SSTable part (test
infrastructure, like oracle/).  scan_oracle.c is compiled together with oracle/dbeel_oracle.c, with the oracle's own flags
(oracle/Makefile), on first use into a per-user temporary directory keyed by the sources' contents, so the tree itself is
never written: tests and tools/scan_bench.py may run from a read-only checkout."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "scan_oracle.c")
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_DEPS = [_SRC, os.path.join(_ORACLE, "dbeel_oracle.c"), os.path.join(_ORACLE, "Makefile")]


def _oracle_cflags() -> list:
    """The oracle's own compiler flags (CFLAGS of oracle/Makefile): both libraries are built the same way."""
    for line in open(os.path.join(_ORACLE, "Makefile")):
        if line.startswith("CFLAGS"):
            return line.split("=", 1)[1].split()
    raise RuntimeError("oracle/Makefile has no CFLAGS line")

SCAN_HASH, SCAN_KEY = 0, 1
STOP_NONE, STOP_ERR, STOP_PANIC = 0, 1, 2

_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"dbeel_scan_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, f"libscan_oracle_{h}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", *_oracle_cflags(), "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_scan.restype = C.c_int
        L.orc_scan.argtypes = [C.POINTER(oracle._Run), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                               C.POINTER(oracle._Out), C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        L.orc_between_cmp.restype = C.c_int
        L.orc_between_cmp.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        _lib = L
    return _lib


def between_cmp(h: int, start: int, end: int) -> bool:
    return bool(lib().orc_between_cmp(h, start, end))


def scan(tables, ranges, kind: int = SCAN_HASH):
    """iter_filter over tables = [(data, index, ...)] oldest first.  Returns ([(data, index)] per range, (table, reason,
    record) of the first record the reference's iterator fails on, or (-1, STOP_NONE, 0))."""
    arr, keep = oracle._mk_runs([(t[0], t[1]) for t in tables])
    # every record can be delivered at most once: the sum of full_size bounds the output (records may share bytes)
    dc = sum(int(i[:i.size // 16 * 16].reshape(-1, 16)[:, 12:16].copy().view("<u4").astype(np.uint64).sum()) for _, i in keep)
    ic = sum(i.size for _, i in keep) + 16
    n = len(ranges)
    outs = (oracle._Out * max(1, n))()
    bufs = []
    for d in range(n):
        o, b = oracle._mk_out(dc, ic, 0)
        outs[d] = o
        bufs.append(b)
    if kind == SCAN_HASH:
        hr = np.array([[int(a), int(b)] for a, b in ranges], np.uint32).reshape(-1)
        blob, off = np.zeros(1, np.uint8), np.zeros(1, np.uint64)
    else:
        hr = np.zeros(1, np.uint32)
        parts = [bytes(k) for pair in ranges for k in pair]
        off = np.zeros(len(parts) + 1, np.uint64)
        off[1:] = np.cumsum([len(p) for p in parts]) if parts else []
        blob = np.frombuffer(b"".join(parts) + b"\0", np.uint8).copy()
    t, r, rec = C.c_int32(), C.c_uint32(), C.c_uint64()
    rc = lib().orc_scan(arr, len(keep), kind, hr.ctypes.data, blob.ctypes.data, off.ctypes.data, n, outs, C.byref(t), C.byref(r),
                        C.byref(rec))
    if rc:
        raise oracle.OracleError(f"orc_scan rc={rc}")
    res = [(bufs[d][0][:outs[d].data_len].copy(), bufs[d][1][:outs[d].index_len].copy()) for d in range(n)]
    return res, (int(t.value), int(r.value), int(rec.value))
