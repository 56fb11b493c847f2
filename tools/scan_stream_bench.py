#!/usr/bin/env python
"""Scans of a cfg2-shaped tree on FILES (tmpfs): the 8 runs of cfg4_shard(0) as 8 tables, 2.548 GB, repeated
--multiplier times for larger trees.  Three ways in, alternated and timed on the wall clock after warm-up:
  stream  dbeel_tree_scan_stream  (files pread in pieces, partitions through pinned rings, exact D2H)
  tree    dbeel_tree_scan         (every file read whole into pinned memory, then dbeel_scan)
  host    dbeel_scan              (the tables already in pinned host memory)
Cases: one eighth of the hash space (a node joins), all eight eighths (everything moves), a key range of ~10 %.
Per case and path: median / min / max seconds, GB/s of input, partitions, H2D and D2H bytes, parity of every destination
and the stop against the CPU scan oracle (larger multipliers: the oracle's output of one copy, repeated).  The card's
name and power limit are read in the same run.
Usage: tools/scan_stream_bench.py [--multiplier M ...] [--iters K] [--dir DIR] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import scan_oracle  # noqa: E402  (CPU parity only)
from bench import make_runs_parallel  # noqa: E402
from dbeel_b200 import capi, sstable, storage_engine as se  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return "unknown (no nvidia-smi)"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def expected(exp1, m):
    """The oracle's destinations for m copies of the tree: each copy's bytes again, .index offsets moved by a copy."""
    out = []
    for d, i in exp1:
        recs = np.asarray(i, np.uint8).reshape(-1, 16)
        parts_i = []
        for k in range(m):
            r = recs.copy()
            off = r[:, :8].copy().view("<u8") + np.uint64(k * d.size)
            r[:, :8] = off.view(np.uint8).reshape(-1, 8)
            parts_i.append(r.reshape(-1))
        out.append((np.concatenate([d] * m) if m > 1 else d, np.concatenate(parts_i) if m > 1 else i))
    return out


class Sink:
    """Destination files of a streamed scan in memory, filled by the write callback with memmove (no GIL held while
    copying); sized to each destination's final length, known from a first run."""

    def __init__(self, sizes):
        self.bufs = [{1: np.empty(max(1, dl), np.uint8), 2: np.empty(max(1, il), np.uint8)} for dl, il in sizes]
        self.addr = [{k: b.ctypes.data for k, b in f.items()} for f in self.bufs]
        self.cap = [{k: b.size for k, b in f.items()} for f in self.bufs]

    def write(self, dest, kind, off, src, size):
        if off + size > self.cap[dest][kind]:
            return 4244
        C.memmove(self.addr[dest][kind] + off, src, size)
        return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys-per-run", type=int, default=1_000_000)
    ap.add_argument("--multiplier", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--dir", default="/dev/shm" if os.path.isdir("/dev/shm") else None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = W.cfg4_shard(0)
    if a.keys_per_run != cfg.keys_per_run:
        cfg = W.scaled(cfg, a.keys_per_run)
    runs = make_runs_parallel(cfg)
    gpu = card()
    lo = bytes(W.format_keys(np.array([0]))[0])
    hi = bytes(W.format_keys(np.array([cfg.id_space // 10]))[0])
    cases = [("hash-1/8 (node join)", capi.SCAN_HASH, [(0, 1 << 29)]),
             ("hash-8x1/8 (all move)", capi.SCAN_HASH, [(k << 29, (k + 1) << 29 if k < 7 else 0xFFFFFFFF) for k in range(8)]),
             ("key-10%", capi.SCAN_KEY, [(lo, hi)])]
    eng = capi.Engine(0)
    st = {}
    print(f"card: {gpu}; partition budget {os.environ.get('DBEEL_PARTITION_MB', '256')} MB, ring "
          f"{os.environ.get('DBEEL_STREAM_RING', '3')}", flush=True)
    summary = {"card": gpu, "results": []}
    oracle = {}
    for name, kind, ranges in cases:
        t0 = time.perf_counter()
        oracle[name] = scan_oracle.scan(runs, ranges, kind)
        st[name] = round(time.perf_counter() - t0, 2)
    for m in a.multiplier:
        d = tempfile.mkdtemp(prefix="scan_stream_bench.", dir=a.dir)
        try:
            for k in range(m):
                for r, (dd, ii) in enumerate(runs):
                    idx = 2 * (k * len(runs) + r)
                    np.asarray(dd).tofile(os.path.join(d, sstable.file_name(idx, sstable.DATA_FILE_EXT)))
                    np.asarray(ii).tofile(os.path.join(d, sstable.file_name(idx, sstable.INDEX_FILE_EXT)))
            tree = se.LSMTree.open_or_create(d, eng)
            in_bytes = m * sum(dd.size + ii.size for dd, ii in runs)
            pinned = []
            for dd, ii in runs * m:
                pd, pi = capi.PinnedBuffer(dd.size), capi.PinnedBuffer(ii.size)
                pd.array[:] = dd
                pi.array[:] = ii
                pinned.append((pd, pi))
            host_tables = [(pd.array, pi.array) for pd, pi in pinned]
            print(f"tree x{m}: {len(runs) * m} tables, {in_bytes / 1e9:.3f} GB on {d}", flush=True)
            for name, kind, ranges in cases:
                exp, exp_stop = oracle[name][0], oracle[name][1]
                exp = expected(exp, m)
                sizes = [(e[0].size, e[1].size) for e in exp]
                sink = Sink(sizes)

                def run(path):
                    t0 = time.perf_counter()
                    if path == "stream":
                        rows, stop = tree.scan_stream(ranges, kind, write=sink.write)
                        got = [(sink.bufs[j][1][:r[0]], sink.bufs[j][2][:r[1]]) for j, r in enumerate(rows)]
                    elif path == "tree":
                        got, stop = tree.scan(ranges, kind)
                    else:
                        got, stop = eng.scan(host_tables, ranges, kind)
                    return time.perf_counter() - t0, got, stop, eng.stats()

                paths = ("stream", "tree", "host")
                times = {p: [] for p in paths}
                info = {}
                for it in range(a.iters + 1):  # the first round warms every path up and is not timed
                    for p in (paths if it % 2 == 0 else paths[::-1]):
                        sec, got, stop, stats = run(p)
                        if it == 0:
                            parity = stop == exp_stop and len(got) == len(exp) and all(
                                np.array_equal(g[0], e[0]) and np.array_equal(g[1], e[1]) for g, e in zip(got, exp))
                            out = sum(g[0].size + g[1].size for g in got)
                            info[p] = {"parity": bool(parity), "output_bytes": int(out),
                                       "partitions": int(stats["partitions"]) if p == "stream" else 1,
                                       "h2d_bytes": int(stats["input_bytes"]) if p == "stream" else in_bytes,
                                       "d2h_bytes": int(stats["output_bytes"]) if p == "stream" else None}
                        else:
                            times[p].append(sec)
                for p in paths:
                    ts = times[p]
                    med = float(np.median(ts))
                    res = {"multiplier": m, "case": name, "path": p, "s_median": round(med, 4), "s_min": round(min(ts), 4),
                           "s_max": round(max(ts), 4), "input_GBps": round(in_bytes / med / 1e9, 2), **info[p]}
                    if p == "stream":
                        res["d2h_is_selected_output"] = res["d2h_bytes"] == res["output_bytes"]
                    summary["results"].append(res)
                    print(json.dumps(res), flush=True)
            del tree
        finally:
            shutil.rmtree(d, ignore_errors=True)
    summary["parity_all"] = all(r["parity"] for r in summary["results"])
    summary["cpu_oracle_s"] = st
    print(json.dumps({"parity_all": summary["parity_all"], "card": gpu}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "scan_stream_bench.json"), "w") as f:
            json.dump(summary, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
