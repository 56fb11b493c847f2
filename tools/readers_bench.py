#!/usr/bin/env python
"""Batched reads across readers (dbeel_readers_get_values) against the same batches sent one reader after another
(dbeel_reader_get_values), alternated in one process.  A node holds a tree per shard and collection, all on one engine per
GPU, and a serving loop sends each of them a small get batch; at small batches a reader call is almost all fixed cost
(per table: a filter, a fence descent and a leaf search, each with a stream synchronise), which one call over all
readers pays once per table level instead of once per reader.
Setup: B trees (B = 1, 2, 8, 32), each a copy of reader_bench.py's cfg2-shaped tree scaled to keys_per_run keys per run
(four tables with their filters, on tmpfs), each with a tree reader.  Per reader a batch of 1, 64 or 4,096 keys, half
present (drawn uniformly over the tree's keys), both modes.  Per setting: median wall time over rounds of the B
sequential calls and of the one batched call, which go first on alternate rounds, after a batch per reader and mode that
loads all its fences and a warm-up round; rows, .data and .index of the two are compared on every round.  Prints the GPU name and power limit of the run.
Measured results and the card they were measured on: DESIGN.md section 7, "Reads across readers".
Usage: tools/readers_bench.py [keys_per_run (default 25000)] [--rounds R] [--readers 1,2,8,32] [--out result.json]"""
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi, sstable  # noqa: E402
from dbeel_b200 import storage_engine as se  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402
from reader_bench import card  # noqa: E402

BATCHES = (1, 64, 4096)
MODES = ((capi.LOOKUP_REFERENCE, "reference"), (capi.LOOKUP_EXACT, "exact"))


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds, readers = opt("--out", None), int(opt("--rounds", "15")), opt("--readers", "1,2,8,32")
    pos = [a for i, a in enumerate(argv) if not a.startswith("--") and (i == 0 or not argv[i - 1].startswith("--"))]
    kpr = int(pos[0]) if pos else 25_000
    n_trees = [int(x) for x in readers.split(",")]
    eng = capi.Engine(0)
    gpu, power = card()
    print(f"{gpu}, power limit {power}", flush=True)
    runs = make_runs_parallel(W.scaled(W.CFG2, kpr))
    tables = [eng.compact(runs[k:k + 2], keep_tombstones=True, seed=SEED32)[:3] for k in range(0, len(runs), 2)]
    del runs
    all_keys = []
    for td, ti, _ in tables:
        offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
        all_keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
    all_keys = np.concatenate(all_keys)
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    root = tempfile.mkdtemp(prefix="readers_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "keys_per_run": kpr, "tables_per_tree": len(tables), "rows": []}
    trees, rds = [], []
    try:
        for t in range(max(n_trees)):
            d = os.path.join(root, f"tree{t}")
            os.makedirs(d)
            for k, (td, ti, tb) in enumerate(tables):
                sstable.write_run_files(d, 2 * k, (td, ti), tb)
            trees.append(se.LSMTree.open_or_create(d, eng))
            rds.append(trees[-1].open_reader())
        print(f"{max(n_trees)} trees of {len(tables)} tables on {'tmpfs' if base else 'disk'}, "
              f"{sum(ti.size // 16 for _, ti, _ in tables)} records each", flush=True)
        rng = np.random.default_rng(41)
        for mode, mname in MODES:
            warm = [all_keys[j].tobytes() for j in range(0, len(all_keys), max(1, len(all_keys) // 20000))]
            for r in rds:  # a batch that reaches every table loads all of the reader's fences in the mode
                r.get_values(warm, mode)
            for B in n_trees:
                for nq in BATCHES:
                    t_seq, t_one, parity = [], [], True
                    for rnd in range(rounds + 1):  # round 0 warms up; the two alternate
                        batches = []
                        for b in range(B):
                            npres = (nq + 1) // 2
                            pick = rng.integers(0, len(all_keys), npres)
                            keys = [all_keys[j].tobytes() for j in pick] + [b"\xb0k%015d" % int(x) for x in
                                                                           rng.integers(20_000_000, 1 << 40, nq - npres)]
                            batches.append((rds[b], keys, mode))
                        for first in ((0, 1) if rnd % 2 else (1, 0)):  # which of the two goes first alternates too
                            t0 = time.perf_counter()
                            if first:
                                seq = [r.get_values(keys, m) for r, keys, m in batches]
                            else:
                                one = eng.readers_get_values(batches)
                            if rnd:
                                (t_seq if first else t_one).append(time.perf_counter() - t0)
                        parity = parity and all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and
                                                np.array_equal(a[2], b[2]) for a, b in zip(seq, one))
                    row = {"readers": B, "keys": nq, "mode": mname, "sequential_s": float(np.median(t_seq)),
                           "batched_s": float(np.median(t_one)), "parity": parity}
                    result["rows"].append(row)
                    print(f"{mname:9s} {B:>3} readers x {nq:>5} keys: sequential {row['sequential_s'] * 1e3:9.3f} ms, "
                          f"batched {row['batched_s'] * 1e3:9.3f} ms ({row['sequential_s'] / row['batched_s']:.2f}x) | "
                          f"parity {parity}", flush=True)
    finally:
        for r in rds:
            r.close()
        for t in trees:
            t.close()
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
