#!/usr/bin/env python
"""Range reads across readers (dbeel_readers_get_ranges) against the same batches sent one reader after another
(dbeel_reader_get_ranges / _reverse), alternated in one process.  A node holds a tree per shard and collection, all on one
engine per GPU, and a serving loop sends each of them a page request: the next page from a cursor or the previous one.  A
short limited range read is almost all fixed cost (the bound searches, one merge round and one emission, each with its
stream synchronisations), which one call over all readers pays once instead of once per reader.
Setup: B trees (B = 1, 2, 8, 32), each a copy of readers_bench.py's tree (cfg2-shaped, four tables, on tmpfs), each with a
tree reader whose exact-mode fences are loaded.  Per reader 1 or 64 queries, each a range from a random key of the tree to
the end of the key space, limits 1, 10 and 100, batches all forward, all reverse, or mixed (odd readers reverse).  Per
setting: median wall time over rounds of the B sequential calls and of the one batched call, which go first on alternate
rounds, after a warm-up round; every batch's rows, .data and .index of the two are compared on every round.  Bytes read
and merge rounds are the engine's stats of the last round; callback reads come from an untimed pass of the same batches
through readers over the same files whose callback logs every read.  Prints the GPU name and power limit of the run.
Measured results and the card they were measured on: DESIGN.md section 7, "Range reads across readers".
Usage: tools/readers_ranges_bench.py [keys_per_run (default 25000)] [--rounds R] [--readers 1,2,8,32] [--out result.json]"""
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
from reader_bench import card, file_reader  # noqa: E402

QUERIES = (1, 64)
LIMITS = (1, 10, 100)
DIRECTIONS = ("forward", "reverse", "mixed")


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds, readers = opt("--out", None), int(opt("--rounds", "5")), opt("--readers", "1,2,8,32")
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
    root = tempfile.mkdtemp(prefix="readers_ranges_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "keys_per_run": kpr, "tables_per_tree": len(tables), "rows": []}
    trees, rds, counting, fds = [], [], [], []
    try:
        for t in range(max(n_trees)):
            d = os.path.join(root, f"tree{t}")
            os.makedirs(d)
            for k, (td, ti, tb) in enumerate(tables):
                sstable.write_run_files(d, 2 * k, (td, ti), tb)
            trees.append(se.LSMTree.open_or_create(d, eng))
            rds.append(trees[-1].open_reader())
        read, fds = file_reader(os.path.join(root, "tree0"), [i for i, _ in trees[0].sstable_indices_and_sizes()])
        counting = [eng.open_reader([(td.size, ti.size, None) for td, ti, _ in tables], read=read) for _ in range(max(n_trees))]
        print(f"{max(n_trees)} trees of {len(tables)} tables on {'tmpfs' if base else 'disk'}, "
              f"{sum(ti.size // 16 for _, ti, _ in tables)} records each", flush=True)
        whole = [(b"", b"\xff" * 32)]
        for r in rds + counting:  # a forward and a reverse read over every table load the exact-mode fences
            r.get_ranges(whole, 1)
            r.get_ranges(whole, 1, reverse=True)
        rng = np.random.default_rng(43)
        for B in n_trees:
            for nq in QUERIES:
                for limit in LIMITS:
                    for direction in DIRECTIONS:
                        rev = lambda b: direction == "reverse" or (direction == "mixed" and b % 2 == 1)
                        t_seq, t_one, parity = [], [], True
                        for rnd in range(rounds + 1):  # round 0 warms up; the two alternate
                            batches = []
                            for b in range(B):
                                starts = [all_keys[j].tobytes() for j in rng.integers(0, len(all_keys), nq)]
                                ranges = [(s, b"\xff" * 32) if not rev(b) else (b"", s) for s in starts]
                                batches.append((rds[b], ranges, limit, rev(b), False))
                            for first in ((0, 1) if rnd % 2 else (1, 0)):
                                t0 = time.perf_counter()
                                if first:
                                    seq, st_seq = [], {"input_bytes": 0, "partitions": 0}
                                    for r, ranges, lim, rv, _ in batches:
                                        seq.append(r.get_ranges(ranges, lim, reverse=rv))
                                        if rnd == rounds:
                                            st = eng.stats()
                                            st_seq = {k: st_seq[k] + st[k] for k in st_seq}
                                else:
                                    one = eng.readers_get_ranges(batches)
                                    if rnd == rounds:
                                        st_one = eng.stats()
                                if rnd:
                                    (t_seq if first else t_one).append(time.perf_counter() - t0)
                            parity = parity and all(same(a, b) for a, b in zip(seq, one))
                        # callback reads: the last round's batches again, through the logging readers
                        cb = [(counting[b], ranges, lim, rv, kt) for b, (_, ranges, lim, rv, kt) in enumerate(batches)]
                        n_seq = 0
                        for r, ranges, lim, rv, _ in cb:
                            r.get_ranges(ranges, lim, reverse=rv)
                            n_seq += len(r.last_stream_reads)
                        eng.readers_get_ranges(cb)
                        n_one = sum(len(r.last_stream_reads) for r in counting[:B])
                        row = {"readers": B, "queries": nq, "limit": limit, "direction": direction,
                               "sequential_s": float(np.median(t_seq)), "batched_s": float(np.median(t_one)),
                               "sequential_bytes": int(st_seq["input_bytes"]), "batched_bytes": int(st_one["input_bytes"]),
                               "sequential_reads": n_seq, "batched_reads": n_one,
                               "sequential_rounds": int(st_seq["partitions"]), "batched_rounds": int(st_one["partitions"]),
                               "parity": parity}
                        result["rows"].append(row)
                        print(f"{B:>3} readers x {nq:>2} queries, limit {limit:>3}, {direction:7s}: sequential "
                              f"{row['sequential_s'] * 1e3:8.3f} ms, batched {row['batched_s'] * 1e3:8.3f} ms "
                              f"({row['sequential_s'] / row['batched_s']:.2f}x) | bytes {row['sequential_bytes']} / "
                              f"{row['batched_bytes']} | reads {n_seq} / {n_one} | rounds {row['sequential_rounds']} / "
                              f"{row['batched_rounds']} | parity {parity}", flush=True)
    finally:
        for r in rds + counting:
            r.close()
        for t in trees:
            t.close()
        for fd in fds:
            for x in (fd if isinstance(fd, tuple) else (fd,)):
                os.close(x)
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
