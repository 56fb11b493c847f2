#!/usr/bin/env python
"""Readers with and without a device page cache (dbeel_page_cache_*), alternated in one process, on the tree of
tools/reader_bench.py (the eight cfg2 runs compacted in pairs into four tables with filters, written to tmpfs).  A serving
loop sends batches of 4,096 and 65,536 keys in exact mode, half present (drawn uniformly or Zipf(1.1) over the tree's
keys), to three tree readers: one uncached, one with a 256 MiB cache and one with a 2 GiB cache.  Round 0 of each
(distribution, batch size) warms up; every reader sees the same keys in the same order.
Per reader and batch: median wall time of the synchronous call, bytes read through the callback (median), hit rate over
the timed rounds, and reads issued (counted by replaying the same key sequence through engine readers with a logging
Python callback and caches of the same sizes, untimed).  Rows, .data and .index are compared with the uncached reader's on
every batch.  Then, in a separate pass under torch.profiler, the k_page_copy time per batch of the 256 MiB reader.  Prints
the GPU name and power limit of the run.  Measured results: DESIGN.md section 7, "Readers".
Usage: tools/page_cache_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
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
import torch  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi, sstable  # noqa: E402
from dbeel_b200 import storage_engine as se  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402
from reader_bench import card, file_reader  # noqa: E402

BATCHES = (4096, 65536)
CACHES = (("none", 0), ("256MiB", 256 << 20), ("2GiB", 2 << 30))
MODE = capi.LOOKUP_EXACT


def batch_keys(rng, all_keys, dist, nq):
    npres = (nq + 1) // 2
    pick = rng.integers(0, len(all_keys), npres) if dist == "uniform" else (rng.zipf(1.1, npres) - 1) % len(all_keys)
    return [all_keys[j].tobytes() for j in pick] + [b"\xb0k%015d" % int(x) for x in rng.integers(20_000_000, 1 << 40, nq - npres)]


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds = opt("--out", None), int(opt("--rounds", "10"))
    pos = [a for a in argv if not a.startswith("--") and a not in (out_path, str(rounds))]
    kpr = int(pos[0]) if pos else 1_000_000
    cfg = W.CFG2 if kpr == 1_000_000 else W.scaled(W.CFG2, kpr)
    eng = capi.Engine(0)
    gpu, power = card()
    print(f"{gpu}, power limit {power}", flush=True)
    runs = make_runs_parallel(cfg)
    tables = [eng.compact(runs[k:k + 2], keep_tombstones=True, seed=SEED32)[:3] for k in range(0, len(runs), 2)]
    del runs
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    d = tempfile.mkdtemp(prefix="page_cache_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "rows": [], "k_page_copy": {}}
    parity = True
    try:
        for k, (td, ti, tb) in enumerate(tables):
            sstable.write_run_files(d, 2 * k, (td, ti), tb)
        tree_bytes = sum(td.size + ti.size + (tb.size if tb is not None else 0) for td, ti, tb in tables)
        print(f"cfg2 in {len(tables)} tables on {'tmpfs' if base else 'disk'}: {sum(ti.size // 16 for _, ti, _ in tables)} "
              f"records, {tree_bytes / 1e6:.0f} MB", flush=True)
        all_keys = []
        for td, ti, _ in tables:
            offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
            all_keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
        all_keys = np.concatenate(all_keys)
        tree = se.LSMTree.open_or_create(d, eng)
        caches = {name: eng.open_page_cache(size) if size else None for name, size in CACHES}
        readers = {name: tree.open_reader(page_cache=caches[name]) for name, _ in CACHES}
        for r in readers.values():
            r.get_values([all_keys[0].tobytes()], MODE)  # loads the first table's fences
        rng = np.random.default_rng(41)
        sequences = {}
        for dist in ("uniform", "zipf"):
            for nq in BATCHES:
                seq = [batch_keys(rng, all_keys, dist, nq) for _ in range(rounds + 1)]
                sequences[(dist, nq)] = seq
                t = {n: [] for n, _ in CACHES}
                b = {n: [] for n, _ in CACHES}
                s0 = {}
                for r, keys in enumerate(seq):
                    if r == 1:
                        s0 = {n: caches[n].stats() for n, _ in CACHES if caches[n]}
                    ref = None
                    for name, _ in CACHES:
                        t0 = time.perf_counter()
                        got = readers[name].get_values(keys, MODE)
                        t1 = time.perf_counter()
                        if r:
                            t[name].append(t1 - t0)
                            b[name].append(eng.stats()["input_bytes"])
                        if ref is None:
                            ref = got
                        else:
                            parity = parity and all(np.array_equal(x, y) for x, y in zip(ref, got))
                for name, _ in CACHES:
                    row = {"dist": dist, "keys": nq, "cache": name, "wall_s": float(np.median(t[name])),
                           "bytes": int(np.median(b[name])), "parity": parity}
                    if caches[name]:
                        s1 = caches[name].stats()
                        h, m = s1["hits"] - s0[name]["hits"], s1["misses"] - s0[name]["misses"]
                        row["hit_rate"] = h / max(1, h + m)
                    result["rows"].append(row)
        # reads issued: the same sequences through logging readers with caches of the same sizes
        read, fds = file_reader(d, [i for i, _ in tree.sstable_indices_and_sizes()])
        sized = [(td.size, ti.size, tb) for td, ti, tb in tables]
        for name, size in CACHES:
            c = eng.open_page_cache(size) if size else None
            with eng.open_reader(sized, read=read) as cr:
                if c:
                    cr.attach_page_cache(c)
                cr.get_values([all_keys[0].tobytes()], MODE)
                for (dist, nq), seq in sequences.items():
                    n = []
                    for r, keys in enumerate(seq):
                        cr.get_values(keys, MODE)
                        if r:
                            n.append(len(cr.last_stream_reads))
                    for row in result["rows"]:
                        if (row["dist"], row["keys"], row["cache"]) == (dist, nq, name):
                            row["reads"] = int(np.median(n))
            if c:
                c.close()
        for a, b_ in fds:
            os.close(a)
            os.close(b_)
        for row in result["rows"]:
            hr = f"{row['hit_rate'] * 100:5.1f} %" if "hit_rate" in row else "    - "
            print(f"{row['dist']:7s} {row['keys']:>6} keys, cache {row['cache']:6s}: {row['wall_s'] * 1e3:8.2f} ms | "
                  f"read {row['bytes'] / 1e6:8.2f} MB in {row['reads']:>6} reads | hit rate {hr} | parity {row['parity']}", flush=True)
        # k_page_copy under the profiler, in a pass of its own: the 256 MiB reader on the Zipf batches
        from torch.profiler import ProfilerActivity, profile
        for nq in BATCHES:
            seq = sequences[("zipf", nq)]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for keys in seq[1:]:
                    readers["256MiB"].get_values(keys, MODE)
                torch.cuda.synchronize()
            us = sum(ev.device_time_total for ev in prof.key_averages() if "k_page_copy" in ev.key)
            result["k_page_copy"][str(nq)] = us / 1e3 / len(seq[1:])
            print(f"k_page_copy, 256 MiB cache, Zipf {nq} keys: {result['k_page_copy'][str(nq)]:.3f} ms per batch", flush=True)
        for r in readers.values():
            r.close()
        for c in caches.values():
            if c:
                c.close()
        tree.close()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    result["parity"] = parity
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()
    if not parity:
        sys.exit("parity failed")


if __name__ == "__main__":
    main()
