#!/usr/bin/env python
"""Batched reads from files (row N2): dbeel_tree_get_values_stream against dbeel_tree_get_values, alternated in one process,
on two trees written to tmpfs: the cfg2 compaction output as one table, and the eight input runs of cfg4_shard(0) as an
8-table tree (no filters: every query that misses searches all eight).  Batches of 10^2 .. 4*10^6 keys, half present.
Reports median wall time over rounds after a warm-up, the bytes read (.data / .index through the callback plus the .bloom
files read whole) against the tree's size, and parity of every row, .data and .index with dbeel_tree_get_values
(dbeel_get_values on the files read whole).  Then the synthetic 96 GiB table of tests/test_gpu_get_values_stream.py,
served by a Python callback: time and bytes read for 1,000 keys in both modes.
Usage: tools/get_values_stream_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
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
import torch  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi, sstable  # noqa: E402
from dbeel_b200 import storage_engine as se  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402

BATCHES = (100, 10_000, 1_000_000, 4_000_000)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds = opt("--out", None), int(opt("--rounds", "5"))
    pos = [a for a in argv if not a.startswith("--") and a not in (out_path, str(rounds))]
    kpr = int(pos[0]) if pos else 1_000_000
    cfg = W.CFG2 if kpr == 1_000_000 else W.scaled(W.CFG2, kpr)
    eng = capi.Engine(0)
    gpu, power = card()
    print(f"{gpu}, power limit {power}", flush=True)
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    result = {"gpu": gpu, "power_limit": power, "rows": []}
    gd, gi, gb, n = eng.compact(make_runs_parallel(cfg), keep_tombstones=cfg.keep_tombstones, seed=SEED32)
    shard = W.cfg4_shard(0) if kpr == 1_000_000 else W.scaled(W.cfg4_shard(0), kpr)
    trees = [("cfg2, 1 table", [(gd, gi, gb)]), ("cfg4_shard(0) runs, 8 tables", [(d, i, None) for d, i in make_runs_parallel(shard)])]
    rng = np.random.default_rng(21)
    for label, tables in trees:
        d = tempfile.mkdtemp(prefix="gvs_bench_", dir=base)
        try:
            for k, (td, ti, tb) in enumerate(tables):
                sstable.write_run_files(d, 2 * k, (td, ti), tb)
            tree_bytes = sum(td.size + ti.size + (tb.size if tb is not None else 0) for td, ti, tb in tables)
            bloom_bytes = sum(tb.size for _, _, tb in tables if tb is not None)
            n_all = sum(ti.size // 16 for _, ti, _ in tables)
            print(f"{label} on {'tmpfs' if base else 'disk'}: {n_all} records, {tree_bytes / 1e6:.0f} MB", flush=True)
            tree = se.LSMTree.open_or_create(d, eng)
            for nq in BATCHES:
                t_pick = rng.integers(0, len(tables), nq // 2)
                present = []
                for k, (td, ti, _) in enumerate(tables):
                    rec = ti.view("<u8").reshape(-1, 2)
                    offs = rec[rng.integers(0, rec.shape[0], int((t_pick == k).sum())), 0].astype(np.int64)
                    present += [r.tobytes() for r in np.stack([td[offs + 8 + b] for b in range(17)], axis=1)]  # 17-byte keys
                absent = [b"\xb0k%015d" % int(x) for x in rng.integers(20_000_000, 1 << 40, nq - nq // 2)]
                keys = present + absent
                keys = [keys[j] for j in rng.permutation(nq)]
                for mode, mname in ((capi.LOOKUP_REFERENCE, "reference"), (capi.LOOKUP_EXACT, "exact")):
                    t_s, t_w = [], []
                    for r in range(rounds + 1):  # round 0 warms up; the two entry points alternate
                        t0 = time.perf_counter()
                        rs, ds, is_ = tree.get_values_stream(keys, mode)
                        t1 = time.perf_counter()
                        read = eng.stats()["input_bytes"] + bloom_bytes
                        rw, dw, iw = tree.get_values(keys, mode)
                        t2 = time.perf_counter()
                        if r:
                            t_s.append(t1 - t0)
                            t_w.append(t2 - t1)
                    parity = bool(np.array_equal(rs, rw) and np.array_equal(ds, dw) and np.array_equal(is_, iw))
                    row = {"tree": label, "keys": nq, "mode": mname, "stream_s": float(np.median(t_s)), "whole_s": float(np.median(t_w)),
                           "bytes_read": int(read), "tree_bytes": int(tree_bytes), "entries": int(is_.size // 16), "parity": parity}
                    result["rows"].append(row)
                    print(f"{nq:>8} keys {mname:9s}: stream {row['stream_s'] * 1e3:9.2f} ms, whole files {row['whole_s'] * 1e3:9.2f} ms | "
                          f"read {read / 1e6:9.2f} MB of {tree_bytes / 1e6:.0f} MB ({100 * read / tree_bytes:6.2f} %) | "
                          f"{row['entries']} entries | parity {parity}", flush=True)
            tree.close()
        finally:
            shutil.rmtree(d, ignore_errors=True)
    del trees, gd, gi, gb

    # the synthetic 96 GiB table: time and bytes read
    import test_gpu_get_values_stream as syn
    rec = sorted(int(x) for x in rng.integers(0, syn.SYN_N, 500))
    keys = [syn.syn_key(r) for r in rec] + [syn.syn_key(r) + b"x" for r in rec]
    for mode, mname in ((capi.LOOKUP_REFERENCE, "reference"), (capi.LOOKUP_EXACT, "exact")):
        t0 = time.perf_counter()
        rows, _, _ = eng.get_values_stream([(syn.SYN_N * syn.SYN_F, syn.SYN_N * 16, None)], keys, mode, read=syn.syn_read)
        dt = time.perf_counter() - t0
        read = eng.stats()["input_bytes"]
        row = {"tree": "synthetic 96 GiB table, Python read callback", "keys": len(keys), "mode": mname, "stream_s": dt,
               "bytes_read": int(read), "tree_bytes": int(syn.SYN_N * (syn.SYN_F + 16)), "entries": int((rows["table"] >= 0).sum())}
        result["rows"].append(row)
        print(f"synthetic 96 GiB table, {len(keys)} keys {mname:9s}: {dt * 1e3:9.1f} ms, read {read / 1e6:.1f} MB, "
              f"{row['entries']} found", flush=True)
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
