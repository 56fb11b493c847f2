#!/usr/bin/env python
"""Scans (row N5, LSMTree::iter_filter) of a cfg2-shaped tree resident in HBM: the 8 runs of cfg4_shard(0) as 8 tables.
Cases: one hash range of 1/8 of the space (a node joins), all eight eighths (everything moves), a key range of ~10 %.
Prints per case the CUDA-event ms per scan after warm-up, GB/s of input and output, parity of every destination and the
stop against the CPU scan oracle in the same run, the oracle's one-core rate; then, in a separate profiled pass, the
torch.profiler kernel times and the gather stage against a device-to-device copy of the same byte count.
Usage: tools/scan_bench.py [--keys-per-run N] [--iters K] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import scan_oracle  # noqa: E402  (CPU parity only)
from bench import make_runs_parallel  # noqa: E402
from dbeel_b200 import capi  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys-per-run", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = W.cfg4_shard(0)
    if a.keys_per_run != cfg.keys_per_run:
        cfg = W.scaled(cfg, a.keys_per_run)
    runs = make_runs_parallel(cfg)
    dev = torch.device("cuda:0")
    t_tabs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in runs]
    tabs = [(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_tabs]
    in_bytes = sum(d.size + i.size for d, i in runs)
    entries = sum(i.size // 16 for _, i in runs)
    dc, ic = sum(d.size for d, _ in runs), sum(i.size for _, i in runs)
    od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
    oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
    eng = capi.Engine(0)
    lo = bytes(W.format_keys(np.array([0]))[0])
    hi = bytes(W.format_keys(np.array([cfg.id_space // 10]))[0])
    cases = [("hash-1/8 (node join)", capi.SCAN_HASH, [(0, 1 << 29)]),
             ("hash-8x1/8 (all move)", capi.SCAN_HASH, [(k << 29, (k + 1) << 29 if k < 7 else 0xFFFFFFFF) for k in range(8)]),
             ("key-10%", capi.SCAN_KEY, [(lo, hi)])]
    gpu = card()
    print(f"card: {gpu}; tree: {len(runs)} tables, {entries} entries, {in_bytes / 1e9:.3f} GB", flush=True)
    results = []
    for name, kind, ranges in cases:
        for _ in range(3):
            rows, stop = eng.scan_device(tabs, ranges, (od.data_ptr(), dc, oi.data_ptr(), ic), kind)
        ms = []
        for _ in range(a.iters):
            eng.scan_device(tabs, ranges, (od.data_ptr(), dc, oi.data_ptr(), ic), kind)
            ms.append(eng.stats()["ms_total"])
        out_bytes = sum(r["data_len"] + r["index_len"] for r in rows)
        d_all, i_all = od.cpu().numpy(), oi.cpu().numpy()
        t0 = time.perf_counter()
        exp, exp_stop = scan_oracle.scan(runs, ranges, kind)
        cpu_s = time.perf_counter() - t0
        parity = stop == exp_stop and all(
            np.array_equal(d_all[r["data_off"]:r["data_off"] + r["data_len"]], e[0]) and
            np.array_equal(i_all[r["index_off"]:r["index_off"] + r["index_len"]], e[1]) for r, e in zip(rows, exp))
        med = float(np.median(ms))
        res = {"case": name, "ms_median": round(med, 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3),
               "input_GBps": round(in_bytes / med / 1e6, 1), "output_GB": round(out_bytes / 1e9, 4),
               "output_GBps": round(out_bytes / med / 1e6, 1), "selected": int(sum(r["items_written"] for r in rows)),
               "stop": stop, "parity": bool(parity), "cpu_oracle_s": round(cpu_s, 3),
               "cpu_oracle_input_GBps": round(in_bytes / cpu_s / 1e9, 3)}
        results.append(res)
        print(json.dumps(res), flush=True)

    # profiled pass: kernel times of one scan per case, and a device copy of the gathered byte count (the copy ceiling)
    from torch.profiler import ProfilerActivity, profile
    prof_rows = []
    for name, kind, ranges in cases:
        rows, _ = eng.scan_device(tabs, ranges, (od.data_ptr(), dc, oi.data_ptr(), ic), kind)
        nbytes = sum(r["data_len"] for r in rows)
        src = torch.empty(max(16, nbytes), dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        for _ in range(3):
            dst.copy_(src)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                eng.scan_device(tabs, ranges, (od.data_ptr(), dc, oi.data_ptr(), ic), kind)
                dst.copy_(src)
            torch.cuda.synchronize()
        k = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", 0) or getattr(ev, "cuda_time_total", 0)
            if t:
                k[ev.key] = round(t / ev.count / 1000.0, 4)
        gather = next((v for kk, v in k.items() if "k_gather_h" in kk), None)
        copy = next((v for kk, v in k.items() if kk.startswith("Memcpy DtoD")), None)
        row = {"case": name, "kernel_ms": k, "gather_ms": gather, "copy_ms_same_bytes": copy,
               "gather_vs_copy": round(copy / gather, 3) if gather and copy else None,
               "gather_TBps": round(2 * nbytes / gather / 1e9, 3) if gather else None}
        prof_rows.append(row)
        print(json.dumps(row), flush=True)
    summary = {"card": gpu, "entries": entries, "input_bytes": in_bytes, "cases": results, "profile": prof_rows,
               "parity_all": all(r["parity"] for r in results)}
    print(json.dumps({"parity_all": summary["parity_all"], "card": gpu}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "scan_bench.json"), "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
