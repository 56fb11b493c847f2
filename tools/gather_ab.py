#!/usr/bin/env python
"""Gather A/B on one GPU, all in one process on one cfg2 input:

  1. the practical copy ceiling: a ~2 GB device-to-device torch copy, CUDA events, warmed up, several repeats
     (rate = bytes read + bytes written over time);
  2. the stage times of every spec, the specs alternated for --rounds rounds (spread = max - min over rounds);
  3. with --profile SPEC (repeatable), per-kernel device times from torch.profiler in a run of their own.

A spec is tools/tune.py's: "DBEEL_GATHER=10,DBEEL_BLOOM_SIDE=1", "LIB=<variant>" (a build made by
`python -m dbeel_b200._build --variant <name> -D...`), or "" for the default.
Usage: tools/gather_ab.py --rounds 3 "" "DBEEL_GATHER=10" --profile "DBEEL_GATHER=10,DBEEL_BLOOM_SIDE=1"
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402

STAGES = ("ms_total", "ms_extract", "ms_merge", "ms_resolve", "ms_gather")


def copy_ceiling(dev, nbytes=2 << 30, reps=10, rounds=3):
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev).fill_(1)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            dst.copy_(src)
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b) / reps
        out.append({"ms": round(ms, 4), "TBps_read_plus_write": round(2 * nbytes / ms / 1e9, 3)})
    del src, dst
    torch.cuda.empty_cache()
    return {"bytes_each_way": nbytes, "rounds": out}


class Job:
    def __init__(self, dev):
        cfg = W.CFG2
        runs = make_runs_parallel(cfg)
        self.t_runs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in runs]
        self.opts = capi.make_opts(cfg.keep_tombstones, seed=SEED32)
        dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], self.opts)
        self.od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
        self.oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
        self.ob = torch.empty(bc + 16, dtype=torch.uint8, device=dev)
        self.d_runs = [(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in self.t_runs]
        self.d_out = (self.od.data_ptr(), dc, self.oi.data_ptr(), ic, self.ob.data_ptr(), bc)
        self.default_lib = capi.LIB_PATH
        torch.cuda.synchronize()

    def engine(self, spec):
        env = dict(kv.split("=") for kv in spec.split(",") if kv)
        for k in [k for k in os.environ if k.startswith("DBEEL_")]:
            del os.environ[k]
        lib = env.pop("LIB", None)
        want = os.path.join(ROOT, "dbeel_b200", f"libdbeel_compact.{lib}.so") if lib else self.default_lib
        if want != capi.LIB_PATH:
            capi.LIB_PATH, capi._lib = want, None
        os.environ.update(env)
        return capi.Engine(0)

    def checksum(self, res):
        return (tuple(res), int(self.od[:res[0] // 8 * 8].view(torch.int64).sum().item()),
                int(self.oi[:res[1] // 8 * 8].view(torch.int64).sum().item()),
                int(self.ob[:res[2] // 8 * 8].view(torch.int64).sum().item()))

    def time(self, spec, steps=20):
        eng = self.engine(spec)
        for _ in range(3):
            res = eng.compact_device(self.d_runs, self.d_out, self.opts)
        acc = dict.fromkeys(STAGES, 0.0)
        for _ in range(steps):
            res = eng.compact_device(self.d_runs, self.d_out, self.opts)
            st = eng.stats()
            for k in STAGES:
                acc[k] += st[k]
        torch.cuda.synchronize()
        chk = self.checksum(res)
        eng.close()
        return {k: v / steps for k, v in acc.items()}, chk

    def profile(self, spec, steps=10):
        from torch.profiler import ProfilerActivity, profile
        eng = self.engine(spec)
        for _ in range(3):
            eng.compact_device(self.d_runs, self.d_out, self.opts)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                eng.compact_device(self.d_runs, self.d_out, self.opts)
            torch.cuda.synchronize()
        eng.close()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0:
                per[ev.key] = round(t / 1e3 / steps, 4)
        return dict(sorted(per.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("specs", nargs="*")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--profile", action="append", default=[])
    ap.add_argument("--no-ceiling", action="store_true")
    ap.add_argument("--json", help="write every number here as well")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(0)}
    if not args.no_ceiling:
        out["copy_ceiling"] = copy_ceiling(dev)
        print("copy ceiling:", json.dumps(out["copy_ceiling"]), flush=True)
    job = Job(dev)
    specs = args.specs or [""]
    times = {s: [] for s in specs}
    ref = None
    for r in range(args.rounds):
        for s in specs:
            t, chk = job.time(s, args.steps)
            ref = chk if ref is None else ref
            times[s].append(t)
            print(f"round {r} {s or 'default':50s} " + " ".join(f"{k[3:]}={t[k]:.4f}" for k in STAGES) +
                  ("  same-output" if chk == ref else "  OUTPUT-DIFFERS"), flush=True)
    summary = {}
    print("\nspec: median [min, max] over rounds, ms")
    for s in specs:
        summary[s or "default"] = row = {}
        for k in STAGES:
            v = [t[k] for t in times[s]]
            row[k] = {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
        print(f"{s or 'default':50s} " + "  ".join(f"{k[3:]} {row[k]}" for k in STAGES))
    out["ab"] = summary
    out["profile"] = {}
    for s in args.profile:
        out["profile"][s or "default"] = per = job.profile(s)
        print(f"\nprofile {s or 'default'} (ms per job):")
        for k, v in list(per.items())[:12]:
            print(f"  {v:8.4f}  {k[:110]}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
