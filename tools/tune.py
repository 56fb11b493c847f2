#!/usr/bin/env python
"""Kernel-variant sweep on one GPU: generates the cfg2 workload once, then times the device-resident
pipeline for each environment configuration (variants are read from the environment when an engine
is created; `LIB=<variant>` selects a compile-time variant built by dbeel_b200/_build.py).  Usage: tools/tune.py "" "DBEEL_FUSED_FINAL=0" "DBEEL_EXTRACT_PERSIST=0,DBEEL_NARROW=0" "LIB=<variant>" ..."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402


def main():
    cfg = W.CFG2
    runs = make_runs_parallel(cfg)
    dev = torch.device("cuda:0")
    t_runs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in runs]
    opts = capi.make_opts(cfg.keep_tombstones, seed=SEED32)
    dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], opts)
    od = torch.empty(dc + 16, dtype=torch.uint8, device=dev)
    oi = torch.empty(ic + 16, dtype=torch.uint8, device=dev)
    ob = torch.empty(bc + 16, dtype=torch.uint8, device=dev)
    d_runs = [(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_runs]
    d_out = (od.data_ptr(), dc, oi.data_ptr(), ic, ob.data_ptr(), bc)
    torch.cuda.synchronize()
    ref = None
    default_lib = capi.LIB_PATH
    for spec in sys.argv[1:] or [""]:
        env = dict(kv.split("=") for kv in spec.split(",") if kv)
        for k in [k for k in os.environ if k.startswith("DBEEL_")]:
            del os.environ[k]
        lib = env.pop("LIB", None)  # an A/B build made by `python -m dbeel_b200._build --variant <name> -D...`
        want = os.path.join(ROOT, "dbeel_b200", f"libdbeel_compact.{lib}.so") if lib else default_lib
        if want != capi.LIB_PATH:
            capi.LIB_PATH, capi._lib = want, None
        os.environ.update(env)
        eng = capi.Engine(0)
        for _ in range(3):
            res = eng.compact_device(d_runs, d_out, opts)
        acc = {}
        steps = 10
        for _ in range(steps):
            res = eng.compact_device(d_runs, d_out, opts)
            st = eng.stats()
            for k in ("ms_total", "ms_extract", "ms_merge", "ms_resolve", "ms_gather"):
                acc[k] = acc.get(k, 0.0) + st[k]
        torch.cuda.synchronize()
        chk = (res, int(od[:res[0] // 8 * 8].view(torch.int64).sum().item()), int(oi[:res[1] // 8 * 8].view(torch.int64).sum().item()),
               int(ob[:res[2] // 8 * 8].view(torch.int64).sum().item()))
        if ref is None:
            ref = chk
        ok = "same-output" if chk == ref else "OUTPUT-DIFFERS"
        print(f"{spec or 'default':45s} " + " ".join(f"{k[3:]}={v / steps:.4f}" for k, v in acc.items()) + f"  {ok}", flush=True)
        eng.close()


if __name__ == "__main__":
    main()
