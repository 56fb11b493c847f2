#!/usr/bin/env python
"""Batched reads with values (row N2) on the table a cfg2 compaction leaves in HBM: dbeel_get_values_device next to
dbeel_get_many_device, alternated in one process, on a 50/50 mix of present and absent keys, both search modes.
Reports Mkeys/s, GB/s of entry bytes returned, k_gather_h's share of the get_values kernels (torch.profiler, a run of its
own), and parity of a sample of rows and entries with the CPU oracle (tests/get_values_oracle.c).
Usage: tools/get_values_bench.py [n_queries (default 4000000)] [keys_per_run (default 1000000)] [--out result.json]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import get_values_oracle as gvo  # noqa: E402  (CPU parity only)
from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402

REPS = 9


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    if out_path in args:
        args.remove(out_path)
    nq = int(args[0]) if args else 4_000_000
    kpr = int(args[1]) if len(args) > 1 else 1_000_000
    cfg = W.CFG2 if kpr == 1_000_000 else W.scaled(W.CFG2, kpr)
    runs = make_runs_parallel(cfg)
    dev = torch.device("cuda:0")
    t_runs = [(torch.from_numpy(d).to(dev), torch.from_numpy(i).to(dev)) for d, i in runs]
    opts = capi.make_opts(cfg.keep_tombstones, seed=SEED32)
    dc, ic, bc = capi.compact_bound([(d.size, i.size) for d, i in runs], opts)
    od, oi, ob = (torch.empty(c + 16, dtype=torch.uint8, device=dev) for c in (dc, ic, bc))
    eng = capi.Engine(0)
    dl, il, bl, n = eng.compact_device([(d.data_ptr(), d.numel(), i.data_ptr(), i.numel()) for d, i in t_runs],
                                       (od.data_ptr(), dc, oi.data_ptr(), ic, ob.data_ptr(), bc), opts)
    del t_runs, runs
    gpu, power = card()
    print(f"{gpu}, power limit {power}", flush=True)
    print(f"table: {n} entries, {dl / 1e6:.0f} MB .data, {il / 1e6:.0f} MB .index, {bl / 1e6:.1f} MB .bloom", flush=True)
    rng = np.random.default_rng(11)
    h_index = oi[:il].cpu().numpy()
    h_rec = h_index.view("<u8").reshape(-1, 2)
    h_data = od[:dl].cpu().numpy()
    klen = 17  # every key of this workload is 17 bytes
    pick = rng.integers(0, n, nq // 2)
    offs = h_rec[pick, 0].astype(np.int64)
    present = np.stack([h_data[offs + 8 + b] for b in range(klen)], axis=1)
    absent = np.frombuffer(b"".join(b"\xb0k%015d" % int(x) for x in rng.integers(20_000_000, 1 << 40, nq - nq // 2)),
                           dtype=np.uint8).reshape(-1, klen)
    keys = np.concatenate([present, absent])[rng.permutation(nq)]
    blob = np.ascontiguousarray(keys).reshape(-1)
    off = np.arange(nq + 1, dtype=np.uint64) * klen
    d_keys, d_off = torch.from_numpy(blob.copy()).to(dev), torch.from_numpy(off.view(np.int64)).to(dev)
    data_cap = int((h_rec[pick, 1] >> 32).sum())  # full_size of every present pick: no answered set needs more
    index_cap = 16 * nq
    d_rows_many = torch.zeros(2 * nq, dtype=torch.int64, device=dev)
    d_rows = torch.zeros(2 * nq, dtype=torch.int64, device=dev)
    o_data = torch.empty(data_cap + 16, dtype=torch.uint8, device=dev)
    o_index = torch.empty(index_cap + 16, dtype=torch.uint8, device=dev)
    table = [(od.data_ptr(), dl, oi.data_ptr(), il, ob.data_ptr(), bl)]
    stream = torch.cuda.ExternalStream(eng.stream_ptr())

    def get_many(mode):
        eng.get_many_device(table, d_keys.data_ptr(), d_off.data_ptr(), nq, d_rows_many.data_ptr(), mode)

    def get_values(mode):
        return eng.get_values_device(table, d_keys.data_ptr(), d_off.data_ptr(), nq, d_rows.data_ptr(),
                                     (o_data.data_ptr(), data_cap, o_index.data_ptr(), index_cap), mode)

    def timed(fn, mode):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        r = fn(mode)
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b), r

    result = {"gpu": gpu, "power_limit": power, "n_queries": nq, "table_entries": n, "modes": {}}
    for mode, mname in ((capi.LOOKUP_REFERENCE, "reference"), (capi.LOOKUP_EXACT, "exact")):
        for _ in range(2):
            get_many(mode)
            get_values(mode)
        t_many, t_vals = [], []
        for _ in range(REPS):  # alternated: both see the same machine state
            t_many.append(timed(get_many, mode)[0])
            ms, (dlen, ilen, items) = timed(get_values, mode)
            t_vals.append(ms)
        rows = d_rows.cpu().numpy().view(capi.LOOKUP_DTYPE)
        many = d_rows_many.cpu().numpy().view(capi.LOOKUP_DTYPE).copy()
        masked = rows.copy()
        masked["bloom_rejects"] &= ~np.uint32(capi.LOOKUP_BAD_ENTRY)
        tm, tv = float(np.median(t_many)), float(np.median(t_vals))
        r = {"get_many_ms": tm, "get_values_ms": tv, "get_many_mkeys_s": nq / tm / 1e3, "get_values_mkeys_s": nq / tv / 1e3,
             "entries": items, "entry_bytes": dlen, "entries_gb_s": dlen / tv / 1e6,
             "rows_equal_get_many": bool(np.array_equal(masked, many))}
        result["modes"][mname] = r
        print(f"{mname:9s}: get_many {tm:7.3f} ms = {r['get_many_mkeys_s']:7.1f} Mkeys/s | get_values {tv:7.3f} ms = "
              f"{r['get_values_mkeys_s']:7.1f} Mkeys/s, {items} entries, {dlen / 1e6:.0f} MB = {r['entries_gb_s']:.1f} GB/s | "
              f"rows == get_many's: {r['rows_equal_get_many']}", flush=True)

    # k_gather_h's share of the get_values kernels, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            get_values(capi.LOOKUP_EXACT)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
            kern[ev.key] = kern.get(ev.key, 0.0) + ev.device_time_total
    kern = {k: v for k, v in kern.items() if "emcpy" not in k and "emset" not in k}
    total = sum(kern.values())
    gather = sum(v for k, v in kern.items() if "k_gather_h" in k)
    result["k_gather_h_share"] = gather / total if total else None
    for k, v in sorted(kern.items(), key=lambda kv: -kv[1]):
        print(f"  {v / 3 / 1e3:8.3f} ms/call  {k[:90]}", flush=True)
    print(f"k_gather_h: {100 * result['k_gather_h_share']:.1f} % of the get_values kernel time", flush=True)

    # parity with the CPU oracle on a sample (REFERENCE mode: the oracle restates the reference's loop)
    sample = min(nq, 200_000)
    host_table = [(h_data, h_index, ob[:bl].cpu().numpy())]
    et, er, ej, ed, ei = gvo.get_values(host_table, blob[:sample * klen], off[:sample + 1])
    s_rows = torch.zeros(2 * sample, dtype=torch.int64, device=dev)
    dlen, ilen, items = eng.get_values_device(table, d_keys.data_ptr(), d_off.data_ptr(), sample, s_rows.data_ptr(),
                                              (o_data.data_ptr(), data_cap, o_index.data_ptr(), index_cap), capi.LOOKUP_REFERENCE)
    rows = s_rows.cpu().numpy().view(capi.LOOKUP_DTYPE)
    parity = bool(np.array_equal(rows["table"], et) and np.array_equal(rows["bloom_rejects"], ej) and
                  np.array_equal(np.where(rows["table"] >= 0, rows["record"], 0), er) and
                  np.array_equal(o_data[:dlen].cpu().numpy(), ed) and np.array_equal(o_index[:ilen].cpu().numpy(), ei))
    result["oracle_sample"] = sample
    result["parity"] = parity
    print(f"oracle parity on the first {sample} keys (rows, .data, .index, {items} entries): {parity}", flush=True)
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
