#!/usr/bin/env python
"""Range reads on a tree reader (dbeel_reader_get_range) against the caller's alternative -- dbeel_reader_scan plus an
LSM merge of its output on the host in numpy (group by key, keep the newest table's version, drop tombstones, sort) --
and against dbeel_reader_scan alone, alternated in one process on the cfg2-shaped tree of tools/reader_scan_bench.py
(four tables on tmpfs).  Ranges of about 1, 1,000 and 100,000 keys, and the whole key space.
Per arm and width: median wall time over rounds, bytes read (dbeel_last_stats), reads (a separate untimed pass through a
logging callback), entries and bytes returned, partitions; parity of get_range with the host merge on every round.  A
separate torch.profiler pass sums the merge stage's kernels (k_range_*) and the host-to-device copies of one get_range
call per width.  Prints the GPU name and power limit of the run.  Results: DESIGN.md section 7, "Range reads".
Usage: tools/reader_range_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
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

WIDTHS = (1, 1000, 100_000, None)  # None: the whole key space
CHUNK = 1 << 20


def host_merge(d, ix):
    """The LSM merge of one destination's raw scan output (tables oldest first): last version per key, tombstones
    dropped, keys ascending -- an SSTable pair, numpy throughout."""
    if ix.size == 0:
        return d[:0], ix[:0]
    rec = ix.view("<u8").reshape(-1, 2)
    off = rec[:, 0].astype(np.int64)
    fs = (rec[:, 1] >> np.uint64(32)).astype(np.int64)
    klen = (rec[:, 1] & np.uint64(0xFFFFFFFF)).astype(np.int64) - 8
    kmax = int(klen.max())
    keys = np.zeros((off.size, kmax + 1), np.uint8)  # zero-padded keys, length last: byte order of Vec<u8>
    for b in range(kmax):
        keys[:, b] = np.where(b < klen, d[np.minimum(off + 8 + b, d.size - 1)], 0)
    keys[:, kmax] = klen
    kv = np.ascontiguousarray(keys).view(f"V{kmax + 1}").reshape(-1)
    rev = kv[::-1]
    _, first = np.unique(rev, return_index=True)  # sorted keys, each one's last occurrence in scan order
    pick = off.size - 1 - first
    dl = np.zeros(pick.size, np.int64)
    for b in range(8):
        dl |= d[off[pick] + 8 + klen[pick] + b].astype(np.int64) << (8 * b)
    pick = pick[dl != 0]
    o, f = off[pick], fs[pick]
    start = np.concatenate([[0], np.cumsum(f)[:-1]]) if f.size else f
    out_d = np.empty(int(f.sum()), np.uint8)
    for a in range(0, pick.size, CHUNK):
        oo, ff, ss = o[a:a + CHUNK], f[a:a + CHUNK], start[a:a + CHUNK]
        src = np.repeat(oo - ss, ff) + np.arange(int(ss[0]), int(ss[0] + ff.sum()))
        out_d[int(ss[0]):int(ss[0] + ff.sum())] = d[src]
    out_i = np.empty((pick.size, 2), np.uint64)
    out_i[:, 0] = start.astype(np.uint64)
    out_i[:, 1] = (f.astype(np.uint64) << np.uint64(32)) | (klen[pick] + 8).astype(np.uint64)
    return out_d, out_i.reshape(-1).view(np.uint8)


def profile_merge(reader, ranges, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        reader.get_range(ranges)
        torch.cuda.synchronize()
    k_us, h2d_us, per = 0.0, 0.0, {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "k_range_" in ev.name:
            k_us += us
            per[ev.name.split("(")[0]] = per.get(ev.name.split("(")[0], 0.0) + us
        elif "HtoD" in ev.name or "Host to Device" in ev.name:
            h2d_us += us
    return k_us, h2d_us, per


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
    runs = make_runs_parallel(cfg)
    tables = [eng.compact(runs[k:k + 2], keep_tombstones=True, seed=SEED32)[:3] for k in range(0, len(runs), 2)]
    del runs
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    d = tempfile.mkdtemp(prefix="reader_range_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "rows": []}
    try:
        for k, (td, ti, tb) in enumerate(tables):
            sstable.write_run_files(d, 2 * k, (td, ti), tb)
        keys = []
        for td, ti, _ in tables:
            offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
            keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
        keys = np.unique(np.concatenate(keys).view("V17").reshape(-1))
        print(f"cfg2 in {len(tables)} tables: {sum(ti.size // 16 for _, ti, _ in tables)} records, {keys.size} keys",
              flush=True)
        tree = se.LSMTree.open_or_create(d, eng)
        reader = tree.open_reader()
        read, fds = file_reader(d, [i for i, _ in tree.sstable_indices_and_sizes()])
        counting = eng.open_reader([(td.size, ti.size, None) for td, ti, _ in tables], read=read)
        del tables
        rng = np.random.default_rng(5)
        reader.get_range([(b"", b"\x00")])  # the first call loads the exact-mode fences
        counting.get_range([(b"", b"\x00")])
        for w in WIDTHS:
            t = {"get_range": [], "scan_host_merge": [], "scan": []}
            st, parity = {}, True
            for r in range((rounds if w is not None else min(rounds, 2)) + 1):  # round 0 warms up
                if w is None:
                    ranges = [(b"", b"\xff" * 18)]
                else:
                    j = int(rng.integers(0, len(keys) - w))
                    ranges = [(keys[j].tobytes(), keys[j + w].tobytes())]
                t0 = time.perf_counter()
                got, _ = reader.get_range(ranges)
                t1 = time.perf_counter()
                st["get_range"] = eng.stats()
                raw, _ = reader.scan(ranges)
                merged = host_merge(*raw[0])
                t2 = time.perf_counter()
                st["scan_host_merge"] = eng.stats()
                raw2, _ = reader.scan(ranges)
                t3 = time.perf_counter()
                st["scan"] = eng.stats()
                parity = parity and np.array_equal(got[0][0], merged[0]) and np.array_equal(got[0][1], merged[1])
                if r:
                    t["get_range"].append(t1 - t0)
                    t["scan_host_merge"].append(t2 - t1)
                    t["scan"].append(t3 - t2)
            counting.get_range(ranges)
            n_g = len(counting.last_stream_reads)
            counting.scan(ranges)
            n_s = len(counting.last_stream_reads)
            k_us, h2d_us, per = profile_merge(reader, ranges, None)
            row = {"width": w if w is not None else "all", "parity": bool(parity), "merge_kernels_ms": k_us / 1e3,
                   "h2d_ms": h2d_us / 1e3, "kernels": {k: v / 1e3 for k, v in per.items()}, "arms": {}}
            for arm, out in (("get_range", got[0]), ("scan_host_merge", merged), ("scan", raw2[0])):
                row["arms"][arm] = {"wall_ms": float(np.median(t[arm])) * 1e3, "bytes_read": int(st[arm]["input_bytes"]),
                                    "reads": n_g if arm == "get_range" else n_s, "entries": int(out[1].size // 16),
                                    "bytes_out": int(out[0].size + out[1].size), "partitions": int(st[arm]["partitions"])}
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
        counting.close()
        reader.close()
        tree.close()
        for a, b in fds:
            os.close(a)
            os.close(b)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(result), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()
    if not all(r["parity"] for r in result["rows"]):
        sys.exit("parity failed")


if __name__ == "__main__":
    main()
