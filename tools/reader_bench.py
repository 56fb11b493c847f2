#!/usr/bin/env python
"""Readers (dbeel_tree_reader_open + dbeel_reader_get_values) against dbeel_tree_get_values_stream, alternated in one
process, on a cfg2-shaped tree of four tables written to tmpfs (the eight cfg2 runs compacted in pairs, each table with its
filter).  A serving loop sends many small batches to the same tables, and that is what a reader is for: it uploads every
filter once and keeps each table's fences on the device after its first batch in a mode, where the stream entry point
reads all .bloom files and the fences again on every call.  Batches of 1, 64, 4,096 and 65,536 keys, half present (the
present half drawn uniformly or Zipf(1.1) over the tree's keys), both modes.
Per batch: median wall time of the synchronous call over rounds (the reader after its first batch per mode), bytes read
(.data / .index through the callback, plus for the stream the .bloom files it reads whole), and reads issued (counted
in a separate untimed pass through a logging Python callback, as the tree's own callback has no log).  Rows, .data and
.index of the two are compared on every batch.  Prints the GPU name and power limit of the run.
Small batches are dominated by the filter uploads and the fence reads, which the reader removes; large batches by the
leaves, which both read.  Measured results and the card they were measured on: DESIGN.md section 7, "Readers".
Usage: tools/reader_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import SEED32, make_runs_parallel  # noqa: E402
from dbeel_b200 import capi, sstable  # noqa: E402
from dbeel_b200 import storage_engine as se  # noqa: E402
from dbeel_b200 import workloads as W  # noqa: E402

BATCHES = (1, 64, 4096, 65536)
MODES = ((capi.LOOKUP_REFERENCE, "reference"), (capi.LOOKUP_EXACT, "exact"))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def file_reader(d, indices):
    """read(table, kind, offset, size) over the tree's files, for the counting pass"""
    fds = [(os.open(os.path.join(d, sstable.file_name(i, sstable.DATA_FILE_EXT)), os.O_RDONLY),
            os.open(os.path.join(d, sstable.file_name(i, sstable.INDEX_FILE_EXT)), os.O_RDONLY)) for i in indices]
    return lambda t, kind, off, size: os.pread(fds[t][0 if kind == 1 else 1], size, off), fds


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds = opt("--out", None), int(opt("--rounds", "20"))
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
    d = tempfile.mkdtemp(prefix="reader_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "rows": []}
    try:
        for k, (td, ti, tb) in enumerate(tables):
            sstable.write_run_files(d, 2 * k, (td, ti), tb)
        tree_bytes = sum(td.size + ti.size + (tb.size if tb is not None else 0) for td, ti, tb in tables)
        bloom_bytes = sum(tb.size for _, _, tb in tables if tb is not None)
        print(f"cfg2 in {len(tables)} tables on {'tmpfs' if base else 'disk'}: {sum(ti.size // 16 for _, ti, _ in tables)} "
              f"records, {tree_bytes / 1e6:.0f} MB, filters {bloom_bytes / 1e6:.1f} MB", flush=True)
        all_keys = []
        for td, ti, _ in tables:
            offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
            all_keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
        all_keys = np.concatenate(all_keys)
        tree = se.LSMTree.open_or_create(d, eng)
        reader = tree.open_reader()
        read, fds = file_reader(d, [i for i, _ in tree.sstable_indices_and_sizes()])
        counting = eng.open_reader([(td.size, ti.size, tb) for td, ti, tb in tables], read=read)
        rng = np.random.default_rng(31)
        for mode, mname in MODES:
            reader.get_values([all_keys[0].tobytes()], mode)  # the reader's first batch in the mode loads its fences
            counting.get_values([all_keys[0].tobytes()], mode)
            for dist in ("uniform", "zipf"):
                for nq in BATCHES:
                    t_r, t_s, parity = [], [], True
                    for r in range(rounds + 1):  # round 0 warms up; the two entry points alternate
                        npres = (nq + 1) // 2
                        pick = (rng.integers(0, len(all_keys), npres) if dist == "uniform"
                                else (rng.zipf(1.1, npres) - 1) % len(all_keys))
                        keys = [all_keys[j].tobytes() for j in pick] + [b"\xb0k%015d" % int(x) for x in
                                                                          rng.integers(20_000_000, 1 << 40, nq - npres)]
                        t0 = time.perf_counter()
                        rr, dr, ir = reader.get_values(keys, mode)
                        t1 = time.perf_counter()
                        read_r = eng.stats()["input_bytes"]
                        rs, ds, is_ = tree.get_values_stream(keys, mode)
                        t2 = time.perf_counter()
                        read_s = eng.stats()["input_bytes"] + bloom_bytes
                        parity = parity and bool(np.array_equal(rr, rs) and np.array_equal(dr, ds) and np.array_equal(ir, is_))
                        if r:
                            t_r.append(t1 - t0)
                            t_s.append(t2 - t1)
                    counting.get_values(keys, mode)  # loads the fences of tables no earlier batch reached
                    counting.get_values(keys, mode)
                    n_r = len(counting.last_stream_reads)
                    eng.get_values_stream([(td.size, ti.size, tb) for td, ti, tb in tables], keys, mode, read=read)
                    n_s = len(eng.last_stream_reads)
                    row = {"keys": nq, "mode": mname, "dist": dist, "reader_s": float(np.median(t_r)), "stream_s": float(np.median(t_s)),
                           "reader_bytes": int(read_r), "stream_bytes": int(read_s), "reader_reads": n_r, "stream_reads": n_s,
                           "parity": parity}
                    result["rows"].append(row)
                    print(f"{mname:9s} {dist:7s} {nq:>6} keys: reader {row['reader_s'] * 1e3:8.3f} ms, stream {row['stream_s'] * 1e3:8.3f} ms | "
                          f"read {read_r / 1e6:8.3f} MB vs {read_s / 1e6:8.3f} MB | reads {n_r} vs {n_s} | parity {parity}", flush=True)
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
