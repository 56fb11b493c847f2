#!/usr/bin/env python
"""Reader range scans (dbeel_tree_reader_open + dbeel_reader_scan, DBEEL_SCAN_KEY) against dbeel_tree_scan_stream,
alternated in one process, on a cfg2-shaped tree of four tables written to tmpfs (the eight cfg2 runs compacted in pairs).
The stream reads every .index twice and every .data window whatever the range; the reader seeks each bound on its cached
fences and reads only the records from lower_bound(start) to lower_bound(end) of every table.  Ranges of about 1, 1,000
and 100,000 keys, and the whole key space.
Per width: median wall time of the synchronous call over rounds (results collected in memory by the same Python callback
for both), bytes and reads issued (the reader's counted by dbeel_last_stats and, for reads, in a separate untimed pass
through a logging Python callback; the stream's as the bytes it copies to the device plus its planning pass over the
.index files, and its read callback calls), and parity of the files and the stop on every call.  Prints the GPU name and
power limit of the run.  Measured results and the card they were measured on: DESIGN.md section 7, "Readers".
Usage: tools/reader_scan_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
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


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds = opt("--out", None), int(opt("--rounds", "7"))
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
    d = tempfile.mkdtemp(prefix="reader_scan_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "rows": []}
    try:
        for k, (td, ti, tb) in enumerate(tables):
            sstable.write_run_files(d, 2 * k, (td, ti), tb)
        tree_bytes = sum(td.size + ti.size for td, ti, _ in tables)
        index_bytes = sum(ti.size for _, ti, _ in tables)
        print(f"cfg2 in {len(tables)} tables on {'tmpfs' if base else 'disk'}: {sum(ti.size // 16 for _, ti, _ in tables)} "
              f"records, {tree_bytes / 1e6:.0f} MB of .data + .index", flush=True)
        keys = []
        for td, ti, _ in tables:
            offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
            keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
        keys = np.unique(np.concatenate(keys).view("V17").reshape(-1))
        tree = se.LSMTree.open_or_create(d, eng)
        reader = tree.open_reader()
        read, fds = file_reader(d, [i for i, _ in tree.sstable_indices_and_sizes()])
        counting = eng.open_reader([(td.size, ti.size, None) for td, ti, _ in tables], read=read)
        rng = np.random.default_rng(5)
        reader.scan([(b"", b"\x00")])  # the reader's first scan loads its exact-mode fences
        counting.scan([(b"", b"\x00")])
        for w in WIDTHS:
            t_r, t_s, parity, bytes_r, bytes_s = [], [], True, 0, 0
            for r in range((rounds if w is not None else min(rounds, 3)) + 1):  # round 0 warms up; the two alternate
                if w is None:
                    ranges = [(b"", b"\xff" * 18)]
                else:
                    j = int(rng.integers(0, len(keys) - w))
                    ranges = [(keys[j].tobytes(), keys[j + w].tobytes())]
                t0 = time.perf_counter()
                out_r, stop_r = reader.scan(ranges)
                t1 = time.perf_counter()
                bytes_r = eng.stats()["input_bytes"]
                out_s, stop_s = tree.scan_stream(ranges, capi.SCAN_KEY)
                t2 = time.perf_counter()
                bytes_s = eng.stats()["input_bytes"] + index_bytes
                parity = parity and stop_r == stop_s and all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                                                             for a, b in zip(out_r, out_s))
                if r:
                    t_r.append(t1 - t0)
                    t_s.append(t2 - t1)
            counting.scan(ranges)
            n_r = len(counting.last_stream_reads)
            n_s = None
            if w is not None or tree_bytes < 4 << 30:
                eng.scan_stream([(td, ti) for td, ti, _ in tables], ranges, capi.SCAN_KEY)
                n_s = eng.last_stream_calls[0]
            items = sum(o[1].size // 16 for o in out_r)
            row = {"width": w if w is not None else "all", "entries": items, "reader_s": float(np.median(t_r)),
                   "stream_s": float(np.median(t_s)), "reader_bytes": int(bytes_r), "stream_bytes": int(bytes_s),
                   "reader_reads": n_r, "stream_reads": n_s, "parity": bool(parity)}
            result["rows"].append(row)
            print(f"width {str(row['width']):>7} ({items:>8} entries): reader {row['reader_s'] * 1e3:9.3f} ms, stream "
                  f"{row['stream_s'] * 1e3:9.3f} ms | read {bytes_r / 1e6:10.4f} MB vs {bytes_s / 1e6:9.1f} MB | reads {n_r} vs {n_s} | "
                  f"parity {parity}", flush=True)
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
