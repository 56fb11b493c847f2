#!/usr/bin/env python
"""Limited range reads on a tree reader (dbeel_reader_get_ranges) against what a caller does without them -- get_range in
calls of up to 256 ranges that do not overlap, with each answer cut to the limit on the host -- alternated in one process on the cfg2-shaped
tree of tools/reader_scan_bench.py (four tables on tmpfs).
  - Batches of 1, 64 and 4,096 queries, limits 1, 10 and 100, start keys uniform or Zipf(1.1) over the keys (hot keys
    scattered by a fixed permutation).  get_ranges asks [start, end of the key space); get_range has no limit, so its
    ranges end 2 * limit keys after the start, the end a caller would have to guess.
  - The whole key space with limit 10 against get_range of the whole key space.
Per row and arm: median wall time over rounds, bytes read and rounds (dbeel_last_stats input_bytes / partitions),
callback reads (a separate untimed pass through a logging callback); parity on every round: every query's entries from
get_ranges equal the first entries of get_range's answer (all of it when that answer is shorter than the limit and its
range reached the end of the key space).  Prints the GPU name and power limit of the run.  Results: DESIGN.md section 7,
"Limited range reads".
Usage: tools/reader_ranges_bench.py [keys_per_run (default 1000000)] [--rounds R] [--out result.json]"""
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

BATCHES = (1, 64, 4096)
LIMITS = (1, 10, 100)
TOP = b"\xff" * 18  # above every cfg2 key


def entries(data, index, first, count):
    ix = np.asarray(index, np.uint8).reshape(-1, 16)[first:first + count]
    if not count:
        return b""
    a = int(ix[0, :8].view("<u8")[0])
    b = int(ix[-1, :8].view("<u8")[0]) + int(ix[-1, 12:16].view("<u4")[0])
    return bytes(data[a:b])


def truncated_get_range(reader, ranges, limit):
    """get_range in calls of up to 256 ranges that do not overlap (calls_of), every answer cut to its first `limit` entries on the host:
    [(entry bytes, entries in the whole answer)], and the calls' dbeel_last_stats summed."""
    uniq = sorted(set(ranges))  # a caller asks a repeated range once
    out, tot = {}, {"input_bytes": 0, "entries_out": 0, "partitions": 0, "reads": 0}  # reads: the counting reader's
    for call in calls_of(uniq):
        got, _ = reader.get_range([uniq[q] for q in call])
        st = dict(reader._engine.stats(), reads=len(reader.last_stream_reads or ()))
        for k in tot:
            tot[k] += int(st[k])
        for q, (d, i) in zip(call, got):
            n = i.size // 16
            out[uniq[q]] = (entries(d, i, 0, min(n, limit)), n)
    return [out[x] for x in ranges], tot


def calls_of(ranges):
    """The ranges in calls of at most 256 (DBEEL_MAX_SCAN_RANGES) whose ranges do not overlap: get_range gives a key to
    the first range of a call that takes it, so a caller must keep overlapping ranges apart."""
    import bisect
    calls, spans = [], []  # per call: query numbers, sorted (start, end)
    for q, (s, e) in enumerate(ranges):
        for c, sp in zip(calls, spans):
            k = bisect.bisect_left(sp, (s, e))
            if len(c) < 256 and (k == len(sp) or e <= sp[k][0]) and (k == 0 or sp[k - 1][1] <= s):
                c.append(q)
                sp.insert(k, (s, e))
                break
        else:
            calls.append([q])
            spans.append([(s, e)])
    return calls


def main():
    argv = sys.argv[1:]
    opt = lambda k, d: argv[argv.index(k) + 1] if k in argv else d
    out_path, rounds = opt("--out", None), int(opt("--rounds", "3"))
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
    d = tempfile.mkdtemp(prefix="reader_ranges_bench_", dir=base)
    result = {"gpu": gpu, "power_limit": power, "rows": []}
    try:
        for k, (td, ti, tb) in enumerate(tables):
            sstable.write_run_files(d, 2 * k, (td, ti), tb)
        keys = []
        for td, ti, _ in tables:
            offs = ti.view("<u8").reshape(-1, 2)[:, 0].astype(np.int64)
            keys.append(np.stack([td[offs + 8 + b] for b in range(17)], axis=1))  # cfg2's 17-byte keys
        keys = np.unique(np.concatenate(keys).view("V17").reshape(-1))
        nk = keys.size
        print(f"cfg2 in {len(tables)} tables: {sum(ti.size // 16 for _, ti, _ in tables)} records, {nk} keys", flush=True)
        tree = se.LSMTree.open_or_create(d, eng)
        reader = tree.open_reader()
        read, fds = file_reader(d, [i for i, _ in tree.sstable_indices_and_sizes()])
        counting = eng.open_reader([(td.size, ti.size, None) for td, ti, _ in tables], read=read)
        del tables
        rng = np.random.default_rng(5)
        perm = rng.permutation(nk)
        for r in (reader, counting):  # the first calls load the exact-mode fences
            r.get_range([(b"", b"\x00")])
            r.get_ranges([(b"", b"\x00")], 1)

        def starts(n, dist):
            j = rng.integers(0, nk, n) if dist == "uniform" else perm[np.minimum(rng.zipf(1.1, n) - 1, nk - 1)]
            return [int(x) for x in j]

        def run_row(name, make, limit, r_count):
            t = {"get_ranges": [], "get_range_truncated": []}
            st, parity = {}, True
            for r in range(r_count + 1):  # round 0 warms up
                qs, gr = make()
                t0 = time.perf_counter()
                rows, data, index = reader.get_ranges(qs, limit)
                t1 = time.perf_counter()
                st["get_ranges"] = eng.stats()
                want, st["get_range_truncated"] = truncated_get_range(reader, gr, limit)
                t2 = time.perf_counter()
                for q, (w, n_all) in enumerate(want):
                    got = entries(data, index, int(rows[q]["first"]), int(rows[q]["count"]))
                    more = bool(rows[q]["flags"] & capi.RANGE_MORE)
                    if gr[q][1] == TOP:  # both asked the rest of the key space
                        parity = parity and got == w and more == (n_all > limit)
                    elif n_all >= limit:
                        parity = parity and got == w and (more or n_all == limit)
                    else:  # the guessed end cut get_range's answer short
                        parity = parity and got[:len(w)] == w
                if r:
                    t["get_ranges"].append(t1 - t0)
                    t["get_range_truncated"].append(t2 - t1)
            counting.get_ranges(qs, limit)
            n_a = len(counting.last_stream_reads)
            ra = eng.stats()["partitions"]
            n_b = truncated_get_range(counting, gr, limit)[1]["reads"]
            row = {"row": name, "parity": bool(parity), "arms": {}}
            for arm, n_reads in (("get_ranges", n_a), ("get_range_truncated", n_b)):
                row["arms"][arm] = {"wall_ms": float(np.median(t[arm])) * 1e3, "bytes_read": int(st[arm]["input_bytes"]),
                                    "reads": n_reads, "rounds": int(st[arm]["partitions"]) if arm == "get_ranges" else None,
                                    "entries": int(st[arm]["entries_out"])}
            row["arms"]["get_ranges"]["rounds_counting_reader"] = int(ra)
            result["rows"].append(row)
            print(json.dumps(row), flush=True)

        for batch in BATCHES:
            for limit in LIMITS:
                for dist in ("uniform", "zipf"):
                    def make(batch=batch, limit=limit, dist=dist):
                        js = starts(batch, dist)
                        qs = [(keys[j].tobytes(), TOP) for j in js]
                        gr = [(keys[j].tobytes(), keys[j + 2 * limit].tobytes() if j + 2 * limit < nk else TOP) for j in js]
                        return qs, gr
                    run_row(f"batch {batch}, limit {limit}, {dist}", make, limit, rounds)
        run_row("whole key space, limit 10", lambda: ([(b"", TOP)], [(b"", TOP)]), 10, min(rounds, 2))
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
