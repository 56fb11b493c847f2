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
With --reverse, range reads from the end (dbeel_reader_get_ranges_reverse) on the same tree: per batch, limit and end
key distribution (uniform or Zipf(1.1), as the starts above), the last `limit` entries below each end key against the
forward mirror -- get_ranges of the same number of entries from the other side of the same key -- and against get_range
in non-overlapping calls reversed and cut on the host, its ranges starting 2 * limit keys below the end; and the last 10
entries of the whole key space against its first 10 and against get_range of the whole key space plus a host tail cut.
Parity on every round: every reverse query's entries equal the last entries of get_range's answer, reversed (all of it
when that answer is shorter than the limit and its range started at the bottom of the key space).  Results: DESIGN.md
section 7, "Range reads from the end".
Usage: tools/reader_ranges_bench.py [keys_per_run (default 1000000)] [--rounds R] [--reverse] [--out result.json]"""
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


def last_entries(data, index, n, limit):
    """The last `limit` of the n entries of one get_range answer, in descending key order, as one byte string."""
    ix = np.asarray(index, np.uint8).reshape(-1, 16)
    out = []
    for k in range(n - 1, max(0, n - limit) - 1, -1):
        off, fs = int(ix[k, :8].view("<u8")[0]), int(ix[k, 12:16].view("<u4")[0])
        out.append(bytes(data[off:off + fs]))
    return b"".join(out)


def truncated_get_range(reader, ranges, limit, reverse=False):
    """get_range in calls of up to 256 ranges that do not overlap (calls_of), every answer cut to its first `limit` entries
    on the host (reverse: its last, in descending order): [(entry bytes, entries in the whole answer)], and the calls'
    dbeel_last_stats summed."""
    uniq = sorted(set(ranges))  # a caller asks a repeated range once
    out, tot = {}, {"input_bytes": 0, "entries_out": 0, "partitions": 0, "reads": 0}  # reads: the counting reader's
    for call in calls_of(uniq):
        got, _ = reader.get_range([uniq[q] for q in call])
        st = dict(reader._engine.stats(), reads=len(reader.last_stream_reads or ()))
        for k in tot:
            tot[k] += int(st[k])
        for q, (d, i) in zip(call, got):
            n = i.size // 16
            out[uniq[q]] = (last_entries(d, i, n, limit) if reverse else entries(d, i, 0, min(n, limit)), n)
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
    reverse = "--reverse" in argv
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
    result = {"gpu": gpu, "power_limit": power, "reverse": reverse, "rows": []}
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

        def run_row_reverse(name, make, limit, r_count):
            arms = ("get_ranges_reverse", "get_ranges_forward_mirror", "get_range_reversed")
            t = {a: [] for a in arms}
            st, parity = {}, True
            for r in range(r_count + 1):  # round 0 warms up
                rq, fq, gr = make()
                t0 = time.perf_counter()
                rows, data, index = reader.get_ranges(rq, limit, reverse=True)
                t1 = time.perf_counter()
                st[arms[0]] = eng.stats()
                reader.get_ranges(fq, limit)
                t2 = time.perf_counter()
                st[arms[1]] = eng.stats()
                want, st[arms[2]] = truncated_get_range(reader, gr, limit, reverse=True)
                t3 = time.perf_counter()
                for q, (w, n_all) in enumerate(want):
                    got = entries(data, index, int(rows[q]["first"]), int(rows[q]["count"]))
                    more = bool(rows[q]["flags"] & capi.RANGE_MORE)
                    if gr[q][0] == b"":  # both asked the rest of the key space below the end
                        parity = parity and got == w and more == (n_all > limit)
                    elif n_all >= limit:
                        parity = parity and got == w and (more or n_all == limit)
                    else:  # the guessed start cut get_range's answer short
                        parity = parity and got[:len(w)] == w
                if r:
                    t[arms[0]].append(t1 - t0)
                    t[arms[1]].append(t2 - t1)
                    t[arms[2]].append(t3 - t2)
            counting.get_ranges(rq, limit, reverse=True)
            n_reads = {arms[0]: len(counting.last_stream_reads)}
            rounds_c = {arms[0]: int(eng.stats()["partitions"])}
            counting.get_ranges(fq, limit)
            n_reads[arms[1]] = len(counting.last_stream_reads)
            rounds_c[arms[1]] = int(eng.stats()["partitions"])
            n_reads[arms[2]] = truncated_get_range(counting, gr, limit, reverse=True)[1]["reads"]
            row = {"row": name, "parity": bool(parity), "arms": {}}
            for arm in arms:
                row["arms"][arm] = {"wall_ms": float(np.median(t[arm])) * 1e3, "bytes_read": int(st[arm]["input_bytes"]),
                                    "reads": n_reads[arm], "rounds": int(st[arm]["partitions"]) if arm in rounds_c else None,
                                    "entries": int(st[arm]["entries_out"])}
                if arm in rounds_c:
                    row["arms"][arm]["rounds_counting_reader"] = rounds_c[arm]
            result["rows"].append(row)
            print(json.dumps(row), flush=True)

        for batch in BATCHES:
            for limit in LIMITS:
                for dist in ("uniform", "zipf"):
                    if reverse:  # the last `limit` entries below keys[j]; the mirror: the first `limit` from keys[j] on
                        def make(batch=batch, limit=limit, dist=dist):
                            js = starts(batch, dist)
                            rq = [(b"", keys[j].tobytes()) for j in js]
                            fq = [(keys[j].tobytes(), TOP) for j in js]
                            gr = [(keys[j - 2 * limit].tobytes() if j >= 2 * limit else b"", keys[j].tobytes()) for j in js]
                            return rq, fq, gr
                        run_row_reverse(f"batch {batch}, limit {limit}, {dist} ends", make, limit, rounds)
                        continue

                    def make(batch=batch, limit=limit, dist=dist):
                        js = starts(batch, dist)
                        qs = [(keys[j].tobytes(), TOP) for j in js]
                        gr = [(keys[j].tobytes(), keys[j + 2 * limit].tobytes() if j + 2 * limit < nk else TOP) for j in js]
                        return qs, gr
                    run_row(f"batch {batch}, limit {limit}, {dist}", make, limit, rounds)
        if reverse:
            run_row_reverse("whole key space, last 10", lambda: ([(b"", TOP)], [(b"", TOP)], [(b"", TOP)]), 10, min(rounds, 2))
        else:
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
