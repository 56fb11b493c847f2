"""The host side of dbeel_scan_stream on a box without a GPU (tests/scan_stream_host_test.cc): the stream pump's
per-destination output pieces, and the partition planner (dbeel_b200/csrc/host/scan_plan.h) on random and damaged trees,
checked against the records themselves and against the scan oracle's PANIC stops."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import scan_oracle
from scan_cases import DAMAGES, ERR, HASH, PANIC, damage, eighths, random_tree

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("scan_stream_host") / "scan_stream_host_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(HERE, "scan_stream_host_test.cc"), "-o", out])
    return out


def test_pump_delivers_every_destination_piece_once_and_stops_on_errors(exe):
    out = subprocess.run([exe, "pump"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")


def _plan(exe, tmp_path, tables, budgets):
    lines = [str(len(tables))]
    for t, (d, i) in enumerate(tables):
        p = tmp_path / f"t{t}.index"
        p.write_bytes(bytes(np.asarray(i, np.uint8)))
        lines.append(f"{d.size} {p}")
    out = subprocess.run([exe, "plan", *map(str, budgets)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stderr
    plans, cur = [], None
    for ln in out.stdout.split("\n"):
        f = ln.split()
        if not f:
            continue
        if f[0] == "budget":
            cur = {"budget": int(f[1]), "panic": (int(f[5]), int(f[6])), "parts": []}
            plans.append(cur)
        elif f[0] == "part":
            cur["parts"].append({"n_rec": int(f[1]), "data_bound": int(f[2]), "slices": []})
        elif f[0] == "slice":
            cur["parts"][-1]["slices"].append(tuple(int(x) for x in f[1:]))
        elif f[0] == "max_read":
            assert int(f[1]) <= 1 << 20  # the index is read in pieces, never whole
    assert len(plans) == len(budgets)
    return plans


def _records(tables):
    """(table, record, offset, full_size) in iteration order, every record of every table."""
    out = []
    for t, (_, i) in enumerate(tables):
        ix = bytes(np.asarray(i, np.uint8))
        for r in range(len(ix) // 16):
            off, _, fs = struct.unpack_from("<QII", ix, 16 * r)
            out.append((t, r, off, fs))
    return out


def _check_plan(tables, plan):
    recs = _records(tables)
    budget = plan["budget"]
    pos = 0  # next record of the sequence a partition must start at
    for part in plan["parts"]:
        n_rec = bound = win = 0
        for (t, lo, hi, wlo, whi) in part["slices"]:
            assert lo < hi and wlo < whi
            for r in range(lo, hi):  # partitions tile the sequence exactly, in order
                assert recs[pos][:2] == (t, r), (recs[pos], t, r)
                _, _, off, fs = recs[pos]
                assert wlo <= off and off + fs <= whi, "a record outside its window"
                bound += fs
                pos += 1
            n_rec += hi - lo
            win += whi - wlo
            assert whi <= tables[t][0].size
        assert n_rec == part["n_rec"] and bound == part["data_bound"]
        if n_rec > 1:
            assert win <= budget and bound + 16 * n_rec <= budget, "over budget"
        assert [s[0] for s in part["slices"]] == sorted({s[0] for s in part["slices"]})
    # the plan ends at the first record the reference would panic on, or at the end
    pt, pr = plan["panic"]
    if pt < 0:
        assert pos == len(recs)
    else:
        first_of_table = sum(1 for t, *_ in recs if t < pt)
        assert pos == first_of_table + pr
        if tables[pt][1].size < 16:  # a table with no index record
            assert pr == 0
        else:
            t, r, off, fs = recs[pos]
            assert (t, r) == (pt, pr) and (fs == 0 or off + fs > tables[t][0].size)
    return pos


def _check_against_oracle(tables, plan):
    """Where no ERR precedes it, the plan's PANIC is the oracle's stop; an earlier ERR is before the plan's end."""
    _, (st, reason, rec) = scan_oracle.scan(tables, eighths(), HASH)
    pt, pr = plan["panic"]
    if reason == PANIC:
        assert (pt, pr) == (st, rec)
    elif reason == ERR:
        assert pt < 0 or (pt, pr) > (st, rec)
    else:
        assert pt < 0


@pytest.mark.parametrize("n_tables,big", [(1, False), (8, False), (37, False), (8, True)])
def test_plan_tiles_the_records_within_budget(exe, tmp_path, n_tables, big):
    rng = np.random.default_rng(900 + n_tables + big)
    tables = random_tree(rng, n_tables, max_entries=200, big=big)
    total = sum(d.size + i.size for d, i in tables)
    budgets = [1, 40, 200, 1000, 5000, 64 << 10, total, 4 * total]
    plans = _plan(exe, tmp_path, tables, budgets)
    parts = [len(p["parts"]) for p in plans]
    assert parts[0] == len(_records(tables))  # a budget below one record: a partition per record
    assert parts[-1] == 1 and parts == sorted(parts, reverse=True)
    for plan in plans:
        _check_plan(tables, plan)
        _check_against_oracle(tables, plan)


def test_plan_of_files_the_writer_produced_has_disjoint_windows(exe, tmp_path):
    rng = np.random.default_rng(4)
    tables = random_tree(rng, 1, max_entries=400)
    for plan in _plan(exe, tmp_path, tables, [700, 3000]):
        _check_plan(tables, plan)
        wins = sorted((s[3], s[4]) for p in plan["parts"] for s in p["slices"])
        assert wins[0][0] == 0 and wins[-1][1] == tables[0][0].size
        assert all(a[1] == b[0] for a, b in zip(wins, wins[1:])), "windows of running offsets tile .data"


@pytest.mark.parametrize("kind", DAMAGES)
def test_plan_ends_at_the_first_panic(exe, tmp_path, kind):
    rng = np.random.default_rng(77)
    tables = random_tree(rng, 6, max_entries=120)
    for t, rec in [(0, 0), (2, 5), (3, 10 ** 6 + 7), (5, 119)]:
        bad = damage(tables, kind, t, rec)
        for plan in _plan(exe, tmp_path, bad, [1, 300, 4096, 1 << 30]):
            _check_plan(bad, plan)
            _check_against_oracle(bad, plan)


def test_pump_writes_at_offsets_past_4gib(exe):
    """Destination files larger than 4 GiB: pieces and their kPiece-sized calls cross 2^32 and 2^33, for the scan's
    per-destination pieces and the compaction's OutPart, and every byte lands at its full 64-bit offset once."""
    out = subprocess.run([exe, "pump-far"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")


class _Virtual:
    """A .data file that only has a length: the planner never reads .data."""

    def __init__(self, size: int):
        self.size = size


def _virtual_table(rng, panic=None):
    """About 6 GiB of .data as index records only: small records with every ~800th one a ~270 MiB record, running offsets.
    panic = (record, kind) damages one record past 2^32: "past_end" points it past the end of .data with a nonzero high
    word (truncated to 32 bits it would point inside the file), "zero" gives it full_size 0."""
    n = 20_000
    fs = rng.integers(40, 300, n).astype(np.int64)
    fs[400::800] = (270 << 20) + rng.integers(1, 4096, fs[400::800].size)
    off = np.zeros(n, np.int64)
    np.cumsum(fs[:-1], out=off[1:])
    data_len = int(off[-1] + fs[-1]) + 123
    assert data_len > 6 << 30
    if panic is not None:
        r, kind = panic
        assert off[r] > 1 << 32
        if kind == "past_end":
            off[r] = (2 << 32) | (int(off[r]) & 0xFFFFFFFF)
            assert off[r] > data_len and off[r] & 0xFFFFFFFF < data_len
        else:
            fs[r] = 0
    idx = np.zeros((n, 4), "<u4")
    idx[:, 0:2] = off.astype("<u8").view("<u4").reshape(n, 2)
    idx[:, 2] = 20
    idx[:, 3] = fs
    return data_len, off, fs, idx.view(np.uint8).reshape(-1)


def _plan_model(data_len, off, fs, budget):
    """plan_scan restated for one table: cut before the record that would take the window or the output bound
    (sum of full_size + 16) past the budget; end before the first record the reference would panic on."""
    parts, cur = [], None

    def close():
        if cur is not None:
            parts.append({"n_rec": cur[1] - cur[0], "data_bound": cur[4], "slices": [(0, cur[0], cur[1], cur[2], cur[3])]})

    for r in range(off.size):
        o, f = int(off[r]), int(fs[r])
        if f == 0 or o > data_len or f > data_len - o:
            close()
            return parts, (0, r)
        if cur is not None and (max(o + f, cur[3]) - min(o, cur[2]) > budget or cur[5] + f + 16 > budget):
            close()
            cur = None
        if cur is None:
            cur = [r, r, o, o + f, 0, 0]   # rec_lo, rec_hi, win_lo, win_hi, data_bound, out_bound
        cur[1], cur[2], cur[3] = r + 1, min(cur[2], o), max(cur[3], o + f)
        cur[4] += f
        cur[5] += f + 16
    close()
    return parts, (-1, 0)


@pytest.mark.parametrize("panic", [None, "past_end", "zero"])
def test_plan_of_a_virtual_6gib_table(exe, tmp_path, panic):
    """plan_scan over a 6 GiB table that exists only as index records: partition windows, index slices and the PANIC cut
    past 2^32 equal the Python restatement, at budgets below, at and above one large record and above 4 GiB."""
    rng = np.random.default_rng(61)
    data_len, off, fs, idx = _virtual_table(rng)
    if panic:
        r = int(np.searchsorted(off, (1 << 32) + (700 << 20)))
        data_len, off, fs, idx = _virtual_table(np.random.default_rng(61), (r, panic))
    budgets = [64 << 20, 256 << 20, 1 << 30, 5 << 30, 8 << 30]
    plans = _plan(exe, tmp_path, [(_Virtual(data_len), idx)], budgets)
    for plan in plans:
        parts, stop = _plan_model(data_len, off, fs, plan["budget"])
        assert plan["panic"] == stop
        assert plan["parts"] == parts, f"budget {plan['budget']}"
        if panic:
            assert stop[1] == r
        wins = [s[3:] for p in plan["parts"] for s in p["slices"]]
        assert any(hi > 1 << 32 for _, hi in wins), "no window reaches past 2^32"
        if plan["budget"] <= 256 << 20:
            assert any(lo > 1 << 32 for lo, _ in wins), "no window starts past 2^32"
    assert len(plans[-1]["parts"]) <= 2 and max(p["data_bound"] for p in plans[-1]["parts"]) > 4 << 30
