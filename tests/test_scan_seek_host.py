"""plan_scan with record spans (dbeel_reader_scan's key ranges, dbeel_b200/csrc/host/scan_plan.h) on a box without a GPU
(tests/scan_seek_host_test.cc): the plan of the spans is the plan of the tables cut down to them with record numbers mapped
back, whole-table spans give today's plan, and only the span slices are read."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from scan_cases import DAMAGES, damage, random_tree

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("scan_seek_host") / "scan_seek_host_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "scan_seek_host_test.cc"), "-o", out])
    return out


def _check(exe, tmp_path, tables, spans, budgets):
    lines = [str(len(tables))]
    for t, ((d, i), sp) in enumerate(zip(tables, spans)):
        p = tmp_path / f"t{t}.index"
        p.write_bytes(bytes(np.asarray(i, np.uint8)))
        lines.append(f"{d.size} {p} {len(sp)} " + " ".join(f"{lo} {hi}" for lo, hi in sp))
    out = subprocess.run([exe, "spans", *map(str, budgets)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def random_spans(rng, n):
    """Ascending disjoint record intervals of a table of n records: none, all, single records, gaps, adjacent pieces."""
    style = int(rng.integers(0, 5))
    if n == 0 or style == 0:
        return []
    if style == 1:
        return [(0, n)]
    cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, int(rng.integers(2, 12)))))
    sp = []
    for a, b in zip(cuts, cuts[1:]):
        if rng.random() < 0.6:
            if sp and sp[-1][1] == a and rng.random() < 0.5:
                sp[-1] = (sp[-1][0], b)  # spans are merged: neighbours that touch are one span
            else:
                sp.append((a, b))
    return sp


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("big", [False, True])
def test_span_plan_is_the_plan_of_the_cut_tables(exe, tmp_path, seed, big):
    rng = np.random.default_rng(3100 + seed + 100 * big)
    tables = random_tree(rng, int(rng.integers(1, 7)), max_entries=150, big=big)
    spans = [random_spans(rng, i.size // 16) for _, i in tables]
    total = sum(d.size + i.size for d, i in tables)
    _check(exe, tmp_path, tables, spans, [1, 40, 300, 2000, 64 << 10, total])


@pytest.mark.parametrize("kind", [k for k in DAMAGES if k != "ragged_index"])
def test_span_plan_with_panics_inside_between_and_outside_spans(exe, tmp_path, kind):
    rng = np.random.default_rng(57)
    tables = random_tree(rng, 5, max_entries=100)
    for t, rec in [(0, 0), (2, 7), (3, 40), (4, 99)]:
        bad = damage(tables, kind, t, rec)
        n = bad[t][1].size // 16
        r = rec % max(1, n)
        for sp_t in ([(0, n)], [(r, min(n, r + 3))], [(0, r), (min(n, r + 1), n)], [(max(0, r - 2), r)], []):
            spans = [random_spans(rng, i.size // 16) for _, i in bad]
            spans[t] = [(a, b) for a, b in sp_t if a < b]
            _check(exe, tmp_path, bad, spans, [1, 300, 4096, 1 << 30])


def test_empty_tables_and_whole_spans(exe, tmp_path):
    rng = np.random.default_rng(8)
    tables = random_tree(rng, 4, max_entries=60)
    tables[2] = (tables[2][0], tables[2][1][:0])  # no index record: a PANIC at (2, 0) whatever the spans
    _check(exe, tmp_path, tables, [[(0, i.size // 16)] for _, i in tables], [1, 500, 1 << 30])
    _check(exe, tmp_path, tables, [[], [(1, 3)], [], [(0, 2)]], [1, 500, 1 << 30])
