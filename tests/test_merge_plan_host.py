"""plan_merge (dbeel_b200/csrc/host/scan_plan.h), the key-aligned partition planner of dbeel_reader_get_range, on a box
without a GPU (tests/merge_plan_test.cc): tiling, key intervals, the budget bound with long shared-prefix keys, monotone
cuts on shuffled tables, and no planner reads when the spans fit one partition."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("merge_plan") / "merge_plan_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "merge_plan_test.cc"), "-o", out])
    return out


@pytest.mark.parametrize("mode", ["random", "prefix", "shuffled", "damaged", "one"])
def test_merge_plan(exe, mode):
    out = subprocess.run([exe, mode], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
