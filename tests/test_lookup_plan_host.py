"""The read plan of dbeel_get_values_stream on a box without a GPU (tests/lookup_plan_test.cc): the fence descent plus the
resume from a leaf probes exactly what the whole-table search probes, in both modes and at every depth; that search
against the oracle's orc_sstable_lookup on real tables; leaf windows on
damaged index slices; merging of read ranges; the depth's clamps."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None or shutil.which("gcc") is None, reason="needs gcc and g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("lookup_plan")
    out, obj = str(d / "lookup_plan_test"), str(d / "dbeel_oracle.o")
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(HERE, "..", "oracle", "dbeel_oracle.c"), "-o", obj])
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "lookup_plan_test.cc"), obj, "-lm", "-o", out])
    return out


@pytest.mark.parametrize("what", ["descent", "oracle", "windows", "merge", "depth"])
def test_lookup_plan(exe, what):
    out = subprocess.run([exe, what], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
