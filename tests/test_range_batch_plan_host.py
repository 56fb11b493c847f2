"""The packing of dbeel_readers_get_ranges' seek batches and query groups on a box without a GPU
(tests/range_batch_plan_test.cc): every unit in exactly one group, each batch's solo groups kept, the budget and each page
cache's capacity respected, and one batch grouped exactly as its solo call groups it."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("range_batch_plan") / "range_batch_plan_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", os.path.join(HERE, "range_batch_plan_test.cc"), "-o", out])
    return out


@pytest.mark.parametrize("what", ["cover", "solo", "budget", "single"])
def test_range_batch_plan(exe, what):
    out = subprocess.run([exe, what], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
