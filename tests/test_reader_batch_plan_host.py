"""The leaf grouping of dbeel_readers_get_values on a box without a GPU (tests/reader_batch_plan_test.cc): every touched
leaf in exactly one group, each pair's solo cuts kept, the budget and each page cache's capacity respected, and one pair
grouped exactly as group_leaves groups it."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("reader_batch_plan") / "reader_batch_plan_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", os.path.join(HERE, "reader_batch_plan_test.cc"), "-o", out])
    return out


@pytest.mark.parametrize("what", ["cover", "solo", "budget", "single"])
def test_reader_batch_plan(exe, what):
    out = subprocess.run([exe, what], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
