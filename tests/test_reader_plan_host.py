"""The plan rules of readers (dbeel_reader_*) on a box without a GPU (tests/reader_plan_test.cc): the fence depth of every
table and its bounds, the exactness premise of cached fences, and when a batch falls back to reading fences per call."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("reader_plan") / "reader_plan_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "reader_plan_test.cc"), "-o", out])
    return out


@pytest.mark.parametrize("what", ["depths", "premise", "fallback"])
def test_reader_plan(exe, what):
    out = subprocess.run([exe, what], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
