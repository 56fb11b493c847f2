"""Builds libdbeel_compact.so in-tree with nvcc for sm_90a (no JIT cache, no torch extension:
the library is a plain C-ABI shared object).  `python -m dbeel_b200._build` or
__graft_entry__.build()."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdbeel_compact.so")
SOURCES = ["dbeel_compact.cu", os.path.join("host", "lsm_tree_host.cc"), os.path.join("host", "numa_bind.cc")]


def deps() -> list[str]:
    """Every file the library is compiled from: csrc/**/*.{cu,cuh,cc,h} and include/*.h."""
    out = []
    for root, _, files in os.walk(CSRC):
        out += [os.path.join(root, f) for f in files if f.endswith((".cu", ".cuh", ".cc", ".h"))]
    inc = os.path.join(HERE, "..", "include")
    out += [os.path.join(inc, f) for f in os.listdir(inc) if f.endswith(".h")]
    return out


NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libdbeel_compact.so must be built where the CUDA toolkit is")


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in deps())


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    cmd = [nvcc_path(), *NVCC_FLAGS, "-o", LIB, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd += ["-Xptxas", "-v"]
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB


def build_variant(name: str, defines: list[str]) -> str:
    """A/B builds for tools/tune.py (`LIB=<path>` in a spec): same sources, extra -D flags, own file name."""
    out = os.path.join(HERE, f"libdbeel_compact.{name}.so")
    cmd = [nvcc_path(), *NVCC_FLAGS, *[f"-D{d}" for d in defines], "-o", out, *[os.path.join(CSRC, s) for s in SOURCES]]
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    if "--variant" in sys.argv:  # python -m dbeel_b200._build --variant vpt2 DBEEL_GATHER_H_VPT=2
        k = sys.argv.index("--variant")
        print(build_variant(sys.argv[k + 1], sys.argv[k + 2:]))
    else:
        print(build(force="--force" in sys.argv, verbose=True))
