"""CPU checks of the 16-byte boundary-vector helpers of k_gather_h (dbeel_b200/csrc/device_fns.cuh, compiled here by g++):
chunks16 picks which aligned source chunks hold the wanted bytes, realign16 shifts them into place, blend16 joins the tail
of one entry with the head of the next."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r"""
#include <stdint.h>
#include <string.h>
#include "device_fns.cuh"
using namespace dbeel;
extern "C" {
uint32_t shim_chunks16(uint32_t s0, uint32_t lo, uint32_t hi) { return chunks16(s0, lo, hi); }
// realign16 over a window where only the chunks chunks16 asks for are loaded; the others hold `junk`
void shim_lean16(const uint8_t src32[32], uint32_t s0, uint32_t lo, uint32_t hi, uint8_t junk, uint8_t out16[16]) {
    uint8_t w[32];
    memset(w, junk, 32);
    const uint32_t m = chunks16(s0, lo, hi);
    if (m & 1u) memcpy(w, src32, 16);
    if (m & 2u) memcpy(w + 16, src32 + 16, 16);
    uint32_t A[4], B[4], O[4];
    memcpy(A, w, 16);
    memcpy(B, w + 16, 16);
    realign16(A, B, s0, O);
    memcpy(out16, O, 16);
}
void shim_blend16(const uint8_t t16[16], const uint8_t h16[16], uint32_t t, uint8_t out16[16]) {
    uint32_t T[4], H[4], O[4];
    memcpy(T, t16, 16);
    memcpy(H, h16, 16);
    blend16(T, H, t, O);
    memcpy(out16, O, 16);
}
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("gather16")
    src, so = d / "shim.cc", d / "shim.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dbeel_b200", "csrc"),
                           "-x", "c++", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.shim_chunks16.restype = C.c_uint32
    L.shim_chunks16.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    L.shim_lean16.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint8, C.c_char_p]
    L.shim_blend16.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_char_p]
    return L


def test_chunks16_loads_only_chunks_with_wanted_bytes(shim):
    for s0 in range(16):
        for lo in range(16):
            for hi in range(lo + 1, 17):
                m = shim.shim_chunks16(s0, lo, hi)
                want = {(s0 + b) // 16 for b in range(lo, hi)}
                assert m == sum(1 << c for c in want), (s0, lo, hi)


def test_lean16_yields_the_wanted_bytes_whatever_the_skipped_chunk_holds(shim):
    rng = np.random.default_rng(23)
    out = C.create_string_buffer(16)
    for _ in range(20):
        src = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        for s0 in range(16):
            for lo, hi in [(0, t) for t in range(1, 16)] + [(t, 16) for t in range(1, 16)] + [(0, 16)]:
                for junk in (0x00, 0xA5):
                    shim.shim_lean16(src, s0, lo, hi, junk, out)
                    assert out.raw[lo:hi] == src[s0 + lo:s0 + hi], (s0, lo, hi)


def test_blend16(shim):
    rng = np.random.default_rng(29)
    out = C.create_string_buffer(16)
    for _ in range(50):
        t16, h16 = bytes(rng.integers(0, 256, 16, dtype=np.uint8)), bytes(rng.integers(0, 256, 16, dtype=np.uint8))
        for t in range(17):
            shim.shim_blend16(t16, h16, t, out)
            assert out.raw == t16[:t] + h16[t:], t
