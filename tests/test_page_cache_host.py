"""The policy of the readers' device page cache (dbeel_b200/csrc/host/page_cache.h) on a box without a GPU
(tests/page_cache_test.cc): plans checked on a byte model of the slots, and the eviction order against a short Python
restatement of CLOCK."""
import json
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PAGE = 4096
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("page_cache") / "page_cache_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "page_cache_test.cc"), "-o", out])
    return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_page_cache_plans(exe, seed):
    out = subprocess.run([exe, "check", str(seed)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")


class Clock:
    """Second chance over `capacity` slots: a page's bit is set when it is inserted or hit; the hand passes over the
    request's own pages, clears set bits and takes the first free slot or clear bit."""

    def __init__(self, capacity):
        self.slot = [None] * capacity  # [key, ref] or None
        self.where = {}
        self.hand = 0

    def request(self, parts, ok):
        keys = []
        for table, kind, _length, ranges in parts:
            pages = sorted({p for lo, hi in ranges if lo < hi for p in range(lo // PAGE, (hi - 1) // PAGE + 1)})
            keys += [(table, kind, p) for p in pages if (table, kind, p) not in keys]
        if len(keys) > len(self.slot):
            return None
        pinned = set()
        hits = [k for k in keys if k in self.where]
        for k in hits:
            self.slot[self.where[k]][1] = True
            pinned.add(self.where[k])
        evicted, fresh = [], []
        for k in keys:  # parts in order, each part's missing pages ascending
            if k in self.where:
                continue
            while True:
                s = self.hand
                self.hand = (self.hand + 1) % len(self.slot)
                if s in pinned:
                    continue
                if self.slot[s] is None:
                    break
                if self.slot[s][1]:
                    self.slot[s][1] = False
                    continue
                evicted.append(self.slot[s][0])
                del self.where[self.slot[s][0]]
                self.slot[s] = None
                break
            pinned.add(s)
            fresh.append((k, s))
        for k, s in fresh:
            if ok:
                self.slot[s] = [k, True]
                self.where[k] = s
        return len(hits), len(fresh), evicted


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_page_cache_eviction_order_is_clock(exe, seed):
    out = subprocess.run([exe, "trace", str(seed)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    lines = [json.loads(x) for x in out.stdout.splitlines()]
    clock = Clock(lines[0]["capacity"])
    evictions = 0
    for n, req in enumerate(lines[1:]):
        parts = [(t, k, length, [tuple(r) for r in rs]) for t, k, length, rs in req["parts"]]
        got = clock.request(parts, req["ok"])
        if got is None:
            assert req["bypass"], n
            continue
        assert not req["bypass"], n
        hits, misses, evicted = got
        assert (hits, misses) == (req["hits"], req["misses"]), n
        assert [tuple(e) for e in req["evicted"]] == evicted, n
        evictions += len(evicted)
    assert evictions > 50  # the trace exercises eviction, not just a cold fill
