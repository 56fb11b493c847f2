#!/usr/bin/env python
"""SASS evidence for DESIGN.md's hardware claims: per kernel of libdbeel_compact.so, how many bulk-copy (UBLKCP / UTMALDG),
mbarrier (SYNCS), cp.async (LDGSTS), 128- and 256-bit global load / store and warp-reduction (REDUX) instructions the sm_90a
binary holds, plus the first occurrences verbatim.  Usage: tools/sass_evidence.py [kernel ...]"""
import os
import re
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dbeel_b200", "libdbeel_compact.so")
PATTERNS = OrderedDict([
    ("UBLKCP (cp.async.bulk, TMA 1-D)", r"\bUBLKCP"), ("UTMALDG/UTMASTG (tensor TMA)", r"\bUTMA(LDG|STG)"),
    ("SYNCS (mbarrier)", r"\bSYNCS"), ("LDGSTS (cp.async)", r"\bLDGSTS"), ("LDG.E.*128", r"\bLDG\.E[\w.]*\.128"),
    ("LDG.E.*256", r"\bLDG\.E[\w.]*\.256"), ("STG.E.*128", r"\bSTG\.E[\w.]*\.128"), ("STG.E.*256", r"\bSTG\.E[\w.]*\.256"),
    ("LDS.128", r"\bLDS\.128"), ("REDUX", r"\bREDUX"), ("SHF (funnel shift)", r"\bSHF\."), ("ATOMG/RED (global atomics)", r"\b(ATOMG|RED)\."),
])


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    kernels = OrderedDict()
    cur = None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
            kernels[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4}\*/", ln):
            kernels[cur].append(re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ln).strip())
    print(f"# {os.path.relpath(LIB, ROOT)}: {len(kernels)} kernels, sm_90a SASS (cuobjdump -sass)\n")
    want = sys.argv[1:] or ["k_gather_h", "k_merge_final", "k_merge_tma", "k_extract", "k_resolve", "k_emit", "k_route_hash",
                            "k_memtable_cuts"]
    for name, lines in kernels.items():
        short = name.split("::")[-1].split("<")[0]
        if short not in want:
            continue
        print(f"## {name}  ({len(lines)} instructions)")
        for label, pat in PATTERNS.items():
            hits = [l for l in lines if re.search(pat, l)]
            if hits:
                print(f"  {label:32s} x{len(hits):<4d} e.g. {hits[0]}")
        print()


if __name__ == "__main__":
    main()
