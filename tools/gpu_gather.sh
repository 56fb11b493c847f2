#!/bin/bash
# Gather attribution on one GPU in one call: the card, the practical copy ceiling, the stage times of gather variants
# alternated round by round on the same cfg2 input, and per-kernel times from torch.profiler in a run of their own.
# With arguments they replace the default spec list (tools/gather_ab.py's syntax); LIB=<name> specs need their builds
# (python -m dbeel_b200._build --variant <name> -D...) in the tree first.  Results go to $GATHER_OUT (default gather_out/).
OUT=${GATHER_OUT:-gather_out}
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee "$OUT/gpu.csv"
if [ $# -eq 0 ]; then
    set -- "" "DBEEL_GATHER=10" "DBEEL_GATHER=0" "DBEEL_GATHER=1" "DBEEL_GATHER=4" "DBEEL_GATHER=6" "DBEEL_GATHER=10,DBEEL_BLOOM_SIDE=1" \
        --profile "" --profile "DBEEL_BLOOM_SIDE=1"
fi
timeout 1200 python tools/gather_ab.py --rounds 3 --json "$OUT/gather_ab.json" "$@" 2>&1 | grep -v "^\[" | tee "$OUT/gather_ab.txt"
nvidia-smi --query-gpu=name,power.limit,clocks.sm --format=csv,noheader | tee -a "$OUT/gpu.csv"
