#!/bin/bash
# One run that validates a build end to end on an H100:
#   ./tools/gpu_round.sh
# parity tests, smoke, the bench line, the reference arm, cfg5, the ncu launch list and one --set full capture
# of the pipeline's kernels (summarise with tools/ncu_summary.py / tools/sass_hotspots.py).
set -u
mkdir -p gpurun_out
nvidia-smi -L
echo "=== pytest -m gpu (full)"
timeout 900 python -m pytest tests -m gpu -q 2>&1 | tail -4
echo "=== smoke"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
echo "=== bench (default)"
timeout 1200 python bench.py > gpurun_out/bench.json 2> gpurun_out/bench.err; tail -4 gpurun_out/bench.err; cut -c1-1500 gpurun_out/bench.json
echo "=== bench reference arm"
timeout 900 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/bench_ref.json 2> gpurun_out/bench_ref.err; tail -2 gpurun_out/bench_ref.err; cut -c1-600 gpurun_out/bench_ref.json
echo "=== cfg5 (BASELINE configs[4]), full stream on this one GPU"
timeout 1200 python bench.py --workload cfg5 --steps 2 --warmup 1 > gpurun_out/bench_cfg5.json 2> gpurun_out/bench_cfg5.err; tail -3 gpurun_out/bench_cfg5.err; cut -c1-900 gpurun_out/bench_cfg5.json
echo "=== ncu launch list (DBEEL_PIPELINE=0 keeps the host-path part of bench.py to one job per call)"
DBEEL_PIPELINE=0 timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 200 --csv --log-file gpurun_out/launches.csv \
    python bench.py --steps 2 --warmup 1 --no-cpu > gpurun_out/bench_under_ncu.log 2>&1
grep -c . gpurun_out/launches.csv
echo "=== ncu full (one cfg2 job, every kernel of the pipeline; then the fused variant's kernel)"
timeout 1500 ncu --set full --clock-control none --import-source on -s 57 -c 19 -f -o gpurun_out/prof_full python tools/tune.py "" > gpurun_out/prof_full.log 2>&1
DBEEL_FUSED_FINAL=1 timeout 900 ncu --set full --clock-control none --import-source on -k regex:k_merge_final -s 3 -c 1 -f -o gpurun_out/prof_fused python tools/tune.py "DBEEL_FUSED_FINAL=1" > gpurun_out/prof_fused.log 2>&1
echo "=== memcheck: one scaled cfg2 job through the default path and the fused one"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 python -c "
import os, numpy as np
from dbeel_b200 import capi, workloads as W
import oracle
runs = W.make_merge_runs(W.scaled(W.CFG2, 30000)); seed = bytes(range(32))
exp = oracle.compact(runs, False, seed=seed)
for env in ({}, {'DBEEL_FUSED_FINAL': '1'}):
    os.environ.update(env); e = capi.Engine(0); g = e.compact(runs, False, seed=seed); e.close()
    for k in env: del os.environ[k]
    print(env, all(np.array_equal(a, b) for a, b in zip(g[:3], exp[:3])))
" 2>&1 | tail -8 | tee gpurun_out/sanitizer.txt
ls -la gpurun_out/ | tail -12
