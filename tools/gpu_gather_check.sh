#!/bin/bash
# k_gather_h (the default gather) against k_gather32 (DBEEL_GATHER=10) in one call: GPU suite and parity sweep with the default,
# bench.py outputs of both compared file by file, bench headline and gather stage times alternated, smoke().
# The full bench line (parity of every rank, other_configs) is a separate bench.py run.  Results go to $GATHER_OUT
# (default gather_out/).
OUT=${GATHER_OUT:-gather_out}
mkdir -p "$OUT"
DUMP=$(mktemp -d)
trap 'rm -rf "$DUMP"' EXIT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/check_gpu.csv
# an unset variable selects the default; DBEEL_GATHER= (empty) would select variant 0
run() { if [ -n "$1" ]; then env DBEEL_GATHER=$1 "${@:2}"; else "${@:2}"; fi; }
echo "=== pytest -m gpu (default)"
timeout 300 python -m pytest tests -m gpu -q 2>&1 | tail -2 | tee -a $OUT/check_pytest.txt
echo "=== parity sweep (default)"
timeout 300 python tools/parity_sweep.py 200 2>&1 | tail -2 | tee $OUT/check_sweep.txt
for r in 1 2 3; do
    for v in 10 ""; do
        run "$v" timeout 120 python bench.py --gpus 1 --steps 10 --warmup 3 --no-cpu --no-others 2>&1 | tail -1 |
            python -c "import json,sys; d=json.loads(sys.stdin.read()); print('DBEEL_GATHER=${v:-default}', d['value'], d['stage_ms'])" |
            tee -a $OUT/check_bench_ab.txt
    done
done
for v in 10 ""; do
    run "$v" timeout 120 python bench.py --gpus 1 --steps 2 --warmup 1 --no-cpu --no-others --dump-outputs "$DUMP/${v:-new}" > /dev/null 2>&1
done
DUMP="$DUMP" python - <<'EOF' 2>&1 | tee $OUT/check_dump.txt
import glob, os
import numpy as np
d = os.environ["DUMP"]
a, b = sorted(glob.glob(f"{d}/10/*.npy")), sorted(glob.glob(f"{d}/new/*.npy"))
assert a and [os.path.basename(x) for x in a] == [os.path.basename(x) for x in b], (len(a), len(b))
bad = [os.path.basename(x) for x, y in zip(a, b) if not np.array_equal(np.load(x), np.load(y))]
print(f"{len(a)} dump files, identical: {not bad}", bad)
EOF
timeout 120 python tools/gather_ab.py --rounds 3 --json $OUT/check_gather_ab.json "DBEEL_GATHER=10" "" 2>&1 | grep -v "^\[" | tee $OUT/check_gather_ab.txt
python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" 2>&1 | tail -1 | tee $OUT/check_smoke.txt
nvidia-smi --query-gpu=name,power.limit,clocks.sm --format=csv,noheader | tee -a $OUT/check_gpu.csv
