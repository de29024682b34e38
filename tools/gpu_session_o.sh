#!/usr/bin/env bash
# Session O: Modular walk tables (tests + config 5), where the end-to-end leg's unexplained tail comes from.
set -u
OUT=gpurun_out/session_r02o
mkdir -p "$OUT"
timeout 600 python -m pytest tests/test_gpu_modular.py -m gpu -x -q > "$OUT/tests_modular.log" 2>&1; echo "modular tests rc=$?" | tee -a "$OUT/session.log"
tail -2 "$OUT/tests_modular.log" | tee -a "$OUT/session.log"
for T in 1 0; do
  echo "=== config 5, walk tables=$T" | tee -a "$OUT/session.log"
  JXG_MODULAR_WALK_TABLES=$T timeout 400 python bench.py --config 5 --steps 4 --warmup 3 > "$OUT/bench5_T$T.log" 2>&1
  grep -h '^{' "$OUT/bench5_T$T.log" | python -c "
import json,sys
for l in sys.stdin:
    d=json.loads(l); print('   value %.0f MP/s, %.2f ms/step, e2e %s' % (d['value'], d['ms_per_step'], d['e2e']))" | tee -a "$OUT/session.log"
done
run() {  # name depth env...
  local name=$1; shift
  local depth=$1; shift
  echo "=== $name depth=$depth ($(date +%T))" | tee -a "$OUT/session.log"
  env "$@" E2E_STAGING=8 E2E_MARKS=1 timeout 300 python tools/e2e_profile4.py 64 16 $depth > "$OUT/$name.log" 2>&1
  grep -h "ms/step\|main thread" "$OUT/$name.log" | tee -a "$OUT/session.log"
}
run fifo_d4 4
run fifo_d5 5
run fifo_d5_nomarks 5 E2E_MARKS=
echo "=== done ($(date +%T))" | tee -a "$OUT/session.log"
