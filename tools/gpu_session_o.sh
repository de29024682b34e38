#!/usr/bin/env bash
# Session O: Modular tests, and where the end-to-end leg's unexplained tail comes from.
set -u
OUT=gpurun_out/session_r02o
mkdir -p "$OUT"
timeout 600 python -m pytest tests/test_gpu_modular.py -m gpu -x -q > "$OUT/tests_modular.log" 2>&1; echo "modular tests rc=$?" | tee -a "$OUT/session.log"
tail -2 "$OUT/tests_modular.log" | tee -a "$OUT/session.log"
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
