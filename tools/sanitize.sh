#!/usr/bin/env bash
# Race / memory checking of the single-GPU kernels (run on an H100):
#   gpurun --timeout 1500 -- tools/sanitize.sh          (SAN_TIMEOUT=<s> bounds each run; rc=124 = cut off, not an error)
# Writes gpurun_out/sanitizer_<tool>_<suite>.log plus a one-line-per-run summary (sanitizer_summary.txt) and
# FAILS (exit 1) when a tool reports an error.  The reference has no sanitizer usage at all (SURVEY.md §5.2).
# Cross-GPU flag protocols (system-scope release/acquire over NVLink) are outside what racecheck models: the
# protocol is model-checked on the CPU (tests/test_barrier_protocol_model.py, every interleaving) and the
# multi-GPU kernels are covered by tests/gpu/comm_check.py + ddp_check.py (pytest -m gpu on a multi-GPU box).
set -uo pipefail
OUT=${1:-gpurun_out}
mkdir -p "$OUT"
SUMMARY="$OUT/sanitizer_summary.txt"
: > "$SUMMARY"
status=0
run() {  # tool suite command...
  local tool=$1 suite=$2; shift 2
  local log="$OUT/sanitizer_${tool}_${suite}.log"
  timeout ${SAN_TIMEOUT:-1200} compute-sanitizer --tool "$tool" --error-exitcode 99 --log-file "$log" "$@" > "$OUT/sanitizer_${tool}_${suite}.out" 2>&1
  local rc=$?
  local verdict
  verdict=$(grep -E "ERROR SUMMARY|RACECHECK SUMMARY" "$log" | tail -1)
  echo "$tool $suite rc=$rc :: ${verdict:-no summary line}" | tee -a "$SUMMARY"
  if [ $rc -ne 0 ] && [ $rc -ne 124 ]; then status=1; fi
}
K="nn_kernels or fused_step_local or wgmma or dense_head or dense_backward"
run memcheck  engine python -m pytest tests/test_gpu_engine.py -m gpu -q -x -k "$K"
run racecheck engine python -m pytest tests/test_gpu_engine.py -m gpu -q -x -k "$K"
run memcheck  conv   python tests/gpu/conv_check.py 2
run racecheck conv   python tests/gpu/conv_check.py 2
run initcheck engine python -m pytest tests/test_gpu_engine.py -m gpu -q -x -k "dense_backward or 2cta"
exit $status
