#!/usr/bin/env bash
# Validation of programmatic dependent launch for every kernel (TFY_PDL=1) before making it the default:
#   gpurun --timeout 900 -- tools/validate_pdl.sh 1 TAG          # one GPU: GPU test-suite + A/B bench
#   gpurun --gpus N --timeout 900 -- tools/validate_pdl.sh N TAG # N GPUs: comm / DDP checks + A/B bench (params_in_sync)
set -uo pipefail
N=${1:-1}; TAG=${2:-pdl}; OUT=gpurun_out; mkdir -p $OUT
R="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
status=0
if [ "$N" = "1" ]; then
  TFY_PDL=1 timeout 600 python -m pytest tests -m gpu -x -q 2>&1 | tail -3 | tee $OUT/${TAG}_pytest_pdl.log
  grep -q " passed" $OUT/${TAG}_pytest_pdl.log && ! grep -q "failed" $OUT/${TAG}_pytest_pdl.log || status=1
  for e in 0 1 0 1; do
    TFY_PDL=$e timeout 120 python bench.py --steps 200 --warmup 10 --repeats 7 2>/dev/null | grep "^{" | tail -1 \
      > $OUT/${TAG}_bench_N1_pdl$e.json
    python - $OUT/${TAG}_bench_N1_pdl$e.json $e <<'PY'
import json, sys
d = json.load(open(sys.argv[1]))
print(f"PDL={sys.argv[2]} us/step={d['ms_per_step'] * 1e3:.2f} e2e={d['e2e']['value']:.0f} loss_fell={d['e2e'].get('loss_fell')}")
PY
  done
else
  TFY_PDL=1 timeout 300 $R --master-port 29721 tests/gpu/comm_check.py --quick 2>&1 | grep -E "FAIL|SUMMARY" | tail -3 \
    | tee $OUT/${TAG}_comm_check_pdl.log
  grep -q "failed=0" $OUT/${TAG}_comm_check_pdl.log || status=1
  TFY_PDL=1 timeout 200 $R --master-port 29722 tests/gpu/ddp_check.py 2>&1 | grep -E "PASS|FAIL|DDP CHECK" | tail -3
  port=29730
  for e in 0 1 0 1; do
    port=$((port+1))
    TFY_PDL=$e timeout 200 $R --master-port $port bench.py --gpus $N --steps 200 --warmup 10 --repeats 7 2>/dev/null \
      | grep "^{" | tail -1 > $OUT/${TAG}_bench_N${N}_pdl$e.json
    python - $OUT/${TAG}_bench_N${N}_pdl$e.json $e <<'PY'
import json, sys
d = json.load(open(sys.argv[1]))
print(f"PDL={sys.argv[2]} us/step={d['ms_per_step'] * 1e3:.2f} sync={d.get('params_in_sync')} "
      f"loss_fell={d['e2e'].get('loss_fell')} exposed_us={d.get('exposed_comm_ms', 0) * 1e3:.1f}")
sys.exit(0 if d.get("params_in_sync") and d["e2e"].get("loss_fell") else 1)
PY
    [ $? -eq 0 ] || status=1
  done
fi
echo "validate_pdl status=$status"
exit $status
