# round-end evidence on ONE H100: the bench lines of both workloads, the GPU test suite (one pytest process per
# file under its own timeout: a hang in one file does not hide the others), the reference arm and the ncu launch list of the default
# bench command. Outputs under gpurun_out/ (copied to profiles/ afterwards).
export CCSIM_NO_REBUILD=1
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm --format=csv,noheader
timeout 400 python bench.py --steps 5 --warmup 3 > gpurun_out/r2_bench_c4.json 2> gpurun_out/r2_bench_c4.err; echo "bench c4 rc=$?"; tail -2 gpurun_out/r2_bench_c4.err
timeout 400 python bench.py --workload c5 --steps 3 --warmup 3 --no-objects > gpurun_out/r2_bench_c5.json 2> gpurun_out/r2_bench_c5.err; echo "bench c5 rc=$?"; tail -2 gpurun_out/r2_bench_c5.err
: > gpurun_out/r2_pytest_gpu.log
for f in tests/test_gpu_fullsize.py tests/test_gpu_parity.py tests/test_gpu_stress.py tests/test_gpu_sharded_one_gpu.py tests/test_gpu_framework.py tests/test_pod_list.py tests/test_golden.py tests/test_reference_outputs.py tests/test_gpu_sharded.py; do
  s=$(date +%s)
  timeout 420 python -m pytest $f -m gpu -q --durations=3 2>&1 | tail -12 > gpurun_out/_t.log
  echo "== $f rc=${PIPESTATUS[0]} $(( $(date +%s) - s ))s" | tee -a gpurun_out/r2_pytest_gpu.log
  cat gpurun_out/_t.log >> gpurun_out/r2_pytest_gpu.log; tail -1 gpurun_out/_t.log
done
rm -f gpurun_out/_t.log
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/r2_launches.csv python bench.py --steps 2 --warmup 3 --no-objects --no-parity > gpurun_out/r2_bench_under_ncu.log 2>&1; echo "ncu rc=$?"
timeout 300 python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/r2_bench_c4_ref.json 2> gpurun_out/r2_bench_c4_ref.err; echo "ref rc=$?"
python - <<PY
import json
for f in ("r2_bench_c4","r2_bench_c5","r2_bench_c4_ref"):
    try:
        d=json.loads(open("gpurun_out/%s.json"%f).read().strip().splitlines()[-1])
        print(f, {k:d.get(k) for k in ("value","ms_per_step","placements_per_sec")}, (d.get("parity") or {}).get("ok"), (d.get("e2e_objects") or {}).get("ms_per_step"), (d.get("clocks")))
    except Exception as e: print(f, "ERR", e)
PY
