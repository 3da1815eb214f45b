# development check of the wave kernels on ONE H100: randomized differential tests, parity suites, full-size runs, then the C4 bench line
export CCSIM_NO_REBUILD=1
for f in tests/test_gpu_stress.py tests/test_gpu_parity.py tests/test_gpu_sharded_one_gpu.py tests/test_gpu_fullsize.py; do
  timeout 300 python -m pytest $f -m gpu -q -x 2>&1 | tail -3
done
timeout 300 python bench.py --steps 5 --warmup 3 --no-objects > /tmp/dev_bench_c4.json 2> /tmp/dev_bench_c4.err; echo "bench rc=$?"; tail -2 /tmp/dev_bench_c4.err
python - <<PY
import json
d=json.loads(open("/tmp/dev_bench_c4.json").read().strip().splitlines()[-1])
print({k:d.get(k) for k in ("value","ms_per_step","placements_per_sec")}, d["parity"]["ok"], json.dumps(d["roofline"]["latency"]))
PY
CCSIM_DEBUG_FLAGS=8 timeout 200 python scripts/perf_probe.py c4 2>&1 | tail -4
