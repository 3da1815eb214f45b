#!/bin/sh
# Round profile of the multi-commit replay on C4 (one H100): builds a profiling libccsim.so (-DMULTI_ROUND_PROFILE) in a temporary
# directory, or takes the one given as $1, and prints CTA 0's split of the replay ("Round profile" in csrc/ccsim_multi.cuh) next to
# the per-phase cycles of scripts/perf_probe.py. The shipped library is neither rebuilt nor touched. PROFILE_DEFINE picks another
# profiling build (scripts/gather_profile.sh).
set -e
PROFILE_DEFINE="${PROFILE_DEFINE:--DMULTI_ROUND_PROFILE}"
cd "$(dirname "$0")/.."
SO="$1"
if [ -z "$SO" ]; then
  TMP=$(mktemp -d)
  SO="$TMP/libccsim_profile.so"
  python - "$SO" "$PROFILE_DEFINE" <<'PY'
import importlib.util, os, subprocess, sys
spec = importlib.util.spec_from_file_location("ccbuild", "cluster-capacity_b200/build.py")
b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)
nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
subprocess.check_call([nvcc] + b.NVCC_FLAGS + [sys.argv[2], "-o", sys.argv[1]] + b.SRC)
PY
fi
CCSIM_SO="$SO" CCSIM_DEBUG_FLAGS=8 python scripts/perf_probe.py c4
