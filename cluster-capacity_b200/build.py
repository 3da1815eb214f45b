"""Builds libccsim.so in-tree for sm_90a (H100; nvcc cross-compiles without a GPU)."""
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = [os.path.join(_HERE, "csrc", "ccsim_engine.cu")]
import glob
DEPS = SRC + sorted(glob.glob(os.path.join(_HERE, "csrc", "*.cuh"))) + [os.path.join(_HERE, "..", "include", "ccsim.h")]
OUT = os.path.join(_HERE, "libccsim.so")
# -fmad=false: the float64 scorers (BalancedAllocation, Go's math.Log) must round every operation on its own, like Go on amd64;
# they use __dmul_rn/__dadd_rn intrinsics already, the flag keeps a plain a*b+c written later from being contracted silently
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC", "-lcudart", "-ldl"]


HOST_DIR = os.path.join(_HERE, "csrc", "host")
HOST_SRC = [os.path.join(HOST_DIR, "cchost.cpp")]
HOST_DEPS = HOST_SRC + [os.path.join(HOST_DIR, f) for f in ("json.hpp", "quantity.hpp", "objects.hpp", "encoder.hpp")] + [
    os.path.join(_HERE, "..", "include", "cchost.h"), os.path.join(_HERE, "..", "include", "ccsim.h")]
HOST_OUT = os.path.join(_HERE, "libcchost.so")


def build(force=False, verbose=False):
    """libccsim.so (CUDA, sm_90a) then libcchost.so (C++ host side, links libccsim via $ORIGIN rpath).
    CCSIM_NO_REBUILD=1 (set by GPU-box job scripts): use the shipped libraries as they are, whatever the source mtimes say."""
    if os.environ.get("CCSIM_NO_REBUILD") and os.path.exists(OUT) and os.path.exists(HOST_OUT) and not force:
        return OUT
    newest = max(os.path.getmtime(p) for p in DEPS)
    if force or not os.path.exists(OUT) or os.path.getmtime(OUT) < newest:
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT + ".tmp"] + SRC
        subprocess.check_call(cmd)
        os.replace(OUT + ".tmp", OUT)      # atomic: a concurrent snapshot of the tree never sees a half-written library
    newest = max([os.path.getmtime(p) for p in HOST_DEPS] + [os.path.getmtime(OUT)])
    if force or not os.path.exists(HOST_OUT) or os.path.getmtime(HOST_OUT) < newest:
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-shared", "-fPIC", "-o", HOST_OUT + ".tmp"] + HOST_SRC +
                              ["-L" + _HERE, "-lccsim", "-Wl,-rpath,$ORIGIN"])
        os.replace(HOST_OUT + ".tmp", HOST_OUT)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose=True))
