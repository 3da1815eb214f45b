"""Per-analysis runs of coupled podspecs (ccsim_set_analyses + ccsim_run_each) against one ccsim_run per template, on C4's 100k-node
snapshot. Prints one JSON line.

Workload: T C4-family templates (C4's three hard spread constraints and hostname anti-affinity, requests and maxSkew drawn per
template), T = 8 and 64, every analysis run to Unschedulable. One launch of the per-analysis kernel is timed with device events
(ccsim_result.run_ms) against the sum of the T ccsim_run launches (multi-commit kernel), alternately after a warm-up. Every timed batch
is compared bit-exact with the single-template runs of the same round: sequence, stop code, FitError histogram.

    python scripts/each_coupled_bench.py [--reps 2] [--sizes 8,64]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
abi = importlib.import_module("cluster-capacity_b200._abi")
engine = importlib.import_module("cluster-capacity_b200.engine")
synth = importlib.import_module("cluster-capacity_b200.synth")


def gpu_info():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def family(snap_t0_ctr, k, seed=11):
    _, t0, _ = snap_t0_ctr
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(k):
        t = abi.Template.from_buffer_copy(t0)
        t.req_cpu = t.least_cpu = t.bal_cpu = t.nz_cpu = int(rng.integers(100, 400))
        t.req_mem = t.least_mem = t.bal_mem = t.nz_mem = int(rng.integers(64, 256)) * synth.MiB
        for c in range(3):
            t.pts[c].max_skew = int(rng.integers(1, 5))
        out.append(t)
    return out


def same(a, b):
    return a.placed == b.placed and a.stop_code == b.stop_code and np.array_equal(a.pod_node, b.pod_node) and \
        np.array_equal(a.reason_hist, b.reason_hist)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sizes", default="8,64")
    a = ap.parse_args()
    name, power = gpu_info()
    snap, (t0,), ctr = synth.c4()
    base = (snap, t0, ctr)
    res = {"gpu": name, "power_limit": power, "workload": "C4 family, 100k nodes, to Unschedulable", "sizes": {}}
    with engine.Engine(device=0) as each, engine.Engine(device=0) as one:
        each.load_nodes(snap)
        one.load_nodes(snap)
        for T in [int(x) for x in a.sizes.split(",")]:
            tmpl = family(base, T)
            each.set_analyses(tmpl, [(ctr, snap.topo)] * T)
            each_ms, single_ms, placed = [], [], 0
            for rep in range(a.reps + 1):              # rep 0 warms both paths up
                got = each.run_each(0)
                want, ms = [], 0.0
                for t in tmpl:
                    one.set_templates([t], ctr)
                    r = one.run(0)
                    want.append(r)
                    ms += r.run_ms
                assert one.kernel_name().startswith("multi"), one.kernel_name()
                for t in range(T):
                    assert same(got[t], want[t]), "analysis %d differs from ccsim_run" % t
                if rep:
                    each_ms.append(got[0].run_ms)
                    single_ms.append(ms)
                placed = sum(g.placed for g in got)
            res["sizes"][str(T)] = {"each_launch_ms": each_ms, "single_runs_ms": single_ms, "placed_total": placed,
                                    "rebuilds": each.run_stats()["rebuilds"], "bit_exact": True}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
