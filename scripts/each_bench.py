"""Per-analysis runs (ccsim_run_each) against one ccsim_run per template, on the same snapshot. Prints one JSON line.

Workloads:
  (a) C5: 1M nodes and its 64 podspecs (synth.c5), --max-limit 6400 for every analysis;
  (b) a 100k-node C2 cluster and 16 podspecs that differ in their requests, every analysis run to Unschedulable.
The two ways are timed alternately after a warm-up, with device events (ccsim_result.run_ms) and a host clock around each batch
(every call ends in a device synchronise). Every timed batch is compared bit-exact with the single-template runs of the same
round: sequence, stop code, FitError histogram. On (a) four analyses are also compared with the memoised C oracle.

    python scripts/each_bench.py [--reps 3] [--only a|b]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

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


def workload_b():
    snap, _, _ = synth.c2(n=100_000, seed=6)
    rng = np.random.Generator(np.random.PCG64(16))
    tmpl = [abi.default_template(int(rng.integers(1500, 6001)), int(rng.integers(1024, 8193)) * synth.MiB) for _ in range(16)]
    return snap, tmpl, 0


def same(a, b):
    return (a.placed == b.placed and a.stop_code == b.stop_code and np.array_equal(a.pod_node, b.pod_node)
            and np.array_equal(a.reason_hist, b.reason_hist))


def bench(name, snap, tmpl, limit, reps, oracle_checks):
    each = engine.Engine(device=0)
    each.load_nodes(snap)
    each.set_templates(tmpl)
    singles = []
    for t in tmpl:
        e = engine.Engine(device=0)
        e.load_nodes(snap)
        e.set_templates([t])
        singles.append(e)
    # warm-up of both ways (module loads, allocations of every buffer the timed calls use)
    want = [e.run(limit) for e in singles]
    got = each.run_each(limit)
    assert all(same(g, w) for g, w in zip(got, want)), "warm-up: per-analysis runs differ from the single-template runs"
    stats = each.run_stats()
    rows = {"each_ms": [], "each_wall_ms": [], "single_ms": [], "single_wall_ms": []}
    for _ in range(reps):
        t0 = time.perf_counter()
        got = each.run_each(limit)
        rows["each_wall_ms"].append((time.perf_counter() - t0) * 1e3)
        rows["each_ms"].append(got[0].run_ms)
        t0 = time.perf_counter()
        want = [e.run(limit) for e in singles]
        rows["single_wall_ms"].append((time.perf_counter() - t0) * 1e3)
        rows["single_ms"].append(sum(w.run_ms for w in want))
        for t, (g, w) in enumerate(zip(got, want)):
            assert same(g, w), "%s: analysis %d differs from its single-template run" % (name, t)
    checked = []
    if oracle_checks:
        from oracle import binding as oracle
        for t in oracle_checks:
            ref = oracle.run(snap, [tmpl[t]], max_pods=limit, memo=True, threads=8)
            assert same(got[t], ref), "%s: analysis %d differs from the C oracle" % (name, t)
            checked.append(t)
    placed = [g.placed for g in got]
    med = lambda v: float(np.median(v))
    out = {
        "nodes": snap.n, "analyses": len(tmpl), "max_limit": limit, "placed_total": int(sum(placed)),
        "placed_min": int(min(placed)), "placed_max": int(max(placed)),
        "stop_codes": sorted(set(int(g.stop_code) for g in got)),
        "each_ms": [round(x, 3) for x in rows["each_ms"]], "single_ms": [round(x, 3) for x in rows["single_ms"]],
        "each_wall_ms": [round(x, 3) for x in rows["each_wall_ms"]], "single_wall_ms": [round(x, 3) for x in rows["single_wall_ms"]],
        "each_placements_per_s": round(sum(placed) / (med(rows["each_ms"]) / 1e3)),
        "single_placements_per_s": round(sum(placed) / (med(rows["single_ms"]) / 1e3)),
        # one analysis places its clones one after another, concurrently with the others: the launch over its longest analysis
        "each_us_per_placement_per_analysis": round(med(rows["each_ms"]) * 1e3 / max(1, max(placed)), 3),
        "single_us_per_placement": round(med(rows["single_ms"]) * 1e3 / max(1, sum(placed)), 3),
        "speedup_device": round(med(rows["single_ms"]) / med(rows["each_ms"]), 2),
        "tree_levels_global": stats["global_levels"], "tree_levels_shared": stats["shared_levels"], "smem_bytes": stats["smem_bytes"],
        "bit_exact_batches": reps, "oracle_checked_analyses": checked,
    }
    each.close()
    for e in singles:
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", choices=["a", "b"], default=None)
    a = ap.parse_args()
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power}
    if a.only in (None, "a"):
        snap, tmpl, _ = synth.c5()
        res["a_c5_1M_x64_limit6400"] = bench("a", snap, tmpl, 6400, a.reps, oracle_checks=[0, 21, 42, 63])
    if a.only in (None, "b"):
        snap, tmpl, limit = workload_b()
        res["b_c2_100k_x16_unschedulable"] = bench("b", snap, tmpl, limit, a.reps, oracle_checks=[])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
