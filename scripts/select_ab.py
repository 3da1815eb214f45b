"""A/B of the multi-commit kernel's tile selection on C4, inside one build and one process: the sorted-tile prefix selection
(CCSIM_DEBUG_FLAGS unset) and the REDUX rounds with the merge (CCSIM_DEBUG_FLAGS=128), run alternately on one engine with the L2
flushed before every run. One JSON line per run: kernel time, waves, waves that selected from the sorted tile, and CTA 0's cycles
per wave and phase; then the range of each arm, with the card's name, power limit and SM clock (read-only nvidia-smi queries).

    python scripts/select_ab.py [--runs 5] [--warmup 2]
"""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
synth = importlib.import_module("cluster-capacity_b200.synth")
engine = importlib.import_module("cluster-capacity_b200.engine")

PHASES = ("scan_filter_score_top8", "barrier_wait", "merge_publish", "gather_exchange_compact", "replay", "row_updates")
ARMS = (("sorted tile", 0), ("REDUX select", 128))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "sm_mhz": int(out[2]), "sm_max_mhz": int(out[3])}
    except Exception as ex:        # noqa: BLE001
        return {"gpu": None, "error": str(ex)}


def run_once(eng, flags):
    os.environ["CCSIM_DEBUG_FLAGS"] = str(flags)
    eng.flush_l2()
    r = eng.run(0)
    st = eng.run_stats()
    w = max(1, st["waves"])
    return {"flags": flags, "kernel_ms": r.run_ms, "waves": st["waves"], "placed": st["placed"], "sorted_tile_waves": eng.sorted_tile_waves(),
            "cycles_per_wave_cta0": {n: round(st["phase_cycles"][i] / w, 1) for i, n in enumerate(PHASES)},
            "pod_node_sha1": hashlib.sha1(r.pod_node.tobytes()).hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="timed runs per arm")
    ap.add_argument("--warmup", type=int, default=2, help="untimed runs per arm first")
    args = ap.parse_args()
    snap, tmpl, ctr = synth.c4()
    res = {name: [] for name, _ in ARMS}
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        for _ in range(args.warmup):
            for _, flags in ARMS:
                run_once(eng, flags)
        print(json.dumps({"card": card()}), flush=True)
        for _ in range(args.runs):
            for name, flags in ARMS:
                r = run_once(eng, flags)
                res[name].append(r)
                print(json.dumps(dict(r, arm=name)), flush=True)
        os.environ.pop("CCSIM_DEBUG_FLAGS", None)
    summary = {"card": card()}
    for name, rs in res.items():
        ms = [r["kernel_ms"] for r in rs]
        summary[name] = {"kernel_ms_min": min(ms), "kernel_ms_max": max(ms),
                         "select_cycles_per_wave": [round(sum(r["cycles_per_wave_cta0"][n] for n in PHASES[:3]), 1) for r in rs]}
    summary["same_sequence"] = len({r["pod_node_sha1"] for rs in res.values() for r in rs}) == 1
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
