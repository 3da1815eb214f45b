"""Per-analysis runs dealt over several devices (framework.NewEach(devices=...) + RunEach) against the same handle on device 0 alone.
Prints one JSON line.

Workloads, each on one snapshot synced once per handle:
  c2     the 512 genpod-style podspecs of scripts/each_many_bench.py (a pause pod per namespace, requests 1.5-6 CPU and 1-8 GiB) on a
         100k-node C2 cluster as API objects (synth.c2's columns: one pod per node carries the node's requests, its pod capacity is
         lowered by the pods C2 counts), every analysis run to Unschedulable and at --max-limit 1000;
  c4     the C4 family of scripts/each_coupled_bench.py as podspecs (C4's three hard spread constraints and hostname
         anti-affinity, requests and maxSkew drawn per podspec) on synth.c4_objects (100k nodes, 200k pods), 8 and 64 podspecs, to
         Unschedulable.
Each workload is timed with a host clock around RunEach (it ends when every device's share has been copied back), on [0] and on
every visible device alternately, after one warm-up run of each (the first RunEach of a handle encodes the podspecs). With one
visible device the second list is [0, 0]: the split then runs its two shares one after the other on device 0.

Every timed batch is compared with the one-device warm-up batch: stop reason (with the FitError histogram) and placement count of
every analysis, and the whole placement sequence of every analysis, except to Unschedulable on c2 (210 million placements), where the
sequences of 16 analyses spread over the list are compared.

    python scripts/each_devices_bench.py [--reps 3] [--only c2|c4] [--coupled-sizes 8,64]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
fw = importlib.import_module("cluster-capacity_b200.framework")
synth = importlib.import_module("cluster-capacity_b200.synth")
from each_many_bench import genpod_podspecs, T_ANALYSES      # noqa: E402  (the same 512 podspecs)


def gpus():
    """every card nvidia-smi lists: index, name, power limit"""
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"]).decode()
    return [dict(zip(("index", "name", "power_limit"), [x.strip() for x in line.split(",")])) for line in out.strip().splitlines()]


def visible_devices():
    import torch
    return torch.cuda.device_count()


def c2_objects(n=100_000, seed=6):
    """synth.c2's cluster as API objects: node i's allocatable, and one pod carrying its requested cpu / memory; the node's pod
    capacity is lowered so that its free pod slots are C2's"""
    snap, _, _ = synth.c2(n=n, seed=seed)
    nodes, pods = [], []
    for i in range(n):
        filler = int(snap.req_cpu[i]) > 0 or int(snap.req_mem[i]) > 0
        free = int(snap.alloc_pods[i]) - int(snap.npods[i])
        nodes.append({"apiVersion": "v1", "kind": "Node", "metadata": {"name": "node-%06d" % i, "labels": {"kubernetes.io/hostname": "node-%06d" % i}},
                      "spec": {}, "status": {"allocatable": {"cpu": "%dm" % snap.alloc_cpu[i], "memory": "%dMi" % (snap.alloc_mem[i] // synth.MiB),
                                                             "pods": str(free + (1 if filler else 0))}}})
        if filler:
            pods.append({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "used-%06d" % i, "namespace": "default"},
                         "spec": {"nodeName": "node-%06d" % i, "containers": [{"name": "c", "image": "img", "resources": {"requests": {
                             "cpu": "%dm" % snap.req_cpu[i], "memory": "%dMi" % (snap.req_mem[i] // synth.MiB)}}}]},
                         "status": {"phase": "Running"}})
    return nodes, pods


def c4_family(template, k, seed=11):
    """k podspecs of the C4 family: requests and the three maxSkews drawn per podspec (scripts/each_coupled_bench.py's draws)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for q in range(k):
        p = json.loads(json.dumps(template))
        p["metadata"]["name"] = "sim-pod-%02d" % q
        p["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "%dm" % int(rng.integers(100, 400)), "memory": "%dMi" % int(rng.integers(64, 256))}}
        for c in range(3):
            p["spec"]["topologySpreadConstraints"][c]["maxSkew"] = int(rng.integers(1, 5))
        out.append(p)
    return out


def batch(cc, seq_of):
    """one timed RunEach: (ms, [(stop reason, placements, sequence or None)] per analysis); seq_of: the analyses whose sequence is read"""
    t0 = time.perf_counter()
    res = cc.RunEach()
    ms = (time.perf_counter() - t0) * 1e3
    lib = fw.lib()
    out = [(r.StopReason(), lib.cc_scheduled_count(r._h), r.ScheduledPods() if t in seq_of else None) for t, r in enumerate(res)]
    return ms, out


def measure(name, specs, nodes, pods, limit, lists, reps, full):
    client = fw.ListClient(nodes, pods, [])
    T = len(specs)
    seq_of = set(range(T)) if full else set(np.linspace(0, T - 1, 16).astype(int).tolist())
    handles = {}
    for devices in lists:
        cc = fw.NewEach(None, None, specs, limit, [], devices=devices)
        cc.SyncWithClient(client)
        handles[tuple(devices)] = cc
    ref = None
    first_ms = {}
    for key, cc in handles.items():     # warm-up: the encoding of the podspecs and every engine
        ms, got = batch(cc, seq_of)
        first_ms[str(list(key))] = round(ms, 1)
        if ref is None:
            ref = got
        assert got == ref, "%s: the warm-up batch on %s differs from the one on [0]" % (name, list(key))
    rows = {str(list(k)): [] for k in handles}
    for _ in range(reps):
        for key, cc in handles.items():
            ms, got = batch(cc, seq_of)
            for t in range(T):
                assert got[t] == ref[t], "%s: analysis %d on %s differs from [0]" % (name, t, list(key))
            rows[str(list(key))].append(round(ms, 1))
    for cc in handles.values():
        cc.Close()
    base = float(np.median(rows[str(lists[0])]))
    return {"analyses": T, "max_limit": limit, "placements": int(sum(r[1] for r in ref)),
            "stop_reasons": sorted({r[0].split(":")[0] for r in ref}), "run_each_ms": rows, "first_run_each_ms": first_ms,
            "speedup_median": {k: round(base / float(np.median(v)), 3) for k, v in rows.items()},
            "bit_exact_batches": reps * len(lists), "sequences_compared": "all" if full else len(seq_of)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", choices=["c2", "c4"], default=None)
    ap.add_argument("--coupled-sizes", default="8,64")
    a = ap.parse_args()
    ndev = visible_devices()
    if ndev < 1:
        raise SystemExit("no CUDA device visible")
    lists = [[0], list(range(ndev)) if ndev > 1 else [0, 0]]
    res = {"gpus": gpus(), "visible_devices": ndev, "device_lists": lists}
    if a.only in (None, "c2"):
        nodes, pods = c2_objects()
        specs = genpod_podspecs(T_ANALYSES)
        for limit in (0, 1000):
            key = "c2_100k_x512_" + ("limit%d" % limit if limit else "unschedulable")
            res[key] = measure(key, specs, nodes, pods, limit, lists, a.reps, full=limit > 0)
            print(json.dumps({key: res[key]}), file=sys.stderr, flush=True)
    if a.only in (None, "c4"):
        nodes, pods, template = synth.c4_objects()
        for k in [int(x) for x in a.coupled_sizes.split(",")]:
            key = "c4_family_100k_x%d" % k
            res[key] = measure(key, c4_family(template, k), nodes, pods, 0, lists, a.reps, full=True)
            print(json.dumps({key: res[key]}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
