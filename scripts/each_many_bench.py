"""Per-analysis runs past the SM count: 512 genpod-style podspecs (a pause pod per namespace whose requests are the namespace's
LimitRange maximum) against a 100k-node C2 cluster, every analysis run to Unschedulable and at --max-limit 1000. Prints one JSON line.

Three ways of running the same 512 analyses are timed alternately after a warm-up, with device events (ccsim_result.run_ms: the
per-analysis kernel) and a host clock around each batch (every call ends in a device synchronise):
  packed   one ccsim_run_each over all 512 (node-local analyses beyond the resident CTAs: several per CTA, one warp each);
  queued   the same launch with one CTA per analysis (grid = 512, CCSIM_DEBUG_FLAGS bit 8), for the comparison;
  chunks   eight ccsim_run_each of 64 analyses each (the only way before the bound was raised).
Every timed batch is compared bit-exact with the others (sequence, stop code, FitError histogram, preemption counters); at
--max-limit 1000 every analysis is also compared with ccsim_run of its template alone, to Unschedulable a sample of 8 (a single
run there takes seconds).

The host part times cc_new_each + SyncWithClient + the encoding of 512 podspecs on synth.c4_objects (100k nodes, 200k pods): the
encoding is the first RunEach minus the second one on the same handle (the second reuses the encoding). `--host-root DIR` also
times the host library of another checkout (built there), e.g. the parent commit's, alternately with this one; a build whose
per-analysis handles take 64 podspecs runs eight handles of 64, each syncing and encoding the snapshot, and the times are summed.

    python scripts/each_many_bench.py [--reps 3] [--host-root DIR] [--only engine|host]
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
T_ANALYSES = 512


def gpu_info():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def genpod_requests(k, seed=12):
    """(cpu milli, memory MiB) of k namespaces' LimitRange maxima"""
    rng = np.random.Generator(np.random.PCG64(seed))
    return [(int(rng.integers(15, 61)) * 100, int(rng.integers(4, 33)) * 256) for _ in range(k)]


def genpod_podspecs(k):
    """what genpod writes for k namespaces: a pause pod per namespace, requests == limits"""
    out = []
    for q, (cpu, mem) in enumerate(genpod_requests(k)):
        res = {"cpu": "%dm" % cpu, "memory": "%dMi" % mem}
        out.append({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "cluster-capacity-stub-container", "namespace": "team%03d" % q},
                    "spec": {"containers": [{"name": "cluster-capacity-stub-container", "image": "registry.k8s.io/pause:3.9",
                                             "resources": {"requests": res, "limits": res}}], "restartPolicy": "OnFailure", "dnsPolicy": "Default"}})
    return out


# ---- host: cc_new_each + SyncWithClient + encode ------------------------------------------------------------------------------------
def host_once(root):
    """seconds of NewEach, SyncWithClient and the encoding of 512 podspecs on synth.c4_objects, with the libraries under `root`"""
    sys.path.insert(0, root)
    fw = importlib.import_module("cluster-capacity_b200.framework")
    synth = importlib.import_module("cluster-capacity_b200.synth")
    nodes, pods, _ = synth.c4_objects()
    client = fw.ListClient(nodes, pods, [])
    specs = genpod_podspecs(T_ANALYSES)
    try:
        fw.NewEach(None, None, specs, 1, []).Close()
        chunks = [specs]
    except fw.FrameworkError:      # a build that takes 64 podspecs per handle: eight handles, each syncing and encoding the snapshot
        chunks = [specs[c:c + 64] for c in range(0, len(specs), 64)]
    out = {"new_s": 0.0, "sync_s": 0.0, "encode_s": 0.0, "run_each_s": 0.0, "handles": len(chunks)}
    for part in chunks:
        t0 = time.perf_counter()
        cc = fw.NewEach(None, None, part, 1, [])
        t1 = time.perf_counter()
        cc.SyncWithClient(client)
        t2 = time.perf_counter()
        first = [r.ScheduledPods() for r in cc.RunEach()]    # (a view is valid until the next RunEach)
        t3 = time.perf_counter()
        again = [r.ScheduledPods() for r in cc.RunEach()]
        t4 = time.perf_counter()
        assert first == again
        cc.Close()
        for k, v in (("new_s", t1 - t0), ("sync_s", t2 - t1), ("encode_s", (t3 - t2) - (t4 - t3)), ("run_each_s", t4 - t3)):
            out[k] += v
    return out


def host(roots, reps):
    rows = {r: [] for r in roots}
    for _ in range(reps):
        for r in roots:     # alternately, each in a process of its own (the package of each checkout has the same name)
            out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--host-once", r]).decode().strip().splitlines()[-1]
            rows[r].append(json.loads(out))
    med = lambda r, k: round(float(np.median([x[k] for x in rows[r]])), 3)
    return {("this" if r == ROOT else r): {k: med(r, k) for k in ("new_s", "sync_s", "encode_s", "run_each_s")} | {"handles": rows[r][0]["handles"], "reps": reps}
            for r in roots}


# ---- engine: packed, queued and 64-analysis chunks ----------------------------------------------------------------------------------
def engine_part(reps):
    sys.path.insert(0, ROOT)
    abi = importlib.import_module("cluster-capacity_b200._abi")
    engine = importlib.import_module("cluster-capacity_b200.engine")
    synth = importlib.import_module("cluster-capacity_b200.synth")
    snap, _, _ = synth.c2(n=100_000, seed=6)
    tmpl = [abi.default_template(cpu, mem * synth.MiB) for cpu, mem in genpod_requests(T_ANALYSES)]

    def same(a, b):
        return (a.placed == b.placed and a.stop_code == b.stop_code and np.array_equal(a.pod_node, b.pod_node)
                and np.array_equal(a.reason_hist, b.reason_hist) and a.preempt_no_victims == b.preempt_no_victims)

    def run_whole(eng, limit, queued):
        if queued:
            os.environ["CCSIM_DEBUG_FLAGS"] = "256"
        try:
            t0 = time.perf_counter()
            got = eng.run_each(limit)
            wall = time.perf_counter() - t0
        finally:
            os.environ.pop("CCSIM_DEBUG_FLAGS", None)
        st = eng.run_stats()
        return got, got[0].run_ms, wall * 1e3, (eng.kernel_name(), st["grid"], st["per_cta"], st["global_levels"], st["shared_levels"], st["smem_bytes"])

    def run_chunks(engs, limit):
        got, ms, t0 = [], 0.0, time.perf_counter()
        for e in engs:
            r = e.run_each(limit)
            got += r
            ms += r[0].run_ms
        return got, ms, (time.perf_counter() - t0) * 1e3

    out = {}
    for limit in (0, 1000):
        whole = engine.Engine(device=0)
        whole.load_nodes(snap)
        whole.set_analyses(tmpl, [([], [])] * T_ANALYSES)
        chunks = []
        for c in range(0, T_ANALYSES, 64):
            e = engine.Engine(device=0)
            e.load_nodes(snap)
            e.set_analyses(tmpl[c:c + 64], [([], [])] * 64)
            chunks.append(e)
        # warm-up of every way, then the single-template runs
        p, _, _, pk = run_whole(whole, limit, False)
        q, _, _, qk = run_whole(whole, limit, True)
        c, _, _ = run_chunks(chunks, limit)
        assert pk[0] == "each<packed>" and qk[0] == "each" and qk[1] == T_ANALYSES, (pk, qk)
        check = range(T_ANALYSES) if limit else np.linspace(0, T_ANALYSES - 1, 8).astype(int).tolist()
        with engine.Engine(device=0) as one:
            one.load_nodes(snap)
            for t in check:
                one.set_templates([tmpl[t]])
                w = one.run(limit)
                assert same(p[t], w), "analysis %d differs from ccsim_run of its template" % t
        rows = {k: [] for k in ("packed_ms", "packed_wall_ms", "queued_ms", "queued_wall_ms", "chunks_ms", "chunks_wall_ms")}
        for _ in range(reps):
            gp, ms, wall, _ = run_whole(whole, limit, False)
            rows["packed_ms"].append(ms); rows["packed_wall_ms"].append(wall)
            gq, ms, wall, _ = run_whole(whole, limit, True)
            rows["queued_ms"].append(ms); rows["queued_wall_ms"].append(wall)
            gc, ms, wall = run_chunks(chunks, limit)
            rows["chunks_ms"].append(ms); rows["chunks_wall_ms"].append(wall)
            for t in range(T_ANALYSES):
                assert same(gp[t], p[t]) and same(gq[t], p[t]) and same(gc[t], p[t]), "batch differs at analysis %d" % t
        placed = [g.placed for g in p]
        med = lambda k: float(np.median(rows[k]))
        out["c2_100k_x512_" + ("limit%d" % limit if limit else "unschedulable")] = {
            "nodes": snap.n, "analyses": T_ANALYSES, "max_limit": limit, "placed_total": int(sum(placed)),
            "placed_min": int(min(placed)), "placed_max": int(max(placed)), "stop_codes": sorted(set(int(g.stop_code) for g in p)),
            **{k: [round(x, 3) for x in v] for k, v in rows.items()},
            "packed_over_queued": round(med("queued_ms") / med("packed_ms"), 3),
            "packed_over_chunks": round(med("chunks_ms") / med("packed_ms"), 3),
            "packed_kernel": {"name": pk[0], "grid": pk[1], "per_cta": pk[2], "global_levels": pk[3], "shared_levels": pk[4], "smem_bytes": pk[5]},
            "queued_kernel": {"name": qk[0], "grid": qk[1], "per_cta": qk[2], "global_levels": qk[3], "shared_levels": qk[4], "smem_bytes": qk[5]},
            "bit_exact_batches": reps, "checked_against_ccsim_run": len(check),
        }
        print(json.dumps({k: out[k] for k in list(out)[-1:]}), file=sys.stderr, flush=True)
        whole.close()
        for e in chunks:
            e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", choices=["engine", "host"], default=None)
    ap.add_argument("--host-root", default=None, help="another checkout whose host library is timed alternately with this one's")
    ap.add_argument("--host-once", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.host_once:
        print(json.dumps(host_once(a.host_once)))
        return
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power}
    if a.only in (None, "engine"):
        res.update(engine_part(a.reps))
    if a.only in (None, "host"):
        res["host_c4_objects_x512"] = host([ROOT] + ([os.path.abspath(a.host_root)] if a.host_root else []), a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
