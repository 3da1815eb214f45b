"""GPU: per-analysis runs with more analyses than the device has SMs. Node-local analyses beyond the CTAs the device holds at once
share CTAs (ccsim_each_packed_kernel, one warp's placement loop each); analyses with coupled terms keep one CTA each (grid = T).
Every analysis is checked against ccsim_run of its template alone and, for a sample, the C oracle: placement by placement, stop
code, FitError histogram, preemption counters and ccsim_node_counts."""
import importlib
import io
import json
import os
from contextlib import redirect_stdout

import numpy as np
import pytest

import helpers
from oracle import binding as oracle
from test_each import mask
from test_each_coupled import NO_HARD_WEIGHT, stripped_cluster
from test_each_many import many
from test_gpu_each import nodes_c2, request_templates, same
from test_gpu_each_coupled import alone, c4_family, with_topo

abi = importlib.import_module("cluster-capacity_b200._abi")
engine = importlib.import_module("cluster-capacity_b200.engine")
fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")
genpod = importlib.import_module("cluster-capacity_b200.genpod")

pytestmark = pytest.mark.gpu
MiB = 1 << 20
NODE_LOCAL = ["plain", "tolerations", "extended", "best_effort", "never_preempt", "selector"]


@pytest.fixture(scope="module")
def sms(built):
    return helpers.device_sm_count()


def sample(T, k=16):
    """k analyses spread over 0..T-1, the first and the last included"""
    return sorted(set(np.linspace(0, T - 1, k).astype(int).tolist()))


def run_all(snap, tmpl, limit, terms=None):
    """one ccsim_run_each: (results, run_stats, kernel name, node counts)"""
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        if terms is None:
            eng.set_analyses(tmpl, [([], [])] * len(tmpl))
        else:
            eng.set_analyses(tmpl, terms)
        got = eng.run_each(limit)
        return got, eng.run_stats(), eng.kernel_name(), [eng.node_counts(t) for t in range(len(tmpl))]


def check_all(snap, tmpl, limit, terms=None, oracle_sample=16):
    """every analysis against ccsim_run of its template alone; a sample of at least 16 against the C oracle"""
    got, st, name, counts = run_all(snap, tmpl, limit, terms)
    assert st["placed"] == sum(g.placed for g in got)
    ora = set(sample(len(tmpl), oracle_sample))
    with engine.Engine(device=0) as one:
        for t, g in enumerate(got):
            ctr, cols = terms[t] if terms is not None else ([], [])
            s1 = with_topo(snap, cols) if terms is not None else snap
            t1 = alone(tmpl[t], t)
            one.load_nodes(s1)
            one.set_templates([t1], ctr)
            want = one.run(limit)
            same(g, want, "analysis %d vs ccsim_run" % t)
            wc, wf = one.node_counts(0)
            assert np.array_equal(counts[t][0], wc) and np.array_equal(counts[t][1], wf), t
            if t in ora:
                same(g, oracle.run(s1, [t1], ctr, max_pods=limit), "analysis %d vs oracle" % t)
    return got, st, name


def node_local_templates(T, seed):
    """T node-local templates: requests of every size, some fit-only, some tolerating a PreferNoSchedule taint"""
    tm = request_templates(T, seed=seed)
    for q in range(0, T, 5):
        tm[q].tol_prefer[0] = 1
    return tm


def tainted_nodes(n, seed):
    """a C2-like cluster in which every third node carries one PreferNoSchedule taint (two normalisation classes)"""
    taint = np.zeros((1, n), np.uint64)
    taint[0, ::3] = 1
    return nodes_c2(n, seed=seed, taint_mask=taint, taint_prefer=[1], taint_lists=[[0] if i % 3 == 0 else [] for i in range(n)])


# ---- 1. 2 x SMs + 7 analyses: node-local ones packed, coupled ones one CTA each ----------------------------------------------------
@pytest.mark.parametrize("limit", [0, 300])
def test_node_local_analyses_past_the_sms_are_packed(built, sms, limit):
    T = 2 * sms + 7
    snap = tainted_nodes(3000, seed=31)
    tm = node_local_templates(T, seed=31)
    tm[T - 2] = abi.default_template(100_000, 64 * MiB)     # fits nowhere
    got, st, name = check_all(snap, tm, limit)
    per = -(-T // sms)
    assert name == "each<packed>" and st["per_cta"] == per == 3 and st["grid"] == -(-T // per)
    assert got[T - 2].placed == 0 and got[T - 2].reason_hist[abi.R_INSUFFICIENT_CPU] > 0
    assert all(g.placed > 0 for t, g in enumerate(got) if t != T - 2)
    assert any(g.stop_code == abi.STOP_UNSCHEDULABLE for t, g in enumerate(got) if t != T - 2) == (limit == 0)
    assert all(g.stop_code == abi.STOP_LIMIT_REACHED for t, g in enumerate(got) if t != T - 2) == (limit > 0)


def test_coupled_analyses_past_the_sms_keep_one_cta_each(built, sms):
    T = 2 * sms + 7
    snap, tmpl, terms = c4_family(2500, T - 1, seed=9, zones=8, racks=32, regions=4, n_existing=5000)
    got, st, name = check_all(snap, tmpl, 0, terms)
    assert name == "each" and st["per_cta"] == 1 and st["grid"] == T
    assert all(g.placed > 0 and g.stop_code == abi.STOP_UNSCHEDULABLE for g in got)


# ---- 2. across the selection edge ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [0, 1])
def test_selection_edge(built, sms, extra):
    T = sms + extra
    snap = tainted_nodes(2000, seed=32)
    got, st, name = check_all(snap, node_local_templates(T, seed=32 + extra), 0)
    if extra == 0:    # every CTA resident: today's launch
        assert name == "each" and st["per_cta"] == 1 and st["grid"] == T
    else:
        assert name == "each<packed>" and st["per_cta"] == 2 and st["grid"] == -(-T // 2)


def test_packed_through_the_one_per_analysis_launch_agrees(built, sms, monkeypatch):
    """the same packed analyses launched one CTA each (CCSIM_DEBUG_FLAGS bit 8): every result equal"""
    T = 2 * sms + 7
    snap = tainted_nodes(1500, seed=33)
    tm = node_local_templates(T, seed=33)
    packed, st, name, counts = run_all(snap, tm, 0)
    assert name == "each<packed>"
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", "256")
    queued, qst, qname, qcounts = run_all(snap, tm, 0)
    assert qname == "each" and qst["grid"] == T and qst["per_cta"] == 1
    for t in range(T):
        same(packed[t], queued[t], "analysis %d packed vs one CTA each" % t)
        assert np.array_equal(counts[t][0], qcounts[t][0]) and np.array_equal(counts[t][1], qcounts[t][1])


# ---- 3. mixed analyses at the object level -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("hostports", [False, True])
def test_mixed_object_analyses(built, sms, hostports):
    """one podspec that fits nowhere, one that reaches --max-limit; node-local podspecs only (packed), or with coupled podspecs and
    hostPorts at t = 64 and t = T - 3 (one CTA per analysis)"""
    T = 2 * sms + 7
    nodes, pods = stripped_cluster(41, n_nodes=40, n_pods=60)
    if hostports:     # with spread and pod (anti-)affinity podspecs too
        tm = many(T, hostports=(64, T - 3))
    else:
        tm = [helpers.template(NODE_LOCAL[t % len(NODE_LOCAL)]) for t in range(T)]
        for t, p in enumerate(tm):
            p["metadata"]["name"] = "pod-%03d" % t
    tm[1]["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "100", "memory": "1Gi"}}
    tm[2]["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "10m", "memory": "1Mi"}}
    limit = 60
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, limit, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    res = cc.RunEach()
    assert len(res) == T
    for t, r in enumerate(res):
        one = fw.New(NO_HARD_WEIGHT, None, tm[t], limit, [])
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        one.Run()
        assert r.StopReason() == one.StopReason() and r.ScheduledPods() == one.ScheduledPods(), t
        assert mask(json.dumps(r.Report())) == mask(json.dumps(one.Report())), t
        one.Close()
    assert res[1].ScheduledPods() == [] and "Insufficient cpu" in res[1].StopReason()
    assert res[2].StopReason() == "LimitReached: Maximum number of pods simulated: %d" % limit
    if hostports:
        for t in (64, T - 3):
            placed = res[t].ScheduledPods()
            assert len(placed) == len(set(placed)) > 0 and "node(s) didn't have free ports" in res[t].StopReason()
    cc.Close()


# ---- 4. the device-memory refusal, before any launch -------------------------------------------------------------------------------
def test_state_larger_than_device_memory_is_refused(built):
    n, T = 2_000_000, abi.EACH_MAX_ANALYSES      # T x n x 12 B = 98 GB of clone counts and leaves alone
    snap = abi.Snapshot(n, np.full(n, 4000, np.int64), np.full(n, 16 << 30, np.int64), np.full(n, 110, np.int32))
    tm = [abi.default_template(100 + t % 50, 64 * MiB) for t in range(T)]
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_analyses(tm, [([], [])] * T)
        before = eng.kernel_launches()
        with pytest.raises(engine.EngineError, match=r"per-analysis runs: the per-analysis device state \(4096 analyses x 2000000 nodes: "
                                                     r"clone counts and leaves, .* = [0-9.]+ GiB\) exceeds free device memory \([0-9.]+ GiB\)"):
            eng.run_each(1)
        assert eng.kernel_launches() == before
        eng.set_analyses(tm[:2], [([], [])] * 2)      # the engine stays usable
        assert [g.placed for g in eng.run_each(1)] == [1, 1]


# ---- 5. the command line: genpod over 300 namespaces --------------------------------------------------------------------------------
def test_genpod_cli_each_300_namespaces(built, tmp_path):
    nodes = [helpers.make_node("n%03d" % i, cpu=str(2 + 2 * (i % 5)), mem="%dGi" % (4 + 4 * (i % 3)), pods="30",
                               labels={"pool": "a" if i % 3 else "b"}) for i in range(24)]
    nss, lrs = [], []
    for k in range(300):
        ann = {"openshift.io/node-selector": "pool=a"} if k % 7 == 0 else {}
        nss.append({"apiVersion": "v1", "kind": "Namespace", "metadata": {"name": "team%03d" % k, "annotations": ann}})
        lrs.append({"apiVersion": "v1", "kind": "LimitRange", "metadata": {"name": "lr", "namespace": "team%03d" % k},
                    "spec": {"limits": [{"type": "Pod", "max": {"cpu": "%dm" % (300 + 37 * (k % 97)), "memory": "%dMi" % (256 + 29 * (k % 89))}}]}})
    snap = tmp_path / "cluster.json"
    snap.write_text(json.dumps({"nodes": nodes, "pods": [], "namespaces": nss, "limitranges": lrs}))
    specs = tmp_path / "specs"
    assert genpod.main(["--namespace", ",".join(n["metadata"]["name"] for n in nss), "--snapshot", str(snap), "--output-dir", str(specs)]) == 0
    files = sorted(os.listdir(specs))
    assert len(files) == 300

    def run(args):
        buf = io.StringIO()
        with redirect_stdout(buf):
            assert cli.main(args + ["--snapshot", str(snap), "--max-limit", "200", "-o", "json"]) == 0
        head, body = buf.getvalue().split("\n", 1)
        assert head.startswith("Cluster capacity version")
        return body

    reviews = json.loads(mask(run(["--podspec", str(specs), "--each"])))
    assert isinstance(reviews, list) and len(reviews) == 300
    assert reviews == [json.loads(mask(run(["--podspec", str(specs / f)]))) for f in files]
    assert len({r["status"]["replicas"] for r in reviews}) > 5
