"""GPU: per-analysis runs of podspecs with hard topology spread, required pod (anti-)affinity and hostPorts (ccsim_set_analyses /
cc_new_each / framework.NewEach / `cluster-capacity --each`). Every analysis t is checked against ccsim_run of template t alone with its
own counters and columns, the C oracle and, for object-level cases, objref.Simulator([podspec t]): placement by placement, stop code,
FitError histogram, preemption counters and node counts."""
import copy
import importlib
import io
import json
from contextlib import redirect_stdout

import numpy as np
import pytest

import helpers
from oracle import binding as oracle
from oracle import objref
from test_each import mask
from test_each_coupled import COUPLED, NODE_LOCAL, NO_HARD_WEIGHT, podspecs, stripped_cluster
from test_gpu_each import same

abi = importlib.import_module("cluster-capacity_b200._abi")
engine = importlib.import_module("cluster-capacity_b200.engine")
fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")
synth = importlib.import_module("cluster-capacity_b200.synth")

pytestmark = pytest.mark.gpu
MiB = 1 << 20


def with_topo(snap, cols):
    s = copy.copy(snap)
    s.topo = [np.ascontiguousarray(c, dtype=np.int32) for c in cols]
    return s


def alone(tmpl, t):
    """template t of a per-analysis launch as a run of its own sees it: its hostPort self-conflict on bit 0"""
    one = abi.Template.from_buffer_copy(tmpl)
    one.image_score = tmpl.image_score
    if one.port_tmpl_conflict:
        one.port_tmpl_conflict = 1
    return one


def run_analyses(snap, tmpl, terms, limit):
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_analyses(tmpl, terms)
        got = eng.run_each(limit)
        assert eng.kernel_name() == "each"
        return got, eng.run_stats(), [eng.node_counts(t) for t in range(len(tmpl))]


def check(snap, tmpl, terms, limit, with_oracle=True):
    """every analysis against ccsim_run of its template alone (own counters and columns) and the C oracle"""
    got, st, counts = run_analyses(snap, tmpl, terms, limit)
    assert st["placed"] == sum(g.placed for g in got)
    for t, g in enumerate(got):
        ctr, cols = terms[t]
        s1, t1 = with_topo(snap, cols), alone(tmpl[t], t)
        with engine.Engine(device=0) as one:
            one.load_nodes(s1)
            one.set_templates([t1], ctr)
            want = one.run(limit)
            wc, wf = one.node_counts(0)
        same(g, want, "analysis %d vs ccsim_run" % t)
        assert np.array_equal(counts[t][0], wc) and np.array_equal(counts[t][1], wf), t
        if with_oracle:
            same(g, oracle.run(s1, [t1], ctr, max_pods=limit), "analysis %d vs oracle" % t)
    return got, st


def terms_of(enc):
    out = []
    for a in enc["analyses"]:
        ctr = [abi.make_counter(c["topo_col"], np.array(c["init"], np.int32), n_present=c["n_present"], inc=c["inc"], elig_bit=c["elig_bit"])
               for c in a["counters"]]
        out.append((ctr, [np.array(c, np.int32) for c in a["topo"]]))
    return out


def c4_family(n, k, seed=5, **kw):
    """C4's snapshot and k templates differing in requests and maxSkew, with C4's counters each; plus one template without counters"""
    snap, (t0,), ctr = synth.c4(n=n, **kw)
    rng = np.random.Generator(np.random.PCG64(seed))
    tmpl, terms = [], []
    for q in range(k):
        t = abi.Template.from_buffer_copy(t0)
        t.req_cpu = t.least_cpu = t.bal_cpu = t.nz_cpu = int(rng.integers(100, 600))
        mem = int(rng.integers(64, 512)) * MiB
        t.req_mem = t.least_mem = t.bal_mem = t.nz_mem = mem
        for c in range(3):
            t.pts[c].max_skew = int(rng.integers(1, 5))
        tmpl.append(t)
        terms.append((ctr, snap.topo))
    tmpl.insert(1, abi.default_template(300, 256 * MiB))
    terms.insert(1, ([], []))
    return snap, tmpl, terms


# ---- 1. the C4 family at 2000 nodes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("limit", [0, 300])
def test_c4_family_matches_single_runs_and_oracle(built, limit):
    snap, tmpl, terms = c4_family(2000, 8, zones=8, racks=32, regions=4, n_existing=4000)
    got, st = check(snap, tmpl, terms, limit)
    assert all(g.placed > 0 for g in got)
    if limit:
        assert all(g.stop_code == abi.STOP_LIMIT_REACHED for g in got)
    else:
        assert all(g.stop_code == abi.STOP_UNSCHEDULABLE for g in got)


# ---- 2. object level: every in-scope variant in one NewEach list; the command line ------------------------------------------------
@pytest.mark.parametrize("seed,limit", [(21, 0), (22, 17)])
def test_objects_match_single_runs_objref_and_engine(built, seed, limit):
    nodes, pods = stripped_cluster(seed, n_nodes=40, n_pods=60)
    tm = podspecs(NODE_LOCAL[:2] + COUPLED + ["affinity_zone"] + NODE_LOCAL[2:])
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, limit, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    res = cc.RunEach()
    assert len(res) == len(tm)
    for t, r in enumerate(res):
        one = fw.New(NO_HARD_WEIGHT, None, tm[t], limit, [])
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        one.Run()
        assert r.StopReason() == one.StopReason() and r.ScheduledPods() == one.ScheduledPods(), t
        assert mask(json.dumps(r.Report())) == mask(json.dumps(one.Report()))
        one.Close()
        if "affinity" not in tm[t]["spec"]:      # objref runs the default configuration: the affinity podspec needs the weight 0
            ref = objref.Simulator([tm[t]], limit)
            ref.sync(nodes, pods)
            ref.run()
            assert r.ScheduledPods() == ref.pods_status and r.StopReason() == ref.stop_reason, t
    snap, T, ctr, _, _, _ = helpers.from_encoded(cc.EncodedSnapshot())
    assert not ctr
    check(snap, T, terms_of(cc.EncodedSnapshot()), limit)
    cc.Close()


def test_prefilter_rejected_podspec_ends_its_own_analysis(built):
    """a podspec whose required node affinity pins disjoint node names: PreFilter rejects it, its analysis ends with cc_run's
    message and no placements; the other analyses of the list still run"""
    nodes, pods = stripped_cluster(25, n_nodes=30, n_pods=40)
    tm = podspecs(["spread_zone", "plain", "anti_hostname"])
    tm[1]["spec"]["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
        {"matchFields": [{"key": "metadata.name", "operator": "In", "values": [nodes[0]["metadata"]["name"]]},
                         {"key": "metadata.name", "operator": "In", "values": [nodes[1]["metadata"]["name"]]}]}]}}}
    cc = fw.NewEach(None, None, tm, 0, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    assert cc.EncodedSnapshot()["analyses"][1]["prefilter_msg"]
    res = cc.RunEach()
    for t, r in enumerate(res):
        one = fw.New(None, None, tm[t], 0, [])
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        one.Run()
        assert r.StopReason() == one.StopReason() and r.ScheduledPods() == one.ScheduledPods(), t
        one.Close()
    assert res[1].ScheduledPods() == [] and "didn't match Pod's node affinity/selector" in res[1].StopReason()
    assert res[0].ScheduledPods() and res[2].ScheduledPods()
    cc.Close()


@pytest.mark.parametrize("fmt", ["", "json", "yaml"])
def test_cli_each_takes_coupled_podspecs(built, tmp_path, fmt):
    nodes, pods = stripped_cluster(23, n_nodes=30, n_pods=40)
    (tmp_path / "snap.json").write_text(json.dumps({"nodes": nodes, "pods": pods, "namespaces": []}))
    d = tmp_path / "specs"
    d.mkdir()
    tm = podspecs(COUPLED + NODE_LOCAL[:1])
    for i, p in enumerate(tm):
        (d / ("%02d.json" % i)).write_text(json.dumps(p))

    def run(args):
        out = io.StringIO()
        with redirect_stdout(out):
            assert cli.main(args + ["--snapshot", str(tmp_path / "snap.json"), "--max-limit", "12", "-o", fmt, "--verbose"]) == 0
        return out.getvalue()
    each = run(["--podspec", str(d), "--each"])
    singles = [run(["--podspec", str(d / ("%02d.json" % i))]) for i in range(len(tm))]
    head = "Cluster capacity version "
    body = lambda s: s.split("\n", 1)[1] if s.startswith(head) else s
    singles = [body(s) for s in singles]
    if fmt == "json":
        assert json.loads(mask(body(each))) == [json.loads(mask(s)) for s in singles]
    else:
        assert mask(body(each)) == mask(("---\n" if fmt == "yaml" else "").join(singles))


# ---- 3. edges ----------------------------------------------------------------------------------------------------------------------
def zone_snapshot(n, zones, seed=2, cpu=4000, pods=110, idle=(), **kw):
    """n nodes round-robin over `zones` zones (column 0) and one domain per node (column 1); the nodes in `idle` request nothing"""
    rng = np.random.Generator(np.random.PCG64(seed))
    req = (rng.integers(1, 20, n) * 100).astype(np.int64)
    req[list(idle)] = 0
    return abi.Snapshot(n, np.full(n, cpu, np.int64), np.full(n, 16 << 30, np.int64), np.full(n, pods, np.int32),
                        req_cpu=req, topo=[np.arange(n) % zones, np.arange(n)], **kw)


def spread(t, c, counter, skew, self_match=1, min_zero=0):
    t.n_pts = max(t.n_pts, c + 1)
    t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = counter, skew, self_match, min_zero


def test_hostname_spread_rebuilds(built):
    """hard spread over a column with one node per domain: folded into the leaves; its minimum moves, every move rebuilds"""
    n = 300
    snap = zone_snapshot(n, 6)
    rng = np.random.Generator(np.random.PCG64(4))
    init = rng.integers(0, 3, n).astype(np.int32)
    t = abi.default_template(100, 64 * MiB)
    spread(t, 0, 0, 1)
    got, st = check(snap, [t], [([abi.make_counter(1, init, inc=1)], snap.topo)], 0)
    assert st["rebuilds"] >= 3 and got[0].placed > 0


def test_min_domains_and_missing_keys(built):
    """minDomains above the domain count (global minimum 0); nodes without the spread, affinity or anti-affinity key"""
    n = 240
    snap = zone_snapshot(n, 5)
    zone = snap.topo[0].copy()
    zone[::7] = -1
    cols = [zone, snap.topo[1]]
    z0 = np.zeros(5, np.int32)
    a = abi.default_template(200, 64 * MiB)
    spread(a, 0, 0, 2, min_zero=1)
    b = abi.default_template(200, 64 * MiB)
    b.n_aff, b.aff_counter[0], b.flags, b.aff_total_init = 1, 0, b.flags | abi.TF_AFF_SELF_MATCH_ALL, 0
    c = abi.default_template(200, 64 * MiB)
    c.n_anti, c.anti_counter[0] = 1, 0
    terms = [([abi.make_counter(0, np.array([0, 3, 1, 2, 0], np.int32), inc=1)], cols),
             ([abi.make_counter(0, z0, inc=1)], cols), ([abi.make_counter(0, z0, inc=1)], cols)]
    got, st = check(snap, [a, b, c], terms, 0)
    assert st["rebuilds"] == 1                  # b: the affinity bypass ends with the first clone
    for g in got[:2]:                           # spread and affinity: the nodes without the key never take a clone
        assert not np.isin(g.pod_node, np.arange(0, n, 7)).any()
    assert got[0].reason_hist[abi.R_PTS_MISSING_LABEL] > 0 and got[0].reason_hist[abi.R_PTS_SKEW] > 0
    assert got[1].reason_hist[abi.R_IPA_AFFINITY] > 0
    # anti-affinity: one clone per zone, then only the nodes without the key (they never count)
    assert np.isin(got[2].pod_node, np.arange(0, n, 7)).any() and got[2].reason_hist[abi.R_IPA_ANTI_AFFINITY] > 0


def test_folded_affinity_bypass_ends(built):
    """required affinity keyed on a column with one node per domain (a hostname key): folded into the leaves. With no matching pod
    anywhere the pod that matches its own term may go anywhere; after the first clone only that clone's node matches, so the rebuild
    must close every other leaf"""
    n = 200
    snap = zone_snapshot(n, 4)
    t = abi.default_template(100, 64 * MiB)
    t.n_aff, t.aff_counter[0], t.flags, t.aff_total_init = 1, 0, t.flags | abi.TF_AFF_SELF_MATCH_ALL, 0
    got, st = check(snap, [t], [([abi.make_counter(1, np.zeros(n, np.int32), inc=1)], snap.topo)], 0)
    assert st["rebuilds"] == 1 and got[0].placed > 1
    assert (got[0].pod_node == got[0].pod_node[0]).all() and got[0].reason_hist[abi.R_IPA_AFFINITY] == n - 1


def test_groups_times_classes_and_closed_best_group(built):
    """zone groups x PreferNoSchedule classes with the top class emptying; the best node overall sits in a zone the spread closes"""
    n = 160
    taint = np.zeros((1, n), np.uint64)
    taint[0, n // 2:] = 1        # half the nodes carry one untolerated PreferNoSchedule taint
    taint[0, 10:20] = 3          # ten carry two: the top class, small enough to empty
    # node 5 (zone 1, no PreferNoSchedule taint) alone requests nothing: it scores best, but zone 1 starts above the others
    snap = zone_snapshot(n, 4, idle=[5], taint_mask=taint, taint_prefer=[3], taint_nosched=[0])
    t = abi.default_template(300, 64 * MiB)
    spread(t, 0, 0, 1)
    ctr = [abi.make_counter(0, np.array([2, 4, 2, 2], np.int32), inc=1)]
    got, _ = check(snap, [t, abi.default_template(300, 64 * MiB)], [(ctr, snap.topo), ([], [])], 0)
    assert got[1].pod_node[0] == 5                            # without the spread constraint node 5 wins
    assert got[0].pod_node[0] % 4 != 1 and got[0].placed > 10  # with it the winner comes from an open zone
    assert 5 in got[0].pod_node                               # and node 5 wins once zone 1 opens


def test_hostports_one_clone_per_free_node(built):
    nodes, pods = stripped_cluster(24, n_nodes=30, n_pods=30)
    tm = podspecs(["hostports", "plain"])
    cc = fw.NewEach(None, None, tm, 0, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    r = cc.RunEach()[0]
    placed = r.ScheduledPods()
    assert len(placed) == len(set(placed)) > 0 and "node(s) didn't have free ports" in r.StopReason()
    one = fw.New(None, None, tm[0], 0, [])
    one.SyncWithClient(helpers.list_client(fw, nodes, pods))
    one.Run()
    assert one.ScheduledPods() == placed and one.StopReason() == r.StopReason()
    one.Close()
    cc.Close()


def test_single_node_group_and_empty_segments(built):
    """a group of one node; a domain of no node (a counter entry no group stands for: groups are built from the nodes there are);
    empty segments, which an analysis without group terms has when one of its classes holds no node"""
    n = 64
    zone = (np.arange(n) % 3).astype(np.int32)
    zone[0] = 3                   # domain 3 holds one node; domain 4 holds none
    taint = np.zeros((1, n), np.uint64)
    taint[0, 1::2] = 1            # a PreferNoSchedule taint on every other node: two classes
    snap = zone_snapshot(n, 3, taint_mask=taint, taint_prefer=[1], taint_nosched=[0])
    t = abi.default_template(100, 64 * MiB)
    spread(t, 0, 0, 1)
    ctr = [abi.make_counter(0, np.zeros(5, np.int32), n_present=4, inc=1)]
    tolerant = abi.default_template(100, 64 * MiB)
    tolerant.tol_prefer[0] = 1    # every node in class 0: the segment of class 1 is empty
    got, _ = check(snap, [t, tolerant, abi.default_template(100, 64 * MiB)], [(ctr, [zone]), ([], []), ([], [])], 0)
    assert 0 in got[0].pod_node and got[1].placed > 0 and got[2].placed > 0


# ---- 4. refusals, none of which launches a kernel ----------------------------------------------------------------------------------
def refused(snap, tmpl, terms, limit, match, code=engine.EngineError, **kw):
    with engine.Engine(device=0, **kw) as eng:
        eng.load_nodes(snap)
        before = eng.kernel_launches()
        with pytest.raises(code, match=match):
            eng.set_analyses(tmpl, terms)
            eng.run_each(limit)
        assert eng.kernel_launches() == before


def test_refusals(built):
    n = 2 * abi_groups() + 2
    snap = zone_snapshot(n, 3, pods=4)
    t = abi.default_template(100, 64 * MiB)
    spread(t, 0, 0, 1)
    # domain groups: accepted at the bound, refused one past it
    at = (np.arange(n) // 2).astype(np.int32)
    at[at >= abi_groups()] = abi_groups() - 1
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_analyses([t], [([abi.make_counter(0, np.zeros(abi_groups(), np.int32), inc=1)], [at])])
        eng.run_each(5)
    past = (np.arange(n) // 2).astype(np.int32)
    refused(snap, [t], [([abi.make_counter(0, np.zeros(past.max() + 1, np.int32), inc=1)], [past])], 5,
            "analysis 0 has %d domain groups \\(max %d\\)" % (abi_groups() + 1, abi_groups()))
    # int32 counters: refused exactly where ccsim_run of the template refuses
    big = np.full(3, 2**31 - 3, np.int32)
    with engine.Engine(device=0) as one:
        one.load_nodes(snap)
        one.set_templates([t], [abi.make_counter(0, big, inc=1)])
        with pytest.raises(engine.EngineError, match="counter 0, domain"):
            one.run(0)
    refused(snap, [abi.default_template(100, 64 * MiB), t], [([], []), ([abi.make_counter(0, big, inc=1)], [snap.topo[0]])], 0,
            "analysis 1: counter 0, domain")
    # soft scorers, world 2, reference sampling
    s = abi.default_template(100, 64 * MiB)
    s.n_pref_terms, s.pref_weight[0] = 1, 5
    refused(snap, [s], [([], [])], 5, "template 0 has a normalised soft scorer")
    refused(snap, [t], [([abi.make_counter(0, np.zeros(3, np.int32), inc=1)], [snap.topo[0]])], 5, "node-sharded runs", world=2)
    refused(snap, [t], [([abi.make_counter(0, np.zeros(3, np.int32), inc=1)], [snap.topo[0]])], 5, "reference sampling",
            sampling=abi.SAMPLING_REFERENCE, pct_nodes_to_score=50)
    # malformed terms
    refused(snap, [t], [([abi.make_counter(3, np.zeros(3, np.int32), inc=1)], [snap.topo[0]])], 5, "topo_col")
    refused(snap, [t], [([], [])], 5, "pts counter index")
    # ccsim_run / ccsim_prepare after ccsim_set_analyses
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_analyses([t], [([abi.make_counter(0, np.zeros(3, np.int32), inc=1)], [snap.topo[0]])])
        for call in (lambda: eng.run(5), lambda: eng.prepare(5)):
            with pytest.raises(engine.EngineError, match="rc=-5"):
                call()


def abi_groups():
    """CCSIM_EACH_MAX_GROUPS as include/ccsim.h defines it"""
    import os
    import re
    with open(os.path.join(os.path.dirname(__file__), "..", "include", "ccsim.h")) as f:
        return int(re.search(r"#define CCSIM_EACH_MAX_GROUPS (\d+)", f.read()).group(1))


# ---- 5. full size, once ------------------------------------------------------------------------------------------------------------
def test_c4_full_size_four_analyses(built):
    snap, (t0,), ctr = synth.c4()
    with engine.Engine(device=0) as one:
        one.load_nodes(snap)
        one.set_templates([t0], ctr)
        want = one.run(0)
    assert want.placed == 31071
    got, st, _ = run_analyses(snap, [t0] * 4, [(ctr, snap.topo)] * 4, 0)
    for g in got:
        same(g, want, "C4 analysis vs ccsim_run")
