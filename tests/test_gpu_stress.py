"""Randomized differential tests of the engines ENGINE_AUTO picks (multi-commit waves, tie-run batching, lean, generic) against the
CPU oracle: spread / anti-affinity templates with random domain counts, skews, self-match flags, missing labels, minDomains, limits.
The coupled-template tests also assert which kernel ran; a CPU test checks that the generator keeps reaching the multi-commit one."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
from oracle import binding as oracle  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
H100_SXM_SMS = 132


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def random_case(seed, sm_count):
    """A counter-coupled workload. Cluster sizes run from one CTA to the largest cluster the multi-commit kernel takes on this
    device (sm_count x 768 nodes: every tile full) and one node past it (the lean sequential kernel). Domain counts of 2^b - 1
    make the last domain's payload field all ones; 2^b needs one more bit."""
    rng = np.random.default_rng(1000 + seed)
    largest = sm_count * helpers.MULTI_TILE
    n = int(rng.choice([200, 600, 3000, 9000, 40000, 90000, largest - 1, largest, largest + 1], p=[.1, .1, .1, .1, .1, .1, .15, .2, .05]))
    n_topo = int(rng.integers(1, 4))
    doms = [int(rng.choice([3, 7, 8, 40, 255, 256, 300, 2000, 2047], p=[.14, .14, .14, .14, .12, .12, .1, .05, .05])) for _ in range(n_topo)]
    topo = []
    for d in doms:
        col = rng.integers(0, d, n).astype(np.int32)
        if rng.random() < 0.4:
            col[rng.random(n) < 0.03] = -1            # nodes without the label
        topo.append(col)
    a_cpu = rng.choice([2000, 4000, 8000, 16000], n)
    npods = rng.integers(0, 20, n).astype(np.int32)
    req_cpu = (rng.random(n) * 0.5 * a_cpu).astype(np.int64) // 10 * 10
    a_pods = rng.choice([30, 60, 110], n) if rng.random() < 0.7 else npods + rng.integers(0, 4, n)      # or: room for 0..3 more pods
    snap = abi.Snapshot(n, a_cpu, a_cpu * (2 * MiB), a_pods, req_cpu=req_cpu, req_mem=req_cpu * (1 * MiB),
                        npods=npods, topo=topo)
    ctr, t = [], abi.default_template(int(rng.choice([100, 250, 700])), int(rng.choice([64, 256, 1024])) * MiB)
    if rng.random() < 0.3:
        t.w_fit, t.w_balanced = int(rng.integers(1, 5)), int(rng.integers(1, 5))
    n_pts = 0
    for c, d in enumerate(doms):
        init = rng.integers(0, 4, d).astype(np.int32) if rng.random() < 0.7 else np.full(d, int(rng.integers(0, 3)), np.int32)
        self_match = int(rng.random() < 0.85)
        n_present = d if rng.random() < 0.8 else max(1, d - int(rng.integers(1, 3)))
        ctr.append(abi.make_counter(c, init, n_present=n_present, inc=self_match))
        t.pts[n_pts].counter, t.pts[n_pts].max_skew = c, int(rng.choice([1, 1, 2, 5]))
        t.pts[n_pts].self_match, t.pts[n_pts].min_zero = self_match, int(rng.random() < 0.1)
        n_pts += 1
    t.n_pts = n_pts
    kind = rng.random()
    if kind < 0.5:                                    # required anti-affinity on the hostname: node-local counter
        ctr.append(abi.make_counter(-1, (rng.random(n) < 0.1).astype(np.int32), inc=1))
        t.n_anti, t.anti_counter[0] = 1, len(ctr) - 1
    elif kind < 0.7 and doms[0] >= 40:                # ... or on the first topology key (its own counter on the same column)
        ctr.append(abi.make_counter(0, (rng.random(doms[0]) < 0.2).astype(np.int32), inc=1))
        t.n_anti, t.anti_counter[0] = 1, len(ctr) - 1
    limit = int(rng.choice([0, 0, 1, 37, 1500]))
    return snap, [t], ctr, limit


def test_random_cases_reach_the_multi_commit_kernel():
    """At least 42 of the 48 coupled cases run on the multi-commit kernel of an H100 SXM, and at least one is a deliberate fallback:
    a change to the generator must not quietly move the stress tests back onto the lean kernel."""
    elig = [helpers.multi_eligible(*random_case(seed, H100_SXM_SMS)[:3], H100_SXM_SMS) for seed in range(48)]
    assert sum(elig) >= 42, [s for s, e in enumerate(elig) if not e]
    assert not all(elig)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(48))
def test_random_coupled_templates(built, sm_count, seed):
    snap, tmpl, ctr, limit = random_case(seed, sm_count)
    cap = limit or 4000                               # keep the single-thread oracle in seconds
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, threads=8)
    engine = importlib.import_module("cluster-capacity_b200.engine")
    for kind in (abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL):
        with engine.Engine(device=0, engine=kind) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(cap)
            stats = helpers.run_stats(eng)
        assert got.placed == want.placed and got.stop_code == want.stop_code, (seed, kind)
        assert np.array_equal(got.pod_node, want.pod_node), (seed, kind)
        assert np.array_equal(got.reason_hist, want.reason_hist), (seed, kind)
        if kind == abi.ENGINE_AUTO:
            assert stats["engine"] == helpers.expected_engine(snap, tmpl, ctr, sm_count), (seed, snap.n, stats)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(48))
def test_random_coupled_templates_forced_look_ahead(built, sm_count, seed, monkeypatch):
    """The multi-commit kernel with its look-ahead forced on for every PodTopologySpread term in every wave (CCSIM_DEBUG_FLAGS=32):
    candidates published from closed cells start dormant, wake up when a minimum move lifts the limit over their cell, crowd the
    tiles' lists (waves without a placement are repeated strictly) — the pod -> node sequence must not change."""
    snap, tmpl, ctr, limit = random_case(seed, sm_count)
    cap = limit or 4000
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, threads=8)
    engine = importlib.import_module("cluster-capacity_b200.engine")
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", "32")
    with engine.Engine(device=0, engine=abi.ENGINE_AUTO) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        got = eng.run(cap)
        stats = helpers.run_stats(eng)
    assert stats["engine"] == helpers.expected_engine(snap, tmpl, ctr, sm_count), (seed, snap.n, stats)
    assert got.placed == want.placed and got.stop_code == want.stop_code, seed
    assert np.array_equal(got.pod_node, want.pod_node), seed
    assert np.array_equal(got.reason_hist, want.reason_hist), seed


def random_node_local_case(seed):
    """Templates whose predicates and scorers are node-local (tie-run batching when there is one template and no
    PreferNoSchedule class; lean / generic kernels otherwise): taints, tolerations, selector bits, scalar resources,
    ephemeral storage, best-effort pods, score weights, several templates."""
    rng = np.random.default_rng(5000 + seed)
    n = int(rng.choice([700, 5000, 30000]))
    a_cpu = rng.choice([1000, 2000, 4000, 8000, 64000], n)
    a_mem = a_cpu * int(rng.choice([1, 2, 4])) * MiB
    a_pods = rng.choice([4, 16, 110], n)
    req_cpu = (rng.random(n) * 0.6 * a_cpu).astype(np.int64) // 10 * 10
    req_mem = (rng.random(n) * 0.6 * a_mem).astype(np.int64)
    npods = np.minimum(rng.integers(0, 30, n), a_pods).astype(np.int32)
    taint = np.zeros(n, np.uint64)
    for tid in range(4):
        taint |= (rng.random(n) < 0.08).astype(np.uint64) << np.uint64(tid)
    prefer_on = rng.random() < 0.4
    nosched, prefer = (0b0011, 0b1100) if prefer_on else (0b1111, 0)
    taint |= (rng.random(n) < 0.02).astype(np.uint64) << np.uint64(abi.TAINT_UNSCHEDULABLE_BIT)
    static = (rng.random(n) < 0.5).astype(np.uint64) | ((rng.random(n) < 0.7).astype(np.uint64) << np.uint64(1))
    scal = [(rng.integers(0, 9, n).astype(np.int64), rng.integers(0, 3, n).astype(np.int64))] if rng.random() < 0.3 else []
    snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, alloc_eph=np.full(n, 100 * GiB), req_cpu=req_cpu, req_mem=req_mem, npods=npods,
                        scalars=scal, taint_mask=taint.reshape(1, n), taint_nosched=[nosched], taint_prefer=[prefer],
                        static_mask=static.reshape(1, n), taint_lists=[[t for t in range(4) if (int(x) >> t) & 1] for x in taint])
    tmpl = []
    for _ in range(int(rng.choice([1, 1, 1, 3]))):
        t = abi.default_template(int(rng.choice([0, 100, 250, 1500])), int(rng.choice([0, 64, 512])) * MiB)
        if t.req_cpu == 0 and t.req_mem == 0:
            t = abi.default_template(0, 0)
        if rng.random() < 0.5:
            t.flags |= abi.TF_HAS_NODE_SELECTOR
            t.sel_mask[0] = int(rng.choice([1, 2, 3]))
        t.tol_nosched[0] = int(rng.integers(0, 16)) & nosched
        t.tol_prefer[0] = int(rng.integers(0, 16)) & prefer
        if scal and rng.random() < 0.7:
            t.req_scalar[0] = int(rng.integers(1, 3))
        if rng.random() < 0.2:
            t.req_eph = int(rng.integers(1, 40)) * GiB
        if rng.random() < 0.3:
            t.w_fit, t.w_balanced = int(rng.integers(1, 4)), int(rng.integers(1, 4))
        tmpl.append(t)
    return snap, tmpl, [], int(rng.choice([0, 0, 0, 57, 333, 5000]))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(16))
def test_random_node_local_templates(built, seed):
    snap, tmpl, ctr, limit = random_node_local_case(seed)
    cap = limit or 6000
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, threads=8)
    engine = importlib.import_module("cluster-capacity_b200.engine")
    for kind in (abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL):
        with engine.Engine(device=0, engine=kind) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(cap)
        assert got.placed == want.placed and got.stop_code == want.stop_code, (seed, kind)
        assert np.array_equal(got.pod_node, want.pod_node), (seed, kind)
        assert np.array_equal(got.reason_hist, want.reason_hist), (seed, kind)
        assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful), (seed, kind)
