"""GPU: the CUDA hot path (through the C-ABI) against the CPU oracle — bit-exact placement sequence, stop code and
FitError histogram on the same seeded snapshots. Sizes are chosen so the single-thread oracle finishes in seconds."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
GiB, MiB = 1 << 30, 1 << 20


def gpu_run(snap, tmpl, ctr=(), max_pods=0, engine_kind=abi.ENGINE_SEQUENTIAL, stats=None):
    """One run; `stats`, when given, is a dict that receives the run's statistics (helpers.run_stats)."""
    engine = importlib.import_module("cluster-capacity_b200.engine")
    with engine.Engine(device=0, engine=engine_kind) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        res = eng.run(max_pods)
        counts, first = eng.node_counts(0)
        if stats is not None:
            stats.update(helpers.run_stats(eng), sm_count=eng.device_info()["sm_count"])
    return res, counts, first


def check(snap, tmpl, ctr=(), max_pods=0, threads=4, auto_engine=None, kernel=None):
    """Sequential engine (one winner per wave: evals/waves equal the reference-equivalent count) AND the default engine
    (AUTO: batched tie-run waves when the template is node-local) against the oracle. `auto_engine`: the engine AUTO must run;
    `kernel`: its kernel instantiation (Engine.kernel_name)."""
    want = oracle.run(snap, tmpl, ctr, max_pods=max_pods, threads=threads)
    stats = {}
    auto, acounts, _ = gpu_run(snap, tmpl, ctr, max_pods, abi.ENGINE_AUTO, stats)
    assert auto_engine is None or stats["engine"] == auto_engine, stats
    assert kernel is None or stats["kernel"] == kernel, stats
    assert auto.placed == want.placed and auto.stop_code == want.stop_code
    assert np.array_equal(auto.pod_node, want.pod_node), "AUTO engine: placement sequence differs from the oracle"
    assert np.array_equal(auto.reason_hist, want.reason_hist)
    assert (auto.preempt_no_victims, auto.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful)
    assert auto.waves <= want.waves
    got, counts, first = gpu_run(snap, tmpl, ctr, max_pods, abi.ENGINE_SEQUENTIAL)
    assert got.placed == want.placed
    assert got.stop_code == want.stop_code
    assert np.array_equal(got.pod_node, want.pod_node)
    assert np.array_equal(got.reason_hist, want.reason_hist)
    assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful)
    assert got.evals == want.evals and got.waves == want.waves
    if len(tmpl) == 1:
        assert np.array_equal(counts, np.bincount(want.pod_node, minlength=snap.n))
        # ReplicasOnNodes order = order of first placement (report.go:157-171)
        seen = {}
        for k, w in enumerate(want.pod_node.tolist()):
            seen.setdefault(w, k)
        for w, k in seen.items():
            assert first[w] == k
    return got


def test_c1_readme(built):
    got = check(*synth.c1())
    assert got.placed == 52


def test_c1_limit(built):
    snap, tmpl, ctr = synth.c1()
    got = check(snap, tmpl, ctr, max_pods=5)
    assert got.stop_code == abi.STOP_LIMIT_REACHED and got.placed == 5


def test_testprediction_nodes(built):
    snap = abi.Snapshot(3, np.array([300, 400, 1200]), np.array([10**9, 2 * 10**9, 10**9]), np.array([3, 3, 3]))
    t = abi.default_template(100, 5 * 10**6)
    assert check(snap, [t]).placed == 9
    assert check(snap, [t], max_pods=6).stop_code == abi.STOP_LIMIT_REACHED


@pytest.mark.parametrize("n", [1, 31, 513, 2000])
def test_c2_fit_only(built, n):
    check(*synth.c2(n=n, seed=n))


def test_c2_default_profile(built):
    check(*synth.c2(n=1500, fit_only=False))


@pytest.mark.parametrize("prefer", [False, True])
def test_c3_full_filter_set(built, prefer):
    got = check(*synth.c3(n=4000, prefer_taints=prefer))
    assert got.reason_hist[abi.R_NODE_AFFINITY] > 0 and got.reason_hist[abi.R_UNSCHEDULABLE] > 0


def test_c4_spread_and_anti_affinity(built):
    got = check(*synth.c4(n=4000, n_existing=8000, zones=8, racks=64, regions=4))
    assert got.placed > 100


def test_c4_large_domain_set_uses_global_replicas(built):
    # 20000 racks > the 16384-int shared-memory counter area: per-CTA replicas in global memory
    check(*synth.c4(n=30000, n_existing=30000, zones=16, racks=20000, regions=4), max_pods=300, kernel="wave<true>")


def test_c5_multi_template_round_robin(built):
    snap, tmpl, ctr = synth.c5(n=3000, n_templates=7)
    check(snap, tmpl, ctr, max_pods=4000, kernel="stream<2>")


def test_colocation_affinity(built):
    zone = [0, 0, 0, 1, 1, 1, 2, 2, 2]
    snap = abi.Snapshot(9, np.full(9, 1000), np.full(9, 1000), np.full(9, 30), topo=[np.asarray(zone, np.int32)])
    t = abi.default_template(10, 10)
    t.flags |= abi.TF_AFF_SELF_MATCH_ALL
    t.n_aff = 1
    t.aff_counter[0] = 0
    ctr = [abi.make_counter(0, np.zeros(3, np.int32), inc=1)]
    got = check(snap, [t], ctr, max_pods=100)
    assert got.placed == 90 and len({zone[i] for i in got.pod_node.tolist()}) == 1


def test_scalar_resources_and_ephemeral(built):
    rng = np.random.default_rng(7)
    n = 700
    snap = abi.Snapshot(n, np.full(n, 64000), np.full(n, 256 * GiB), np.full(n, 110),
                        alloc_eph=rng.integers(10, 100, n) * GiB,
                        scalars=[(rng.integers(0, 9, n), rng.integers(0, 3, n))])
    t = abi.default_template(500, 1 * GiB, eph=7 * GiB)
    t.req_scalar[0] = 2
    got = check(snap, [t], kernel="wave<true>")
    assert got.reason_hist[abi.R_SCALAR0] > 0


def test_best_effort_pod(built):
    n = 300
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.random.default_rng(3).integers(0, 20, n))
    check(snap, [abi.default_template(0, 0)])


def test_host_ports_one_clone_per_node(built):
    n = 200
    static = (np.random.default_rng(5).random(n) < 0.3).astype(np.uint64)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 110), static_mask=static.reshape(1, n),
                        has_placed_mask=True)
    t = abi.default_template(100, 100 * MiB)
    t.flags |= abi.TF_HAS_HOST_PORTS
    t.port_static_mask[0] = 1
    t.port_tmpl_conflict = 1
    got = check(snap, [t], kernel="wave<true>")
    assert got.placed == int((static == 0).sum())
    assert got.reason_hist[abi.R_NODE_PORTS] == n


def test_full_size_c2_properties(built):
    """BASELINE config C2 at full size (10k nodes): closed-form count and per-node distribution (KA5), no oracle run;
    the batched engine and the sequential engine must produce the same pod -> node sequence."""
    snap, tmpl, ctr = synth.c2()
    got, counts, _ = gpu_run(snap, tmpl, ctr)
    cap = synth.closed_form_capacity(snap, tmpl[0])
    assert got.placed == int(cap.sum()) and np.array_equal(counts, cap)
    assert got.evals == (got.placed + 1) * snap.n
    bat, bcounts, _ = gpu_run(snap, tmpl, ctr, 0, abi.ENGINE_BATCHED)
    assert np.array_equal(bat.pod_node, got.pod_node) and np.array_equal(bcounts, cap)
    assert bat.waves < got.waves // 50


@pytest.mark.parametrize("limit", [1, 2, 7, 63, 64, 65, 500, 4093, 4096, 10007])
def test_batched_limit_truncates_mid_wave(built, limit):
    snap, tmpl, ctr = synth.c2(n=3000, seed=11)
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=4)
    bat, _, _ = gpu_run(snap, tmpl, ctr, limit, abi.ENGINE_BATCHED)
    assert bat.stop_code == want.stop_code == abi.STOP_LIMIT_REACHED and bat.placed == limit
    assert np.array_equal(bat.pod_node, want.pod_node)


def test_batched_refuses_coupled_templates(built):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    snap, tmpl, ctr = synth.c4(n=2000, n_existing=4000, zones=4, racks=16, regions=2)
    with engine.Engine(device=0, engine=abi.ENGINE_BATCHED) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        with pytest.raises(engine.EngineError, match="batched engine needs"):
            eng.run(0)


def test_identical_nodes_all_tied(built):
    # 500 identical nodes: every wave ties all feasible nodes (worst case for the tie-run ordering)
    n = 500
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 30))
    check(snap, [abi.default_template(150, 100 * MiB)])


@pytest.mark.parametrize("gen,kw,pct", [("c2", dict(n=1500), 0), ("c2", dict(n=1500), 10), ("c2", dict(n=99), 0),
                                        ("c3", dict(n=4000, prefer_taints=True), 0), ("c3", dict(n=4000), 30),
                                        ("c4", dict(n=4000, n_existing=8000, zones=8, racks=64, regions=4), 0), ("c2", dict(n=700), 100)])
def test_reference_sampling_mode(built, gen, kw, pct):
    """A4: adaptive numFeasibleNodesToFind + rotating start index (schedule_one.go:538-539,697-723), as the deterministic
    sequential scan the oracle's mode=1 restates: same pod -> node sequence, same number of nodes examined."""
    engine = importlib.import_module("cluster-capacity_b200.engine")
    snap, tmpl, ctr = getattr(synth, gen)(**kw)
    limit = 3000
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, mode=1, pct=pct)
    with engine.Engine(device=0, sampling=abi.SAMPLING_REFERENCE, pct_nodes_to_score=pct) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        got = eng.run(limit)
    assert got.placed == want.placed and got.stop_code == want.stop_code
    assert np.array_equal(got.pod_node, want.pod_node)
    assert np.array_equal(got.reason_hist, want.reason_hist)
    assert got.examined == want.evals
    if pct == 100 or snap.n < 100:
        canon = oracle.run(snap, tmpl, ctr, max_pods=limit)
        assert np.array_equal(got.pod_node, canon.pod_node)


def test_preferred_node_affinity_two_phase(built):
    """NodeAffinity preferred terms (A18): raw = sum of matching weights, normalised by the max over the feasible nodes of
    each cycle — as the best nodes fill up the maximum (and with it every node's score) changes."""
    rng = np.random.default_rng(17)
    n = 2500
    a_cpu = rng.choice([2000, 4000, 8000], n)
    static = (rng.random(n) < 0.2).astype(np.uint64) | ((rng.random(n) < 0.5).astype(np.uint64) << np.uint64(1)) | ((rng.random(n) < 0.1).astype(np.uint64) << np.uint64(2))
    taint = ((rng.random(n) < 0.3).astype(np.uint64) << np.uint64(0))
    snap = abi.Snapshot(n, a_cpu, np.full(n, 16 * GiB), np.full(n, 12), static_mask=static.reshape(1, n),
                        taint_mask=taint.reshape(1, n), taint_prefer=[1], taint_lists=[[0] if int(x) else [] for x in taint])
    t = abi.default_template(500, 512 * MiB)
    t.n_pref_terms = 3
    for k, (bit, w) in enumerate([(0, 60), (1, 25), (2, 9)]):
        t.pref_weight[k] = w
        t.pref_mask[k][0] = 1 << bit
    check(snap, [t], max_pods=6000, kernel="wave<true>")


@pytest.mark.parametrize("system_default", [False, True])
def test_soft_scorers_three_phase(built, system_default):
    """PodTopologySpread score (log weights from the feasible set, min/max normalisation), InterPodAffinity score (float
    normalisation), ImageLocality column and PreferNoSchedule classes together: every wave runs the three-pass pipeline."""
    snap, tmpl, ctr = helpers.soft_cluster(5 if system_default else 4, system_default=system_default)
    got = check(snap, tmpl, ctr, max_pods=5000, kernel="wave<true>")
    assert got.placed > 1000


def test_soft_scorers_until_full(built):
    snap, tmpl, ctr = helpers.soft_cluster(6, n=700)
    got = check(snap, tmpl, ctr, kernel="wave<true>")
    assert got.stop_code == abi.STOP_UNSCHEDULABLE


def test_image_locality_only_multi_template(built):
    """ImageLocality is a static per-node, per-template column: no extra pass, also with several templates."""
    rng = np.random.default_rng(8)
    n = 2000
    snap = abi.Snapshot(n, rng.choice([2000, 4000], n), np.full(n, 8 * GiB), np.full(n, 10))
    tm = []
    for k in range(3):
        t = abi.default_template(200 + 100 * k, 128 * MiB)
        img = np.where(rng.random(n) < 0.4, rng.integers(1, 101, n), 0).astype(np.uint8)
        t._keep_img = img
        t.image_score = img.ctypes.data_as(abi.C.POINTER(abi.C.c_uint8))
        tm.append(t)
    check(snap, tm, max_pods=3000, kernel="wave<true>")


@pytest.mark.parametrize("limit", [1, 2, 7, 64, 1001, 0])
def test_multi_commit_waves_match_the_sequential_loop(built, limit):
    """Multi-commit waves (ccsim_multi.cuh; picked by ENGINE_AUTO for counter-coupled templates): several reference cycles
    per exchange, pod -> node sequence identical to one-winner-per-wave, --max-limit cuts in the middle of a wave."""
    snap, tmpl, ctr = synth.c4(n=60000, n_existing=90000, zones=32, racks=512, regions=8)
    want = oracle.run(snap, tmpl, ctr, max_pods=limit or 2500, threads=8)
    stats = {}
    got, counts, _ = gpu_run(snap, tmpl, ctr, limit or 2500, abi.ENGINE_AUTO, stats)
    assert stats["engine"] == helpers.expected_engine(snap, tmpl, ctr, stats["sm_count"]) == "multi-commit", stats
    assert got.placed == want.placed and got.stop_code == want.stop_code
    assert np.array_equal(got.pod_node, want.pod_node)
    if got.placed > 100:
        assert got.waves * 3 < want.waves          # it really batched
    assert np.array_equal(counts, np.bincount(want.pod_node, minlength=snap.n))


def test_multi_commit_zone_anti_affinity_and_missing_keys(built):
    """Required anti-affinity on a zone key (limit 0 on a replicated counter: one clone per zone) next to a spread constraint
    whose key some nodes lack, run until Unschedulable: the terminal histogram comes from the state the multi-commit
    kernel left behind."""
    rng = np.random.default_rng(31)
    n = 20000
    zone = rng.integers(0, 300, n).astype(np.int32)
    zone[rng.random(n) < 0.05] = -1
    rack = rng.integers(0, 40, n).astype(np.int32)
    snap = abi.Snapshot(n, rng.choice([2000, 4000, 8000], n), np.full(n, 16 * GiB), np.full(n, 20), topo=[zone, rack])
    ctr = [abi.make_counter(0, (rng.random(300) < 0.1).astype(np.int32), inc=1),
           abi.make_counter(1, rng.integers(0, 3, 40), inc=1)]
    t = abi.default_template(200, 128 * MiB)
    t.n_anti = 1
    t.anti_counter[0] = 0
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 1, 3, 1, 0
    got = check(snap, [t], ctr, auto_engine="multi-commit", kernel="multi<false>")
    assert got.stop_code == abi.STOP_UNSCHEDULABLE and got.placed > 200   # nodes without the zone label are not bound by the anti-affinity term
