"""The Filter and the FitError diagnosis of every wave-kernel instantiation, against the plain Go-semantics model (tests/scoremodel.py).

Each ladder is a small deterministic workload built at the edges where a kernel's incremental Filter state can drift from the
per-cycle recount the reference does, or where a kernel's write-back feeds the terminal diagnosis a stale value:
- node-local: every node-local reason at the terminal cycle (taints whose Spec order differs from their bit order, in one and in
  two taint words; NodeUnschedulable, tolerated and not; selector, required terms, nodeName and PreFilter bits; static host
  ports; existing pods' anti-affinity; cpu, memory, ephemeral-storage and scalar shortages; requests above the allocatable;
  nodes already overcommitted);
- spread: zone and rack constraints at maxSkew 1, 3 and INT32_MAX, self_match 0 and 1, min_zero with a true minimum above 0, a
  domain outside n_present, nodes without the key, and a minimum that moves on the run's last placement, so that the terminal
  diagnosis of some nodes depends on the new minimum;
- anti-affinity: hostname counters (node-local, in the lean tile) and a zone term that nodes without the zone key pass;
- affinity: required zone affinity through the first-pod bypass, from existing pods, and without self-match;
- pod-list ports: three templates of which two conflict on a host port, through the placed-template mask.

CPU: the C oracle equals the model on every case (sequence, stop code, FitError histogram, preemption split); every Filter mutation
of the model changes at least one prediction; the generators meet the edges they are written for.
GPU: every case on each instantiation it can reach, under ENGINE_AUTO and ENGINE_SEQUENTIAL, against the model and the oracle:
sequence, stop code, histogram, preemption split and per-node counts; the instantiation is asserted, and the last test checks
that the file ran all ten."""
import importlib

import numpy as np
import pytest

import helpers
import scoremodel as sm

abi = importlib.import_module("cluster-capacity_b200._abi")
from oracle import binding as oracle  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
AUTO, SEQ = abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL
INT32_MAX = 2 ** 31 - 1
UNSCHED_BIT = np.uint64(1) << np.uint64(abi.TAINT_UNSCHEDULABLE_BIT)


def _bits(*b):
    return sum(1 << x for x in b)


# ---- node-local ladder ---------------------------------------------------------------------------------------------------------
LOCAL_KINDS = ["pods4", "cpu3", "mem2", "full", "overcommit", "cpu_beyond",                  # NodeResourcesFit
               "unschedulable", "taints", "no_selector", "port", "existing_anti", "tolerated"]
EXTRA_KINDS = ["prefilter", "no_term", "term1_only", "eph2", "eph_beyond", "scalar1", "scalar_beyond"]


def node_local(words=1, n=612, templates=1, fit_only=False, nodename=False, fillers=0):
    """Nodes of every node-local kind, round-robin. words=1: one taint and one static word (the lean and streaming kernels);
    words=2: two of each plus the extras that send a workload to the generic kernel (PreFilter set, required terms, ephemeral
    storage, a scalar resource). templates=3: three templates (the streaming kernels), the third too big for many nodes, so the
    run stops on it while the others still fit. fit_only: only the NodeResourcesFit kinds (no mask column). fillers: nodes
    appended without a free pod slot."""
    kinds = LOCAL_KINDS[:6] if fit_only else LOCAL_KINDS + (EXTRA_KINDS if words == 2 else [])
    N = n + fillers
    kind = np.array([kinds[i % len(kinds)] for i in range(n)] + ["filler"] * fillers)
    k = lambda name: kind == name
    a_cpu, a_mem, a_pods = np.full(N, 4000), np.full(N, 8 * GiB), np.full(N, 4, np.int32)
    r_cpu, r_mem, npods = np.zeros(N, np.int64), np.zeros(N, np.int64), np.zeros(N, np.int32)
    a_eph = np.full(N, 100 * GiB)
    a_pods[k("filler")] = 0
    a_cpu[k("cpu3")] = 350                                   # three clones of 100m, then Insufficient cpu
    a_mem[k("mem2")] = 300 * MiB                             # two clones of 128Mi
    a_pods[k("full")] = npods[k("full")] = 5                 # Too many pods from the start
    r_cpu[k("overcommit")], a_cpu[k("overcommit")] = 1500, 1000          # requested above allocatable already: two reasons
    r_mem[k("overcommit")] = 9 * GiB
    a_cpu[k("cpu_beyond") | k("port")] = 50                  # the request exceeds the allocatable itself: Unresolvable
    a_pods[k("tolerated")] = 2
    taint = np.zeros((words, N), np.uint64)
    taint[0][k("unschedulable")] |= UNSCHED_BIT
    t_hi = 64 if words == 2 else 2                           # the Spec-first taint: in word 1, or a higher bit of word 0
    lists = [[] for _ in range(N)]
    for i in np.nonzero(k("taints"))[0]:
        taint[t_hi >> 6][i] |= np.uint64(1) << np.uint64(t_hi & 63)
        taint[0][i] |= np.uint64(2)
        lists[i] = [t_hi, 1]                                 # Spec order: t_hi first; bit order would name taint 1
    for i in np.nonzero(k("tolerated"))[0]:
        taint[0][i] |= np.uint64(8)
        lists[i] = [3]
    nosched = [_bits(1, 2, 3)] + ([_bits(0)] if words == 2 else [])
    static = np.zeros((words, N), np.uint64)
    static[0] |= np.uint64(1)                                # bit 0: the selector's label
    static[0][k("no_selector")] &= ~np.uint64(1)
    static[0][k("port")] |= np.uint64(2)                     # bit 1: host port 8080 taken by a pod already there
    static[0][k("existing_anti")] |= np.uint64(4)            # bit 2: an existing pod's anti-affinity matches the pod
    kw = {}
    if words == 2:
        static[1] |= np.uint64(1)                            # bit 64: inside the PreFilter node set
        static[1][k("prefilter")] = 0
        static[0] |= np.uint64(8)                            # bit 3: the first required term
        static[0][k("no_term") | k("term1_only")] &= ~np.uint64(8)
        static[1][k("term1_only")] |= np.uint64(2)           # bit 65: the second required term
        a_eph[k("eph2")], a_eph[k("eph_beyond")] = int(2.5 * GiB), GiB // 2
        sc = np.full(N, 100)
        sc[k("scalar1")], sc[k("scalar_beyond")] = 1, 0
        kw["scalars"] = [(sc, np.zeros(N))]
        kw["alloc_eph"] = a_eph
    snap = abi.Snapshot(N, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, taint_mask=taint, taint_nosched=nosched,
                        static_mask=static, taint_lists=lists, **kw)
    tmpl = []
    for q in range(templates):
        t = abi.default_template((100, 200, 700)[q], (128, 64, 128)[q] * MiB, eph=GiB if words == 2 else 0)
        if not fit_only:
            t.flags |= abi.TF_HAS_NODE_SELECTOR | abi.TF_HAS_HOST_PORTS
            t.sel_mask[0], t.port_static_mask[0], t.existing_anti_mask[0], t.tol_nosched[0] = 1, 2, 4, 8
            if q == 1:
                t.flags |= abi.TF_TOLERATES_UNSCHEDULABLE
        if words == 2:
            t.flags |= abi.TF_PREFILTER_NODES | abi.TF_HAS_AFFINITY_TERMS
            t.prefilter_bit, t.n_aff_terms = 64, 2
            t.aff_term_mask[0][0], t.aff_term_mask[1][1] = 8, 2
            t.req_scalar[0] = 1
        if nodename:
            t.nodename_idx = int(np.nonzero(k("pods4"))[0][3])
        tmpl.append(t)
    return snap, tmpl, []


# ---- spread ladder -------------------------------------------------------------------------------------------------------------
def spread(n=480):
    """Three hard constraints: zone at maxSkew 1 (self_match 1, zone 5 outside n_present = 5, every 17th node without a zone),
    rack at maxSkew 3 with min_zero and every rack's count above 0 (self_match 0: static counts), and zone again at maxSkew
    INT32_MAX. Zone 3 starts far above the others; every present zone has room for the same final count, so the run's last
    placement raises the zone minimum. Every 23rd zoned node has no rack label and never takes a clone: at the terminal cycle it
    passes the zone constraint with the new minimum and stops at the rack constraint's missing label (Unresolvable), while the
    minimum before the last placement would fail it on zone skew (Unschedulable)."""
    i = np.arange(n)
    zone = (i % 6).astype(np.int32)
    zone[i % 17 == 16] = -1
    rack = (i % 20).astype(np.int32)
    rack[(i % 23 == 22) & (zone >= 0)] = -1
    rng = np.random.default_rng(41)
    racks = rng.integers(1, 6, 20).astype(np.int32)
    zones = np.array([3, 1, 2, 9, 1, 0], np.int32)
    a_pods = np.where(zone == 5, 1, 2).astype(np.int32)
    open_ = (zone >= 0) & (rack >= 0) & (racks[rack] <= 3)          # nodes the rack constraint lets in
    final = [zones[z] + int(a_pods[open_ & (zone == z)].sum()) for z in range(5)]
    top = max(final)
    for z in range(5):                                # top up one node per present zone to the same final count
        a_pods[np.nonzero(open_ & (zone == z))[0][0]] += top - final[z]
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), a_pods, topo=[zone, rack])
    ctr = [abi.make_counter(0, zones, n_present=5, inc=1), abi.make_counter(1, racks),
           abi.make_counter(0, zones.copy(), n_present=5, inc=1)]
    t = abi.default_template(100, 128 * MiB)
    t.n_pts = 3
    for c, (j, skew, self_match, min_zero) in enumerate(((0, 1, 1, 0), (1, 3, 0, 1), (2, INT32_MAX, 1, 0))):
        t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = j, skew, self_match, min_zero
    return snap, [t], ctr


# ---- anti-affinity ladder ------------------------------------------------------------------------------------------------------
def anti(n=300):
    """Required anti-affinity of the pod to its own kind on the hostname (node-local counter; every 11th node holds a matching pod
    already) and on the zone (zone 1 holds one; every 7th node has no zone label and passes that term)."""
    i = np.arange(n)
    zone = (i % 5).astype(np.int32)
    zone[i % 7 == 6] = -1
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 3, np.int32), topo=[zone])
    ctr = [abi.make_counter(-1, (i % 11 == 10).astype(np.int32), inc=1),
           abi.make_counter(0, np.array([0, 1, 0, 0, 0], np.int32), inc=1)]
    t = abi.default_template(100, 128 * MiB)
    t.n_anti, t.anti_counter[0], t.anti_counter[1] = 2, 0, 1
    return snap, [t], ctr


# ---- affinity ladder -----------------------------------------------------------------------------------------------------------
AFFINITY_FORMS = ["bypass", "existing", "no_self_match"]


def affinity(form, n=200):
    """Required zone affinity. bypass: no matching pod anywhere and the pod matches its own term, so the first clone may go to any
    node with a zone and the rest follow it; existing: zone 2 holds 3 matching pods; no_self_match: no matching pod and the pod
    does not match its own term, so nothing is placed. Every 9th node has no zone label."""
    i = np.arange(n)
    zone = (i % 4).astype(np.int32)
    zone[i % 9 == 8] = -1
    a_pods = np.full(n, 2, np.int32)
    a_pods[zone == 3] = 3
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), a_pods, topo=[zone])
    init = np.array([0, 0, 3 if form == "existing" else 0, 0], np.int32)
    ctr = [abi.make_counter(0, init, inc=1)]
    t = abi.default_template(100, 128 * MiB)
    t.n_aff, t.aff_counter[0] = 1, 0
    t.aff_total_init = int(init.sum())
    if form != "no_self_match":
        t.flags |= abi.TF_AFF_SELF_MATCH_ALL
    return snap, [t], ctr


# ---- pod-list port ladder ------------------------------------------------------------------------------------------------------
def ports(n=300, fillers=0):
    """A pod list of three podspecs: the first two both want host port 8080 (each conflicts with the other's clones and its own),
    the third has no port. Every 5th node has 8080 taken by a pod already there."""
    N = n + fillers
    i = np.arange(N)
    a_pods = np.where(i < n, 3, 0).astype(np.int32)
    static = ((i % 5 == 4) & (i < n)).astype(np.uint64).reshape(1, N)
    snap = abi.Snapshot(N, np.full(N, 4000), np.full(N, 8 * GiB), a_pods, static_mask=static, has_placed_mask=True)
    tmpl = []
    for q, cpu in enumerate((100, 300, 200)):
        t = abi.default_template(cpu, 128 * MiB)
        if q < 2:
            t.flags |= abi.TF_HAS_HOST_PORTS
            t.port_static_mask[0], t.port_tmpl_conflict = 1, 0b011
        tmpl.append(t)
    return snap, tmpl, []


# ---- seeded random hard workloads ----------------------------------------------------------------------------------------------
def random_hard(seed):
    """A counter-coupled workload with random domain counts, skews, self-match and min_zero flags, n_present, missing labels, a
    selector and NoSchedule taints; one to four free slots per node. seed % 3 picks the pod (anti-)affinity: hostname
    anti-affinity to its own kind, zone anti-affinity to existing pods only, or zone affinity to its own kind over a column of
    three zones (large zones: the run goes on after the bypass)."""
    rng = np.random.default_rng(7000 + seed)
    n = int(rng.choice([150, 400, 1200]))
    doms = [int(rng.choice([3, 7, 40])) for _ in range(int(rng.integers(1, 3)))]
    topo = []
    for d in doms:
        col = rng.integers(0, d, n).astype(np.int32)
        col[rng.random(n) < 0.05] = -1
        topo.append(col)
    kind = seed % 3
    if kind == 2:
        aff = rng.integers(0, 3, n).astype(np.int32)
        aff[rng.random(n) < 0.05] = -1
        topo.append(aff)
    static = (rng.random(n) < 0.9).astype(np.uint64).reshape(1, n)
    taint = (rng.random(n) < 0.1).astype(np.uint64).reshape(1, n)
    snap = abi.Snapshot(n, rng.choice([1000, 4000], n), np.full(n, 8 * GiB), rng.integers(1, 5, n).astype(np.int32),
                        static_mask=static, taint_mask=taint, taint_nosched=[1], topo=topo,
                        taint_lists=[[0] if int(x) else [] for x in taint[0]])
    t = abi.default_template(int(rng.choice([100, 300])), 128 * MiB)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    ctr = []
    for c, d in enumerate(doms):
        self_match = int(rng.random() < 0.8)
        ctr.append(abi.make_counter(c, rng.integers(0, 4, d).astype(np.int32), n_present=d - int(rng.random() < 0.3), inc=self_match))
        t.pts[c].counter, t.pts[c].max_skew = c, int(rng.choice([1, 2, 3]))
        t.pts[c].self_match, t.pts[c].min_zero = self_match, int(rng.random() < 0.2)
    t.n_pts = len(doms)
    if kind == 0:
        ctr.append(abi.make_counter(-1, (rng.random(n) < 0.1).astype(np.int32), inc=1))
        t.n_anti, t.anti_counter[0] = 1, len(ctr) - 1
    elif kind == 1:
        ctr.append(abi.make_counter(0, (rng.random(doms[0]) < 0.3).astype(np.int32)))
        t.n_anti, t.anti_counter[0] = 1, len(ctr) - 1
    else:
        ctr.append(abi.make_counter(len(topo) - 1, np.zeros(3, np.int32), inc=1))
        t.n_aff, t.aff_counter[0] = 1, len(ctr) - 1
        t.flags |= abi.TF_AFF_SELF_MATCH_ALL
    return snap, [t], ctr


RANDOM_SEEDS = [3, 4, 5, 27, 32, 43]       # two of each kind, every one placing tens of pods

CASES = {"local1": lambda: node_local(1), "local2": lambda: node_local(2), "local2_nodename": lambda: node_local(2, nodename=True),
         "local1_3tmpl": lambda: node_local(1, templates=3), "fit_3tmpl": lambda: node_local(1, templates=3, fit_only=True),
         "spread": spread, "anti": anti, "ports": ports}
CASES.update({"affinity_" + f: (lambda f=f: affinity(f)) for f in AFFINITY_FORMS})
CASES.update({"random%d" % s: (lambda s=s: random_hard(s)) for s in RANDOM_SEEDS})

_PRED = {}


def predicted(name, max_pods=0, mutate=None):
    key = (name, max_pods, mutate)
    if key not in _PRED:
        _PRED[key] = sm.run(*CASES[name](), max_pods=max_pods, mutate=mutate)
    return _PRED[key]


def inside_limit(name):
    """A --max-limit inside the run: about half of it, and odd, so that it need not fall on a wave edge."""
    placed = predicted(name).placed
    return max(1, min(placed, (placed // 2) | 1))


def _assert_equal(got, want, who):
    m = min(got.placed, want.placed)
    diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
    assert (got.placed, got.stop_code) == (want.placed, want.stop_code), (who, got.placed, want.placed, diff[:1])
    assert np.array_equal(got.pod_node, want.pod_node), (who, "first difference at pod", diff[:1])
    assert np.array_equal(got.reason_hist, want.reason_hist), (who, {r: (int(a), int(b)) for r, (a, b) in
                                                                     enumerate(zip(got.reason_hist, want.reason_hist)) if a != b})
    assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful), who


def _same(a, b):
    return ((a.placed, a.stop_code, a.preempt_no_victims, a.preempt_not_helpful) == (b.placed, b.stop_code, b.preempt_no_victims,
                                                                                  b.preempt_not_helpful)
            and np.array_equal(a.pod_node, b.pod_node) and np.array_equal(a.reason_hist, b.reason_hist))


# ---- CPU -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("limit", [False, True], ids=["unschedulable", "limit"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_model(built, name, limit):
    """The oracle's run equals the model's: sequence, stop code, FitError histogram, preemption split."""
    mp = inside_limit(name) if limit else 0
    want = predicted(name, mp)
    assert want.stop_code == (abi.STOP_LIMIT_REACHED if limit and predicted(name).placed else abi.STOP_UNSCHEDULABLE)
    _assert_equal(oracle.run(*CASES[name](), max_pods=mp, threads=8), want, "oracle")


MUTATION_ORDER = ["local1", "local2", "local1_3tmpl", "spread", "anti", "ports"] + ["affinity_" + f for f in AFFINITY_FORMS]


@pytest.mark.parametrize("mutation", sm.FILTER_MUTATIONS)
def test_filter_mutation_changes_a_prediction(built, mutation):
    """A model wrong in this one way predicts a different sequence, histogram or preemption split on at least one ladder: the
    suite would notice a kernel, or a diagnosis, with the same defect."""
    for name in MUTATION_ORDER:
        if not _same(predicted(name, 0, mutation), predicted(name)):
            print("\n  %s: %s" % (mutation, name), end="")
            return
    pytest.fail("no ladder notices the mutation %s" % mutation)


def test_generators_reach_their_edges(built):
    """Each ladder meets the edges it is written for, in some cycle or at its terminal one."""
    hist = lambda name: predicted(name).reason_hist
    for name in ("local1", "local2", "local1_3tmpl"):      # every node-local reason at the terminal cycle
        h = hist(name)
        for r in (abi.R_TOO_MANY_PODS, abi.R_INSUFFICIENT_CPU, abi.R_INSUFFICIENT_MEMORY, abi.R_UNSCHEDULABLE, abi.R_NODE_AFFINITY,
                  abi.R_NODE_PORTS, abi.R_IPA_EXISTING_ANTI):
            assert h[r] > 0, (name, abi.REASON_TEXT[r])
    assert hist("local1")[abi.R_TAINT0 + 2] > 0 and hist("local1")[abi.R_TAINT0 + 1] == 0          # Spec order, not bit order
    assert hist("local2")[abi.R_TAINT0 + 64] > 0 and hist("local2")[abi.R_TAINT0 + 1] == 0
    for r in (abi.R_PREFILTER_NODES, abi.R_INSUFFICIENT_EPHEMERAL, abi.R_SCALAR0):
        assert hist("local2")[r] > 0, abi.REASON_TEXT.get(r, r)
    assert hist("local2_nodename")[abi.R_NODE_NAME] > 500 and predicted("local2_nodename").placed == 4
    for name in ("local1", "local2", "fit_3tmpl"):      # Unresolvable Fit (cpu_beyond) next to Unschedulable Fit (overcommit)
        p = predicted(name)
        assert p.preempt_no_victims > 0 and p.preempt_not_helpful > 0
    for name in ("local1_3tmpl", "fit_3tmpl"):           # the run stops on the third template, which has reasons of its own
        p = predicted(name)
        assert p.placed % 3 == 2 and hist(name)[abi.R_INSUFFICIENT_CPU] > 0
    s = predicted("spread").hard
    for edge in ("skew_at_max", "skew_one_over", "missing_key", "outside_present", "min_zero_above", "min_moved_last"):
        assert s[edge] > 0, edge
    assert hist("spread")[abi.R_PTS_SKEW] > 0 and hist("spread")[abi.R_PTS_MISSING_LABEL] > 0
    stale = predicted("spread", 0, "diag_ptsmin_stale")       # the diagnosis depends on the minimum the last placement moved
    assert stale.placed == predicted("spread").placed and not np.array_equal(stale.reason_hist, hist("spread"))
    assert stale.preempt_no_victims != predicted("spread").preempt_no_victims
    a = predicted("anti")
    assert a.hard["anti_missing_key"] > 0 and hist("anti")[abi.R_IPA_ANTI_AFFINITY] > 0
    assert a.reason_hist[abi.R_IPA_ANTI_AFFINITY] == a.preempt_no_victims
    b = predicted("affinity_bypass")
    assert b.hard["bypass"] == 1 and b.hard["bypass_ended"] == 1 and b.placed > 1
    assert len({int(x) % 4 for x in b.pod_node}) == 1                    # every clone follows the first into its zone
    assert predicted("affinity_existing").hard["bypass"] == 0
    assert predicted("affinity_existing").placed > 0
    ns = predicted("affinity_no_self_match")
    assert ns.placed == 0 and ns.preempt_not_helpful == 200 and hist("affinity_no_self_match")[abi.R_IPA_AFFINITY] == 200
    assert hist("ports")[abi.R_NODE_PORTS] > 0
    p = predicted("ports")
    on = lambda q: set(int(x) for x in p.pod_node[q::3])
    assert not (on(0) & on(1)) and (on(2) & (on(0) | on(1)))             # port holders never share a node; the third joins them
    stops = {predicted("random%d" % s).stop_code for s in RANDOM_SEEDS}
    assert stops == {abi.STOP_UNSCHEDULABLE}
    assert min(predicted("random%d" % s).placed for s in RANDOM_SEEDS) >= 20      # long enough for the counters to drift
    assert {s % 3 for s in RANDOM_SEEDS} == {0, 1, 2}
    assert sum(predicted("random%d" % s).hard["outside_present"] > 0 for s in RANDOM_SEEDS) >= 2
    assert sum(predicted("random%d" % s).hard["skew_at_max"] > 0 for s in RANDOM_SEEDS) >= 3


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
RAN = set()
ALL_INSTANTIATIONS = {"lean<false>", "lean<true>", "batched", "multi<false>", "multi<true>", "stream<0>", "stream<1>", "stream<2>",
                      "wave<true>", "wave<false>"}


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def _engine():
    return importlib.import_module("cluster-capacity_b200.engine")


def _check_counts(eng, want, n, n_tmpl, who):
    """ccsim_node_counts per template: the clones of template q on each node, from the model's sequence."""
    for q in range(n_tmpl):
        counts, _ = eng.node_counts(q)
        assert np.array_equal(counts, np.bincount(want.pod_node[q::n_tmpl], minlength=n)), (who, "node_counts of template", q)


def _run_engines(snap, tmpl, ctr, want, kernels, max_pods=0, sampling=False):
    """ENGINE_AUTO and ENGINE_SEQUENTIAL against the model's result; kernels: {engine: the instantiation it must run}."""
    engine = _engine()
    for kind in (AUTO, SEQ):
        kw = dict(sampling=abi.SAMPLING_REFERENCE, pct_nodes_to_score=100) if sampling else {}
        with engine.Engine(device=0, engine=kind, **kw) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(max_pods)
            st = eng.run_stats()
            print("\n  %-4s %-12s waves %6d placed %6d" % ("AUTO" if kind == AUTO else "SEQ", st["kernel"], got.waves, got.placed), end="")
            assert st["kernel"] == kernels[kind], (kind, st)
            RAN.add(st["kernel"])
            _assert_equal(got, want, st["kernel"])
            _check_counts(eng, want, snap.n, len(tmpl), st["kernel"])


LEAN = {AUTO: "lean<false>", SEQ: "lean<false>"}
SAMPLED = {AUTO: "lean<true>", SEQ: "lean<true>"}
GENERIC = {AUTO: "wave<true>", SEQ: "wave<true>"}
COUPLED = {AUTO: "multi<false>", SEQ: "lean<false>"}
RUNS = [      # id, case, {engine: instantiation}, reference sampling at 100 %, CCSIM_STREAM_ALL
    ("local1-batched", "local1", {AUTO: "batched", SEQ: "lean<false>"}, False, False),
    ("local1-sampling", "local1", SAMPLED, True, False),
    ("local2-generic", "local2", GENERIC, False, False),
    ("local2_nodename-generic", "local2_nodename", GENERIC, False, False),
    ("local1_3tmpl-stream1", "local1_3tmpl", {AUTO: "stream<1>", SEQ: "stream<1>"}, False, False),
    ("fit_3tmpl-stream2", "fit_3tmpl", {AUTO: "stream<2>", SEQ: "stream<2>"}, False, False),
    ("fit_3tmpl-stream0", "fit_3tmpl", {AUTO: "stream<0>", SEQ: "stream<0>"}, False, True),
    ("spread-multi", "spread", COUPLED, False, False),
    ("spread-sampling", "spread", SAMPLED, True, False),
    ("anti-multi", "anti", COUPLED, False, False),
    ("anti-sampling", "anti", SAMPLED, True, False),
    ("ports-generic", "ports", GENERIC, False, False),
] + [("affinity_%s-lean" % f, "affinity_" + f, LEAN, False, False) for f in AFFINITY_FORMS] + [
    ("random%d" % s, "random%d" % s, None, False, False) for s in RANDOM_SEEDS]


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [False, True], ids=["unschedulable", "limit"])
@pytest.mark.parametrize("name,case,kernels,sampling,stream_all", RUNS, ids=[r[0] for r in RUNS])
def test_ladder(built, sm_count, monkeypatch, name, case, kernels, sampling, stream_all, limit):
    if stream_all:
        monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    snap, tmpl, ctr = CASES[case]()
    if kernels is None:       # random workloads: the multi-commit kernel where the host's rule takes them
        kernels = COUPLED if helpers.multi_eligible(snap, tmpl, ctr, sm_count) else LEAN
    elif kernels is COUPLED:
        assert helpers.multi_eligible(snap, tmpl, ctr, sm_count)
    mp = inside_limit(case) if limit else 0
    want = predicted(case, mp)
    _assert_equal(oracle.run(snap, tmpl, ctr, max_pods=mp, threads=8), want, "oracle")
    _run_engines(snap, tmpl, ctr, want, kernels, mp, sampling)


SHARDED = [("spread", 2, {AUTO: "multi<true>", SEQ: "lean<false>"}), ("spread", 3, {AUTO: "multi<true>", SEQ: "lean<false>"}),
           ("anti", 2, {AUTO: "multi<true>", SEQ: "lean<false>"}),
           ("local2", 2, GENERIC), ("local2", 3, GENERIC), ("ports", 3, GENERIC)]


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [False, True], ids=["unschedulable", "limit"])
@pytest.mark.parametrize("case,world,kernels", SHARDED, ids=["%s-world%d" % (c, w) for c, w, _ in SHARDED])
def test_ladder_sharded(built, sm_count, case, world, kernels, limit):
    """The ladder over `world` node shards of this one device: every rank reports the whole sequence and stop code and its own
    shard's share of the histogram and the preemption split."""
    snap, tmpl, ctr = CASES[case]()
    mp = inside_limit(case) if limit else 0
    want = predicted(case, mp)
    for kind in (AUTO, SEQ):
        engs = helpers.sharded_engines(snap, tmpl, ctr, world, kind)
        try:
            res = helpers.run_sharded_once(engs, mp)
            names = [e.run_stats()["kernel"] for e in engs]
            print("\n  %s world %d: %s" % ("AUTO" if kind == AUTO else "SEQ", world, names), end="")
            assert names == [kernels[kind]] * world, names
            RAN.update(names)
            for r, e in zip(res, engs):
                assert (r.placed, r.stop_code) == (want.placed, want.stop_code)
                assert np.array_equal(r.pod_node, want.pod_node)
                _check_counts(e, want, snap.n, len(tmpl), names[0])
            assert np.array_equal(sum(r.reason_hist for r in res), want.reason_hist)
            assert (sum(r.preempt_no_victims for r in res), sum(r.preempt_not_helpful for r in res)) == (
                want.preempt_no_victims, want.preempt_not_helpful)
        finally:
            for e in engs:
                e.close()


_FIRST_STREAMED = {}
PAST_TILE = {"local2": lambda fillers: node_local(2, fillers=fillers), "ports": lambda fillers: ports(fillers=fillers)}
PAST_TILE_BASE = {"local2": 612, "ports": 300}


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [False, True], ids=["unschedulable", "limit"])
@pytest.mark.parametrize("case", sorted(PAST_TILE))
def test_ladder_streamed_generic_tile(built, sm_count, case, limit):
    """wave<false>: the ladder followed by nodes without a free pod slot, one node past the generic kernel's resident tile."""
    base = PAST_TILE_BASE[case]
    make = lambda n: PAST_TILE[case](max(0, n - base))
    if case not in _FIRST_STREAMED:
        _FIRST_STREAMED[case] = helpers.largest_n(make, "wave<true>", 50_000, 2_000_000) + 1
    n = _FIRST_STREAMED[case]
    print("\n  first wave<false>: N = %d" % n, end="")
    snap, tmpl, ctr = make(n)
    mp = inside_limit(case) if limit else 0
    want = sm.run(snap, tmpl, ctr, max_pods=mp)
    short = predicted(case, mp)                  # the fillers take nothing and only add Too many pods
    assert np.array_equal(want.pod_node, short.pod_node)
    _assert_equal(oracle.run(snap, tmpl, ctr, max_pods=mp, threads=8), want, "oracle")
    _run_engines(snap, tmpl, ctr, want, {AUTO: "wave<false>", SEQ: "wave<false>"}, mp)


@pytest.mark.gpu
def test_every_instantiation_ran(built):
    """The cases above ran all ten wave-kernel instantiations (multi<true> and the sharded wave<true> through one-device
    shards)."""
    assert ALL_INSTANTIATIONS <= RAN, sorted(ALL_INSTANTIATIONS - RAN)
