"""The normalised soft scorers on the generic wave kernel's three-pass waves, against the plain Go-semantics model
(tests/scoremodel.py): NodeAffinity preferred terms, PodTopologySpread ScheduleAnyway / system-default spreading on any topology
column, the InterPodAffinity score, with counters that change at every commit, and PreferNoSchedule classes.

CPU: the C oracle equals the model on every case below; each of the model's mutations (a soft path wrong in one named way)
changes at least one predicted sequence, so the cases would notice a kernel with that defect; the generators reach the edges
they are written for; counters that could leave int32 are refused by the encoder (by topology key) and by the oracle.

GPU: ENGINE_AUTO and ENGINE_SEQUENTIAL run every case on wave<true>, or on wave<false> one node past the resident tile (found by
bisection over ccsim_prepare), and give the model's pod -> node sequence, stop code, FitError histogram and preemption counts."""
import functools
import importlib

import numpy as np
import pytest

import helpers
import scoremodel as sm

abi = importlib.import_module("cluster-capacity_b200._abi")
fw = importlib.import_module("cluster-capacity_b200.framework")
from oracle import binding as oracle  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
AUTO, SEQ = abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL
SMEM_CNT_MAX_INTS = 16384       # counters beyond this many ints live as per-CTA replicas in global memory (ccsim_wave.cuh)

# static bits of the generated snapshots
B_IGNORED, B_HOST = 0, 1        # IgnoredNodes of explicit constraints; "node carries kubernetes.io/hostname"
B_PREF = (2, 3, 4, 5)           # labels that preferred node-affinity terms select
B_ELIG0 = 8                     # B_ELIG0 + j: counter j's elig_bit (has the key and passes the inclusion policies)
HOST = "host"


# ---- generators ----------------------------------------------------------------------------------------------------------------
def build(rng, live, fillers=0, system_default=False, cols=(("zone", 6, 0.1), ("rack", 40, 0.05)), spts=None, ipa=(),
          n_pref=0, n_hard=0, host_missing=0.0, taint_words=1, max_pods=0, pod=(300, 512 * MiB), slots=(1, 5),
          weights=None, spread_init=20, spread_inc=(0, 1, 1), elig_p=0.5, ipa_inc=(-7, -3, 0, 2, 5)):
    """(snapshot, [template], counters, max_pods) of one soft workload. `live` nodes with room for slots[0]..slots[1]-1 clones sit
    evenly among `fillers` nodes that are full on pods. cols: (name, values, p_missing) topology columns; spts: [(column name or
    HOST, maxSkew)] (the system defaults when None and system_default); ipa: column names or HOST; n_hard: non-binding hard spread
    terms on a column every node carries. Every per-node value of a filler comes from a second generator, and the main one draws
    a fixed number of values whatever N is: make(N) = build(same seed, fillers = N - live) is one workload that only grows."""
    N = live + fillers
    frng = np.random.default_rng(int(rng.integers(1 << 30)))
    pos = (np.arange(live) * N) // max(1, live)
    is_live = np.zeros(N, bool)
    is_live[pos] = True

    def column(k, p):
        v = np.empty(N, np.int32)
        v[pos] = rng.integers(0, k, live)
        v[~is_live] = frng.integers(0, k, N - live)
        m = np.zeros(N, bool)
        m[pos] = rng.random(live) < p
        m[~is_live] = frng.random(N - live) < p
        v[m] = -1
        return v

    def per_node(draw):
        """A length-N column: the live nodes' values drawn from rng, the fillers' from frng."""
        v = draw(rng, live)
        out = np.empty(N, v.dtype)
        out[pos] = v
        out[~is_live] = draw(frng, N - live)
        return out

    topo, colidx, values = [], {}, {}
    for name, k, p in cols:
        colidx[name], values[name] = len(topo), k
        topo.append(column(k, p))
    if n_hard:
        colidx["hard"], values["hard"] = len(topo), 4
        topo.append(column(4, 0.0))
    has_host = np.ones(N, bool)
    has_host[pos] = rng.random(live) >= host_missing
    if spts is None:
        spts = [(HOST, 3), ("zone", 5)] if system_default else []

    a_pods = np.ones(N, np.int32)
    npods = np.ones(N, np.int32)
    a_pods[pos] = rng.integers(slots[0], slots[1], live)
    npods[pos] = 0
    a_cpu = np.full(N, 4000, np.int64)
    a_mem = np.full(N, 16 * GiB, np.int64)
    a_cpu[pos] = rng.choice([1000, 2000, 4000, 8000], live)
    a_mem[pos] = rng.choice([2, 4, 8, 16], live) * GiB
    r_cpu = np.zeros(N, np.int64)
    r_mem = np.zeros(N, np.int64)
    r_cpu[pos] = (rng.random(live) * 0.5 * a_cpu[pos]).astype(np.int64)
    r_mem[pos] = (rng.random(live) * 0.5 * a_mem[pos]).astype(np.int64)

    static = np.zeros(N, np.uint64)
    put = lambda b, m: np.uint64(1 << b) * m.astype(np.uint64)
    static |= put(B_HOST, has_host)
    for b in B_PREF:
        static |= put(b, per_node(lambda g, k: g.random(k) < 0.4))
    ctr = []

    def counter(col, init, inc, elig=None):
        j = len(ctr)
        eb = -1
        if elig is not None:
            nonlocal static
            static |= put(B_ELIG0 + j, elig)
            eb = B_ELIG0 + j
        ctr.append(abi.make_counter(col, init, inc=inc, elig_bit=eb))
        return j

    t = abi.default_template(*pod)
    if weights is None:
        weights = rng.integers(1, 6, 7)
    t.w_taint, t.w_node_affinity, t.w_fit, t.w_pts, t.w_ipa, t.w_balanced, t.w_image = [int(x) for x in weights]
    t.n_spts = len(spts)
    for c, (key, skew) in enumerate(spts):
        sc = t.spts[c]
        sc.max_skew = skew
        inc = int(rng.choice(spread_inc))
        if key == HOST:
            sc.hostname, sc.has_key_bit = 1, (B_HOST if not has_host.all() else -1)
            sc.counter = counter(-1, per_node(lambda g, k: g.integers(0, min(4, spread_init + 1), k)), inc)
        else:
            sc.hostname, sc.has_key_bit = 0, -1
            col, k = colidx[key], values[key]
            elig = (topo[col] >= 0) & per_node(lambda g, k: g.random(k) < 0.7) if inc and rng.random() < elig_p else None
            sc.counter = counter(col, rng.integers(0, spread_init + 1, k), inc, elig)
    if spts and not system_default:       # requireAllTopologies: the nodes that miss a constraint key are ignored
        miss = np.zeros(N, bool)
        for key, _ in spts:
            miss |= ~has_host if key == HOST else topo[colidx[key]] < 0
        static |= put(B_IGNORED, miss)
        t.spts_ignored_bit = B_IGNORED
    t.n_ipa_score = len(ipa)
    for q, key in enumerate(ipa):
        inc = int(rng.choice(ipa_inc))
        if key == HOST:
            t.ipa_score_counter[q] = counter(-1, per_node(lambda g, k: g.integers(-60, 61, k)), inc)
        else:
            t.ipa_score_counter[q] = counter(colidx[key], rng.integers(-60, 61, values[key]), inc)
    t.n_pts = n_hard
    for c in range(n_hard):       # coupled but never binding: maxSkew above any count the run can reach
        t.pts[c].counter = counter(colidx["hard"], rng.integers(0, 5, 4), 1)
        t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = 10 ** 6, 1, 0
    t.n_pref_terms = n_pref
    for q in range(n_pref):
        bits = rng.choice(B_PREF, int(rng.integers(1, 3)), replace=False)
        t.pref_mask[q][0] = int(sum(1 << int(b) for b in bits))
        t.pref_weight[q] = int(rng.integers(1, 101))

    # PreferNoSchedule classes: three taints, spread over the taint words; the pod tolerates one of them half of the time
    ids = [0, 1, 2] if taint_words == 1 else [0, 64 + 5, 64 + 40]
    tmask = np.zeros((taint_words, N), np.uint64)
    prefer = [0] * taint_words
    for tid in ids:
        w, b = tid >> 6, tid & 63
        prefer[w] |= 1 << b
        tmask[w] |= put(b, per_node(lambda g, k: g.random(k) < 0.25))
    if rng.random() < 0.5:
        tid = int(rng.choice(ids))
        t.tol_prefer[tid >> 6] = 1 << (tid & 63)
    img = per_node(lambda g, k: np.where(g.random(k) < 0.3, g.integers(1, 101, k), 0)).astype(np.uint8)
    t._keep_img = img
    t.image_score = img.ctypes.data_as(abi.C.POINTER(abi.C.c_uint8))
    snap = abi.Snapshot(N, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, static_mask=static.reshape(1, N),
                        topo=topo, taint_mask=tmask, taint_prefer=prefer)
    if max_pods == "mid":
        max_pods = max(1, int(a_pods[pos].sum()) // 2)
    return snap, [t], ctr, max_pods


SEEDS = range(24)
LIVE = [40, 150, 400, 600]
FILLERS = [0, 0, 100, 600, 3000, 9000, 20000, 60000]
PAST_TILE = (22, 23)            # these seeds run one node past the resident tile on the GPU
CPU_PAST_TILE_N = 260_000       # ... and at about that size on the CPU, where the tile's size is not known


def random_case(seed, n_total=None):
    """Randomized soft workload `seed`: zone / rack / region spreading with random maxSkew, inclusion policies (elig_bit) and
    missing labels, the system defaults against explicit constraints, hostname constraints with and without has_key_bit,
    InterPodAffinity counters with positive and negative increments, preferred node-affinity terms, PreferNoSchedule classes
    in one or two taint words, --max-limit 0, 1 or mid-run. n_total: the node count (fillers added); default: by seed."""
    rng = np.random.default_rng(7000 + seed)
    system_default = seed % 2 == 0
    live = LIVE[seed % len(LIVE)] if seed not in PAST_TILE else 150
    cols = (("zone", int(rng.integers(2, 9)), float(rng.choice([0, 0.05, 0.2]))),
            ("rack", int(rng.integers(5, 80)), float(rng.choice([0, 0.03]))),
            ("region", 3, float(rng.choice([0, 0.1]))))
    spts = None
    if not system_default:
        keys = list(rng.choice(["zone", "rack", "region", HOST], int(rng.integers(1, 5)), replace=False))
        spts = [(str(k), int(rng.integers(1, 6))) for k in keys]
    ipa = [str(k) for k in rng.choice(["zone", "rack", HOST], int(rng.integers(0, 4)), replace=False)]
    limit = ["mid", 0, 1][seed % 3] if seed not in PAST_TILE else "mid"
    fillers = FILLERS[(seed // 2) % len(FILLERS)]
    if n_total is not None:
        fillers = n_total - live
    return build(rng, live, fillers, system_default, cols, spts, ipa, n_pref=int(rng.integers(0, 4)),
                 host_missing=float(rng.choice([0, 0.05])), taint_words=1 + seed % 2 if seed % 3 else 1, max_pods=limit)


def _chunks(n):
    grid = -(-n // helpers.GRID_NODES)      # the persistent grid of a small cluster: one CTA per 512 nodes
    chunk = -(-n // grid)
    return grid, chunk


def edge_cta_dead():
    """4100 nodes over nine CTAs: every node of CTA 2 is full, every node of CTA 4 misses the zone label (ignored)."""
    rng = np.random.default_rng(11)
    snap, tmpl, ctr, mp = build(rng, 4100, 0, False, spts=[("zone", 2), (HOST, 1)], ipa=("rack",), n_pref=2, max_pods=900,
                                slots=(1, 3))
    grid, chunk = _chunks(snap.n)
    assert grid >= 5
    full = np.arange(2 * chunk, 3 * chunk)
    snap.npods[full] = snap.alloc_pods[full]
    ign = np.arange(4 * chunk, 5 * chunk)
    snap.topo[0][ign] = -1
    snap.static_mask[0][ign] |= np.uint64(1 << B_IGNORED)
    return snap, tmpl, ctr, mp


def edge_all_ignored():
    """Every feasible node is ignored: the explicit constraint's key is only on the full fillers."""
    rng = np.random.default_rng(12)
    snap, tmpl, ctr, mp = build(rng, 300, 900, False, spts=[("zone", 1)], ipa=("zone",), n_pref=1, slots=(1, 4))
    snap.topo[0][snap.npods == 0] = -1
    snap.static_mask[0] |= np.uint64(1 << B_IGNORED) * (snap.topo[0] < 0).astype(np.uint64)
    return snap, tmpl, ctr, mp


def edge_spread_raws_zero():
    """Every spread raw is 0 (counts 0 that never move, maxSkew 1): max == 0 gives every scored node 100."""
    rng = np.random.default_rng(13)
    return build(rng, 400, 200, False, spts=[("zone", 1), ("rack", 1), (HOST, 1)], ipa=("rack",), n_pref=2,
                 spread_init=0, spread_inc=(0,), slots=(1, 4))


def edge_node_affinity_max_zero():
    """The preferred terms match only full nodes: NodeAffinity max == 0 every cycle (raw 0 for all)."""
    rng = np.random.default_rng(14)
    snap, tmpl, ctr, mp = build(rng, 400, 400, True, ipa=("zone",), n_pref=3, slots=(1, 4))
    live = snap.npods == 0
    snap.static_mask[0][live] &= ~np.uint64(sum(1 << b for b in B_PREF))
    return snap, tmpl, ctr, mp


def edge_truncation():
    """Small NodeAffinity weights (2, 3, 4): 100 * raw meets multiples of max and one below them (the guards assert both; the
    spread normalisation's 100 * (max + min - r) meets both across the edge cases)."""
    rng = np.random.default_rng(15)
    snap, tmpl, ctr, mp = build(rng, 300, 0, False, spts=[("rack", 1)], n_pref=3, spread_init=3, slots=(1, 6),
                                cols=(("zone", 3, 0.0), ("rack", 12, 0.0)))
    t = tmpl[0]
    for q, w in enumerate((2, 3, 4)):     # raws 0..9: 100 * 3 % 7 == 6, 100 * 2 % 4 == 0, ...
        t.pref_weight[q] = w
    return snap, tmpl, ctr, mp


def edge_domain_ladder():
    """Six zones of one to three small nodes: as a zone's last feasible node fills, size and with it w drop mid-run."""
    rng = np.random.default_rng(16)
    snap, tmpl, ctr, mp = build(rng, 14, 50, False, spts=[("zone", 2)], cols=(("zone", 6, 0.0),), slots=(1, 3),
                                spread_inc=(1,), elig_p=0.0)
    snap.topo[0][snap.npods == 0] = np.array([0, 0, 0, 1, 1, 2, 2, 2, 3, 4, 4, 5, 5, 5], np.int32)
    return snap, tmpl, ctr, mp


def limit_many_domains():
    """A zone column with 20000 values: the soft zone counter (and an InterPodAffinity one) exceed the shared-memory counters
    and live as per-CTA replicas in global memory; the domain stamps are 20001 long."""
    rng = np.random.default_rng(17)
    snap, tmpl, ctr, mp = build(rng, 500, 24000, True, cols=(("zone", 20000, 0.02),), ipa=("zone",), n_pref=1, max_pods=600)
    assert max(c.n_domains for c in ctr if c.topo_col >= 0) > SMEM_CNT_MAX_INTS
    return snap, tmpl, ctr, mp


def limit_max_counters():
    """8 soft constraints, 8 InterPodAffinity keys and 8 never-binding hard spread terms: 24 counters, the commit's
    one-lane-per-counter update at its limit."""
    rng = np.random.default_rng(18)
    cols = tuple(("c%d" % k, 2 + 3 * k, 0.05 * (k % 3)) for k in range(7))
    spts = [("c%d" % k, 1 + k % 4) for k in range(7)] + [(HOST, 2)]
    ipa = ["c%d" % k for k in range(7)] + [HOST]
    snap, tmpl, ctr, mp = build(rng, 400, 300, False, cols=cols, spts=spts, ipa=ipa, n_pref=2, n_hard=8, max_pods="mid",
                                host_missing=0.05)
    assert len(ctr) == abi.MAX_COUNTERS == 24 and tmpl[0].n_spts == 8 and tmpl[0].n_ipa_score == 8
    return snap, tmpl, ctr, mp


def edge_unresolvable():
    """Some nodes can never hold the pod: allocatable cpu (200m) or memory (256Mi) below its request. The run ends with them
    UnschedulableAndUnresolvable ("Preemption is not helpful") next to nodes that only ran out of pod slots ("No preemption
    victims")."""
    rng = np.random.default_rng(19)
    snap, tmpl, ctr, mp = build(rng, 300, 300, True, ipa=("rack",), n_pref=2, slots=(1, 4))
    live = np.nonzero(snap.npods == 0)[0]
    small_cpu, small_mem = live[::5], live[1::5]
    snap.alloc_cpu[small_cpu], snap.req_cpu[small_cpu], snap.nz_cpu[small_cpu] = 200, 0, 0
    snap.alloc_mem[small_mem], snap.req_mem[small_mem], snap.nz_mem[small_mem] = 256 * MiB, 0, 0
    return snap, tmpl, ctr, mp


EDGES = {"unresolvable": edge_unresolvable, "cta_dead": edge_cta_dead, "all_ignored": edge_all_ignored, "spread_raws_zero": edge_spread_raws_zero,
         "node_affinity_max_zero": edge_node_affinity_max_zero, "truncation": edge_truncation, "domain_ladder": edge_domain_ladder,
         "many_domains": limit_many_domains, "max_counters": limit_max_counters}


def case(name):
    if name.startswith("seed"):
        seed = int(name[4:])
        return random_case(seed, CPU_PAST_TILE_N if seed in PAST_TILE else None)
    return EDGES[name]()


CASES = ["seed%d" % s for s in SEEDS] + sorted(EDGES)


@functools.lru_cache(maxsize=None)
def predicted(name):
    snap, tmpl, ctr, mp = case(name)
    return sm.run(snap, tmpl, ctr, max_pods=mp)


def _same(a, b):
    return (a.placed, a.stop_code) == (b.placed, b.stop_code) and np.array_equal(a.pod_node, b.pod_node)


def _assert_equal(got, want, who):
    m = min(got.placed, want.placed)
    diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
    assert (got.placed, got.stop_code) == (want.placed, want.stop_code), (who, got.placed, want.placed, diff[:1])
    assert np.array_equal(got.pod_node, want.pod_node), (who, "first difference at pod", diff[:1])
    assert np.array_equal(got.reason_hist, want.reason_hist), who
    assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful), who


# ---- CPU -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_model(built, name):
    """The oracle's run equals the model's: sequence, stop code, FitError histogram, preemption counts."""
    snap, tmpl, ctr, mp = case(name)
    want = predicted(name)
    assert want.placed > 0
    got = oracle.run(snap, tmpl, ctr, max_pods=mp, threads=8, memo=True)
    _assert_equal(got, want, "oracle")


def test_generators_reach_their_edges(built):
    """Each edge case meets the edge it is written for, and the randomized seeds cover both modes, both kernels' sizes and every
    --max-limit kind."""
    soft = {name: predicted(name).soft for name in EDGES}
    cycles = lambda name: predicted(name).placed + (predicted(name).stop_code == abi.STOP_UNSCHEDULABLE)
    assert soft["all_ignored"]["no_scored"] == cycles("all_ignored") - 1      # (the terminal cycle has no feasible node)
    z = soft["spread_raws_zero"]
    assert z["pts_max0"] > 0 and z["pts_max0"] + z["no_scored"] == len(z["sizes"])
    assert soft["node_affinity_max_zero"]["na_max0"] == cycles("node_affinity_max_zero") - 1
    assert {"at", "below"} <= soft["truncation"]["na_edges"]
    assert {"at", "below"} <= set().union(*(s["pts_edges"] for s in soft.values()))
    sizes = [s[0] for s in soft["domain_ladder"]["sizes"]]
    assert max(sizes) == 6 and any(b < a for a, b in zip(sizes, sizes[1:])) and min(sizes) < 6, sizes
    assert soft["cta_dead"]["no_scored"] == 0 and len(set(soft["cta_dead"]["sizes"])) > 1
    u = predicted("unresolvable")
    assert u.stop_code == abi.STOP_UNSCHEDULABLE and u.preempt_not_helpful == 120 and u.preempt_no_victims == 600 - 120
    modes = {random_case(s)[1][0].spts_ignored_bit >= 0 for s in SEEDS if s not in PAST_TILE}
    incs = {c.inc for s in SEEDS if s not in PAST_TILE for c in random_case(s)[2]}
    assert modes == {False, True} and min(incs) < 0 < max(incs)
    assert {random_case(s)[3] == 0 for s in SEEDS} == {True, False} and any(random_case(s)[3] == 1 for s in SEEDS)


def test_past_tile_workload_only_grows():
    """make(N) of the wave<false> bisection is one workload that only grows: the template, the counters' increments, eligibility
    bits and topology-domain counts, and every live node are the same at two sizes."""
    def view(n):
        snap, tmpl, ctr, mp = random_case(PAST_TILE[0], n)
        t = abi.Template.from_buffer_copy(tmpl[0])
        t.image_score = None
        live = np.nonzero(snap.npods == 0)[0]
        cols = [snap.alloc_cpu, snap.alloc_mem, snap.alloc_pods, snap.req_cpu, snap.req_mem, snap.static_mask[0], snap.taint_mask[0],
                tmpl[0]._keep_img] + snap.topo
        nodes = [np.asarray(c)[live] for c in cols] + [np.asarray(c._keep)[live] for c in ctr if c.topo_col < 0]
        shared = [(c.topo_col, c.inc, c.elig_bit) + ((c.n_domains, bytes(np.asarray(c._keep))) if c.topo_col >= 0 else ()) for c in ctr]
        return bytes(t), shared, nodes, mp
    a, b = view(60_000), view(61_237)
    assert a[0] == b[0] and a[1] == b[1] and a[3] == b[3]
    assert len(a[2]) == len(b[2]) and all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))


MUTATION_ORDER = [n for n in CASES if not (n.startswith("seed") and int(n[4:]) in PAST_TILE)]


@pytest.mark.parametrize("mutation", sm.MUTATIONS)
def test_mutation_changes_a_prediction(built, mutation):
    """A model wrong in this one way predicts a different sequence on at least one case: the suite would notice a kernel with
    the same defect."""
    for name in MUTATION_ORDER:
        snap, tmpl, ctr, mp = case(name)
        bad = sm.run(snap, tmpl, ctr, max_pods=mp, mutate=mutation)
        if not _same(bad, predicted(name)):
            print("\n  %s: %s" % (mutation, name), end="")
            return
    pytest.fail("no case notices the mutation %s" % mutation)


# ---- int32 counters ------------------------------------------------------------------------------------------------------------
def overflow_case(init_hi=2 ** 31 - 5000, inc=1000, max_pods=0):
    """Preferred pod affinity of the pod to its own labels with weight 1000 per clone on a zone key: zone 0 starts 5000 below
    INT32_MAX. In exact arithmetic (the reference's int64) zone 0 keeps the highest InterPodAffinity raw and takes every clone;
    an int32 counter wraps at the fifth clone and sends the sixth to zone 1."""
    n = 8
    zone = (np.arange(n) % 2).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 16 * GiB), np.full(n, 8), topo=[zone])
    t = abi.default_template(100, 128 * MiB)
    t.n_ipa_score, t.ipa_score_counter[0] = 1, 0
    t.w_ipa = 5
    return snap, [t], [abi.make_counter(0, np.array([init_hi, 0], np.int32), inc=inc)], max_pods


def per_node_case(slots_last):
    """Soft hostname anti-affinity of weight 1000 (inc -1000) on four nodes whose counts start at -(2^31 - 10 000): a node's count
    stays exact for 9 more clones. Three nodes hold 8 pods and the last one `slots_last`. The cluster's 24 + slots_last slots
    would take any one count out of int32, but a node-local count only receives its own node's clones."""
    n = 4
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 16 * GiB), np.array([8, 8, 8, slots_last]))
    t = abi.default_template(100, 128 * MiB)
    t.n_ipa_score, t.ipa_score_counter[0] = 1, 0
    t.w_ipa = 5
    return snap, [t], [abi.make_counter(-1, np.full(n, -(2 ** 31 - 10_000), np.int32), inc=-1000)]


def test_overflow_refused_by_the_oracle(built):
    """The model (int64 counts) fills zone 0 first; the oracle refuses the counter (rc=-4) instead of wrapping it. The boundary is
    exact: 4 placements keep zone 0 inside int32 and run (equal to the model), 5 reach 2^31 and are refused."""
    snap, tmpl, ctr, _ = overflow_case()
    want = sm.run(snap, tmpl, ctr)
    assert want.placed == 64 and set(snap.topo[0][want.pod_node[:32]]) == {0}      # zone 0 first, until it is full
    for mp in (0, 6, 5):
        with pytest.raises(RuntimeError, match="rc=-4"):
            oracle.run(snap, tmpl, ctr, max_pods=mp)
    _assert_equal(oracle.run(snap, tmpl, ctr, max_pods=4), sm.run(snap, tmpl, ctr, max_pods=4), "oracle")
    neg = overflow_case(init_hi=-(2 ** 31) + 5000, inc=-1000)
    for mp in (0, 5):
        with pytest.raises(RuntimeError, match="rc=-4"):
            oracle.run(*neg[:3], max_pods=mp)
    _assert_equal(oracle.run(*neg[:3], max_pods=4), sm.run(*neg[:3], max_pods=4), "oracle")


def test_overflow_bound_is_per_domain(built):
    """Each domain is bounded by its own free pod slots: 9 slots on the last node run (33 placements in all, equal to the model),
    10 are refused."""
    snap, tmpl, ctr = per_node_case(9)
    want = sm.run(snap, tmpl, ctr)
    assert want.placed == 33
    _assert_equal(oracle.run(snap, tmpl, ctr), want, "oracle")
    with pytest.raises(RuntimeError, match="rc=-4"):
        oracle.run(*per_node_case(10))


def _encode(nodes, pods, pod):
    cc = fw.New(None, None, pod, 0, [])
    try:
        cc.SyncWithClient(fw.ListClient(nodes, pods))
        return helpers.from_encoded(cc.EncodedSnapshot())
    finally:
        cc.Close()


def test_encoder_refuses_a_count_outside_int32(built):
    """Existing pods whose preferred pod-affinity terms match the new pod add their weights to their zone's counter, summed in
    int64. Three weights of 2^30 - 1 in one zone sum past INT32_MAX, and so does one pod with two terms of 2^30 (its own
    contribution is 2^31): the encoder refuses both by topology key instead of narrowing; two weights of 2^30 - 1 are kept. A
    weight outside int32 does not decode (the API's field is int32) and is refused. (The API server caps these weights at 100;
    large weights reach the sum without 21 million pods.)"""
    zone = "topology.kubernetes.io/zone"
    term = lambda w: {"weight": w, "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": zone}}
    nodes = [helpers.make_node("n%d" % i, labels={zone: "z%d" % (i % 2)}) for i in range(4)]
    pod = helpers.make_pod("p", cpu="100m", mem="64Mi", labels={"app": "sim"})
    existing = lambda k, terms: [helpers.make_pod("e%d" % q, cpu="10m", node="n0", affinity={"podAffinity": {
        "preferredDuringSchedulingIgnoredDuringExecution": terms}}) for q in range(k)]
    with pytest.raises(fw.UnsupportedError, match=r'topology key "topology.kubernetes.io/zone": a per-domain count of 3221225469 is outside int32'):
        _encode(nodes, existing(3, [term((1 << 30) - 1)]), pod)
    with pytest.raises(fw.UnsupportedError, match=r'topology key "topology.kubernetes.io/zone": a per-domain count of 2147483648 is outside int32'):
        _encode(nodes, existing(1, [term(1 << 30), term(1 << 30)]), pod)
    _, ts, ctr, _, _, _ = _encode(nodes, existing(2, [term((1 << 30) - 1)]), pod)
    assert ts[0].n_ipa_score == 1 and int(ctr[ts[0].ipa_score_counter[0]]._keep.max()) == 2 ** 31 - 2
    with pytest.raises(fw.FrameworkError, match=r"a preferred term's weight 4294967396 is outside int32"):
        _encode(nodes, existing(1, [term((1 << 32) + 100)]), pod)


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
def _engine():
    return importlib.import_module("cluster-capacity_b200.engine")


def _run_engines(snap, tmpl, ctr, max_pods, want, kernel):
    engine = _engine()
    for kind in (AUTO, SEQ):
        with engine.Engine(device=0, engine=kind) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(max_pods)
            st = eng.run_stats()
        print("\n  %-4s %-12s n %7d waves %6d placed %6d" % ("AUTO" if kind == AUTO else "SEQ", st["kernel"], snap.n, got.waves, got.placed),
              end="")
        assert st["kernel"] == kernel, (kind, st)
        _assert_equal(got, want, "AUTO" if kind == AUTO else "SEQ")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in CASES if not (n.startswith("seed") and int(n[4:]) in PAST_TILE)])
def test_soft_case(built, name):
    """The generic kernel's resident instantiation gives the model's result on every case."""
    snap, tmpl, ctr, mp = case(name)
    _run_engines(snap, tmpl, ctr, mp, predicted(name), "wave<true>")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", PAST_TILE)
def test_soft_case_past_the_resident_tile(built, seed):
    """wave<false>: the randomized workload one node past the largest cluster whose tiles stay resident."""
    make = lambda n: random_case(seed, n)[:3]
    n = helpers.largest_n(make, "wave<true>", 50_000, 2_000_000) + 1
    snap, tmpl, ctr, mp = random_case(seed, n)
    want = sm.run(snap, tmpl, ctr, max_pods=mp)
    _assert_equal(oracle.run(snap, tmpl, ctr, max_pods=mp, threads=8, memo=True), want, "oracle")
    _run_engines(snap, tmpl, ctr, mp, want, "wave<false>")


@pytest.mark.gpu
def test_overflow_refused_before_any_launch(built):
    """ccsim_prepare / ccsim_run refuse the wrapping counter by counter and domain; nothing is launched. The boundary is exact: a
    --max-limit of 5 is refused, 4 runs and equals the model. A node-local count is bounded by its own node's slots."""
    engine = _engine()
    snap, tmpl, ctr, _ = overflow_case()
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        for mp, m in ((0, 32), (6, 6), (5, 5)):      # zone 0 has 32 free slots
            with pytest.raises(engine.EngineError, match=r"counter 0, domain 0: \|initial count\| 2147478648 \+ %d placements x "
                                                         r"\|increment\| 1000 can leave int32" % m):
                eng.prepare(mp)
            with pytest.raises(engine.EngineError, match="can leave int32"):
                eng.run(mp)
        assert helpers.kernel_name(eng) == "" and eng.kernel_launches() == 0
        got = eng.run(4)
    _assert_equal(got, sm.run(snap, tmpl, ctr, max_pods=4), "engine")
    with engine.Engine(device=0) as eng:
        eng.load_nodes(per_node_case(10)[0])
        eng.set_templates(*per_node_case(10)[1:])
        with pytest.raises(engine.EngineError, match=r"counter 0, domain 3: \|initial count\| 2147473648 \+ 10 placements x "
                                                     r"\|increment\| 1000 can leave int32"):
            eng.prepare(0)
    snap, tmpl, ctr = per_node_case(9)
    _run_engines(snap, tmpl, ctr, 0, sm.run(snap, tmpl, ctr), "wave<true>")
