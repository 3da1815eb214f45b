"""GPU: the lean (and its reference-sampling variant), tie-run, streaming and generic wave kernels at their edges: the full grid,
the largest tile each kernel still holds (found by bisection over ccsim_prepare, not restated from byte counts), the taint-class,
term and slot limits, a tile streamed from global memory, the TMA ring wrapping in each of its modes, the padded last tile, one node
that wins every wave, and the 12-bit score field at its budget.

Every case runs the CPU oracle, ENGINE_AUTO and ENGINE_SEQUENTIAL and compares the pod -> node sequence, the stop code, the FitError
histogram, the preemption counters and the per-node counts (reference sampling: also the nodes examined). Each asserts the kernel
instantiation of each run (Engine.kernel_name) and, where it matters, the shape fact that makes the case an edge."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
engine = importlib.import_module("cluster-capacity_b200.engine")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
GiB, MiB = 1 << 30, 1 << 20
AUTO, SEQ = abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL
STREAM_TILE, STREAM_STAGES = 1024, 4        # ccsim_stream.cuh: nodes per ring stage, stages when every column is streamed


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def run_all(snap, tmpl, ctr, cap, kernel, pct=None):
    """Oracle, ENGINE_AUTO and ENGINE_SEQUENTIAL on one workload. `kernel`: the instantiation both engines must run, or a dict
    {engine: instantiation}. `pct`: reference sampling mode with that pct_nodes_to_score. Returns the oracle's result and the
    statistics of each run."""
    kernels = kernel if isinstance(kernel, dict) else {AUTO: kernel, SEQ: kernel}
    sampling = pct is not None
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, mode=1 if sampling else 0, pct=pct or 0, threads=8, memo=True)
    nt = len(tmpl)
    stats = {}
    for kind in (AUTO, SEQ):
        with engine.Engine(device=0, engine=kind, sampling=abi.SAMPLING_REFERENCE if sampling else abi.SAMPLING_CANONICAL,
                           pct_nodes_to_score=pct or 0) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(cap)
            counts, _ = eng.node_counts(0)
            st = stats[kind] = helpers.run_stats(eng)
        print("\n  %-4s %-12s grid %3d waves %6d placed %6d" % ("AUTO" if kind == AUTO else "SEQ", st["kernel"], st["grid"], got.waves, got.placed),
              end="")
        assert st["kernel"] == kernels[kind], (kind, st)
        assert got.placed == want.placed and got.stop_code == want.stop_code, (kind, got.placed, want.placed, got.stop_code)
        m = min(got.placed, want.placed)
        diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
        assert np.array_equal(got.pod_node, want.pod_node), (kind, "first difference at pod", diff[:1])
        assert np.array_equal(got.reason_hist, want.reason_hist), kind
        assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful), kind
        assert np.array_equal(counts, np.bincount(want.pod_node[0::nt], minlength=snap.n)), kind
        if sampling:
            assert got.examined == want.evals, (kind, got.examined, want.evals)
    return want, stats


def _nodes(n, seed, **kw):
    """C2's node distribution (4..64 cores, 0-70 % used) as a Snapshot; kw adds columns."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a_cpu, a_mem, a_pods, r_cpu, r_mem, npods = synth._c2_nodes(n, rng)
    return abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, **kw), rng


# ---- lean kernel, reference sampling, on the full grid ------------------------------------------------------------------
@pytest.mark.parametrize("pct", [0, 1, 100])
def test_sampling_full_grid(built, sm_count, pct):
    """100k nodes: every CTA runs, and the rotation start crosses every tile boundary; the gather reads all 132 CTAs' words."""
    snap, tmpl, ctr = synth.c2(n=100_000, seed=71)
    _, st = run_all(snap, tmpl, ctr, 3000, "lean<true>", pct=pct)
    assert st[AUTO]["grid"] == sm_count


def test_sampling_sparse_feasible_set(built, sm_count):
    """The node selector matches 1 node in 50: K (5 % of 100k) exceeds the 2000 feasible nodes, so every cycle examines all nodes."""
    n = 100_000
    snap, _ = _nodes(n, 72, static_mask=(np.arange(n) % 50 == 0).astype(np.uint64).reshape(1, n))
    t = abi.default_template(150, 100 * MiB)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    want, st = run_all(snap, [t], [], 1000, "lean<true>", pct=0)
    assert st[AUTO]["grid"] == sm_count and want.placed == 1000
    assert want.evals == n * st[AUTO]["waves"]


def test_sampling_with_taint_classes(built, sm_count):
    """PreferNoSchedule classes (three): the class words and the sampling words (K-th node, part counts) are gathered together."""
    snap, tmpl, ctr = synth.c3(n=100_000, prefer_taints=True)
    _, st = run_all(snap, tmpl, ctr, 3000, "lean<true>", pct=0)
    assert st[AUTO]["grid"] == sm_count


def test_sampling_largest_lean_tile(built, sm_count):
    """The largest cluster the sampling kernel holds: its two part counts travel as 22-bit fields of one word, whose sums over the
    grid must stay below 2^22. One node more and reference sampling is refused (it needs the lean resident kernel)."""
    make = lambda n: synth.c2(n=n, seed=73)
    n = helpers.largest_n(make, "lean<true>", 150_000, 1_000_000, sampling=abi.SAMPLING_REFERENCE)
    print("\n  largest lean<true>: N = %d" % n, end="")
    assert n < 1 << 22
    run_all(*make(n), 2000, "lean<true>", pct=0)
    with pytest.raises(engine.EngineError, match="reference sampling mode needs the lean resident kernel"):
        helpers.prepared_kernel(*make(n + 1), sampling=abi.SAMPLING_REFERENCE)


# ---- the class pick of the lean and the generic kernel --------------------------------------------------------------------
def _class_case(n, extended=False, taint_score=True, top_only=False, seed=81):
    """Nodes carrying 0..7 untolerated PreferNoSchedule taints (eight normalisation classes). `extended`: an extended-resource
    request moves the workload to the generic kernel. `top_only`: every node below the top class is unschedulable, so the highest
    class present (maxraw) is the only one."""
    rng = np.random.Generator(np.random.PCG64(seed))
    cls = rng.integers(0, 8, n)
    taint = ((np.uint64(1) << cls.astype(np.uint64)) - np.uint64(1)).astype(np.uint64)
    if top_only:
        taint[cls < 7] |= np.uint64(1) << np.uint64(abi.TAINT_UNSCHEDULABLE_BIT)
    kw = dict(taint_mask=taint.reshape(1, n), taint_prefer=[0x7F])
    if extended:
        kw["scalars"] = [(rng.integers(0, 40, n), rng.integers(0, 4, n))]
    snap, _ = _nodes(n, seed + 1, **kw)
    t = abi.default_template(150, 100 * MiB)
    if extended:
        t.req_scalar[0] = 1
    if not taint_score:
        t.score_enable &= ~abi.PL_TAINT_TOLERATION
    return snap, [t], []


@pytest.mark.parametrize("taint_score,top_only", [(True, False), (False, False), (True, True)])
@pytest.mark.parametrize("kernel", ["lean<false>", "wave<true>"])
def test_class_pick_full_grid(built, sm_count, kernel, taint_score, top_only):
    """Eight classes (CCSIM_MAX_CLASSES) on the full grid, on the lean kernel and on the generic one (the same snapshot plus an
    extended-resource request): both must match the oracle, and so each other. Also with TaintToleration scoring off while the
    classes exist, and with every feasible node in the top class."""
    snap, tmpl, ctr = _class_case(80_000, extended=kernel == "wave<true>", taint_score=taint_score, top_only=top_only)
    _, st = run_all(snap, tmpl, ctr, 2000, kernel)
    assert st[AUTO]["grid"] == sm_count


def test_eighth_prefer_taint_refused(built):
    n = 100
    taint = np.zeros(n, np.uint64)
    taint[7] = np.uint64(0xFF)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 30), taint_mask=taint.reshape(1, n), taint_prefer=[0xFF])
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        with pytest.raises(engine.EngineError, match=r"PreferNoSchedule taints \(max 7\)"):
            eng.set_templates([abi.default_template(150, 100 * MiB)], [])


def test_class_pick_second_taint_word(built, sm_count):
    """More than 64 distinct taints: PreferNoSchedule taints in taint word 1 (and one in word 0) set the class, next to 64
    tolerated NoSchedule taints in word 0. Generic kernel only."""
    n = 80_000
    rng = np.random.Generator(np.random.PCG64(83))
    w0 = rng.integers(0, 1 << 62, n, dtype=np.uint64) & ~np.uint64(1)
    w0 |= (rng.random(n) < 0.3).astype(np.uint64)                    # bit 0: PreferNoSchedule
    w1 = rng.integers(0, 16, n).astype(np.uint64)                     # taints 64..67: PreferNoSchedule
    snap, _ = _nodes(n, 84, taint_mask=np.stack([w0, w1]), taint_nosched=[(1 << 62) - 2, 0], taint_prefer=[1, 0xF])
    t = abi.default_template(150, 100 * MiB)
    t.tol_nosched[0] = (1 << 62) - 2
    _, st = run_all(snap, [t], [], 2000, "wave<true>")
    assert st[AUTO]["grid"] == sm_count


# ---- lean term and slot limits -------------------------------------------------------------------------------------------------
def _terms_case(n_pts, n_anti_topo, n_anti_local, n_aff=0, seed=85):
    """Spread constraints on topology columns 0..n_pts-1 (one slot each), anti-affinity on the first columns (no new slots) and on
    node-local counters (one slot each), and optionally required pod affinity that every node passes."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n, doms = 20_000, 200
    snap, _ = _nodes(n, seed + 1, topo=[rng.integers(0, doms, n).astype(np.int32) for _ in range(max(1, n_pts))])
    t = abi.default_template(150, 100 * MiB)
    ctr = []
    for c in range(n_pts):
        t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = len(ctr), 2 + c, 1, 0
        ctr.append(abi.make_counter(c, rng.integers(0, 3, doms).astype(np.int32), inc=1))
    t.n_pts = n_pts
    for a in range(n_anti_topo):          # existing pods' domains only (inc 0): about one domain in ten closed
        t.anti_counter[a] = len(ctr)
        ctr.append(abi.make_counter(a % max(1, n_pts), (rng.random(doms) < 0.1).astype(np.int32)))
    for a in range(n_anti_local):         # hostname anti-affinity against clones of this pod: one clone per node
        t.anti_counter[n_anti_topo + a] = len(ctr)
        ctr.append(abi.make_counter(-1, (rng.random(n) < 0.05).astype(np.int32), inc=1 if a == 0 else 0))
    t.n_anti = n_anti_topo + n_anti_local
    for a in range(n_aff):
        t.aff_counter[a] = len(ctr)
        ctr.append(abi.make_counter(0, np.ones(doms, np.int32), inc=1))
    t.n_aff = n_aff
    return snap, [t], ctr


@pytest.mark.parametrize("n_aff,kernel", [(0, "lean<false>"), (1, "wave<true>")])
def test_lean_term_limit(built, n_aff, kernel):
    """8 spread + 8 anti-affinity terms are LEAN_MAX_TERMS = 16: lean. One required affinity term more: generic."""
    snap, tmpl, ctr = _terms_case(8, 6, 2, n_aff=n_aff)
    assert tmpl[0].n_pts + tmpl[0].n_anti + tmpl[0].n_aff == 16 + n_aff
    run_all(snap, tmpl, ctr, 1500, kernel)


@pytest.mark.parametrize("n_local,kernel", [(4, "lean<false>"), (5, "wave<true>")])
def test_lean_slot_limit(built, n_local, kernel):
    """6 topology columns + 4 node-local counters are LEAN_MAX_SLOTS = 10 record slots: lean. An eleventh: generic."""
    snap, tmpl, ctr = _terms_case(6, 0, n_local)
    run_all(snap, tmpl, ctr, 1500, kernel)


# ---- the lean and tie-run tiles at their largest -------------------------------------------------------------------------------
def test_lean_resident_boundary(built, sm_count):
    """The largest cluster the lean kernel holds (node-local template, sequential engine), and one node more. The tie-run kernel
    needs 12 bytes more per node, so at that size ENGINE_AUTO runs the lean kernel too; one node more, both stream."""
    make = lambda n: synth.c2(n=n, seed=79)
    n = helpers.largest_n(make, "lean<false>", 100_000, 1_000_000, engine=SEQ)
    nxt = helpers.prepared_kernel(*make(n + 1), engine=SEQ)
    print("\n  largest lean<false>: N = %d, N + 1 runs %s" % (n, nxt), end="")
    run_all(*make(n), 2000, "lean<false>")
    run_all(*make(n + 1), 2000, "stream<2>")


def test_tie_run_band(built, sm_count):
    """The largest cluster the tie-run kernel holds, and one node more: it falls back to the lean kernel, which still holds it."""
    make = lambda n: synth.c2(n=n, seed=79)
    n = helpers.largest_n(make, "batched", 100_000, 1_000_000)
    print("\n  largest batched: N = %d, N + 1 runs %s" % (n, helpers.prepared_kernel(*make(n + 1))), end="")
    run_all(*make(n), 2000, {AUTO: "batched", SEQ: "lean<false>"})
    run_all(*make(n + 1), 2000, "lean<false>")


# ---- tie-run batching on the full grid ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("limit", [1, 131, 132, 133, 4096, 0])
def test_tie_run_full_grid_all_tied(built, sm_count, limit):
    """Identical nodes on every CTA, the last CTA's chunk short: every wave ties all feasible nodes. One pod per node, so an
    unlimited run ends when every node is full."""
    n = (sm_count - 1) * (helpers.GRID_NODES + 1) + 1
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 1))
    want, st = run_all(snap, [abi.default_template(150, 100 * MiB)], [], limit, {AUTO: "batched", SEQ: "lean<false>"})
    chunk = -(-n // sm_count)
    assert st[AUTO]["grid"] == sm_count and n - (sm_count - 1) * chunk < chunk
    assert want.placed == (limit or n)


# ---- generic kernel with its tile streamed from global memory ----------------------------------------------------------------
def _extended(n, seed=87):
    rng = np.random.Generator(np.random.PCG64(seed))
    snap, _ = _nodes(n, seed + 1, scalars=[(rng.integers(0, 6, n), rng.integers(0, 2, n))])
    t = abi.default_template(150, 100 * MiB)
    t.req_scalar[0] = 2
    return snap, [t], []


@pytest.mark.parametrize("workload", ["extended", "soft"])
def test_generic_tile_not_resident(built, sm_count, workload):
    """The first cluster too large for the generic kernel's resident tile, and one far past it."""
    make = _extended if workload == "extended" else (lambda n: helpers.soft_cluster(89, n=n))
    n = helpers.largest_n(make, "wave<true>", 50_000, 1_000_000, max_pods=300) + 1
    print("\n  first wave<false> (%s): N = %d" % (workload, n), end="")
    for m in (n, 2 * n):
        run_all(*make(m), 300, "wave<false>")


# ---- streaming kernel: each mode with a wrapping ring ---------------------------------------------------------------------------
def _tiles(n, grid):
    """Ring tiles per CTA of the streaming kernel."""
    return -(-(-(-n // grid)) // STREAM_TILE)


def test_stream_resident_columns_boundary(built, sm_count):
    """The largest cluster whose free columns stay resident next to the memo ring (stream<2>), and one node more (stream<0>:
    every column streamed through the 4-stage ring)."""
    make = lambda n: synth.c5(n=n, n_templates=4, seed=91)
    n = helpers.largest_n(make, "stream<2>", 200_000, 2_000_000, max_pods=2000)
    print("\n  largest stream<2>: N = %d" % n, end="")
    run_all(*make(n), 2000, "stream<2>")
    _, st = run_all(*make(n + 1), 2000, "stream<0>")
    assert _tiles(n + 1, st[AUTO]["grid"]) > STREAM_STAGES


def test_stream_all_columns_forced(built, sm_count, monkeypatch):
    """CCSIM_STREAM_ALL at 600k nodes: more than four tiles per CTA, so the 4-stage ring wraps inside every wave."""
    monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    n = 600_000
    _, st = run_all(*synth.c5(n=n, n_templates=4, seed=92), 2000, "stream<0>")
    assert st[AUTO]["grid"] == sm_count and _tiles(n, sm_count) > STREAM_STAGES


def test_stream_mask_columns_wrap(built, sm_count):
    """stream<1> at 600k nodes: untolerated NoSchedule taints and node selectors in some templates put the mask columns into the
    ring, which wraps (five tiles per CTA)."""
    n = 600_000
    rng = np.random.Generator(np.random.PCG64(93))
    taint = (rng.random(n) < 0.1).astype(np.uint64) | ((rng.random(n) < 0.05).astype(np.uint64) << np.uint64(1))
    static = (rng.random(n) < 0.5).astype(np.uint64) | ((rng.random(n) < 0.3).astype(np.uint64) << np.uint64(1))
    snap, _ = _nodes(n, 94, taint_mask=taint.reshape(1, n), taint_nosched=[0b11], static_mask=static.reshape(1, n))
    tmpl = []
    for k in range(4):
        t = abi.default_template(100 + 150 * k, (64 + 100 * k) * MiB)
        t.tol_nosched[0] = 0b10 if k % 2 else 0
        if k >= 2:
            t.flags |= abi.TF_HAS_NODE_SELECTOR
            t.sel_mask[0] = 1 << (k - 2)
        tmpl.append(t)
    _, st = run_all(snap, tmpl, [], 2000, "stream<1>")
    assert st[AUTO]["grid"] == sm_count and _tiles(n, sm_count) > STREAM_STAGES


@pytest.mark.parametrize("stream_all", [False, True])
def test_stream_padded_last_tile(built, sm_count, monkeypatch, stream_all):
    """Every CTA's chunk (the last one's included) ends one node past a tile boundary: its last tile holds one real node and 1023
    padding nodes, which must never win."""
    if stream_all:
        monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    chunk = 4 * STREAM_TILE + 1
    n = sm_count * chunk
    _, st = run_all(*synth.c5(n=n, n_templates=3, seed=95), 2000, "stream<0>" if stream_all else "stream<2>")
    assert st[AUTO]["grid"] == sm_count and -(-n // st[AUTO]["grid"]) % STREAM_TILE == 1


@pytest.mark.parametrize("stream_all", [False, True])
def test_stream_repeat_winner(built, sm_count, monkeypatch, stream_all):
    """One node far larger than the rest wins every wave for every template: each commit must invalidate that node's memo entry
    of every template before the next wave reads it, also while the commit queue is full."""
    if stream_all:
        monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    n = 200_000
    rng = np.random.Generator(np.random.PCG64(96))
    a_cpu, a_mem, a_pods, _, _, _ = synth._c2_nodes(n, rng)
    r_cpu, r_mem = a_cpu * 17 // 20, a_mem * 17 // 20          # every other node 85 % used: about 115 points against the big node's 198
    big = n // 2 + 17
    a_cpu[big], a_mem[big], a_pods[big], r_cpu[big], r_mem[big] = 10 ** 8, 1 << 50, 100_000, 0, 0
    snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem)
    tmpl = synth.c5(n=1, n_templates=5, seed=96)[1]
    want, _ = run_all(snap, tmpl, [], 600, "stream<0>" if stream_all else "stream<2>")
    assert (want.pod_node == big).sum() >= 300


# ---- the key's score field at its budget ----------------------------------------------------------------------------------------
def _budget_template(w_taint=1, w_fit=20, w_balanced=19, scalar=False):
    t = abi.default_template(150, 100 * MiB)
    t.w_taint, t.w_node_affinity, t.w_pts, t.w_ipa, t.w_image = w_taint, 0, 0, 0, 0
    t.w_fit, t.w_balanced = w_fit, w_balanced
    if scalar:
        t.req_scalar[0] = 1
    return t


def _budget_nodes(n, classes=False, scalar=False, seed=97):
    """Big, nearly empty nodes: total scores near 4000, above 2048 (bit 11 of the 12-bit score field)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    kw = {}
    if classes:
        cls = rng.integers(0, 3, n)
        kw.update(taint_mask=((np.uint64(1) << cls.astype(np.uint64)) - np.uint64(1)).reshape(1, n), taint_prefer=[0b11])
    if scalar:
        kw["scalars"] = [(np.full(n, 100), np.zeros(n))]
    return abi.Snapshot(n, rng.choice([64000, 128000], n), np.full(n, 512 * GiB), np.full(n, 110),
                        req_cpu=rng.integers(0, 40, n) * 100, **kw)


@pytest.mark.parametrize("kernels", ["lean<false>", "batched", "stream<2>", "wave<true>"])
def test_score_field_at_budget(built, kernels):
    """Weights summing to 40 on every kernel that packs the score: the lean kernel with TaintToleration classes (the class pick
    adds w_taint * norm after the gather), the tie-run kernel, the streaming kernel (three templates) and the generic kernel."""
    n = 20_000
    if kernels == "lean<false>":
        snap, tmpl, want_k = _budget_nodes(n, classes=True), [_budget_template(w_taint=3, w_balanced=17)], "lean<false>"
    elif kernels == "batched":
        snap, tmpl, want_k = _budget_nodes(n), [_budget_template()], {AUTO: "batched", SEQ: "lean<false>"}
    elif kernels == "stream<2>":
        snap, tmpl, want_k = _budget_nodes(n), [_budget_template(w_fit=20 - k, w_balanced=19 + k) for k in range(3)], "stream<2>"
    else:
        snap, tmpl, want_k = _budget_nodes(n, scalar=True), [_budget_template(scalar=True)], "wave<true>"
    for t in tmpl:
        assert t.w_taint + t.w_fit + t.w_balanced == 40
    want, _ = run_all(snap, tmpl, [], 1500, want_k)
    assert oracle.node_score(snap, tmpl[0], int(want.pod_node[0]), 0)[0] >= 2048


def test_score_weights_over_budget_refused(built):
    snap = _budget_nodes(100)
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        with pytest.raises(engine.EngineError, match="too large for the packed key"):
            eng.set_templates([_budget_template(w_balanced=20)], [])


# ---- kernel names without a launch -----------------------------------------------------------------------------------------------
def test_kernel_name_from_prepare(built):
    """ccsim_kernel_name: "" before any prepare and for an empty cluster; the multi-commit instantiations from prepare() alone
    (the sharded one with two ranks of this process on one device: no kernel is launched)."""
    with engine.Engine(device=0) as eng:
        assert helpers.kernel_name(eng) == ""
        eng.load_nodes(abi.Snapshot(0, np.zeros(0), np.zeros(0), np.zeros(0)))
        eng.set_templates([abi.default_template(150, 100 * MiB)], [])
        eng.prepare(0)
        assert helpers.kernel_name(eng) == ""
    snap, tmpl, ctr = synth.c4(n=3000, n_existing=6000, zones=8, racks=32, regions=4)
    name = helpers.prepared_kernel(snap, tmpl, ctr)
    print("\n  AUTO %-12s (prepare only)" % name, end="")
    assert name == "multi<false>"
    engs = [engine.Engine(device=0, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            e.load_nodes(snap)
            e.set_templates(tmpl, ctr)
        engine.Engine.connect_local(engs)
        for e in engs:
            e.prepare(0)
            print("\n  AUTO %-12s (rank %d of 2, prepare only)" % (helpers.kernel_name(e), engs.index(e)), end="")
            assert helpers.kernel_name(e) == "multi<true>"
    finally:
        for e in engs:
            e.close()
