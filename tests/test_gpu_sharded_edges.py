"""GPU (ONE device is enough): the node-sharded engines at their edges, with every rank a handle of this process on device 0
(helpers.sharded_engines: the in-kernel exchange of a multi-GPU run, wired by pointer). The generic wave kernel over shards
with each of the extras that send a workload to it, ties and PreferNoSchedule classes across a shard boundary, shards of one
node, one node per rank and a refused split, eight ranks, the streaming kernel's three modes over uneven shards, multi-commit
waves at their edges, and one set of handles run past the 8-bit run epoch and past the 12-bit wave tag.

Every case runs the CPU oracle, then the ranks under ENGINE_AUTO and ENGINE_SEQUENTIAL, and compares on every rank the pod -> node
sequence, the stop code, the per-node counts and the kernel instantiation; over the ranks the sums of the FitError histogram,
the preemption counters and (sequential engine) the nodes evaluated. A case whose ranks do not all fit on this device's SMs at
once is skipped. The generic kernel with its tile streamed from global memory (wave<false>) needs a full grid per rank, so it is
only reachable with one device per rank: tests/test_gpu_sharded.py covers it on a 2-GPU box."""
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


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def shard_bases(n, world):
    """First global node index of each rank's shard (contiguous blocks of ceil(n / world) nodes, as ccsim_load_nodes cuts them)."""
    per = -(-n // world)
    return [min(per * r, n) for r in range(world)]


def skip_unless_fits(n, world, sm_count):
    grid = helpers.persistent_grid(n, sm_count, world)      # the ranks' persistent grids run side by side on this one device
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))


def check_sharded(sm_count, snap, tmpl, ctr, limit, world, kernel, want=None):
    """Oracle, then `world` ranks under ENGINE_AUTO and ENGINE_SEQUENTIAL. `kernel`: the instantiation every rank must run, or
    a dict {engine: instantiation}. Returns the oracle's result and each engine's per-rank statistics."""
    skip_unless_fits(snap.n, world, sm_count)
    kernels = kernel if isinstance(kernel, dict) else {AUTO: kernel, SEQ: kernel}
    if want is None:
        want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=8, memo=True)
    per_node = np.bincount(want.pod_node[0::len(tmpl)], minlength=snap.n)
    stats = {}
    for kind in (AUTO, SEQ):
        name = "AUTO" if kind == AUTO else "SEQ"
        engs = helpers.sharded_engines(snap, tmpl, ctr, world, kind)
        try:
            res = helpers.run_sharded_once(engs, limit)
            st = stats[kind] = [e.run_stats() for e in engs]
            counts = [e.node_counts(0)[0] for e in engs]
        finally:
            for e in engs:
                e.close()
        print("\n  %-4s world %d  %s  grid %d  waves %d  placed %d" % (name, world, ",".join(s["kernel"] for s in st), st[0]["grid"],
                                                                      res[0].waves, res[0].placed), end="")
        assert all(s["kernel"] == kernels[kind] for s in st), (name, st)
        for r, got in enumerate(res):
            assert (got.placed, got.stop_code) == (want.placed, want.stop_code), (name, "rank", r, got.placed, want.placed, got.stop_code)
            m = min(got.placed, want.placed)
            diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
            assert np.array_equal(got.pod_node, want.pod_node), (name, "rank", r, "first difference at pod", diff[:1])
            assert np.array_equal(counts[r], per_node), (name, "rank", r, "node counts")
        assert np.array_equal(sum(g.reason_hist for g in res), want.reason_hist), name
        assert sum(g.preempt_no_victims for g in res) == want.preempt_no_victims, name
        assert sum(g.preempt_not_helpful for g in res) == want.preempt_not_helpful, name
        if kind == SEQ:
            assert sum(g.evals for g in res) == want.evals, name
    return want, stats


def _nodes(n, seed, slots=(1, 6), **kw):
    """C2's cpu / memory distribution with 1..5 free pod slots per node (unlimited runs stay short); kw adds columns."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a_cpu, a_mem, a_pods, r_cpu, r_mem, npods = synth._c2_nodes(n, rng)
    npods = np.minimum(npods, a_pods - slots[1])
    a_pods = npods + rng.integers(slots[0], slots[1], n).astype(np.int32)
    return abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, **kw), rng


def _image(t, col):
    col = np.ascontiguousarray(col, np.uint8)
    t._keep_img = col
    t.image_score = col.ctypes.data_as(abi.C.POINTER(abi.C.c_uint8))
    return t


# ---- 1. the generic kernel over shards ------------------------------------------------------------------------------------------
N_GENERIC = 4001


def _generic_ext(world, n=N_GENERIC, seed=101):
    """(a) An extended resource and ephemeral storage: the first half of the nodes runs out of ephemeral storage, the second half
    out of the extended resource."""
    rng = np.random.Generator(np.random.PCG64(seed))
    front = np.arange(n) < n // 2
    eph = np.where(front, rng.integers(5, 21, n), rng.integers(100, 201, n)) * GiB
    sc_alloc = np.where(front, rng.integers(20, 41, n), rng.integers(0, 7, n))
    snap = abi.Snapshot(n, rng.choice([16000, 32000, 64000], n), np.full(n, 256 * GiB), np.full(n, 110), alloc_eph=eph,
                        req_cpu=rng.integers(0, 80, n) * 100, scalars=[(sc_alloc, rng.integers(0, 3, n))])
    t = abi.default_template(500, 1 * GiB, eph=7 * GiB)
    t.req_scalar[0] = 2
    return snap, [t], [], 0


def _generic_ports(world, n=N_GENERIC, seed=102):
    """(b) hostPorts: one clone per node (placed_mask, one word per node of each shard), 30 % of the nodes' ports taken."""
    static = (np.random.default_rng(seed).random(n) < 0.3).astype(np.uint64)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 110), static_mask=static.reshape(1, n),
                        has_placed_mask=True)
    t = abi.default_template(100, 100 * MiB)
    t.flags |= abi.TF_HAS_HOST_PORTS
    t.port_static_mask[0] = 1
    t.port_tmpl_conflict = 1
    return snap, [t], [], 0


def generic_ext_ports(n, seed=109):
    """(a) and (b) in one workload: extended resource, ephemeral storage and hostPorts (tests/test_gpu_sharded.py, real peers)."""
    snap, tmpl, _, _ = _generic_ext(2, n=n, seed=seed)
    snap.static_mask = (np.random.default_rng(seed).random(n) < 0.3).astype(np.uint64).reshape(1, n)
    snap.static_words, snap.has_placed_mask = 1, True
    tmpl[0].flags |= abi.TF_HAS_HOST_PORTS
    tmpl[0].port_static_mask[0] = 1
    tmpl[0].port_tmpl_conflict = 1
    return snap, tmpl, []


def generic_streamed(n, seed=110):
    """An extended-resource request on C2's nodes: the generic kernel, with its tile resident or streamed depending on n."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a_cpu, a_mem, a_pods, r_cpu, r_mem, npods = synth._c2_nodes(n, rng)
    snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods,
                        scalars=[(rng.integers(0, 6, n), rng.integers(0, 2, n))])
    t = abi.default_template(150, 100 * MiB)
    t.req_scalar[0] = 2
    return snap, [t], []


def _generic_nodename(world, n=N_GENERIC, seed=103):
    """(c) nodeName names the second node of the last shard: every other rank has no feasible node in any wave."""
    snap, _ = _nodes(n, seed, slots=(20, 40))
    t = abi.default_template(150, 100 * MiB)
    t.nodename_idx = shard_bases(n, world)[-1] + 1
    return snap, [t], [], 0


def _generic_prefilter(world, n=N_GENERIC, seed=104):
    """(d) PreFilter node names (static bit 0) on 5 % of the nodes, spread over every shard."""
    rng = np.random.Generator(np.random.PCG64(seed))
    snap, _ = _nodes(n, seed, static_mask=(rng.random(n) < 0.05).astype(np.uint64).reshape(1, n))
    t = abi.default_template(150, 100 * MiB)
    t.flags |= abi.TF_PREFILTER_NODES
    t.prefilter_bit = 0
    return snap, [t], [], 0


def _generic_affinity_terms(world, n=N_GENERIC, seed=105):
    """(e) Two nodeAffinity terms over two static words, next to a node selector in word 0."""
    rng = np.random.Generator(np.random.PCG64(seed))
    w0 = rng.integers(0, 16, n).astype(np.uint64)
    w1 = rng.integers(0, 16, n).astype(np.uint64)
    snap, _ = _nodes(n, seed + 1, static_mask=np.stack([w0, w1]))
    t = abi.default_template(150, 100 * MiB)
    t.flags |= abi.TF_HAS_NODE_SELECTOR | abi.TF_HAS_AFFINITY_TERMS
    t.sel_mask[0] = 0b1000
    t.n_aff_terms = 2
    t.aff_term_mask[0][0], t.aff_term_mask[0][1] = 0b0011, 0b0001
    t.aff_term_mask[1][1] = 0b0110
    return snap, [t], [], 0


TAINT_W1 = 64 + 2          # an untolerated NoSchedule taint in taint word 1


def _generic_taint_words(world, n=N_GENERIC, seed=106):
    """(f) Two taint words: untolerated NoSchedule taints 1 (word 0, every node) and 66 (word 1, second half of the nodes: ranks
    >= 1 at every world size tested), next to the tolerated taint 0. A node carrying both lists 66 first when it is in the second
    half, so the diagnosis's first untolerated taint in Spec.Taints order differs from the lowest bit there."""
    rng = np.random.Generator(np.random.PCG64(seed))
    back = np.arange(n) >= n // 2
    t0 = rng.random(n) < 0.2
    t1 = rng.random(n) < 0.25
    t66 = back & (rng.random(n) < 0.4)
    w0 = t0.astype(np.uint64) | (t1.astype(np.uint64) << np.uint64(1))
    w1 = t66.astype(np.uint64) << np.uint64(TAINT_W1 - 64)
    lists = []
    for i in range(n):
        ids = ([0] if t0[i] else []) + ([TAINT_W1] if t66[i] else []) + ([1] if t1[i] else [])
        lists.append(ids)
    snap, _ = _nodes(n, seed + 1, taint_mask=np.stack([w0, w1]), taint_nosched=[0b11, 1 << (TAINT_W1 - 64)], taint_lists=lists)
    t = abi.default_template(150, 100 * MiB)
    t.tol_nosched[0] = 0b01
    return snap, [t], [], 0


def _generic_image(world, n=N_GENERIC, seed=107):
    """(g) ImageLocality columns of two templates (pods alternate): every shard reads its own slice of each column."""
    rng = np.random.Generator(np.random.PCG64(seed))
    snap, _ = _nodes(n, seed + 1)
    tmpl = [_image(abi.default_template(150 + 350 * k, (100 + 200 * k) * MiB),
                   np.where(rng.random(n) < 0.4, rng.integers(1, 101, n), 0)) for k in range(2)]
    return snap, tmpl, [], 0


ZONE_NODES = 300


def _generic_colocation(world, n=N_GENERIC, seed=108, last_shard_pods=False):
    """(h) Required zone pod affinity with the self-match-all bypass: zones are blocks of 300 nodes, and the best node of the
    cluster is the last node of rank 0, whose zone continues on rank 1, so the first placement opens a zone that straddles the
    boundary and every later pod must follow it there. With `last_shard_pods` the affinity is already satisfied by pods of one
    zone that lies in the last shard only (aff_total_init > 0). Ephemeral storage sends the workload to the generic kernel;
    existing anti-affinity pods on a fifth of the nodes (a node-local counter) close those nodes."""
    rng = np.random.Generator(np.random.PCG64(seed))
    zone = (np.arange(n) // ZONE_NODES).astype(np.int32)
    zones = int(zone.max()) + 1
    snap, _ = _nodes(n, seed + 1, topo=[zone], alloc_eph=np.full(n, 100 * GiB))
    big = shard_bases(n, world)[1] - 1
    assert zone[big] == zone[big + 1]
    snap.alloc_cpu[big], snap.alloc_mem[big], snap.req_cpu[big], snap.req_mem[big] = 64000, 256 * GiB, 0, 0
    init = np.zeros(zones, np.int32)
    t = abi.default_template(150, 100 * MiB, eph=1 * GiB)
    t.flags |= abi.TF_AFF_SELF_MATCH_ALL
    if last_shard_pods:
        z = zone[n - 5]
        assert np.all(np.nonzero(zone == z)[0] >= shard_bases(n, world)[-1])
        init[z] = 2
        t.aff_total_init = 2
    t.n_aff, t.aff_counter[0] = 1, 0
    anti = (rng.random(n) < 0.2).astype(np.int32)
    anti[big] = 0
    t.n_anti, t.anti_counter[0] = 1, 1
    ctr = [abi.make_counter(0, init, inc=1), abi.make_counter(-1, anti)]
    return snap, [t], ctr, 0


GENERIC = {"ext": _generic_ext, "ports": _generic_ports, "nodename": _generic_nodename, "prefilter": _generic_prefilter,
           "affinity_terms": _generic_affinity_terms, "taint_words": _generic_taint_words, "image": _generic_image,
           "colocation": _generic_colocation, "colocation_last_shard": lambda w: _generic_colocation(w, last_shard_pods=True)}


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("which", sorted(GENERIC))
def test_generic_kernel_over_shards(built, sm_count, which, world):
    snap, tmpl, ctr, limit = GENERIC[which](world)
    assert helpers.prepared_kernel(snap, tmpl, ctr, max_pods=limit) == "wave<true>"     # on one GPU too: the case is about sharding
    want, _ = check_sharded(sm_count, snap, tmpl, ctr, limit, world, "wave<true>")
    h, bases = want.reason_hist, shard_bases(snap.n, world)
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed > 0
    if which == "ext":
        assert h[abi.R_SCALAR0] > 0 and h[abi.R_INSUFFICIENT_EPHEMERAL] > 0
    elif which == "ports":
        assert want.placed == int((snap.static_mask[0] == 0).sum()) and h[abi.R_NODE_PORTS] == snap.n
    elif which == "nodename":
        assert h[abi.R_NODE_NAME] == snap.n - 1 and set(want.pod_node.tolist()) == {tmpl[0].nodename_idx}
    elif which == "prefilter":
        assert h[abi.R_PREFILTER_NODES] == int((snap.static_mask[0] == 0).sum())
        assert all(np.any((want.pod_node >= lo) & (want.pod_node < lo + bases[1])) for lo in bases)
    elif which == "affinity_terms":
        assert h[abi.R_NODE_AFFINITY] > 0
    elif which == "taint_words":
        assert h[abi.R_TAINT0 + TAINT_W1] > 0 and h[abi.R_TAINT0 + 1] > 0
    elif which.startswith("colocation"):
        zone = snap.topo[0]
        zones = set(zone[want.pod_node].tolist())
        assert len(zones) == 1
        if which == "colocation":
            assert want.pod_node[0] == bases[1] - 1 and np.any(want.pod_node >= bases[1])
        else:
            assert np.all(want.pod_node >= bases[-1])


# ---- 2. ties and classes across a shard boundary --------------------------------------------------------------------------------
def _with_scalar(snap, tmpl):
    """The same workload plus an extended-resource request every node can always take: the generic kernel instead of the lean."""
    snap.scalars = [(np.full(snap.n, 10 ** 6, np.int64), np.zeros(snap.n, np.int64))]
    for t in tmpl:
        t.req_scalar[0] = 1
    return snap, tmpl


def _tied(world, n=2401):
    """Identical nodes with one free pod slot each: every wave ties all free nodes, and the lowest index wins."""
    return abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 1)), [abi.default_template(150, 100 * MiB)]


def _boundary_pairs(world, n=2401, seed=111):
    """At every shard boundary, the last node of one rank and the first node of the next are the best nodes of the cluster, all
    with the same score."""
    snap, _ = _nodes(n, seed)
    for b in shard_bases(n, world)[1:]:
        for i in (b - 1, b):
            snap.alloc_cpu[i], snap.alloc_mem[i], snap.req_cpu[i], snap.req_mem[i] = 64000, 256 * GiB, 0, 0
            snap.nz_cpu[i], snap.nz_mem[i], snap.npods[i], snap.alloc_pods[i] = 0, 0, 0, 3
    return snap, [abi.default_template(150, 100 * MiB)]


def _top_class_last_rank(world, n=2401, seed=112):
    """PreferNoSchedule taints 0..2: every node carries one or two of them, except the last four nodes (on the last rank at every
    world size), which carry all three. So the highest class exists on one rank only, until those nodes fill up mid-run."""
    rng = np.random.Generator(np.random.PCG64(seed))
    taint = np.where(rng.random(n) < 0.5, 0b001, 0b011).astype(np.uint64)
    taint[-4:] = 0b111
    snap, _ = _nodes(n, seed + 1, taint_mask=taint.reshape(1, n), taint_prefer=[0b111])
    snap.alloc_cpu[-4:], snap.req_cpu[-4:], snap.alloc_mem[-4:], snap.req_mem[-4:] = 64000, 0, 256 * GiB, 0
    return snap, [abi.default_template(150, 100 * MiB)]


TIES = {"tied": _tied, "boundary_pairs": _boundary_pairs, "top_class_last_rank": _top_class_last_rank}


@pytest.mark.parametrize("kernel", ["lean<false>", "wave<true>"])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("which", sorted(TIES))
def test_ties_and_classes_across_the_boundary(built, sm_count, which, world, kernel):
    snap, tmpl = TIES[which](world)
    if kernel == "wave<true>":
        snap, tmpl = _with_scalar(snap, tmpl)
    bases = shard_bases(snap.n, world)
    limit = bases[1] + 3 if which == "tied" else 0
    want, _ = check_sharded(sm_count, snap, tmpl, [], limit, world, kernel)
    seq = want.pod_node
    if which == "tied":            # rank 0 fills node by node; the winner moves to rank 1's first node with the next pod
        assert np.array_equal(seq, np.arange(limit))
    elif which == "boundary_pairs":
        assert seq[0] == bases[1] - 1 and bases[1] in seq.tolist()
    else:
        assert np.all(np.bincount(seq, minlength=snap.n)[-4:] == snap.alloc_pods[-4:] - snap.npods[-4:])
        assert want.stop_code == abi.STOP_UNSCHEDULABLE


# ---- 3. shard shapes ------------------------------------------------------------------------------------------------------------
def _shape_n(world, shape):
    if shape == "last_shard_one_node":      # shards of `world` nodes, the last of one node
        return world * (world - 1) + 1
    if shape == "one_node_per_rank":
        return world
    return 1025 * world - (world - 1)       # short_last: three CTAs per rank, while the last shard alone would need two


@pytest.mark.parametrize("kernel", ["lean<false>", "wave<true>"])
@pytest.mark.parametrize("world", [3, 8])
@pytest.mark.parametrize("shape", ["last_shard_one_node", "one_node_per_rank", "short_last"])
def test_shard_shapes(built, sm_count, shape, world, kernel):
    n = _shape_n(world, shape)
    snap, _ = _nodes(n, 120 + n, slots=(3, 9))
    tmpl = [abi.default_template(150, 100 * MiB)]
    if kernel == "wave<true>":
        snap, tmpl = _with_scalar(snap, tmpl)
    sizes = np.diff(shard_bases(n, world) + [n])
    assert sizes.min() >= 1 and (shape != "last_shard_one_node" or sizes[-1] == 1) and (shape != "one_node_per_rank" or sizes.max() == 1)
    want, st = check_sharded(sm_count, snap, tmpl, [], 0, world, kernel)
    assert want.stop_code == abi.STOP_UNSCHEDULABLE
    assert {int(x) for x in want.pod_node} == set(np.nonzero(snap.alloc_pods > snap.npods)[0].tolist())
    if shape == "short_last":
        assert st[AUTO][0]["grid"] == 3 and -(-int(sizes[-1]) // helpers.GRID_NODES) == 2


@pytest.mark.parametrize("world", [3, 8])
def test_split_without_nodes_for_a_rank_refused(built, world):
    """ceil(N / world) x (world - 1) >= N leaves the last rank without nodes: refused at load_nodes, before anything launches."""
    n = 2 * (world - 1)
    snap, _ = _nodes(n, 130)
    for r in range(world):
        with engine.Engine(device=0, rank=r, world=world) as eng:
            with pytest.raises(engine.EngineError, match="leaves a rank without nodes"):
                eng.load_nodes(snap)


@pytest.mark.parametrize("which", ["multi", "lean"])
def test_eight_ranks(built, sm_count, which):
    """CCSIM_MAX_WORLD ranks: the winner exchange reads all eight lanes, and the multi-commit summary has eight source ranks."""
    if which == "multi":
        snap, tmpl, ctr = synth.c4(n=6000, n_existing=12000, zones=8, racks=64, regions=4)
        kernel = {AUTO: "multi<true>", SEQ: "lean<false>"}
    else:
        snap, tmpl, ctr = synth.c3(n=5001, prefer_taints=True)
        kernel = "lean<false>"
    want, st = check_sharded(sm_count, snap, tmpl, ctr, 0, 8, kernel)
    if which == "multi":
        assert want.placed > 100 and all(s["waves"] * 2 < want.waves for s in st[AUTO])


# ---- 4. the streaming kernel over shards ----------------------------------------------------------------------------------------
N_STREAM = 40_961           # an uneven last shard at world 2 and 4; every rank's chunk ends inside a padded ring tile


def _stream_masks(world, n=N_STREAM, seed=141):
    """stream<1>: untolerated NoSchedule taints and node selectors in some of the templates."""
    rng = np.random.Generator(np.random.PCG64(seed))
    taint = (rng.random(n) < 0.1).astype(np.uint64) | ((rng.random(n) < 0.05).astype(np.uint64) << np.uint64(1))
    static = (rng.random(n) < 0.5).astype(np.uint64) | ((rng.random(n) < 0.3).astype(np.uint64) << np.uint64(1))
    a_cpu, a_mem, a_pods, r_cpu, r_mem, npods = synth._c2_nodes(n, rng)
    snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, taint_mask=taint.reshape(1, n),
                        taint_nosched=[0b11], static_mask=static.reshape(1, n))
    tmpl = []
    for k in range(4):
        t = abi.default_template(100 + 150 * k, (64 + 100 * k) * MiB)
        t.tol_nosched[0] = 0b10 if k % 2 else 0
        if k >= 2:
            t.flags |= abi.TF_HAS_NODE_SELECTOR
            t.sel_mask[0] = 1 << (k - 2)
        tmpl.append(t)
    return snap, tmpl


def _stream_dominant(world, n=N_STREAM, seed=142):
    """One dominant node per rank, in the first ring tile of its rank's first CTA, all tied: the winner sits again and again in
    the tile every CTA pre-requests for the next wave, and moves to the next rank's dominant node when one fills up."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a_cpu, a_mem, a_pods, _, _, _ = synth._c2_nodes(n, rng)
    r_cpu, r_mem = a_cpu * 17 // 20, a_mem * 17 // 20
    for b in shard_bases(n, world):
        d = b + 5
        a_cpu[d], a_mem[d], a_pods[d], r_cpu[d], r_mem[d] = 10 ** 7, 1 << 46, 1500 // (world + 1), 0, 0
    snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem)
    return snap, synth.c5(n=1, n_templates=5, seed=142)[1]


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("mode", ["stream<0>", "stream<1>", "stream<2>", "stream<0>:dominant", "stream<2>:dominant"])
def test_streaming_over_shards(built, sm_count, monkeypatch, mode, world):
    kernel = mode.split(":")[0]
    if kernel == "stream<0>":
        monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    if mode.endswith("dominant"):
        snap, tmpl = _stream_dominant(world)
    elif kernel == "stream<1>":
        snap, tmpl = _stream_masks(world)
    else:
        snap, tmpl = synth.c5(n=N_STREAM, n_templates=4, seed=143)[:2]
    bases = shard_bases(snap.n, world)
    assert snap.n - bases[-1] < bases[1]
    want, _ = check_sharded(sm_count, snap, tmpl, [], 1500, world, kernel)
    if mode.endswith("dominant"):
        dom = np.array(bases) + 5
        won = np.isin(want.pod_node, dom)
        assert won.sum() >= 750 and len(set(want.pod_node[won].tolist())) > 1


# ---- 5. multi-commit waves over shards ----------------------------------------------------------------------------------------
N_SPARSE = 61_440


def _spread_last_shard(world, n=6000, seed=151):
    """Zone spread (maxSkew 1) where zone 7 exists only among the last 400 nodes (last shard) and starts empty, next to hostname
    anti-affinity against existing pods."""
    rng = np.random.Generator(np.random.PCG64(seed))
    zone = rng.integers(0, 7, n).astype(np.int32)
    zone[-400:] = 7
    snap, _ = _nodes(n, seed + 1, topo=[zone])
    ctr = [abi.make_counter(0, np.append(rng.integers(3, 6, 7), 0).astype(np.int32), inc=1),
           abi.make_counter(-1, (rng.random(n) < 0.2).astype(np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return snap, [t], ctr


MULTI = {AUTO: "multi<true>", SEQ: "lean<false>"}


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("limit", [0, 63, 64, 65, 129])
def test_multi_commit_cap_and_limit_over_shards(built, sm_count, world, limit):
    """Every 300th node feasible, single-use nodes and a spread constraint that never binds: only the cap of 64 commits ends a
    wave. --max-limit just before, at and after a wave's end."""
    snap, tmpl, ctr = helpers.sparse_eligibility_case(N_SPARSE, max_skew=10 ** 6, every=300)
    want, st = check_sharded(sm_count, snap, tmpl, ctr, limit, world, MULTI)
    for s in st[AUTO]:
        if limit:
            assert want.stop_code == abi.STOP_LIMIT_REACHED and s["waves"] == -(-limit // 64), s
        else:
            assert want.placed == -(-N_SPARSE // 300) and s["waves"] * 64 >= s["placed"] > 32 * s["waves"], s


@pytest.mark.parametrize("world", [2, 3])
def test_multi_commit_spread_domain_on_the_last_shard(built, sm_count, world):
    snap, tmpl, ctr = _spread_last_shard(world)
    assert np.all(np.nonzero(snap.topo[0] == 7)[0] >= shard_bases(snap.n, world)[-1])
    want, st = check_sharded(sm_count, snap, tmpl, ctr, 0, world, MULTI)
    assert snap.topo[0][want.pod_node[0]] == 7 and want.stop_code == abi.STOP_UNSCHEDULABLE
    assert all(s["placed"] > s["waves"] for s in st[AUTO])


# ---- 6. the run epoch and the wave tag wrapping ---------------------------------------------------------------------------------
def _check_ranks(res, want, what):
    for r, got in enumerate(res):
        assert (got.placed, got.stop_code) == (want.placed, want.stop_code), (what, r)
        assert np.array_equal(got.pod_node, want.pod_node), (what, r)
    assert np.array_equal(sum(g.reason_hist for g in res), want.reason_hist), what


def test_run_epoch_wraps(built, sm_count):
    """One set of handles runs 300 times, more than one cycle of the 8-bit run epoch: stale exchange words of a run 255 runs back
    carry the same epoch. The runs alternate between odd and even wave counts, so the buffer parity (xwave0) changes too; every
    fifth run's template fits nowhere (Unschedulable at pod 0: one wave)."""
    world, n = 2, 3001
    skip_unless_fits(n, world, sm_count)
    snap, _ = _nodes(n, 161, slots=(20, 40))
    fits, never = abi.default_template(150, 100 * MiB), abi.default_template(10 ** 6, 100 * MiB)
    plan = [(fits, 1), (fits, 2), (fits, 5), (never, 0), (fits, 64)]
    wants = [oracle.run(snap, [t], [], max_pods=lim, threads=8, memo=True) for t, lim in plan]
    assert wants[3].placed == 0 and [w.waves for w in wants] == [1, 2, 5, 1, 64]
    engs = helpers.sharded_engines(snap, [fits], [], world, AUTO)
    runs = 0
    try:
        for it in range(300):
            t, lim = plan[it % len(plan)]
            if it % len(plan) in (0, 3, 4):        # the template changes before runs 0, 3 and 4 of each cycle
                for e in engs:
                    e.set_templates([t], [])
            res = helpers.run_sharded_once(engs, lim)
            runs += 1
            assert all(e.run_stats()["kernel"] == "lean<false>" for e in engs)
            _check_ranks(res, wants[it % len(plan)], it)
    finally:
        for e in engs:
            e.close()
    print("\n  %d runs on one set of handles" % runs, end="")
    assert runs > 255


def test_wave_tag_wraps(built, sm_count):
    """Sequential engine, 5003 placements per run: more than 4095 waves, so the 12-bit wave tag wraps inside the run. Twice on
    the same handles: the second run starts on the other buffer parity."""
    world = 2
    snap, tmpl, ctr = synth.c2(n=20_000, seed=171)
    skip_unless_fits(snap.n, world, sm_count)
    want = oracle.run(snap, tmpl, ctr, max_pods=5003, threads=8, memo=True)
    engs = helpers.sharded_engines(snap, tmpl, ctr, world, SEQ)
    try:
        for it in range(2):
            res = helpers.run_sharded_once(engs, 5003)
            print("\n  run %d: %s, waves %s" % (it, [e.run_stats()["kernel"] for e in engs], [g.waves for g in res]), end="")
            assert all(e.run_stats()["kernel"] == "lean<false>" for e in engs)
            assert all(g.waves > 4095 for g in res)
            _check_ranks(res, want, it)
            assert sum(g.evals for g in res) == want.evals
    finally:
        for e in engs:
            e.close()
