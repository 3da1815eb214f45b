"""GPU: the multi-commit kernel's node records on the sorted tile (ccsim_multi.cuh). In a single-use launch (required hostname
anti-affinity: a node takes one clone) every node's key, payload and node-local Filter verdict are kept in a record at the node's
rank, rebuilt at every constants build; each wave tests only the replicated counter cells of the records, and a winner's record
dies before the next wave. Every case runs with the default selection and with CCSIM_DEBUG_FLAGS bit 7 (128: REDUX rounds and the
merge, which re-run the whole Filter pass on every row each wave). Both must match the CPU oracle pod by pod, run the same waves
with the same candidates and raised bars, and the default run must select from the sorted tile in every wave."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
REDUX, RECOUNT = 128, 2      # CCSIM_DEBUG_FLAGS bits 7 and 1
H100_SXM_SMS = 132


def _single_use(snap, t, ctr, hostname_init):
    """Adds required anti-affinity on the hostname (a node-local counter) to template t: every node takes one clone at most."""
    ctr.append(abi.make_counter(-1, np.asarray(hostname_init, np.int32), inc=1))
    t.anti_counter[t.n_anti] = len(ctr) - 1
    t.n_anti += 1
    return snap, [t], ctr


def node_local_failures():
    """Nodes that fail a node-local part of the Filter pass from the start — a NoSchedule taint, a missing selector bit, no free
    pod slot (free CPU, so a high score), too little CPU, no zone label under a DoNotSchedule zone spread — and nodes that already
    run a matching pod (hostname anti-affinity), mixed with feasible nodes at random scores: in rank order they sit between
    feasible nodes of higher and lower keys, in every tile."""
    rng = np.random.default_rng(11)
    n, zones = 6000, 8
    i = np.arange(n)
    kind = rng.integers(0, 8, n)                       # 0-1: feasible; 2..7: one reason each
    a_cpu = np.full(n, 8000)
    req_cpu = 10 * rng.integers(0, 600, n)
    req_cpu = np.where(kind == 5, 7950, req_cpu)       # 50m free: the 150m clone does not fit
    npods = rng.integers(0, 10, n).astype(np.int32)
    a_pods = np.where(kind == 4, npods, 110)           # no pod slot left
    taint = (kind == 2).astype(np.uint64)
    static = (kind != 3).astype(np.uint64)
    zone = (i % zones).astype(np.int32)
    zone[kind == 6] = -1
    snap = abi.Snapshot(n, a_cpu, np.full(n, 16 * GiB), a_pods, req_cpu=req_cpu, npods=npods, taint_mask=taint.reshape(1, n),
                        taint_nosched=[1], taint_prefer=[0], static_mask=static.reshape(1, n), topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(zones, np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 2, 1, 0
    return _single_use(snap, t, ctr, (kind == 7).astype(np.int32))


def won_top_ranks():
    """Tile 0 holds the 64 best-scored nodes of the cluster, which win in the first waves: from then on the top of its rank order
    is all dead records, and its list must come from the ranks below them."""
    rng = np.random.default_rng(23)
    n, zones = 4000, 8
    req_cpu = 10 * rng.integers(100, 700, n)
    req_cpu[:64] = 10 * rng.permutation(64)           # the best scores, in a random order
    snap = abi.Snapshot(n, np.full(n, 8000), np.full(n, 16 * GiB), np.full(n, 110), req_cpu=req_cpu,
                        topo=[rng.integers(0, zones, n).astype(np.int32)])
    ctr = [abi.make_counter(0, np.zeros(zones, np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 3, 1, 0
    return _single_use(snap, t, ctr, np.zeros(n, np.int32))


def random_single_use(seed, sm_count):
    """A single-use template in the style of test_gpu_stress.random_case: random spread constraints, domain counts, skews,
    missing labels, minDomains, sometimes anti-affinity on a topology key too, with node-local failures (taints, selector bits,
    full nodes, matching pods already on the node). Sizes up to every tile full."""
    rng = np.random.default_rng(7000 + seed)
    n = int(rng.choice([300, 3000, 20000, 60000, sm_count * helpers.MULTI_TILE]))
    n_topo = int(rng.integers(1, 4))
    doms = [int(rng.choice([3, 8, 40, 255, 256, 2047] if n_topo < 3 else [3, 8, 40, 255])) for _ in range(n_topo)]
    topo = []
    for d in doms:
        col = rng.integers(0, d, n).astype(np.int32)
        if rng.random() < 0.4:
            col[rng.random(n) < 0.03] = -1
        topo.append(col)
    a_cpu = rng.choice([2000, 4000, 8000, 16000], n)
    npods = rng.integers(0, 20, n).astype(np.int32)
    req_cpu = (rng.random(n) * 0.5 * a_cpu).astype(np.int64) // 10 * 10
    a_pods = np.where(rng.random(n) < 0.05, npods, rng.choice([30, 60, 110], n))
    taint = (rng.random(n) < 0.05).astype(np.uint64)
    static = (rng.random(n) < 0.9).astype(np.uint64)
    snap = abi.Snapshot(n, a_cpu, a_cpu * (2 * MiB), a_pods, req_cpu=req_cpu, req_mem=req_cpu * MiB, npods=npods,
                        taint_mask=taint.reshape(1, n), taint_nosched=[1], taint_prefer=[0], static_mask=static.reshape(1, n), topo=topo)
    t = abi.default_template(int(rng.choice([100, 250, 700])), int(rng.choice([64, 256, 1024])) * MiB)
    if rng.random() < 0.5:
        t.flags |= abi.TF_HAS_NODE_SELECTOR
        t.sel_mask[0] = 1
    if rng.random() < 0.3:
        t.w_fit, t.w_balanced = int(rng.integers(1, 5)), int(rng.integers(1, 5))
    ctr = []
    for c, d in enumerate(doms):
        init = rng.integers(0, 4, d).astype(np.int32) if rng.random() < 0.7 else np.full(d, int(rng.integers(0, 3)), np.int32)
        self_match = int(rng.random() < 0.85)
        n_present = d if rng.random() < 0.8 else max(1, d - int(rng.integers(1, 3)))
        ctr.append(abi.make_counter(c, init, n_present=n_present, inc=self_match))
        t.pts[c].counter, t.pts[c].max_skew = c, int(rng.choice([1, 1, 2, 5]))
        t.pts[c].self_match, t.pts[c].min_zero = self_match, int(rng.random() < 0.1)
    t.n_pts = len(doms)
    if doms[0] >= 40 and rng.random() < 0.3:         # anti-affinity on the first topology key (its own counter on the same column)
        ctr.append(abi.make_counter(0, (rng.random(doms[0]) < 0.2).astype(np.int32), inc=1))
        t.n_anti, t.anti_counter[0] = 1, len(ctr) - 1
    snap, tmpl, ctr = _single_use(snap, t, ctr, (rng.random(n) < 0.1).astype(np.int32))
    return snap, tmpl, ctr, int(rng.choice([0, 0, 37, 1500]))


CASES = {
    "node_local_failures": (node_local_failures, 0, 0),
    "c4_small_recount_every_wave": (lambda: synth.c4(n=30000, n_existing=60000, zones=32, racks=256, regions=8), 0, RECOUNT),
    "won_top_ranks": (won_top_ranks, 0, 0),
}
N_RANDOM = 24


def _run(snap, tmpl, ctr, limit, flags, monkeypatch):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        got = eng.run(limit)
        st = eng.run_stats()
        return got, st, eng.sorted_tile_waves()


def check(snap, tmpl, ctr, limit, flags, monkeypatch):
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=8, memo=True)
    runs = [_run(snap, tmpl, ctr, limit, f, monkeypatch) for f in (flags, flags | REDUX)]
    for got, st, _ in runs:
        assert st["engine"] == "multi-commit", st
        assert got.placed == want.placed and got.stop_code == want.stop_code, (got.placed, want.placed)
        assert np.array_equal(got.pod_node, want.pod_node)
        assert np.array_equal(got.reason_hist, want.reason_hist)
    (_, srt, srt_waves), (_, rdx, rdx_waves) = runs
    stats = lambda s: [s[k] for k in ("waves", "placed", "candidates", "bar_raised_waves")]
    assert stats(srt) == stats(rdx), (stats(srt), stats(rdx))
    assert srt_waves == srt["waves"] and rdx_waves == 0, (srt_waves, srt["waves"], rdx_waves)
    return want, srt


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_node_records(built, monkeypatch, case):
    make, limit, flags = CASES[case]
    want, st = check(*make(), limit, flags, monkeypatch)
    print("\n  %s: waves %d placed %d" % (case, st["waves"], want.placed))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(N_RANDOM))
def test_random_single_use_templates(built, monkeypatch, seed):
    sm_count = helpers.device_sm_count()
    snap, tmpl, ctr, limit = random_single_use(seed, sm_count)
    check(snap, tmpl, ctr, limit or 4000, 0, monkeypatch)       # (a cap keeps the oracle in seconds)


def test_random_single_use_cases_reach_the_multi_commit_kernel():
    """Every random case runs on the multi-commit kernel of an H100 SXM, so every one of them exercises the node records."""
    elig = [helpers.multi_eligible(*random_single_use(seed, H100_SXM_SMS)[:3], H100_SXM_SMS) for seed in range(N_RANDOM)]
    assert all(elig), [s for s, e in enumerate(elig) if not e]
