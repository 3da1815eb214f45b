"""GPU: the multi-commit kernel's key-order replay (ccsim_multi.cuh). Single-use templates (required hostname anti-affinity: a node
takes one clone) rank their wave's candidates once and take each winner with a ballot; CCSIM_DEBUG_FLAGS bit 6 (64) keeps the
arg-max round. Every case runs the CPU oracle and the kernel with and without bit 6: both must match the oracle pod by pod, match
each other byte for byte, and run the same waves. The key-order counter (Engine.key_order_waves) shows which round ran."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
GiB, MiB = 1 << 30, 1 << 20
ARGMAX = 64          # CCSIM_DEBUG_FLAGS bit 6: the arg-max round on single-use waves
LOOK_AHEAD = 32      # CCSIM_DEBUG_FLAGS bit 5: look-ahead on every spread term in every wave (wake-ups)


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def _gpu(snap, tmpl, ctr, cap, flags, monkeypatch):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        got = eng.run(cap)
        counts, _ = eng.node_counts(0)
        return got, counts, eng.run_stats(), eng.key_order_waves()


def _same(got, want, what, hist=True):
    assert got.placed == want.placed and got.stop_code == want.stop_code, (what, got.placed, want.placed, got.stop_code, want.stop_code)
    m = min(got.placed, want.placed)
    diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
    assert np.array_equal(got.pod_node, want.pod_node), (what, "first difference at pod", diff[:1])
    if hist:
        assert np.array_equal(got.reason_hist, want.reason_hist), what


def check(snap, tmpl, ctr, cap, monkeypatch, flags=0, single_use=True):
    """Oracle, key order (`flags`) and the arg-max round (`flags` | 64) on one workload; returns the oracle's result and the
    key-order run's statistics."""
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, threads=8, memo=True)
    ko, ko_counts, ko_st, ko_waves = _gpu(snap, tmpl, ctr, cap, flags, monkeypatch)
    am, am_counts, am_st, am_waves = _gpu(snap, tmpl, ctr, cap, flags | ARGMAX, monkeypatch)
    _same(ko, want, "key order")
    _same(am, want, "arg-max round")
    assert ko.pod_node.tobytes() == am.pod_node.tobytes() and ko.reason_hist.tobytes() == am.reason_hist.tobytes()
    assert np.array_equal(ko_counts, np.bincount(want.pod_node, minlength=snap.n)) and np.array_equal(ko_counts, am_counts)
    assert ko_st["engine"] == am_st["engine"] == "multi-commit", (ko_st, am_st)
    # the same waves, candidates and raised bars: the round changes how a wave is decided, not what it decides
    for key in ("waves", "placed", "candidates", "bar_raised_waves"):
        assert ko_st[key] == am_st[key], (key, ko_st[key], am_st[key])
    assert am_waves == 0
    if single_use:
        assert ko_waves > 0
    else:
        assert ko_waves == 0
    print("\n  waves %d placed %d candidates/wave %.1f bar raised %d key-order waves %d" % (
        ko_st["waves"], ko_st["placed"], ko_st["candidates"] / max(1, ko_st["waves"]), ko_st["bar_raised_waves"], ko_waves))
    return want, ko_st, ko_waves


def _random_single_use(seed):
    """Hostname anti-affinity plus 1-3 spread constraints: mixed maxSkew and domain counts, some nodes without the key."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(3000, 12000))
    terms = int(rng.integers(1, 4))
    t = abi.default_template(int(rng.choice([100, 200, 500])), int(rng.choice([64, 128, 256])) * MiB)
    topo, ctr = [], []
    for c in range(terms):
        d = int(rng.choice([3, 8, 17, 64, 200]))
        col = rng.integers(0, d, n).astype(np.int32)
        col[rng.random(n) < float(rng.choice([0.0, 0.02, 0.1]))] = -1
        topo.append(col)
        ctr.append(abi.make_counter(c, rng.integers(0, 4, d).astype(np.int32), inc=1))
        t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = c, int(rng.choice([1, 2, 3, 5, 1000])), 1, 0
    t.n_pts = terms
    ctr.append(abi.make_counter(-1, (rng.random(n) < 0.05).astype(np.int32), inc=1))      # pods of the same app already on 5% of the nodes
    t.n_anti, t.anti_counter[0] = 1, terms
    a_cpu = rng.choice([2000, 4000, 8000], n)
    req_cpu = (rng.random(n) * 0.5 * a_cpu).astype(np.int64) // 10 * 10
    snap = abi.Snapshot(n, a_cpu, np.full(n, 16 * GiB), np.full(n, 110), req_cpu=req_cpu, topo=topo)
    return snap, [t], ctr, int(rng.choice([0, 1500]))


@pytest.mark.parametrize("flags", [0, LOOK_AHEAD])
@pytest.mark.parametrize("seed", range(6))
def test_random_single_use_templates(built, monkeypatch, seed, flags):
    """With look-ahead forced, minimum moves wake dormant candidates up in rows above the replay's position, and the nodes that
    already won must stay out."""
    snap, tmpl, ctr, cap = _random_single_use(100 + seed)
    check(snap, tmpl, ctr, cap, monkeypatch, flags)


@pytest.mark.parametrize("max_skew", [1, 10 ** 6])
@pytest.mark.parametrize("cands", [5, 31, 32, 33])
def test_candidates_at_row_edges(built, monkeypatch, cands, max_skew):
    """Every 40th node feasible, one score for all, no tile with more than 16: the wave's candidates are exactly the feasible
    nodes. Fewer than a row, one full row, and a row and one."""
    snap, tmpl, ctr = helpers.sparse_eligibility_case(40 * cands, max_skew=max_skew)
    want, st, _ = check(snap, tmpl, ctr, 0, monkeypatch)
    assert want.placed == cands and st["candidates"] >= cands


@pytest.mark.parametrize("max_skew", [1, 10 ** 6])
def test_full_rows_with_the_bar_raised(built, sm_count, monkeypatch, max_skew):
    """A full grid with far more candidates than the replay's 256 slots: the bar is raised and all eight rows are filled."""
    snap, tmpl, ctr = helpers.sparse_eligibility_case(sm_count * helpers.GRID_NODES, max_skew=max_skew)
    _, st, _ = check(snap, tmpl, ctr, 300, monkeypatch)
    assert st["bar_raised_waves"] > 0


def _commit_cap_case(sm_count):
    """About 226 candidates per wave on a full grid, none of them ever killed: only the 64-commit cap or the limit ends a wave."""
    return helpers.sparse_eligibility_case(sm_count * helpers.GRID_NODES, max_skew=10 ** 6, every=300)


def test_commits_per_wave_cap(built, sm_count, monkeypatch):
    snap, tmpl, ctr = _commit_cap_case(sm_count)
    want, st, _ = check(snap, tmpl, ctr, 0, monkeypatch)
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed == (snap.n + 299) // 300
    assert st["waves"] * 64 >= st["placed"] > 32 * st["waves"]


@pytest.mark.parametrize("limit", [5, 31, 33, 63, 64, 65])
def test_limit_inside_a_row_and_at_the_cap(built, sm_count, monkeypatch, limit):
    snap, tmpl, ctr = _commit_cap_case(sm_count)
    want, st, _ = check(snap, tmpl, ctr, limit, monkeypatch)
    assert want.stop_code == abi.STOP_LIMIT_REACHED and want.placed == limit
    assert st["waves"] == -(-limit // 64)


def test_spread_only_keeps_the_arg_max_round(built, monkeypatch):
    """No hostname term: a winner may come back in its wave (second life), so no wave is replayed in key order."""
    snap, tmpl, ctr = synth.c4(n=7000, n_existing=9000, zones=8, racks=64, regions=4)
    tmpl[0].n_anti = 0
    check(snap, tmpl, ctr[:3], 900, monkeypatch, single_use=False)


SHARDED = {
    "c4": (lambda: synth.c4(n=6000, n_existing=12000, zones=8, racks=64, regions=4), 0),
    "sparse": (lambda: helpers.sparse_eligibility_case(40000, max_skew=10 ** 6), 500),
}


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("which", sorted(SHARDED))
def test_node_shards_on_one_gpu(built, sm_count, monkeypatch, which, world):
    """Node shards: every rank ranks the union of the ranks' summaries and replays it alike."""
    make, limit = SHARDED[which]
    snap, tmpl, ctr = make()
    grid = helpers.persistent_grid(snap.n, sm_count, world)
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=8, memo=True)
    seqs = []
    for flags in (0, ARGMAX):
        monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
        engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
        try:
            res = helpers.run_sharded_once(engs, limit)
            stats = [e.run_stats() for e in engs]
            ko = [e.key_order_waves() for e in engs]
        finally:
            for e in engs:
                e.close()
        for r in res:           # replicated parts: identical on every rank; the FitError histogram is per shard
            _same(r, want, ("flags", flags), hist=False)
        assert np.array_equal(sum(r.reason_hist for r in res), want.reason_hist)
        assert all(s["engine"] == "multi-commit" for s in stats), stats
        assert all(k > 0 for k in ko) if flags == 0 else all(k == 0 for k in ko), ko
        seqs.append(res[0].pod_node.tobytes())
    assert seqs[0] == seqs[1]


def test_c4_full(built, monkeypatch):
    """The bench workload: 100k nodes, three spread constraints and hostname anti-affinity, to Unschedulable. Every wave is
    single-use, so every wave is replayed in key order."""
    snap, tmpl, ctr = synth.c4()
    want, st, ko = check(snap, tmpl, ctr, 0, monkeypatch)
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed > 30000
    assert ko == st["waves"]
