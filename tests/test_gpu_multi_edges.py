"""GPU: the multi-commit wave kernel (ccsim_multi.cuh) at the edges of its packed formats and its per-wave limits: full tiles, a
domain-id payload at its 27-bit budget, two terms on one payload field, the replicated-term limit, the top of the 12-bit score field,
all-tied keys, the candidate cap, second lives, the commits-per-wave cap and --max-limit at a wave edge.

Every case runs the CPU oracle, ENGINE_AUTO and ENGINE_SEQUENTIAL and compares the pod -> node sequence, the stop code, the FitError
histogram and the per-node counts. Each also asserts which kernel ran and the wave statistic that shows the targeted path was taken."""
import importlib

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
GiB, MiB = 1 << 30, 1 << 20


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def run_all(snap, tmpl, ctr, cap, engine_name):
    """Oracle, ENGINE_AUTO and ENGINE_SEQUENTIAL on one workload; returns the oracle's result and the AUTO run's statistics."""
    want = oracle.run(snap, tmpl, ctr, max_pods=cap, threads=8, memo=True)
    engine = importlib.import_module("cluster-capacity_b200.engine")
    stats = {}
    for kind in (abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL):
        with engine.Engine(device=0, engine=kind) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            got = eng.run(cap)
            counts, _ = eng.node_counts(0)
            stats[kind] = helpers.run_stats(eng)
        assert got.placed == want.placed and got.stop_code == want.stop_code, (kind, got.placed, want.placed, got.stop_code)
        m = min(got.placed, want.placed)
        diff = np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0]
        assert np.array_equal(got.pod_node, want.pod_node), (kind, "first difference at pod", diff[:1])
        assert np.array_equal(got.reason_hist, want.reason_hist), kind
        assert np.array_equal(counts, np.bincount(want.pod_node, minlength=snap.n)), kind
    st = stats[abi.ENGINE_AUTO]
    print("\n  %s: waves %d placed %d bar_raised_waves %d candidates %d" % (st["engine"], st["waves"], st["placed"], st["bar_raised_waves"], st["candidates"]))
    assert st["engine"] == engine_name, st
    assert st["placed"] == want.placed
    return want, st


@pytest.mark.parametrize("extra", [0, 1])
def test_full_tiles(built, sm_count, extra):
    """sm_count x 768 nodes: every tile, the last one included, holds exactly one node per thread. One node more does not fit."""
    n = sm_count * helpers.MULTI_TILE + extra
    snap, tmpl, ctr = synth.c4(n=n, n_existing=2 * n, zones=32, racks=512, regions=8)
    name = "lean sequential" if extra else "multi-commit"
    assert helpers.expected_engine(snap, tmpl, ctr, sm_count) == name
    _, st = run_all(snap, tmpl, ctr, 1500, name)
    assert st["grid"] == sm_count


def _payload_case(doms, seed=41):
    """Three spread constraints whose columns have `doms` domains. About a tenth of the nodes sit in the last domain of each column
    and score best (more room): they win, fill their cells, and the other candidates in those cells must die."""
    rng = np.random.default_rng(seed)
    n = 20000
    topo, hot = [], np.zeros(n, bool)
    for d in doms:
        col = rng.integers(0, d - 1, n).astype(np.int32)
        last = rng.random(n) < 0.1
        col[last] = d - 1
        hot |= last
        topo.append(col)
    a_cpu = np.where(hot, 32000, 4000)
    req_cpu = (rng.random(n) * 0.4 * 4000).astype(np.int64) // 10 * 10
    snap = abi.Snapshot(n, a_cpu, a_cpu * (2 * MiB), np.full(n, 110), req_cpu=req_cpu, req_mem=req_cpu * (2 * MiB), topo=topo)
    ctr = []
    t = abi.default_template(200, 400 * MiB)
    for c, d in enumerate(doms):
        init = rng.integers(0, 3, d).astype(np.int32)
        init[d - 1] = 0
        ctr.append(abi.make_counter(c, init, inc=1))
        t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = c, 2, 1, 0
    t.n_pts = len(doms)
    return snap, [t], ctr


@pytest.mark.parametrize("doms,bits,name", [((255, 255, 255), 27, "multi-commit"), ((255, 255, 256), 28, "lean sequential")])
def test_payload_at_the_budget(built, sm_count, doms, bits, name):
    """255 domains take 8 bits + a guard bit: three columns fill the 27-bit payload exactly, and domain 254's field is all ones.
    256 domains need one bit more, and the workload falls back to the lean kernel."""
    assert sum(d.bit_length() + 1 for d in doms) == bits
    snap, tmpl, ctr = _payload_case(doms)
    assert helpers.expected_engine(snap, tmpl, ctr, sm_count) == name
    want, _ = run_all(snap, tmpl, ctr, 1500, name)
    for c, d in enumerate(doms):       # the last domain's cell closed, and a node in it that outranked a later winner was passed over
        assert _closed_cell_skips(snap, tmpl[0], ctr, c, d - 1, want.pod_node) > 0, c


def _closed_cell_skips(snap, t, ctr, col, dom, seq):
    """Pods of `seq` won by a node that ranks below some never-placed node B of cell (col, dom), at a time when that cell was over its
    spread limit (maxSkew - 1 + the column's minimum; column c has constraint t.pts[c] on counter ctr[c]) and B's cells in the other
    columns were not. B still had room (it was never placed), so the oracle passed it over only because of that cell: the kernel
    must have killed B's candidate there."""
    limit = lambda c: t.pts[c].max_skew - t.pts[c].self_match + cnt[c].min()
    score = lambda i, clones: oracle.node_score(snap, t, int(i), int(clones))[0]
    members = np.nonzero(snap.topo[col] == dom)[0]
    members = members[~np.isin(members, seq)]
    mscore = np.array([score(i, 0) for i in members])
    cnt = [np.array(c._keep, np.int64) for c in ctr]
    skips = 0
    for k, w in enumerate(seq.tolist()):
        if cnt[col][dom] > limit(col):
            live = np.ones(len(members), bool)
            for c in range(len(ctr)):
                if c != col:
                    live &= cnt[c][snap.topo[c][members]] <= limit(c)
            ws = score(w, (seq[:k] == w).sum())
            skips += bool(np.any(live & ((mscore > ws) | ((mscore == ws) & (members < w)))))
        for c in range(len(ctr)):
            cnt[c][snap.topo[c][w]] += 1
    return skips


def test_two_terms_on_one_payload_field(built):
    """Zone anti-affinity and zone spread (maxSkew 1) on two counters of the same column share one payload field; a commit in a
    zone at the spread minimum fills both cells at once. Run until Unschedulable."""
    rng = np.random.default_rng(43)
    n, zones = 20000, 300
    zone = rng.integers(0, zones, n).astype(np.int32)
    zone[rng.random(n) < 0.03] = -1
    snap = abi.Snapshot(n, rng.choice([2000, 4000, 8000], n), np.full(n, 16 * GiB), np.full(n, 30), topo=[zone])
    ctr = [abi.make_counter(0, rng.integers(0, 2, zones).astype(np.int32), inc=1),
           abi.make_counter(0, (rng.random(zones) < 0.2).astype(np.int32), inc=1)]
    t = abi.default_template(200, 128 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    want, _ = run_all(snap, [t], ctr, 0, "multi-commit")
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed >= 10


@pytest.mark.parametrize("terms", [6, 7])
def test_replicated_term_limit(built, sm_count, terms):
    """Six spread constraints on replicated counters is the most the kernel takes (MULTI_GT); a seventh falls back. Three domains
    per column keep the payload at 3 bits per term, so only the term count decides."""
    rng = np.random.default_rng(47)
    n = 6000
    topo = [rng.integers(0, 3, n).astype(np.int32) for _ in range(terms)]
    snap = abi.Snapshot(n, rng.choice([4000, 8000], n), np.full(n, 16 * GiB), np.full(n, 110), topo=topo)
    t = abi.default_template(150, 100 * MiB)
    ctr = []
    for c in range(terms):
        ctr.append(abi.make_counter(c, rng.integers(0, 3, 3).astype(np.int32), inc=1))
        t.pts[c].counter, t.pts[c].max_skew, t.pts[c].self_match, t.pts[c].min_zero = c, 1 + c % 4, 1, 0
    t.n_pts = terms
    name = "multi-commit" if terms <= helpers.MULTI_GT else "lean sequential"
    assert helpers.expected_engine(snap, [t], ctr, sm_count) == name
    run_all(snap, [t], ctr, 1500, name)


def _score_top_case(w_fit):
    """Big, nearly empty nodes and score weights summing to 40 (w_fit + w_balanced + w_taint): scores near 4000. Spread only, with a
    maxSkew that never binds and no hostname term, so a winner comes back in its wave with its second-life key."""
    rng = np.random.default_rng(59)
    n = 8000
    zone = rng.integers(0, 16, n).astype(np.int32)
    snap = abi.Snapshot(n, rng.choice([64000, 128000], n), np.full(n, 512 * GiB), np.full(n, 110),
                        req_cpu=rng.integers(0, 40, n) * 100, topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(16, np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.w_taint, t.w_node_affinity, t.w_pts, t.w_ipa, t.w_image = 1, 0, 0, 0, 0
    t.w_fit, t.w_balanced = w_fit, 19
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1000, 1, 0
    return snap, [t], ctr


def test_score_field_top(built):
    """Scores above 2048 set the top bit of the 12-bit score field in the key and in the second-life key (`cnext`): a node that wins
    twice in a row wins the second time with its post-clone score. A weight sum of 41 could overflow the field and is refused."""
    snap, tmpl, ctr = _score_top_case(20)
    want, st = run_all(snap, tmpl, ctr, 1500, "multi-commit")
    seq = want.pod_node
    assert oracle.node_score(snap, tmpl[0], int(seq[0]), 0)[0] >= 2048
    rep = np.nonzero(seq[1:] == seq[:-1])[0]
    assert len(rep), "no node wins twice in a row"
    k = int(rep[0]) + 1                # pod k goes to the node of pod k - 1, with the score it has after its earlier clones
    assert oracle.node_score(snap, tmpl[0], int(seq[k]), int((seq[:k] == seq[k]).sum()))[0] >= 2048
    assert st["placed"] > st["waves"]  # second lives were taken inside waves
    snap, tmpl, ctr = _score_top_case(21)
    engine = importlib.import_module("cluster-capacity_b200.engine")
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        with pytest.raises(engine.EngineError, match="too large for the packed key"):
            eng.set_templates(tmpl, ctr)


def test_all_keys_tied(built):
    """Identical nodes: keys differ only in the node index, so tile 0 holds the 16 best keys and its 16th key is the bar. No wave
    may commit more than the 16 candidates above it."""
    rng = np.random.default_rng(61)
    n = 20000
    zone = rng.integers(0, 64, n).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 30), topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(64, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    want, st = run_all(snap, [t], ctr, 300, "multi-commit")
    assert want.placed == 300 and st["placed"] <= helpers.MULTI_M * st["waves"]


def test_candidate_cap_raises_the_bar(built, sm_count):
    """At most 16 feasible nodes per tile on a full grid and one score for all: every published entry clears the first bar, far
    more than the replay's 256 slots, so the bar must be raised (bar_raised_waves)."""
    snap, tmpl, ctr = helpers.sparse_eligibility_case(sm_count * helpers.GRID_NODES, max_skew=1)
    _, st = run_all(snap, tmpl, ctr, 300, "multi-commit")
    assert st["grid"] == sm_count and st["bar_raised_waves"] > 0


def test_node_wins_again_within_a_wave(built):
    """Spread only (no hostname term), three nodes with ~100x the room of the rest: the same node wins with its first key, again
    with its second-life key, and the wave ends at its second win."""
    rng = np.random.default_rng(53)
    n = 20000
    a_cpu = rng.choice([4000, 8000], n)
    big = np.array([n // 3, n // 2, n - 5])
    a_cpu[big] = 400000
    a_pods = np.full(n, 110)
    a_pods[big] = 5000
    req_cpu = (rng.random(n) * 0.5 * a_cpu).astype(np.int64) // 10 * 10
    req_cpu[big] = 0
    zone = rng.integers(0, 8, n).astype(np.int32)
    snap = abi.Snapshot(n, a_cpu, a_cpu * (2 * MiB), a_pods, req_cpu=req_cpu, req_mem=req_cpu * (2 * MiB), topo=[zone])
    ctr = [abi.make_counter(0, rng.integers(0, 5, 8).astype(np.int32), inc=1)]
    t = abi.default_template(150, 300 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1000, 1, 0
    want, st = run_all(snap, [t], ctr, 600, "multi-commit")
    assert st["placed"] > st["waves"]      # several commits per wave: the winners came back with their second-life keys
    seq = want.pod_node
    assert np.any((seq[2:] == seq[1:-1]) & (seq[1:-1] == seq[:-2])), "no node wins three times in a row"


def _commit_cap_case(sm_count):
    """Every 300th node feasible on a full grid: about 226 candidates, all above the first bar and within the replay's 256 slots.
    Single-use nodes and a spread constraint that never binds keep every candidate feasible, so only the cap of 64 commits ends a
    wave until the candidates run out."""
    return helpers.sparse_eligibility_case(sm_count * helpers.GRID_NODES, max_skew=10 ** 6, every=300)


def test_commits_per_wave_cap(built, sm_count):
    snap, tmpl, ctr = _commit_cap_case(sm_count)
    want, st = run_all(snap, tmpl, ctr, 0, "multi-commit")
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed == (snap.n + 299) // 300
    assert st["bar_raised_waves"] == 0
    assert st["waves"] * 64 >= st["placed"] > 32 * st["waves"]


@pytest.mark.parametrize("limit", [63, 64, 65, 128, 129])
def test_limit_at_a_wave_edge(built, sm_count, limit):
    """--max-limit just before, at and just after the end of a 64-commit wave."""
    snap, tmpl, ctr = _commit_cap_case(sm_count)
    want, st = run_all(snap, tmpl, ctr, limit, "multi-commit")
    assert want.stop_code == abi.STOP_LIMIT_REACHED and want.placed == limit
    assert st["waves"] == -(-limit // 64)
