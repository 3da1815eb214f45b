"""The multi-commit kernel's two-level gather over node shards (ccsim_multi.cuh), against a plain model of it.

Level 1: every rank compacts its own tiles' lists: the candidates keyed >= T_r = max(Tlist_r, kbest_r - delta), at most
MULTI_LEVELS score levels below its best key (else the bar rises to the lowest level kept), at most 256 (else the bar is the key
of rank 255). Level 2: every rank sends that summary to every peer, and every CTA compacts the summaries concatenated in rank
order with the same rules, from T = max(max_r T_r, kbest - delta) and the global best key. The concatenation is in key order
within a score level only because rank r holds the nodes [per * r, per * (r + 1)); the model below sorts the union by key
instead, so it does not share that assumption with the kernel.

The cases are single-use (required hostname anti-affinity, a zone spread that never binds) and no tile holds more than 16
feasible nodes, so no tile has unseen nodes (Tlist = 0) and a node's key does not change until it wins: the model knows every
wave's candidates from the nodes not yet placed. Every wave line of every rank (CCSIM_DEBUG_FLAGS bit 2) must show the same wave,
and every wave the C and T the model gives for its first pod and its bar distance. The ranks ranked the same waves the same
way: each wave's raised bar is counted once per rank, when either of its levels had more than 256 candidates. A spread-only
case with second lives checks the second-life key carried in the summaries."""
import importlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import helpers
import scoremodel

abi = importlib.import_module("cluster-capacity_b200._abi")
from oracle import binding as oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ARGMAX, WAVE_LINES = 64, 4          # CCSIM_DEBUG_FLAGS bits 6 and 2
CAP, LEVELS, M, IDX_BITS = 256, 4, helpers.MULTI_M, helpers.MULTI_IDX_BITS
MASK = (1 << IDX_BITS) - 1
DELTA0 = 1 << IDX_BITS              # the bar distance of a run's first wave: one score level
NODE_CPU, NODE_MEM = 8000, 16 << 30


# ---- the model ---------------------------------------------------------------------------------------------------------------
def key(score, i):
    return ((score + 1) << IDX_BITS) | (MASK - i)


def key_node(k):
    return MASK - (k & MASK)


def below(k, delta):
    return k - delta if k > delta else 0


def compact(keys, T, kbest):
    """One gather level: the keys >= T in key order, on at most LEVELS score levels from the best key's (more: the bar rises to
    the lowest level kept), at most CAP of them (more: the bar is the key of rank CAP - 1). Returns (kept keys, bar, > CAP)."""
    cand = sorted((k for k in keys if k and k >= T), reverse=True)
    kbl = kbest >> IDX_BITS
    if any(kbl - (k >> IDX_BITS) >= LEVELS for k in cand):
        T = (kbl - (LEVELS - 1)) << IDX_BITS
        cand = [k for k in cand if k >= T]
    over = len(cand) > CAP
    if over:
        T = cand[CAP - 1]
        cand = cand[:CAP]
    return cand, T, over


def model_wave(n, world, nodes, scores, delta=DELTA0):
    """The two-level gather of a wave whose feasible nodes are `nodes` (global indices) with `scores`, when no tile has unseen
    nodes. Returns {C, T, kbest, bar (node of the global rank-255 candidate, or None), raised (per rank: a level had > CAP)}."""
    per = -(-n // world)
    keys = [key(int(s), int(i)) for i, s in zip(nodes, scores)]
    kept, bars, bests, over1 = [], [], [], []
    for r in range(world):
        mine = [k for k in keys if per * r <= key_node(k) < per * (r + 1)]
        kb = max(mine, default=0)
        c, t, o = compact(mine, below(kb, delta), kb)
        kept += c
        bars.append(t)
        bests.append(kb)
        over1.append(o)
    kbest = max(bests)
    cand, T, over2 = compact(kept, max(max(bars), below(kbest, delta)), kbest)
    return dict(C=len(cand), T=T, kbest=kbest, bar=key_node(T) if over2 else None, raised=[o or over2 for o in over1])


# ---- the cases ---------------------------------------------------------------------------------------------------------------
def _template():
    t = abi.default_template(100, 128 << 20)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 10 ** 6, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return t


def model_score(t, req_cpu):
    """The score a key carries for a NODE_CPU / NODE_MEM node with `req_cpu` milli-CPU requested (and as non-zero request), from
    the Go-semantics model: NodeResourcesFit and BalancedAllocation. The other scorers give every node the same score here
    (TaintToleration 100: no PreferNoSchedule taint; the rest nothing to score), and the kernel leaves such a term out of its keys."""
    a = (NODE_CPU, NODE_MEM)
    return (t.w_fit * scoremodel.least_allocated(a, (req_cpu + t.least_cpu, t.least_mem), (t.least_w_cpu, t.least_w_mem))
            + t.w_balanced * scoremodel.balanced(a, (req_cpu + t.bal_cpu, t.bal_mem)))


def req_for_level(off):
    """The smallest requested milli-CPU (a multiple of 10) whose score is `off` levels from an empty node's."""
    t = _template()
    top = model_score(t, 0)
    for r in range(0, NODE_CPU, 10):
        if model_score(t, r) == top + off:
            return r
    raise AssertionError("no request scores %d levels from the top" % off)


A, B, BURIED = 0, -1, -12           # score levels, relative to an empty node's


class Case:
    """Identical nodes of which `groups` {level: node indices} match the template's node selector, each group on its score
    level. Required anti-affinity on the hostname (a node takes one clone) and a zone spread that never binds."""

    def __init__(self, n, world, groups):
        feas = np.zeros(n, bool)
        req = np.zeros(n, np.int64)
        for lv, idx in groups.items():
            assert not feas[idx].any()
            feas[idx] = True
            req[idx] = req_for_level(lv)
        zone = (np.arange(n) % 8).astype(np.int32)
        self.n, self.world = n, world
        self.snap = abi.Snapshot(n, np.full(n, NODE_CPU), np.full(n, NODE_MEM), np.full(n, 110), req_cpu=req,
                                 static_mask=feas.astype(np.uint64).reshape(1, n), topo=[zone])
        self.ctr = [abi.make_counter(0, np.zeros(8, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
        self.tmpl = [_template()]
        self.nodes = np.nonzero(feas)[0]
        self.scores = np.array([model_score(self.tmpl[0], int(r)) for r in req[self.nodes]], np.int64)
        top = model_score(self.tmpl[0], 0)
        for lv, idx in groups.items():            # every group on the score level it is meant for
            assert set(self.scores[np.isin(self.nodes, idx)].tolist()) == {top + lv}, lv

    def ranks(self):
        per = -(-self.n // self.world)
        return [(per * r, min(self.n, per * (r + 1))) for r in range(self.world)]

    def most_per_tile(self, sm_count):
        """The most feasible nodes in one tile of any rank (the kernel's grid and chunk rule)."""
        grid = helpers.persistent_grid(self.n, sm_count, self.world)
        most = 0
        for lo, hi in self.ranks():
            chunk = -(-(hi - lo) // grid)
            most = max(most, int(np.bincount((self.nodes[(self.nodes >= lo) & (self.nodes < hi)] - lo) // chunk).max(initial=0)))
        return most

    def first_wave(self):
        return model_wave(self.n, self.world, self.nodes, self.scores)


def union(count):
    """One score, every 40th node feasible, `count` in all: no rank has more than 256 of them."""
    return lambda world: Case(40 * count, world, {A: np.arange(0, 40 * count, 40)})


def rank_overflows_alone(world):
    """One score, every 32nd node feasible, 288 per rank: every rank keeps its first 256, the union only rank 0's."""
    n = 9216 * world
    return Case(n, world, {A: np.arange(0, n, 32)})


def full_summaries(levels):
    """65 536 nodes over 8 ranks of 16 tiles of 512: every 32nd node feasible, exactly 16 per tile and 256 per rank, 2 048
    summary entries. `levels`: the nodes from 28 672 on (the second half of rank 3 and ranks 4-7) one level higher, so the bar
    falls inside rank 4."""
    def make(world):
        idx = np.arange(0, 65536, 32)
        return Case(65536, world, {A: idx[idx >= 28672], B: idx[idx < 28672]} if levels else {A: idx})
    return make


def tie_at_the_bar(world):
    """100 nodes on level A at the end of the last rank, 292 on level B below them, spread over every rank: the union's rank 255
    is the 156th B node, inside a middle rank."""
    return Case(32000, world, {A: np.arange(28000, 32000, 40), B: np.arange(0, 28000, 96)})


def empty_and_buried_ranks(world):
    """Rank 0's nodes 12 levels below everyone's (below the global bar), rank 1 without a feasible node, every 40th node of the
    later ranks on the top level."""
    n = 24000
    per = -(-n // world)
    return Case(n, world, {BURIED: np.arange(0, per, 40), A: np.arange(2 * per, n, 40)})


def double_overflow(world):
    """Rank 0: 300 nodes on level B (more than 256 on its own). Rank 1: 10 nodes on level A. The union of rank 0's 256 and rank
    1's 10 overflows again."""
    return Case(19200, world, {B: np.arange(0, 9600, 32), A: 9600 + 40 * np.arange(10)})


def levels_by_rank(world):
    """Four nodes on each of 4 x world score levels, four levels per rank, rank r's below rank r - 1's: a rank's own candidates
    span at most four levels, so once the bar distance has grown the union's levels are clamped at level 2 only."""
    per = 16 * 40
    return Case(world * per, world, {-4 * r - q: per * r + 40 * (4 * q + np.arange(4)) for r in range(world) for q in range(4)})


CASES = {
    "union_256": (union(256), (2, 3, 4)),
    "union_257": (union(257), (2, 3, 4)),
    "rank_overflows_alone": (rank_overflows_alone, (2, 4)),
    "full_summaries": (full_summaries(False), (8,)),
    "full_summaries_levels": (full_summaries(True), (8,)),
    "tie_at_the_bar": (tie_at_the_bar, (3, 4, 8)),
    "empty_and_buried_ranks": (empty_and_buried_ranks, (3, 4)),
    "double_overflow": (double_overflow, (2,)),
    "levels_by_rank": (levels_by_rank, (3, 4)),
}
PARAMS = [(c, w) for c, (_, worlds) in sorted(CASES.items()) for w in worlds]


def make_case(name, world):
    return CASES[name][0](world)


# ---- the model on its own (no GPU) -------------------------------------------------------------------------------------------
def test_model_hand_worked():
    s = 400
    # rank 0: 300 nodes on level s (more than 256 on its own: its bar is its 256th, node 32 * 255); rank 1: 10 nodes one level
    # higher. The union of 10 + 256 overflows again: its rank 255 is rank 0's 246th node. Each rank raised a bar once.
    nodes = np.concatenate([np.arange(0, 9600, 32), 9600 + 40 * np.arange(10)])
    m = model_wave(19200, 2, nodes, np.where(nodes < 9600, s, s + 1))
    assert (m["C"], m["T"], m["kbest"], m["bar"], m["raised"]) == (256, key(s, 32 * 245), key(s + 1, 9600), 32 * 245, [True, True])
    # 257 tied nodes, every 40th, over three ranks of 3 427: 85 + 86 + 86, none overflows alone. The bar is the 256th node, on the
    # last rank; the first wave's bar before the compaction is one level below the best key, node 0's.
    m = model_wave(40 * 257, 3, np.arange(0, 40 * 257, 40), np.full(257, s))
    assert (m["C"], m["T"], m["bar"], m["raised"]) == (256, key(s, 40 * 255), 40 * 255, [True] * 3)
    m = model_wave(40 * 256, 3, np.arange(0, 40 * 256, 40), np.full(256, s))
    assert (m["C"], m["T"], m["bar"], m["raised"]) == (256, key(s - 1, 0), None, [False] * 3)
    # at equal score a lower node index ranks higher, whichever rank it is on: rank 1's node 600 falls below the bar of 256 from
    # rank 0's 255 nodes and rank 1's node 500
    nodes = np.concatenate([np.arange(0, 255), [500, 600]])
    m = model_wave(1000, 2, nodes, np.full(len(nodes), s))
    assert (m["C"], m["bar"]) == (256, 500)
    # a rank far below the bar adds nothing; the first bar admits the next level down only up to the best node's index (node
    # 1500), so rank 2's nodes 2100 and 2200 need a wider bar distance
    nodes = np.array([10, 20, 1500, 2100, 2200, 2300])
    m = model_wave(3000, 3, nodes, np.array([s - 12, s - 12, s, s - 1, s - 1, s]))
    assert (m["C"], m["T"], m["kbest"]) == (2, key(s - 1, 1500), key(s, 1500))
    m = model_wave(3000, 3, nodes, np.array([s - 12, s - 12, s, s - 1, s - 1, s]), delta=4 << IDX_BITS)
    assert (m["C"], m["T"]) == (4, key(s - 4, 1500))
    # more than LEVELS levels in the union, at most LEVELS on each rank: the clamp of level 2 raises the bar to level s - 3
    m = model_wave(6000, 2, np.array([0, 1, 2, 3000, 3001, 3002]), np.array([s, s - 1, s - 2, s - 3, s - 4, s - 5]), delta=8 << IDX_BITS)
    assert (m["C"], m["T"], m["bar"]) == (4, (s + 1 - 3) << IDX_BITS, None)
    cand, T, over = compact([key(s - v, v) for v in range(6)], 0, key(s, 0))
    assert (len(cand), T, over) == (4, (s + 1 - 3) << IDX_BITS, False)


@pytest.mark.parametrize("case,world", PARAMS)
def test_cases_reach_their_edge(case, world):
    """Each case's first wave, by the model, is the edge it is named for; no tile holds more than 16 feasible nodes."""
    c = make_case(case, world)
    assert c.most_per_tile(helpers.MAX_GRID) <= M
    m = c.first_wave()
    ranks = c.ranks()
    rank_of = lambda i: next(r for r, (lo, hi) in enumerate(ranks) if lo <= i < hi)
    if case == "union_256":
        assert (m["C"], m["bar"], m["raised"]) == (256, None, [False] * world)
    elif case == "union_257":
        assert (m["C"], m["bar"], rank_of(m["bar"]), m["raised"]) == (256, 40 * 255, world - 1, [True] * world)
    elif case == "rank_overflows_alone":
        assert (m["C"], m["T"], m["bar"], m["raised"]) == (256, key(c.scores[0], 32 * 255), None, [True] * world)
    elif case.startswith("full_summaries"):
        assert all((hi - lo) // 32 == 256 for lo, hi in ranks) and m["C"] == 256 and m["raised"] == [True] * world
        bar = 28672 + 32 * 255 if case.endswith("levels") else 32 * 255
        assert m["bar"] == bar and rank_of(bar) == (4 if case.endswith("levels") else 0)
    elif case == "tie_at_the_bar":
        assert m["bar"] == 96 * 155 and 0 < rank_of(m["bar"]) < world - 1
    elif case == "empty_and_buried_ranks":
        lo1, hi1 = ranks[1]
        assert not np.any((c.nodes >= lo1) & (c.nodes < hi1))
        assert all(key(s, i) < m["T"] for i, s in zip(c.nodes, c.scores) if i < ranks[0][1])
        assert m["bar"] == (2 * 6000 + 40 * 255 if world == 4 else None)
    elif case == "double_overflow":
        assert (m["C"], m["bar"], m["raised"]) == (256, 32 * 245, [True, True])
    elif case == "levels_by_rank":
        assert m["C"] < 16 and not any(m["raised"])


def test_model_scores_match_the_oracle(built):
    """The model's scores of every level the cases use, plus the TaintToleration score every node has, are the reference's (the
    CPU oracle's node score)."""
    for case in (levels_by_rank(4), empty_and_buried_ranks(3)):
        t = case.tmpl[0]
        same = t.w_taint * int(scoremodel.taint_norm(np.zeros(1, np.int64))[0])
        for i, s in zip(case.nodes, case.scores):
            assert oracle.node_score(case.snap, t, int(i), 0)[0] == s + same, i


# ---- the kernel against the model (one GPU: the ranks are handles of this process) ------------------------------------------
@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def skip_unless_fits(n, world, sm_count):
    grid = helpers.persistent_grid(n, sm_count, world)      # the ranks' persistent grids run side by side on this one device
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))


def second_life_case():
    """Spread only (no hostname term) with scores above 2048: a winner comes back in its wave with its second-life key, whose
    top bit (bit 11 of the 12-bit field) is set."""
    from test_gpu_multi_edges import _score_top_case
    return _score_top_case(20)


SECOND_LIFE_LIMIT = 1500


def workload(name, world):
    if name == "second_life":
        return second_life_case()
    c = make_case(name, world)
    return c.snap, c.tmpl, c.ctr


def run_ranks(snap, tmpl, ctr, world, limit, flags, monkeypatch):
    """One run of `world` ranks under ENGINE_AUTO: per rank its RunResult, run_stats, node counts and key-order waves."""
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
    engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
    try:
        res = helpers.run_sharded_once(engs, limit)
        return res, [e.run_stats() for e in engs], [e.node_counts(0)[0] for e in engs], [e.key_order_waves() for e in engs]
    finally:
        for e in engs:
            e.close()


def check_ranks(want, n, res, stats, counts):
    """tests/test_gpu_sharded_edges.py's check_sharded for one engine: every rank's pod -> node sequence, stop code and node
    counts, the sums of the FitError histogram and preemption counters; every rank ran multi<true> and the same waves."""
    per_node = np.bincount(want.pod_node, minlength=n)
    for r, got in enumerate(res):
        assert (got.placed, got.stop_code) == (want.placed, want.stop_code), ("rank", r, got.placed, want.placed, got.stop_code)
        m = min(got.placed, want.placed)
        assert np.array_equal(got.pod_node, want.pod_node), ("rank", r, "first difference at pod", np.nonzero(got.pod_node[:m] != want.pod_node[:m])[0][:1])
        assert np.array_equal(counts[r], per_node), ("rank", r, "node counts")
    assert np.array_equal(sum(g.reason_hist for g in res), want.reason_hist)
    assert sum(g.preempt_no_victims for g in res) == want.preempt_no_victims
    assert sum(g.preempt_not_helpful for g in res) == want.preempt_not_helpful
    assert all(s["kernel"] == "multi<true>" for s in stats), [s["kernel"] for s in stats]
    for k in ("waves", "placed", "candidates"):
        assert len({s[k] for s in stats}) == 1, (k, [s[k] for s in stats])
    assert all(s["bar_raised_waves"] <= s["waves"] for s in stats), [(s["bar_raised_waves"], s["waves"]) for s in stats]


LINE = re.compile(r"wave (\d+) k=(\d+) acc=(\d+) C=(\d+) T=([0-9a-f]+) Tlist=([0-9a-f]+) kbest=([0-9a-f]+) delta=([0-9a-f]+) "
                  r"ran_dry=\d+ look_ahead=\d+ first=(-?\d+) last=(-?\d+)")
FIELDS = ("k", "acc", "C", "T", "Tlist", "kbest", "delta", "first", "last")


def _run_workload(name, world, limit):
    snap, tmpl, ctr = workload(name, world)
    engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
    try:
        helpers.run_sharded_once(engs, limit)
    finally:
        for e in engs:
            e.close()


def wave_lines(name, world, limit=0):
    """The wave lines (CCSIM_DEBUG_FLAGS bit 2) of a run of `world` ranks, from a process of its own (device printf is flushed when
    it ends). CTA 0 of every rank prints one line per wave: every wave must have exactly `world` lines, all the same. Returns
    the waves in order, one dict each."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_multi_shard_merge as m; m._run_workload(%r, %d, %d)" % (
        HERE, ROOT, name, world, limit)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, CCSIM_DEBUG_FLAGS=str(WAVE_LINES)))
    assert r.returncode == 0, r.stderr[-2000:]
    waves = {}
    for m in LINE.finditer(r.stdout):
        v = [int(m.group(i)) for i in (2, 3, 4)] + [int(m.group(i), 16) for i in (5, 6, 7, 8)] + [int(m.group(9)), int(m.group(10))]
        waves.setdefault(int(m.group(1)), []).append(dict(zip(FIELDS, v)))
    assert sorted(waves) == list(range(len(waves)))
    for w, ls in waves.items():
        assert len(ls) == world and all(x == ls[0] for x in ls), ("wave", w, ls)
    return [waves[w][0] for w in range(len(waves))]


def check_wave_lines(lines, stats):
    """Every wave keeps at most 256 candidates above a bar no lower than the one it starts from; the lines add up to the run's
    statistics."""
    assert len(lines) == stats[0]["waves"]
    for i, w in enumerate(lines):
        assert w["C"] <= CAP and w["T"] >= max(w["Tlist"], below(w["kbest"], w["delta"])), (i, w)
    assert sum(w["C"] for w in lines) == stats[0]["candidates"]
    assert sum(w["acc"] for w in lines) == stats[0]["placed"]


@pytest.mark.gpu
@pytest.mark.parametrize("case,world", PARAMS)
def test_gather_over_shards_matches_the_model(built, sm_count, monkeypatch, case, world):
    """The oracle's placements on every rank, with the key-order round and the arg-max round alike; every wave line of every rank
    the same, and every wave's C, T and best key the model's; each rank's raised bars counted once per wave."""
    c = make_case(case, world)
    skip_unless_fits(c.n, world, sm_count)
    assert c.most_per_tile(sm_count) <= M
    want = oracle.run(c.snap, c.tmpl, c.ctr, threads=8, memo=True)
    ko = run_ranks(c.snap, c.tmpl, c.ctr, world, 0, 0, monkeypatch)
    am = run_ranks(c.snap, c.tmpl, c.ctr, world, 0, ARGMAX, monkeypatch)
    for res, stats, counts, _ in (ko, am):
        check_ranks(want, c.n, res, stats, counts)
    assert ko[0][0].pod_node.tobytes() == am[0][0].pod_node.tobytes()
    for a, b in zip(ko[1], am[1]):        # the arg-max round replays the same candidates: the same waves
        assert all(a[k] == b[k] for k in ("waves", "placed", "candidates", "bar_raised_waves")), (a, b)
    assert ko[3] == [s["waves"] for s in ko[1]] and am[3] == [0] * world

    lines = wave_lines(case, world)
    check_wave_lines(lines, ko[1])
    # every wave, from the nodes not placed before it and its bar distance, as the model sees it; each wave counts a raised bar
    # once on a rank, whichever of its levels went over 256
    placed = want.pod_node
    raised = np.zeros(world, np.int64)
    for i, w in enumerate(lines):
        left = ~np.isin(c.nodes, placed[:w["k"]])
        m = model_wave(c.n, world, c.nodes[left], c.scores[left], w["delta"])
        assert (w["C"], w["T"], w["kbest"], w["Tlist"]) == (m["C"], m["T"], m["kbest"], 0), (i, w, m)
        raised += m["raised"]
    assert lines[0]["delta"] == DELTA0
    assert [s["bar_raised_waves"] for s in ko[1]] == raised.tolist()
    first = c.first_wave()
    print("\n  world %d waves %d placed %d candidates %d | first wave C %d T %08x (rank-255 node %s) | raised bars per rank %s" % (
        world, len(lines), want.placed, ko[1][0]["candidates"], lines[0]["C"], lines[0]["T"], first["bar"], raised.tolist()), end="")
    if case == "levels_by_rank":        # the union spanned more than LEVELS levels while no rank's own candidates did
        assert any(w["T"] == ((w["kbest"] >> IDX_BITS) - (LEVELS - 1)) << IDX_BITS and w["T"] > below(w["kbest"], w["delta"])
                   for w in lines)


@pytest.mark.gpu
def test_double_overflow_raises_one_bar(built, sm_count, monkeypatch):
    """One wave (--max-limit 1) in which rank 0's own lists and then the union both hold more than 256 candidates: every rank
    counts one raised bar."""
    c = double_overflow(2)
    skip_unless_fits(c.n, 2, sm_count)
    want = oracle.run(c.snap, c.tmpl, c.ctr, max_pods=1, threads=8, memo=True)
    res, stats, counts, _ = run_ranks(c.snap, c.tmpl, c.ctr, 2, 1, 0, monkeypatch)
    check_ranks(want, c.n, res, stats, counts)
    assert c.first_wave()["raised"] == [True, True]
    assert [(s["waves"], s["bar_raised_waves"]) for s in stats] == [(1, 1), (1, 1)], stats


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_second_lives_over_shards(built, sm_count, monkeypatch, world):
    snap, tmpl, ctr = second_life_case()
    skip_unless_fits(snap.n, world, sm_count)
    want = oracle.run(snap, tmpl, ctr, max_pods=SECOND_LIFE_LIMIT, threads=8, memo=True)
    res, stats, counts, _ = run_ranks(snap, tmpl, ctr, world, SECOND_LIFE_LIMIT, 0, monkeypatch)
    check_ranks(want, snap.n, res, stats, counts)
    seq = want.pod_node
    rep = np.nonzero(seq[1:] == seq[:-1])[0] + 1            # pod k won by the node of pod k - 1
    assert len(rep) and oracle.node_score(snap, tmpl[0], int(seq[rep[0]]), int((seq[:rep[0]] == seq[rep[0]]).sum()))[0] >= 2048
    assert all(s["placed"] > s["waves"] for s in stats)      # second lives were taken inside waves
    lines = wave_lines("second_life", world, SECOND_LIFE_LIMIT)
    check_wave_lines(lines, stats)
    print("\n  world %d waves %d placed %d candidates %d raised bars %s" % (world, len(lines), want.placed, stats[0]["candidates"],
                                                                           [s["bar_raised_waves"] for s in stats]), end="")
