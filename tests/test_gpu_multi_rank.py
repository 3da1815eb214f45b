"""GPU: the multi-commit kernel's compaction in key order (ccsim_multi.cuh). After the gather every thread ranks its own entries of
the tiles' sorted lists — per-level ballots, one barrier, a sum over the groups before its own — and stores each candidate at its rank;
more than 256 candidates put the bar at the key of rank 255, and candidates on more than MULTI_LEVELS score levels below the best key
raise the bar to the lowest level kept. Every case runs the CPU oracle and the kernel with and without CCSIM_DEBUG_FLAGS bit 6 (the
arg-max round, which does not depend on the order of the candidates): both must match the oracle pod by pod and each other byte for
byte. A third run with bit 2 (one line per wave) shows which bars the waves took."""
import importlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import helpers

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ARGMAX, WAVE_LINES = 64, 4          # CCSIM_DEBUG_FLAGS bits 6 and 2
CAP, LEVELS, IDX_BITS = 256, 4, helpers.MULTI_IDX_BITS
MASK = (1 << IDX_BITS) - 1


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


def selector_case(n, feasible, req_cpu=None, max_skew=10 ** 6, zones=8):
    """Identical 8-CPU nodes of which those in `feasible` match the template's node selector; `req_cpu` (milli-CPU already
    requested per node) sets the scores. Required anti-affinity on the hostname (a node takes one clone: every wave is replayed in
    key order) and a zone spread constraint with the given maxSkew."""
    i = np.arange(n)
    zone = (i % zones).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 8000), np.full(n, 16 << 30), np.full(n, 110), req_cpu=req_cpu, static_mask=np.asarray(feasible, np.uint64).reshape(1, n),
                        topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(zones, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
    t = abi.default_template(100, 128 << 20)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, max_skew, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return snap, [t], ctr


def score_groups(groups, n=20000, every=40, step=100):
    """Every `every`-th node feasible (at most 16 per tile: no unseen nodes), cycling through `groups` requested-CPU values `step`
    milli-CPU apart, about one score level each: the best key's level and the ones below it are each held by a few nodes, so the
    replay runs dry above the bar and the bar distance grows until the candidates span more levels than the compaction ranks."""
    i = np.arange(n)
    feas = i % every == 0
    return selector_case(n, feas, req_cpu=np.where(feas, step * ((i // every) % groups), 0))


def tile_edges():
    """A grid of 18 CTAs (chunk 488) with a short last tile (481 nodes): tiles 0-1 with every 4th node feasible (more than 16:
    unseen nodes, T from the lists), tiles 2-4 empty, the rest every 40th (fewer than 16 each); three score groups."""
    n, chunk = 8777, 488
    i = np.arange(n)
    tile = i // chunk
    feas = np.where(tile < 2, i % 4 == 0, i % 40 == 0) & ((tile < 2) | (tile > 4))
    return selector_case(n, feas, req_cpu=np.where(feas, 150 * (i % 3), 0))


CASES = {
    "one_score_255": lambda: helpers.sparse_eligibility_case(40 * 255, max_skew=10 ** 6),
    "one_score_256": lambda: helpers.sparse_eligibility_case(40 * 256, max_skew=10 ** 6),
    "one_score_257": lambda: helpers.sparse_eligibility_case(40 * 257, max_skew=10 ** 6),
    "levels_2": lambda: score_groups(2),
    "levels_4": lambda: score_groups(4),
    "levels_40": lambda: score_groups(40),
    "far_more": lambda: score_groups(3, n=60000),
    "tile_edges": tile_edges,
    "c4_small": lambda: synth.c4(n=30000, n_existing=60000, zones=32, racks=256, regions=8),
}


def _gpu(snap, tmpl, ctr, flags, monkeypatch):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        got = eng.run(0)
        return got, eng.run_stats(), eng.key_order_waves()


def wave_lines(case):
    """The kernel's wave lines (CCSIM_DEBUG_FLAGS bit 2) for CASES[case], from a process of its own (device printf is flushed when
    it ends): per wave {C, T, Tlist, kbest, delta}."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_multi_rank as m; m._run_case(%r)" % (HERE, ROOT, case)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=dict(os.environ, CCSIM_DEBUG_FLAGS=str(WAVE_LINES)))
    assert r.returncode == 0, r.stderr[-2000:]
    pat = re.compile(r"wave \d+ k=\d+ acc=\d+ C=(\d+) T=([0-9a-f]+) Tlist=([0-9a-f]+) kbest=([0-9a-f]+) delta=([0-9a-f]+)")
    return [dict(C=int(m.group(1)), T=int(m.group(2), 16), Tlist=int(m.group(3), 16), kbest=int(m.group(4), 16), delta=int(m.group(5), 16))
            for m in pat.finditer(r.stdout)]


def _run_case(case):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    snap, tmpl, ctr = CASES[case]()
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        eng.run(0)


def first_bar(w):
    """The bar before the compaction: the largest last key of a list with unseen nodes, or delta below the best key."""
    return max(w["Tlist"], w["kbest"] - w["delta"] if w["kbest"] > w["delta"] else 0)


def clamped(w):
    """The wave's candidates spanned more than LEVELS score levels: the bar went up to the lowest key of the lowest level kept."""
    return w["T"] > first_bar(w) and w["C"] < CAP and w["T"] == ((w["kbest"] >> IDX_BITS) - (LEVELS - 1)) << IDX_BITS


@pytest.mark.parametrize("case", sorted(CASES))
def test_compaction_in_key_order(built, sm_count, monkeypatch, case):
    snap, tmpl, ctr = CASES[case]()
    assert helpers.multi_eligible(snap, tmpl, ctr, sm_count)
    want = oracle.run(snap, tmpl, ctr, threads=8, memo=True)
    ko, ko_st, ko_waves = _gpu(snap, tmpl, ctr, 0, monkeypatch)
    am, am_st, am_waves = _gpu(snap, tmpl, ctr, ARGMAX, monkeypatch)
    for got, what in ((ko, "key order"), (am, "arg-max round")):
        assert got.placed == want.placed and got.stop_code == want.stop_code, (what, got.placed, want.placed)
        assert np.array_equal(got.pod_node, want.pod_node), (what, np.nonzero(got.pod_node != want.pod_node)[0][:1])
        assert np.array_equal(got.reason_hist, want.reason_hist), what
    assert ko.pod_node.tobytes() == am.pod_node.tobytes() and ko.reason_hist.tobytes() == am.reason_hist.tobytes()
    assert ko_st["kernel"] == am_st["kernel"] == "multi<false>", (ko_st["kernel"], am_st["kernel"])
    for key in ("waves", "placed", "candidates", "bar_raised_waves"):
        assert ko_st[key] == am_st[key], (key, ko_st[key], am_st[key])
    assert ko_waves == ko_st["waves"] and am_waves == 0

    lines = wave_lines(case)
    assert len(lines) == ko_st["waves"]
    assert all(w["C"] <= CAP and w["T"] >= first_bar(w) for w in lines)
    assert sum(w["C"] for w in lines) == ko_st["candidates"]
    exact = [w for w in lines if w["C"] == CAP and w["T"] > first_bar(w)]
    n_clamped = sum(clamped(w) for w in lines)
    print("\n  waves %d placed %d candidates/wave %.1f bar at rank 255 in %d waves, level clamp in %d" % (
        ko_st["waves"], ko_st["placed"], ko_st["candidates"] / max(1, ko_st["waves"]), ko_st["bar_raised_waves"], n_clamped))
    if case.startswith("one_score_"):
        # all feasible nodes share one score and no tile has unseen nodes: the first wave's candidates are exactly the feasible nodes
        c = int(case.rsplit("_", 1)[1])
        assert lines[0]["C"] == min(c, CAP) and n_clamped == 0
        assert (ko_st["bar_raised_waves"] > 0) == (c > CAP)
        if c > CAP:    # the bar is the key of rank 255: node 40 * 255, same score as the best
            assert lines[0]["T"] >> IDX_BITS == lines[0]["kbest"] >> IDX_BITS and MASK - (lines[0]["T"] & MASK) == 40 * 255
    if case == "levels_40":
        assert n_clamped > 0
    if case == "far_more":      # 500 feasible nodes on each of three levels, no unseen nodes: far more than 256 candidates
        assert ko_st["bar_raised_waves"] > 0 and len(exact) > 0


SHARDED = ("levels_40", "one_score_257", "tile_edges")


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case", SHARDED)
def test_node_shards_on_one_gpu(built, sm_count, monkeypatch, case, world):
    """Node shards: every rank compacts its own lists in key order, then the ranks' summaries are merged (gather level 2)."""
    snap, tmpl, ctr = CASES[case]()
    grid = helpers.persistent_grid(snap.n, sm_count, world)
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))
    want = oracle.run(snap, tmpl, ctr, threads=8, memo=True)
    seqs = []
    for flags in (0, ARGMAX):
        monkeypatch.setenv("CCSIM_DEBUG_FLAGS", str(flags))
        engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
        try:
            res = helpers.run_sharded_once(engs, 0)
            stats = [e.run_stats() for e in engs]
        finally:
            for e in engs:
                e.close()
        for r in res:
            assert r.placed == want.placed and r.stop_code == want.stop_code and np.array_equal(r.pod_node, want.pod_node), ("flags", flags)
        assert np.array_equal(sum(r.reason_hist for r in res), want.reason_hist)
        assert all(s["kernel"] == "multi<true>" for s in stats), [s["kernel"] for s in stats]
        seqs.append(res[0].pod_node.tobytes())
    assert seqs[0] == seqs[1]
