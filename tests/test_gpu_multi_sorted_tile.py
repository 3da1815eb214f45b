"""GPU: the multi-commit kernel's selection from the sorted tile (ccsim_multi.cuh). Single-use templates (required hostname
anti-affinity: a node takes one clone) sort each tile by key once per launch and publish the first 16 feasible nodes in key order;
CCSIM_DEBUG_FLAGS bit 7 (128) keeps the per-warp REDUX rounds and the merge. Every case runs the CPU oracle and the kernel with and
without bit 7, each in a process of its own with the wave lines on (bit 2: device printf is flushed when the process ends). Both
runs must match the oracle pod by pod and each other byte for byte, run the same waves with the same candidates and raised bars,
and print the same wave lines: the published lines are word for word the same, so everything after them is too. The sorted-tile
counter (Engine.sorted_tile_waves) shows which selection ran."""
import importlib
import os
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
GiB, MiB = 1 << 30, 1 << 20
REDUX, LOOK_AHEAD, WAVE_LINES = 128, 32, 4      # CCSIM_DEBUG_FLAGS bits 7, 5 and 2


def selector_case(feasible, req_cpu, zones=8, max_skew=10 ** 6):
    """Identical 8-CPU nodes of which those in `feasible` match the node selector; `req_cpu` (milli-CPU already requested) sets
    the scores. Hostname anti-affinity (single use) and a zone spread constraint."""
    n = len(feasible)
    zone = (np.arange(n) % zones).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 8000), np.full(n, 16 * GiB), np.full(n, 110), req_cpu=np.asarray(req_cpu, np.int64),
                        static_mask=np.asarray(feasible, np.uint64).reshape(1, n), topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(zones, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
    t = abi.default_template(100, 128 * MiB)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, max_skew, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return snap, [t], ctr


def tiles_16_17_empty():
    """18 CTAs of 488 nodes and a short last tile of 481: tile 0 with exactly 16 feasible nodes (no more-bit), tile 1 with 17 (the
    16th entry carries the more-bit and is the bar), tiles 2-4 without a feasible node, the rest every 40th. Scores are random, so
    key order is not slot order."""
    n, chunk = 8777, 488
    rng = np.random.default_rng(7)
    i = np.arange(n)
    tile = i // chunk
    feas = np.where(tile >= 5, i % 40 == 0, False)
    feas[rng.choice(chunk, 16, replace=False)] = True
    feas[chunk + rng.choice(chunk, 17, replace=False)] = True
    return selector_case(feas, np.where(feas, 10 * rng.integers(0, 500, n), 0))


def all_tied():
    """Identical nodes, all feasible: keys differ only in the node index, so key order is slot order."""
    rng = np.random.default_rng(61)
    n = 20000
    zone = rng.integers(0, 64, n).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 4000), np.full(n, 8 * GiB), np.full(n, 30), topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(64, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
    t = abi.default_template(150, 100 * MiB)
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, 1, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return snap, [t], ctr


def spread_only():
    """No hostname term: a winner may come back in its wave (second life), so no tile is sorted."""
    snap, tmpl, ctr = synth.c4(n=7000, n_existing=9000, zones=8, racks=64, regions=4)
    tmpl[0].n_anti = 0
    return snap, tmpl, ctr[:3]


# name -> (workload, --max-limit, flags of both runs, single-use template)
CASES = {
    "c4_small": (lambda: synth.c4(n=30000, n_existing=60000, zones=32, racks=256, regions=8), 0, 0, True),
    "c4_full": (synth.c4, 0, 0, True),
    "sparse": (lambda: helpers.sparse_eligibility_case(40 * 300, max_skew=1), 0, 0, True),
    "tiles_16_17_empty": (tiles_16_17_empty, 0, 0, True),
    "all_tied": (all_tied, 3000, 0, True),
    "short_last_tile": (lambda: synth.c4(n=9001, n_existing=18000, zones=8, racks=64, regions=4), 0, 0, True),
    "look_ahead": (lambda: synth.c4(n=30000, n_existing=60000, zones=32, racks=256, regions=8), 0, LOOK_AHEAD, True),
    "spread_only": (spread_only, 900, 0, False),
}


def _worker(case, limit, world, out):
    """Runs CASES[case] once (CCSIM_DEBUG_FLAGS from the environment) and saves what the parent compares: on one GPU, or as
    `world` node shards of this process on device 0."""
    snap, tmpl, ctr = CASES[case][0]()
    if world == 1:
        engine = importlib.import_module("cluster-capacity_b200.engine")
        with engine.Engine(device=0) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            res = [eng.run(limit)]
            stats, sorted_waves = [eng.run_stats()], [eng.sorted_tile_waves()]
    else:
        engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
        try:
            res = helpers.run_sharded_once(engs, limit)
            stats, sorted_waves = [e.run_stats() for e in engs], [e.sorted_tile_waves() for e in engs]
        finally:
            for e in engs:
                e.close()
    np.savez(out, pod_node=np.stack([r.pod_node for r in res]), reason_hist=np.stack([r.reason_hist for r in res]),
             placed=[r.placed for r in res], stop_code=[r.stop_code for r in res], sorted_waves=sorted_waves,
             engine=[s["engine"] for s in stats],
             stats=[[s[k] for k in ("waves", "placed", "candidates", "bar_raised_waves")] for s in stats])


def _run(tmp_path, case, flags, limit, world=1):
    out = str(tmp_path / ("%s_%d_%d_%d.npz" % (case, flags, limit, world)))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_multi_sorted_tile as m; m._worker(%r, %d, %d, %r)" % (HERE, ROOT, case, limit, world, out)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, CCSIM_DEBUG_FLAGS=str(flags | WAVE_LINES)))
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("wave ")]
    return dict(np.load(out)), lines


def _matches_oracle(got, want, world):
    for r in range(world):          # node shards: the replicated parts are identical on every rank; the FitError histogram is per shard
        assert int(got["placed"][r]) == want.placed and int(got["stop_code"][r]) == want.stop_code, (r, got["placed"], want.placed)
        assert np.array_equal(got["pod_node"][r], want.pod_node), r
    assert np.array_equal(got["reason_hist"].sum(axis=0), want.reason_hist)


def check(tmp_path, case, limit=None, world=1):
    make, case_limit, flags, single_use = CASES[case]
    limit = case_limit if limit is None else limit
    snap, tmpl, ctr = make()
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=8, memo=True)
    srt, srt_lines = _run(tmp_path, case, flags, limit, world)
    rdx, rdx_lines = _run(tmp_path, case, flags | REDUX, limit, world)
    _matches_oracle(srt, want, world)
    _matches_oracle(rdx, want, world)
    for key in ("pod_node", "reason_hist", "placed", "stop_code"):
        assert srt[key].tobytes() == rdx[key].tobytes(), key
    assert all(e == "multi-commit" for e in list(srt["engine"]) + list(rdx["engine"])), (srt["engine"], rdx["engine"])
    # waves, placed, candidates, raised bars: the selection changes how a tile's list is found, not what it holds
    assert np.array_equal(srt["stats"], rdx["stats"]), (srt["stats"], rdx["stats"])
    # node shards: every rank's CTA 0 prints; the ranks run side by side, so their lines interleave
    if world > 1:
        srt_lines, rdx_lines = sorted(srt_lines), sorted(rdx_lines)
    assert len(srt_lines) == world * int(srt["stats"][0][0])
    assert srt_lines == rdx_lines
    waves = srt["stats"][:, 0]
    assert np.array_equal(srt["sorted_waves"], waves if single_use else np.zeros_like(waves)), (srt["sorted_waves"], waves)
    assert not rdx["sorted_waves"].any()
    print("\n  %s: waves %d placed %d sorted-tile waves %s" % (case, waves[0], want.placed, list(srt["sorted_waves"])))
    return want, srt


@pytest.mark.parametrize("case", sorted(set(CASES) - {"c4_full"}))
def test_same_lists_both_ways(built, tmp_path, case):
    check(tmp_path, case)


def test_c4_full(built, tmp_path):
    """The bench workload: 100k nodes, three spread constraints and hostname anti-affinity, to Unschedulable."""
    want, srt = check(tmp_path, "c4_full")
    assert want.stop_code == abi.STOP_UNSCHEDULABLE and want.placed == 31071
    assert int(srt["stats"][0][0]) == 1406


def test_limit_at_a_wave_edge(built, tmp_path):
    """--max-limit equal to the pods placed before some wave: the run stops at the top of that wave, right after the row updates
    of the wave before it."""
    _, lines = _run(tmp_path, "c4_small", 0, 0)
    ks = [int(ln.split()[2][2:]) for ln in lines]
    edge = ks[len(ks) // 2]
    assert edge > 0
    want, srt = check(tmp_path, "c4_small", limit=edge)
    assert want.stop_code == abi.STOP_LIMIT_REACHED and want.placed == edge


@pytest.mark.parametrize("world", [2, 4])
def test_node_shards_on_one_gpu(built, tmp_path, world):
    """Node shards: tiles are per rank, so every rank selects from its sorted tiles; the lines stay on each GPU."""
    sm_count = helpers.device_sm_count()
    snap, _, _ = CASES["short_last_tile"][0]()
    grid = helpers.persistent_grid(snap.n, sm_count, world)
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))
    check(tmp_path, "short_last_tile", world=world)
