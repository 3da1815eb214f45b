"""GPU (ONE device is enough): the node-sharded engines with all ranks on device 0. Every rank is a handle of this process, the
exchange buffers are wired by pointer (ccsim_peer_import_local) and the ranks' persistent kernels run concurrently on different
streams (small clusters: every rank needs only a few SMs), started from one host thread per rank. The same in-kernel exchange
as across GPUs — candidate lines of every CTA into every rank's buffer (multi-commit), winner words (lean, streaming) — only
the stores do not cross NVLink. Results must equal the oracle's, like tests/test_gpu_sharded.py on a multi-GPU box."""
import importlib

import numpy as np
import pytest

import helpers
from helpers import run_sharded

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
from oracle import binding as oracle  # noqa: E402

pytestmark = pytest.mark.gpu


CASES = {
    "c3": (lambda: synth.c3(n=5001, prefer_taints=True), 0, None),
    "c4": (lambda: synth.c4(n=6000, n_existing=12000, zones=8, racks=64, regions=4), 0, "multi-commit"),
    "c4_limit": (lambda: synth.c4(n=9000, n_existing=15000, zones=16, racks=128, regions=4), 700, "multi-commit"),
    "spread": (lambda: (lambda s, t, c: (s, [_no_anti(t[0])], c[:3]))(*synth.c4(n=7000, n_existing=9000, zones=8, racks=64, regions=4)), 900, "multi-commit"),
    "c5": (lambda: synth.c5(n=9001, n_templates=9), 1200, "streaming"),
    # every 40th node feasible, one score for all: each rank publishes more than 256 candidates (40 CTAs per rank at world 2), so the
    # bar is raised on the ranks and again over the union of their summaries (at world 4 the union alone overflows)
    "sparse": (lambda: helpers.sparse_eligibility_case(40000, max_skew=10 ** 6), 500, "multi-commit"),
}
BAR_RAISED = {"sparse"}


def _no_anti(t):
    t.n_anti = 0
    return t


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("which", sorted(CASES))
def test_sharded_engines_on_one_gpu_match_the_oracle(built, sm_count, which, world):
    make, limit, engine_name = CASES[which]
    snap, tmpl, ctr = make()
    grid = helpers.persistent_grid(snap.n, sm_count, world)     # the ranks' persistent grids run side by side on this one device
    if world * grid > sm_count:
        pytest.skip("%d ranks x %d CTAs do not fit on %d SMs" % (world, grid, sm_count))
    runs = [limit, (limit or 0) // 2 + 7, limit]        # several runs per handle: epoch / buffer parity carry over
    wants = [oracle.run(snap, tmpl, ctr, max_pods=lim, threads=4, memo=True) for lim in runs]
    for kind in (abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL):
        for (res, stats), w in zip(run_sharded(snap, tmpl, ctr, limit, world, kind, runs), wants):
            for r in res:       # replicated parts: identical on every rank
                assert r.placed == w.placed and r.stop_code == w.stop_code
                assert np.array_equal(r.pod_node, w.pod_node), "rank sequence differs from the oracle at pod %d" % int(
                    np.nonzero(r.pod_node[:min(len(r.pod_node), len(w.pod_node))] != w.pod_node[:min(len(r.pod_node), len(w.pod_node))])[0][0])
            # per-shard parts sum up
            assert np.array_equal(sum(r.reason_hist for r in res), w.reason_hist)
            assert sum(r.preempt_no_victims for r in res) == w.preempt_no_victims
            assert sum(r.preempt_not_helpful for r in res) == w.preempt_not_helpful
            if kind == abi.ENGINE_SEQUENTIAL:
                assert sum(r.evals for r in res) == w.evals
            elif engine_name:
                assert all(engine_name in s["engine"] for s in stats), stats
                if which in BAR_RAISED:
                    assert all(s["bar_raised_waves"] > 0 for s in stats), stats
