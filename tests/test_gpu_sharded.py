"""GPU (needs >= 2 devices, skipped otherwise): the node-sharded run — one process per GPU, per-wave exchange of the shard
winners through peer memory inside the persistent kernel — must give exactly the single-GPU / oracle result."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _worker(rank, world, port, which, q, n=0):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    synth = importlib.import_module("cluster-capacity_b200.synth")
    engine = importlib.import_module("cluster-capacity_b200.engine")
    sharded = importlib.import_module("cluster-capacity_b200.sharded")
    from oracle import binding as oracle
    abi = importlib.import_module("cluster-capacity_b200._abi")
    limit = 0
    if which == "c3":
        snap, tmpl, ctr = synth.c3(n=5001, prefer_taints=True)
    elif which == "c4":
        snap, tmpl, ctr = synth.c4(n=6000, n_existing=12000, zones=8, racks=64, regions=4)
    elif which == "c5":            # several node-local templates: the streaming (TMA) engine over node shards
        snap, tmpl, ctr = synth.c5(n=300_001, n_templates=9)
        limit = 1500
    elif which == "ext":          # the generic kernel: extended resource, ephemeral storage and hostPorts, resident tiles
        snap, tmpl, ctr = importlib.import_module("test_gpu_sharded_edges").generic_ext_ports(200_001)
        limit = 3000
    elif which == "generic_streamed":     # the generic kernel with each rank's tile streamed from global memory
        snap, tmpl, ctr = importlib.import_module("test_gpu_sharded_edges").generic_streamed(n)
        limit = 300
    elif which == "c4_wide":      # enough nodes per shard for full grids: the multi-commit replay sees 2 x grid candidate lists
        snap, tmpl, ctr = synth.c4(n=120_001, n_existing=200_000, zones=32, racks=1024, regions=8)
        limit = 3000
    else:                          # spread only: nodes take several clones, winners re-enter the replay ("second life")
        snap, tmpl, ctr = synth.c4(n=40_000, n_existing=60_000, zones=16, racks=256, regions=4)
        tmpl[0].n_anti = 0
        ctr = ctr[:3]
        limit = 2500
    torch.cuda.set_device(rank)
    ok = True
    why = []
    want = oracle.run(snap, tmpl, ctr, max_pods=limit, threads=8, memo=True)
    for kind in (abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL):   # AUTO: multi-commit waves over the shards for counter-coupled templates
        eng = engine.Engine(device=rank, engine=kind, rank=rank, world=world)
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        eng.connect_peers(dist)
        for it in range(3):          # several runs per handle: the run epoch / buffer parity must carry over; no host barrier in between
            res = eng.run(limit if it != 1 else (limit or 0) // 2 + 7)
            m = sharded.merge_results(dist, res)
            w = want if it != 1 else oracle.run(snap, tmpl, ctr, max_pods=(limit or 0) // 2 + 7, threads=8, memo=True)
            same = (m["placed"] == w.placed and m["stop_code"] == w.stop_code and np.array_equal(m["pod_node"], w.pod_node)
                    and np.array_equal(m["reason_hist"], w.reason_hist) and m["preempt_no_victims"] == w.preempt_no_victims
                    and m["preempt_not_helpful"] == w.preempt_not_helpful)
            if not same:
                why.append("engine %d run %d: placed %d/%d stop %d/%d seq_equal %s hist_equal %s preempt %d,%d / %d,%d" % (
                    kind, it, m["placed"], w.placed, m["stop_code"], w.stop_code, np.array_equal(m["pod_node"], w.pod_node),
                    np.array_equal(m["reason_hist"], w.reason_hist), m["preempt_no_victims"], m["preempt_not_helpful"], w.preempt_no_victims, w.preempt_not_helpful))
            ok &= same
            if kind == abi.ENGINE_SEQUENTIAL:
                if m["evals"] != w.evals:
                    why.append("engine %d run %d: evals %d != %d" % (kind, it, m["evals"], w.evals))
                ok &= m["evals"] == w.evals
            elif which.startswith("c4") or which == "spread":
                ok &= eng.run_stats()["engine"] == "multi-commit" and (w.placed < 100 or res.waves * 2 < w.waves)
            if which == "c5":
                ok &= eng.run_stats()["engine"].startswith("streaming")
            if which in KERNEL:
                if eng.run_stats()["kernel"] != KERNEL[which]:
                    why.append("engine %d run %d: kernel %s" % (kind, it, eng.run_stats()["kernel"]))
                ok &= eng.run_stats()["kernel"] == KERNEL[which]
        eng.close()
    q.put((rank, bool(ok), int(res.placed), why))
    dist.destroy_process_group()


KERNEL = {"ext": "wave<true>", "generic_streamed": "wave<false>"}     # the instantiation every rank must run


@pytest.mark.parametrize("which", ["c3", "c4", "c4_wide", "spread", "c5", "ext", "generic_streamed"])
def test_two_gpu_sharded_matches_oracle(built, which):
    """generic_streamed: the smallest cluster whose shards no longer fit the generic kernel's resident tile, found by bisection over
    ccsim_prepare with two connected ranks of this process (nothing is launched). Only this test reaches wave<false> over shards:
    a streamed tile needs a full grid per rank, and two full grids do not fit on one device at once."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n = 0
    if which == "generic_streamed":
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        import helpers
        import test_gpu_sharded_edges as edges
        n = helpers.largest_sharded_n(edges.generic_streamed, "wave<true>", 100_000, 2_000_000, 2, max_pods=300) + 1
        n += n % 2          # at odd N the last shard is one node shorter and may stay resident: an even N streams on both ranks
        assert helpers.sharded_kernels(*edges.generic_streamed(n), 2, max_pods=300) == ["wave<false>"] * 2
        print("\n  first sharded wave<false>: N = %d" % n, end="")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + os.getpid() % 1500
    procs = [ctx.Process(target=_worker, args=(r, 2, port, which, q, n)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(o[1] for o in out), out
