"""Quick device-time probe of the wave kernel on the BASELINE configs (not the bench contract; see bench.py)."""
import hashlib, importlib, sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
engine = importlib.import_module("cluster-capacity_b200.engine")

def probe(name, snap, tmpl, ctr, limit, bytes_per_eval, engine_kind=abi.ENGINE_AUTO):
    with engine.Engine(device=0, engine=engine_kind) as eng:
        t0 = time.time(); eng.load_nodes(snap); eng.set_templates(tmpl, ctr); t1 = time.time()
        r = eng.run(limit)
        r = eng.run(limit)
        info = eng.device_info()
        st = eng.run_stats()
    us = r.run_ms * 1e3 / max(1, r.waves)
    print("%-28s n=%-8d grid=%-4d placed=%-8d waves=%-8d run=%9.3f ms  %6.2f us/wave  %.3g evals/s  %.0f GB/s algorithmic  (load %.1f ms)" % (
        name, snap.n, info["grid"], r.placed, r.waves, r.run_ms, us, r.evals / (r.run_ms * 1e-3),
        r.evals * bytes_per_eval / (r.run_ms * 1e-3) / 1e9, (t1 - t0) * 1e3), end="")
    print("  %s  pod->node sha1 %s" % (st["kernel"], hashlib.sha1(r.pod_node.tobytes()).hexdigest()[:16]), flush=True)
    if st["engine"] == "multi-commit":
        w = max(1, st["waves"])
        print("    engine=%s  placements/wave=%.2f  candidates/wave=%.1f  bar raised in %d waves  cycles/wave (CTA 0): scan=%d S1=%d merge+publish=%d gather=%d replay=%d tail=%d  smem=%d B" % (
            st["engine"], st["placed"] / w, st["candidates"] / w, st["bar_raised_waves"], *[c // w for c in st["phase_cycles"][:6]], st["smem_bytes"]), flush=True)
        print("    replay detail: setup=%d cycles/wave  waves ended by a binding minimum move: %d of %d  (rounds: CCSIM_DEBUG_FLAGS=8)" % (st["phase_cycles"][6] // w, st["phase_cycles"][7], w), flush=True)

if __name__ == "__main__":
    which = sys.argv[1:] or ["c2", "c3", "c4", "c5"]
    if "c2" in which: probe("C2 10k fit-only", *synth.c2(), 20000, 72)
    if "c2big" in which: probe("C2 100k fit-only", *synth.c2(n=100_000), 20000, 72)
    if "c3" in which: probe("C3 50k full filters", *synth.c3(), 20000, 88)
    if "c4" in which: probe("C4 100k PTS+IPA", *synth.c4(), 0, 96)
    if "c4spread" in which:      # spread constraints only (no hostname anti-affinity): nodes take several clones, winners can come back
        snap, tmpl, ctr = synth.c4()
        tmpl[0].n_anti = 0
        probe("C4 spread-only", snap, tmpl, ctr[:3], 20000, 92)
        probe("C4 spread-only, sequential", snap, tmpl, ctr[:3], 20000, 92, abi.ENGINE_SEQUENTIAL)
    if "c5" in which: probe("C5 1M x 64 templates", *synth.c5(), 6400, 72)
    if "sharded" in which:       # multi<true>: C4-small over node shards, the ranks as handles of this process on device 0 connected
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        import helpers           # by pointer (tests/helpers.py); a run lasts as long as its slowest rank
        snap, tmpl, ctr = synth.c4(n=30000, n_existing=60000, zones=32, racks=256, regions=8)
        for world in (2, 4):
            engs = helpers.sharded_engines(snap, tmpl, ctr, world, abi.ENGINE_AUTO)
            try:
                for _ in range(2):
                    helpers.run_sharded_once(engs, 0)
                ms = []
                for _ in range(5):
                    res = helpers.run_sharded_once(engs, 0)
                    ms.append(max(r.run_ms for r in res))
                st = engs[0].run_stats()
            finally:
                for e in engs:
                    e.close()
            w = max(1, st["waves"])
            print("%-28s world=%d %s placed=%d waves=%d candidates/wave=%.1f bar raised in %d waves  run %.3f-%.3f ms (5 runs)  pod->node sha1 %s" % (
                "C4-small node shards", world, st["kernel"], st["placed"], st["waves"], st["candidates"] / w, st["bar_raised_waves"], min(ms), max(ms),
                hashlib.sha1(res[0].pod_node.tobytes()).hexdigest()[:16]), flush=True)
    if "generic" in which:       # the generic wave kernel, which bench.py never reaches: normalised soft scorers and eight
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        import helpers           # PreferNoSchedule classes with an extended-resource request, resident and one node past the tile
        def classes(n):
            rng = np.random.Generator(np.random.PCG64(81))
            a_cpu, a_mem, a_pods, r_cpu, r_mem, npods = synth._c2_nodes(n, rng)
            taint = (np.uint64(1) << rng.integers(0, 8, n).astype(np.uint64)) - np.uint64(1)
            snap = abi.Snapshot(n, a_cpu, a_mem, a_pods, req_cpu=r_cpu, req_mem=r_mem, npods=npods, taint_mask=taint.reshape(1, n),
                                taint_prefer=[0x7F], scalars=[(rng.integers(0, 40, n), rng.integers(0, 4, n))])
            t = abi.default_template(150, 100 << 20)
            t.req_scalar[0] = 1
            return snap, [t], []
        probe("generic soft 100k", *helpers.soft_cluster(89, n=100_000), 3000, 0)
        probe("generic 8 classes 100k", *classes(100_000), 5000, 0)
        n = helpers.largest_n(classes, "wave<true>", 100_000, 1_000_000, max_pods=5000) + 1
        probe("generic past the tile", *classes(n), 5000, 0)
