"""GPU: per-analysis runs (ccsim_run_each / cc_run_each / `cluster-capacity --each`). Every analysis t is checked against ccsim_run of
template t alone on the same snapshot, the C oracle with [template t] and, for object-level cases, objref.Simulator([podspec t]):
placement by placement, stop code, FitError histogram, preemption counters and ccsim_node_counts."""
import ctypes as C
import importlib
import io
import json
import os
from contextlib import redirect_stdout

import numpy as np
import pytest

import helpers
from oracle import binding as oracle
from oracle import objref
from test_each import mask
from test_pod_list import LISTS, cluster, templates

abi = importlib.import_module("cluster-capacity_b200._abi")
engine = importlib.import_module("cluster-capacity_b200.engine")
fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")
genpod = importlib.import_module("cluster-capacity_b200.genpod")

pytestmark = pytest.mark.gpu
MiB, GiB = 1 << 20, 1 << 30


def same(got, want, what):
    assert got.placed == want.placed and got.stop_code == want.stop_code, (what, got.placed, want.placed, got.stop_code, want.stop_code)
    assert np.array_equal(got.pod_node, want.pod_node), what
    assert np.array_equal(got.reason_hist, want.reason_hist), what
    assert (got.preempt_no_victims, got.preempt_not_helpful) == (want.preempt_no_victims, want.preempt_not_helpful), what


def run_each(snap, tmpl, limit, eng=None):
    """(results, run_stats, node counts) of one ccsim_run_each"""
    own = eng is None
    eng = eng or engine.Engine(device=0)
    try:
        if own:
            eng.load_nodes(snap)
            eng.set_templates(tmpl)
        got = eng.run_each(limit)
        assert eng.kernel_name() == "each" and eng.run_stats()["engine"] == "per-analysis max-tree"
        return got, eng.run_stats(), [eng.node_counts(t) for t in range(len(tmpl))]
    finally:
        if own:
            eng.close()


def check(snap, tmpl, limit, with_oracle=True):
    """every analysis against ccsim_run of its template alone and the C oracle; returns the per-analysis results"""
    got, st, counts = run_each(snap, tmpl, limit)
    assert st["grid"] == len(tmpl) and st["placed"] == sum(g.placed for g in got)
    for t, g in enumerate(got):
        with engine.Engine(device=0) as one:
            one.load_nodes(snap)
            one.set_templates([tmpl[t]])
            want = one.run(limit)
            wc, wf = one.node_counts(0)
        same(g, want, "analysis %d vs ccsim_run" % t)
        assert np.array_equal(counts[t][0], wc) and np.array_equal(counts[t][1], wf), t
        if with_oracle:
            same(g, oracle.run(snap, [tmpl[t]], max_pods=limit), "analysis %d vs oracle" % t)
    return got, st


def check_analyses_path(snap, tmpl, limit, got, st):
    """the same templates loaded through ccsim_set_analyses with empty terms: every result, the node counts and the tree's shape
    and shared memory equal the ccsim_set_templates run's"""
    _, _, counts = run_each(snap, tmpl, limit)
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_analyses(tmpl, [([], [])] * len(tmpl))
        again, ast, acounts = run_each(snap, tmpl, limit, eng)
    for t in range(len(tmpl)):
        same(again[t], got[t], "analysis %d through ccsim_set_analyses" % t)
        assert np.array_equal(acounts[t][0], counts[t][0]) and np.array_equal(acounts[t][1], counts[t][1]), t
    assert [ast[k] for k in ("global_levels", "shared_levels", "smem_bytes")] == [st[k] for k in ("global_levels", "shared_levels", "smem_bytes")]


def nodes_c2(n, seed=1, **over):
    rng = np.random.Generator(np.random.PCG64(seed))
    cores = rng.choice([4, 8, 16, 32], size=n)
    a_cpu = cores.astype(np.int64) * 1000
    a_mem = cores.astype(np.int64) * rng.choice([2, 4, 8], size=n) * GiB
    d = dict(alloc_cpu=a_cpu, alloc_mem=a_mem, alloc_pods=np.full(n, 30, np.int32),
             req_cpu=(rng.random(n) * 0.7 * a_cpu / 10).astype(np.int64) * 10, req_mem=(rng.random(n) * 0.7 * a_mem / MiB).astype(np.int64) * MiB,
             npods=rng.integers(0, 20, size=n).astype(np.int32))
    d.update(over)
    return abi.Snapshot(n, d.pop("alloc_cpu"), d.pop("alloc_mem"), d.pop("alloc_pods"), **d)


def request_templates(k, seed=7):
    rng = np.random.Generator(np.random.PCG64(seed))
    return [abi.default_template(int(rng.integers(200, 3001)), int(rng.integers(128, 4097)) * MiB, fit_only=bool(q % 2)) for q in range(k)]


# ---- object level: the podspec lists of test_pod_list, one that fits nowhere, every path -----------------------------------------
@pytest.mark.parametrize("key", sorted(LISTS))
@pytest.mark.parametrize("limit", [0, 1, 23])
def test_each_lists_match_single_runs_and_oracles(built, key, limit):
    nodes, pods = cluster(41, 40, 60)
    tm = templates(key)
    huge = helpers.template("plain")
    huge["metadata"]["name"] = "fits-nowhere"
    huge["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "100", "memory": "1Gi"}}
    tm.insert(1, huge)
    cc = fw.New(None, None, tm, limit, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    res = cc.RunEach()
    assert len(res) == len(tm)
    for t, r in enumerate(res):
        ref = objref.Simulator([tm[t]], limit)
        ref.sync(nodes, pods)
        ref.run()
        assert r.ScheduledPods() == ref.pods_status and r.StopReason() == ref.stop_reason, (key, t)
        one = fw.New(None, None, tm[t], limit, [])
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        one.Run()
        assert r.StopReason() == one.StopReason() and r.ScheduledPods() == one.ScheduledPods()
        assert mask(json.dumps(r.Report())) == mask(json.dumps(one.Report()))
        assert r.Print(True, "") == one.Print(True, "")
        one.Close()
    assert res[1].ScheduledPods() == [] and "Insufficient cpu" in res[1].StopReason()
    # the same analyses at the engine on the merged snapshot (static bits of all podspecs side by side)
    snap, T, ctr, _, _, _ = helpers.from_encoded(cc.EncodedSnapshot())
    assert not ctr
    check(snap, T, limit)
    cc.Close()


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("limit", [0, 1, 23])
def test_each_random_clusters(built, seed, limit):
    nodes, pods = cluster(seed, 60, 90)
    tm = templates("selectors") + templates("extended")
    cc = fw.New(None, None, tm, limit, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    snap, T, _, _, _, _ = helpers.from_encoded(cc.EncodedSnapshot())
    check(snap, T, limit)
    cc.Close()


def test_each_without_node_resources_fit_needs_a_limit(built):
    snap = nodes_c2(500)
    tm = request_templates(3)
    tm[1].filter_enable &= ~abi.PL_FIT
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tm)
        with pytest.raises(engine.EngineError, match="template 1: NodeResourcesFit is disabled: the run is unbounded, --max-limit is required"):
            eng.run_each(0)
    got, _ = check(snap, tm, 23)
    assert got[1].placed == 23


# ---- ties, classes, tree edges ---------------------------------------------------------------------------------------------
def test_each_ties_first_node_wins_and_identical_podspecs_agree(built):
    n = 100
    snap = abi.Snapshot(n, np.full(n, 8000), np.full(n, 16 * GiB), np.full(n, 4))
    t = abi.default_template(1000, 1 * GiB)
    got, _ = check(snap, [t, abi.default_template(1000, 1 * GiB), abi.default_template(500, 0)], 0)
    assert got[0].pod_node[0] == 0 and got[0].placed == 4 * n
    same(got[0], got[1], "identical podspecs")
    assert list(got[0].pod_node[:n]) == list(range(n))        # every node drops after its clone: the next in order ties and wins


@pytest.mark.parametrize("taint_words", [1, 2])
def test_each_prefer_no_schedule_classes(built, taint_words):
    """nodes with 0..7 untolerated PreferNoSchedule taints (classes up to the eighth), the top classes fill mid-run so TaintToleration's
    normalisation shifts; with two taint words the taints sit in the second word"""
    n = 700
    rng = np.random.Generator(np.random.PCG64(3))
    cls = np.arange(n) % 8
    bits = np.zeros(n, np.uint64)
    for c in range(1, 8):
        bits |= np.where(cls >= c, np.uint64(1) << np.uint64(c), np.uint64(0)).astype(np.uint64)
    tm = np.zeros((taint_words, n), np.uint64)
    tm[taint_words - 1] = bits
    prefer = [0] * taint_words
    prefer[-1] = 0xFE
    pods = np.where(cls >= 6, 2, 9).astype(np.int32)
    snap = abi.Snapshot(n, rng.choice([4000, 8000], size=n), np.full(n, 32 * GiB), pods, taint_mask=tm, taint_prefer=prefer,
                        taint_lists=[[64 * (taint_words - 1) + c for c in range(1, 8) if (int(bits[i]) >> c) & 1] for i in range(n)])
    plain = abi.default_template(300, 256 * MiB)
    tol = abi.default_template(300, 256 * MiB)
    tol.tol_prefer[taint_words - 1] = 0b110                      # tolerates two of the seven
    noscore = abi.default_template(700, 256 * MiB)
    noscore.score_enable &= ~abi.PL_TAINT_TOLERATION
    got, st = check(snap, [plain, tol, noscore], 0)
    assert all(g.stop_code == abi.STOP_UNSCHEDULABLE for g in got)
    check_analyses_path(snap, [plain, tol, noscore], 0, got, st)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 32769])
def test_each_tree_edges(built, n):
    snap = nodes_c2(n, seed=n)
    if n > 2:      # one node that wins hundreds of times, and over-committed nodes (allocatable < requested)
        b = n // 2
        snap.alloc_cpu[b], snap.alloc_mem[b], snap.alloc_pods[b] = 40_000_000, 40 << 40, 700
        snap.req_cpu[b] = snap.req_mem[b] = snap.nz_cpu[b] = snap.nz_mem[b] = snap.npods[b] = 0
        snap.req_cpu[3::7] = snap.alloc_cpu[3::7] + 1000          # (b is never one of them)
        snap.nz_cpu[3::7] = snap.req_cpu[3::7]
    tm = request_templates(3, seed=n)
    limit = 0 if n <= 1025 else 1500
    got, st = check(snap, tm, limit)
    assert st["global_levels"] + st["shared_levels"] == (0 if n == 1 else int(np.ceil(np.log(n) / np.log(32) - 1e-12)))
    check_analyses_path(snap, tm, limit, got, st)
    if n > 2:
        assert max(np.bincount(g.pod_node, minlength=n)[n // 2] for g in got) >= 100


def test_each_past_the_shared_memory_level_split(built):
    """the largest cluster whose upper tree levels all fit in shared memory, found by bisection, and the next one up: level 1 moves
    to global memory, and the analyses stay exact"""
    tm = request_templates(2, seed=5)

    def make(n):
        return nodes_c2(n, seed=9)

    def stats(n):
        return run_each(make(n), tm, 1)[1]

    lo, hi = 200_000, 1_400_000
    assert stats(lo)["global_levels"] == 0 and stats(hi)["global_levels"] == 1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if stats(mid)["global_levels"] == 0:
            lo = mid
        else:
            hi = mid
    below, above = stats(lo), stats(hi)
    assert below["global_levels"] == 0 and below["shared_levels"] == 4
    assert above["global_levels"] == 1 and above["shared_levels"] == 3 and above["smem_bytes"] < below["smem_bytes"]
    check(make(hi), tm, 40)


# ---- the uncommon predicates, each podspec on its own words of the merged bits ---------------------------------------------------
def test_each_extras(built):
    n = 600
    rng = np.random.Generator(np.random.PCG64(11))
    static = rng.integers(0, 1 << 62, size=(2, n), dtype=np.int64).astype(np.uint64)
    foo = rng.integers(0, 5, size=n).astype(np.int64)
    snap = nodes_c2(n, seed=11, alloc_eph=np.full(n, 100 * GiB), req_eph=rng.integers(0, 90, size=n).astype(np.int64) * GiB,
                    scalars=[(foo, np.zeros(n, np.int64))], static_mask=static)
    sel = abi.default_template(300, 256 * MiB)
    sel.flags |= abi.TF_HAS_NODE_SELECTOR
    sel.sel_mask[1] = 0b1011                                     # nodeSelector bits in the second static word
    terms = abi.default_template(300, 256 * MiB)
    terms.flags |= abi.TF_HAS_AFFINITY_TERMS
    terms.n_aff_terms = 2
    terms.aff_term_mask[0][0] = 0b11
    terms.aff_term_mask[1][1] = 0b110000
    name = abi.default_template(100, 0)
    name.nodename_idx = 17
    res = abi.default_template(200, 128 * MiB, eph=7 * GiB)
    res.req_scalar[0] = 2
    img = abi.default_template(250, 64 * MiB)
    col = rng.integers(0, 101, size=n).astype(np.uint8)
    img._keep_img = col
    img.image_score = col.ctypes.data_as(C.POINTER(C.c_uint8))
    got, _ = check(snap, [sel, terms, name, res, img], 0)
    assert set(got[2].pod_node.tolist()) == {17}
    check(snap, [sel, terms, name, res, img], 23)


# ---- handle reuse ----------------------------------------------------------------------------------------------------------------
def test_each_handle_reuse(built):
    snap = nodes_c2(3000, seed=21)
    tm = request_templates(4, seed=21)
    fresh, _, fresh_counts = run_each(snap, tm, 300)
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tm)
        for _ in range(2):
            got, _, counts = run_each(snap, tm, 300, eng)
            for t in range(len(tm)):
                same(got[t], fresh[t], "repeat")
                assert np.array_equal(counts[t][0], fresh_counts[t][0])
        single = eng.run(300)
        assert eng.kernel_name() != "each"
        with engine.Engine(device=0) as other:
            other.load_nodes(snap)
            other.set_templates(tm)
            same(single, other.run(300), "ccsim_run after ccsim_run_each")
            assert np.array_equal(eng.node_counts(2)[0], other.node_counts(2)[0])
        got, _, _ = run_each(snap, tm, 300, eng)
        for t in range(len(tm)):
            same(got[t], fresh[t], "after ccsim_run")


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def _refused(snap, tmpl, ctr, limit, match, **kw):
    with engine.Engine(device=0, **kw) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        launches = eng.kernel_launches()
        with pytest.raises(engine.EngineError, match=match):
            eng.run_each(limit)
        assert eng.kernel_launches() == launches


def test_each_refusals(built):
    synth = importlib.import_module("cluster-capacity_b200.synth")
    snap, t4, c4 = synth.c4(n=2000, n_existing=4000, zones=8, racks=32, regions=4)
    _refused(snap, t4, c4, 10, r"per-domain counters \(topology spread, pod \(anti-\)affinity\) are not supported")
    snap = nodes_c2(200)
    soft = request_templates(2)
    soft = soft[1:] + soft[:1]           # the template with every scorer enabled second
    soft[1].n_pref_terms = 1
    soft[1].pref_weight[0] = 5
    _refused(snap, soft, (), 10, "template 1 has a normalised soft scorer")
    _refused(nodes_c2(200, has_placed_mask=True), request_templates(2), (), 10, r"hostPorts \(placed mask\)")
    _refused(snap, request_templates(2), (), 10, r"node-sharded runs \(world 2\)", rank=0, world=2)
    _refused(snap, request_templates(2), (), 10, "reference sampling", sampling=abi.SAMPLING_REFERENCE)
    off = request_templates(2)
    off[0].filter_enable &= ~abi.PL_FIT
    _refused(snap, off, (), 10 ** 13, r"sequence buffers \(2 x 10000000000000 x 4 B = [0-9.]+ GiB\) exceed free device memory")


# ---- the command line: genpod over 64 namespaces -------------------------------------------------------------------------------
def test_genpod_cli_each_64_namespaces(built, tmp_path):
    import yaml
    nodes = [helpers.make_node("n%03d" % i, cpu=str(2 + 2 * (i % 5)), mem="%dGi" % (4 + 4 * (i % 3)), pods="30",
                               labels={"pool": "a" if i % 3 else "b"}) for i in range(24)]
    nss, lrs = [], []
    for k in range(64):
        ann = {"openshift.io/node-selector": "pool=a"} if k % 7 == 0 else {}
        nss.append({"apiVersion": "v1", "kind": "Namespace", "metadata": {"name": "team%02d" % k, "annotations": ann}})
        lrs.append({"apiVersion": "v1", "kind": "LimitRange", "metadata": {"name": "lr", "namespace": "team%02d" % k},
                    "spec": {"limits": [{"type": "Pod", "max": {"cpu": "%dm" % (300 + 37 * k), "memory": "%dMi" % (256 + 29 * k)}},
                                        {"type": "Pod", "max": {"cpu": "4", "memory": "8Gi"}}]}})
    snap = tmp_path / "cluster.json"
    snap.write_text(json.dumps({"nodes": nodes, "pods": [], "namespaces": nss, "limitranges": lrs}))
    specs = tmp_path / "specs"
    assert genpod.main(["--namespace", ",".join(n["metadata"]["name"] for n in nss), "--snapshot", str(snap), "--output-dir", str(specs)]) == 0
    files = sorted(os.listdir(specs))
    assert len(files) == 64

    def run(args):
        buf = io.StringIO()
        with redirect_stdout(buf):
            assert cli.main(args + ["--snapshot", str(snap), "--max-limit", "200", "--verbose"]) == 0
        head, body = buf.getvalue().split("\n", 1)
        assert head.startswith("Cluster capacity version")
        return body

    for fmt in ("", "json", "yaml"):
        o = ["-o", fmt] if fmt else []
        singles = [run(["--podspec", str(specs / f)] + o) for f in files]
        got = run(["--podspec", str(specs), "--each"] + o)
        if fmt == "json":
            reviews = json.loads(mask(got))
            assert reviews == [json.loads(mask(s)) for s in singles]
        elif fmt == "yaml":
            assert mask(got) == mask("---\n".join(singles))
        else:
            assert got == "".join(singles)
    for t, f in enumerate(files):
        ref = objref.Simulator([cli.parse_api_spec(str(specs / f))], 200)
        ref.sync(nodes, [], nss)
        ref.run()
        assert reviews[t]["status"]["replicas"] == len(ref.pods_status), f
        assert reviews[t]["status"]["failReason"]["failType"] == ref.stop_reason.split(":")[0]
    assert yaml.safe_load((specs / files[0]).read_text())["spec"]["nodeSelector"] == {"pool": "a"}
