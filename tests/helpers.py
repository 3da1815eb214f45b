"""Shared test helpers: encoded-snapshot -> ctypes structs, object-level scenario generators."""
import ctypes as C
import importlib
import random
import threading

import numpy as np

abi = importlib.import_module("cluster-capacity_b200._abi")


def from_encoded(enc):
    """cc_debug_encoded_snapshot JSON -> (Snapshot, [Template], [Counter], taint_dict, scalar_names, names)."""
    nd = enc["nodes"]
    n = nd["n"]
    u64 = lambda a: np.array([int(x) for x in a], dtype=np.uint64)
    scal = [(np.array(a, np.int64), np.array(r, np.int64)) for a, r in zip(nd["alloc_scalar"], nd["req_scalar"])]
    lists = [nd["taint_list"][nd["taint_off"][i]:nd["taint_off"][i + 1]] for i in range(n)]
    snap = abi.Snapshot(n, np.array(nd["alloc_cpu"], np.int64), np.array(nd["alloc_mem"], np.int64), np.array(nd["alloc_pods"], np.int32),
                        alloc_eph=np.array(nd["alloc_eph"], np.int64), req_cpu=np.array(nd["req_cpu"], np.int64),
                        req_mem=np.array(nd["req_mem"], np.int64), req_eph=np.array(nd["req_eph"], np.int64),
                        npods=np.array(nd["npods"], np.int32), nz_cpu=np.array(nd["nz_cpu"], np.int64), nz_mem=np.array(nd["nz_mem"], np.int64),
                        scalars=scal, taint_mask=u64(nd["taint_mask"]).reshape(nd["taint_words"], n) if n else None,
                        taint_nosched=[int(x) for x in nd["taint_nosched"]], taint_prefer=[int(x) for x in nd["taint_prefer"]],
                        static_mask=u64(nd["static_mask"]).reshape(nd["static_words"], n) if nd["static_words"] else None,
                        topo=[np.array(t, np.int32) for t in nd["topo"]], has_placed_mask=nd["has_placed_mask"],
                        taint_lists=lists, names=enc["names"])
    ts = []
    for k, hx in enumerate(enc.get("templates_hex") or [enc["template_hex"]]):
        t = abi.Template()
        raw = bytes.fromhex(hx)
        assert len(raw) == C.sizeof(abi.Template)
        C.memmove(C.byref(t), raw, len(raw))
        img = np.array((enc.get("image_scores") or [enc.get("image_score") or []])[k], np.uint8)   # the hex carries a pointer of the encoding process: replace it
        t._keep_img = img
        t.image_score = img.ctypes.data_as(C.POINTER(C.c_uint8)) if len(img) else None
        ts.append(t)
    ctr = [abi.make_counter(c["topo_col"], np.array(c["init"], np.int32), n_present=c["n_present"], inc=c["inc"], elig_bit=c.get("elig_bit", -1))
           for c in enc["counters"]]
    return snap, ts, ctr, nd["taint_dict"], nd["scalar_names"], enc["names"]


# ---- which kernel runs a workload ------------------------------------------------------------------------------------
GRID_NODES, MAX_GRID = 512, 160                   # persistent grid: one CTA per SM, one per 512 nodes for small clusters
MULTI_TILE, MULTI_M, MULTI_EPT = 768, 16, 3       # multi-commit kernel: one node per thread, 16 candidates per tile, 3 per thread
MULTI_PAY_BITS, MULTI_GT, MULTI_IDX_BITS = 27, 6, 20


def run_stats(eng):
    """What the last run() of `eng` did: the kernel that ran ("engine") and its wave statistics (Engine.run_stats)."""
    return eng.run_stats()


def kernel_name(eng):
    """The wave-kernel instantiation the last prepare() / run() of `eng` chose, e.g. "lean<true>" (Engine.kernel_name)."""
    return eng.kernel_name()


def prepared_kernel(snap, tmpl, ctr, max_pods=0, **engine_kw):
    """The kernel a workload runs on, from ccsim_prepare alone: nothing is launched."""
    engine = importlib.import_module("cluster-capacity_b200.engine")
    with engine.Engine(device=0, **engine_kw) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        eng.prepare(max_pods)
        return kernel_name(eng)


def largest_n(make, kernel, lo, hi, max_pods=0, **engine_kw):
    """The largest N in [lo, hi) for which the workload make(N) = (snapshot, templates, counters) still runs on `kernel`, by
    bisection over prepare() alone. Where one kernel ends depends on sizeof of the shared-memory structs and on the device's
    opt-in limit, so the tests find it instead of restating it. Requires `kernel` at lo and another kernel (or a refusal) at hi."""
    def on(n):
        try:
            return prepared_kernel(*make(n), max_pods=max_pods, **engine_kw) == kernel
        except RuntimeError:          # EngineError: the configuration refuses the workload
            return False
    assert on(lo), (kernel, lo)
    assert not on(hi), (kernel, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if on(mid):
            lo = mid
        else:
            hi = mid
    return lo


def device_sm_count(device=0):
    engine = importlib.import_module("cluster-capacity_b200.engine")
    with engine.Engine(device=device) as eng:
        return eng.device_info()["sm_count"]


def persistent_grid(n, sm_count, world=1):
    """CTAs per rank of the persistent wave kernels: sized from the largest node shard."""
    shard = -(-n // world)
    return max(1, min(sm_count, MAX_GRID, -(-shard // GRID_NODES)))


# ---- node-sharded ranks on one device -------------------------------------------------------------------------------
def sharded_engines(snap, tmpl, ctr, world, kind, **engine_kw):
    """`world` handles of this process on device 0 (rank r = the r-th), loaded and wired to each other by pointer
    (Engine.connect_local): the same in-kernel exchange as across GPUs, only the stores do not cross NVLink."""
    engine = importlib.import_module("cluster-capacity_b200.engine")
    engs = [engine.Engine(device=0, engine=kind, rank=r, world=world, **engine_kw) for r in range(world)]
    try:
        for e in engs:
            e.load_nodes(snap)
            e.set_templates(tmpl, ctr)
        engine.Engine.connect_local(engs)
    except Exception:
        for e in engs:
            e.close()
        raise
    return engs


def run_sharded_once(engs, lim):
    """One run of every rank: all ranks past their allocations (prepare) before any rank's kernel starts waiting for its peers,
    then the runs side by side, one host thread per rank. Returns the ranks' RunResults."""
    world = len(engs)
    res, errs = [None] * world, []
    for e in engs:
        e.prepare(lim)

    def work(r):
        try:
            res[r] = engs[r].run(lim)
        except Exception as ex:       # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    assert all(r is not None for r in res), "a rank did not finish"
    return res


def run_sharded(snap, tmpl, ctr, limit, world, kind, runs):
    """The ranks of a node-sharded run as handles of this process on device 0, one run per entry of `runs` (its max_pods) on the
    same handles. Returns [(per-rank RunResults, per-rank run_stats)] per run."""
    engs = sharded_engines(snap, tmpl, ctr, world, kind)
    out = []
    for lim in runs:
        res = run_sharded_once(engs, lim)
        out.append((res, [e.run_stats() for e in engs]))
    for e in engs:
        e.close()
    return out


def sharded_kernels(snap, tmpl, ctr, world, max_pods=0, kind=0):
    """The kernel each rank of a node-sharded run would launch, from ccsim_prepare alone (ranks of this process on device 0,
    connected; nothing is launched)."""
    engs = sharded_engines(snap, tmpl, ctr, world, kind)
    try:
        for e in engs:
            e.prepare(max_pods)
        return [kernel_name(e) for e in engs]
    finally:
        for e in engs:
            e.close()


def largest_sharded_n(make, kernel, lo, hi, world, max_pods=0):
    """largest_n for a node-sharded run: the largest N in [lo, hi) for which every rank of make(N) still runs `kernel`."""
    def on(n):
        try:
            return set(sharded_kernels(*make(n), world, max_pods=max_pods)) == {kernel}
        except RuntimeError:          # EngineError: the configuration refuses the workload
            return False
    assert on(lo), (kernel, lo)
    assert not on(hi), (kernel, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if on(mid):
            lo = mid
        else:
            hi = mid
    return lo


def multi_eligible(snap, tmpl, ctr, sm_count):
    """Whether ENGINE_AUTO runs this single-GPU workload on the multi-commit kernel (ccsim_multi.cuh) instead of the lean
    sequential one. This restates the host's rule on purpose, apart from it: if the rule drifts, a test that asserts the engine
    fails. The workload must already be lean-eligible (one template, one taint word, no PreferNoSchedule taints, counters in
    shared memory)."""
    if len(tmpl) != 1 or not ctr or snap.n >= 1 << MULTI_IDX_BITS or tmpl[0].n_aff:       # no required pod affinity
        return False
    t = tmpl[0]
    grid = persistent_grid(snap.n, sm_count)
    if -(-snap.n // grid) > MULTI_TILE or grid * MULTI_M > MULTI_EPT * MULTI_TILE:
        return False
    if any(c.inc < 0 for c in ctr):                   # feasibility must be monotone within a wave
        return False
    reads = [t.pts[c].counter for c in range(t.n_pts)] if t.filter_enable & abi.PL_POD_TOPOLOGY_SPREAD else []
    reads += [t.anti_counter[a] for a in range(t.n_anti)] if t.filter_enable & abi.PL_INTER_POD_AFFINITY else []
    if sum(ctr[j].topo_col >= 0 for j in reads) > MULTI_GT:
        return False
    if any(c.topo_col >= 0 and c.inc != 0 and reads.count(j) != 1 for j, c in enumerate(ctr)):
        return False
    bits = 0                                          # payload: dom + 1 (0..max domains) per topology column + a zero guard bit
    for col in {c.topo_col for c in ctr if c.topo_col >= 0}:
        bits += max([1] + [c.n_domains for c in ctr if c.topo_col == col]).bit_length() + 1
    return bits <= MULTI_PAY_BITS


def expected_engine(snap, tmpl, ctr, sm_count):
    """The kernel ENGINE_AUTO picks for a lean-eligible, counter-coupled workload."""
    return "multi-commit" if multi_eligible(snap, tmpl, ctr, sm_count) else "lean sequential"


def sparse_eligibility_case(n, max_skew, every=40, zones=8):
    """Identical nodes of which every `every`-th matches the template's node selector: with every >= 40 a tile of up to 640 nodes has
    at most 16 feasible nodes, so no tile has unseen candidates and the replay bar comes from the best key alone; all keys share one
    score. Required anti-affinity on the hostname (a node takes one clone) and a zone spread constraint with the given maxSkew."""
    i = np.arange(n)
    static = (i % every == 0).astype(np.uint64)
    zone = ((i // every) % zones).astype(np.int32)
    snap = abi.Snapshot(n, np.full(n, 8000), np.full(n, 16 << 30), np.full(n, 110), static_mask=static.reshape(1, n), topo=[zone])
    ctr = [abi.make_counter(0, np.zeros(zones, np.int32), inc=1), abi.make_counter(-1, np.zeros(n, np.int32), inc=1)]
    t = abi.default_template(100, 128 << 20)
    t.flags |= abi.TF_HAS_NODE_SELECTOR
    t.sel_mask[0] = 1
    t.n_pts = 1
    t.pts[0].counter, t.pts[0].max_skew, t.pts[0].self_match, t.pts[0].min_zero = 0, max_skew, 1, 0
    t.n_anti, t.anti_counter[0] = 1, 1
    return snap, [t], ctr


def soft_cluster(seed, n=3000, system_default=False):
    """Normalised soft scorers on one template: ScheduleAnyway spreading over a zone column (inclusion policies) and the hostname,
    pod (anti-)affinity score weights per rack and per node, an ImageLocality column and PreferNoSchedule classes. Every wave runs
    the generic kernel's three-pass pipeline."""
    rng = np.random.default_rng(seed)
    zone = rng.integers(0, 20, n).astype(np.int32)
    zone[rng.random(n) < 0.07] = -1                        # nodes without the zone label
    rack = rng.integers(0, 200, n).astype(np.int32)
    bit = lambda a, b: a.astype(np.uint64) << np.uint64(b)
    static = bit(zone < 0, 0) | bit(rng.random(n) < 0.9, 1) | bit(rng.random(n) < 0.8, 2)
    taint = bit(rng.random(n) < 0.25, 0)
    snap = abi.Snapshot(n, rng.choice([2000, 4000, 8000], n), np.full(n, 16 << 30), rng.choice([6, 10, 14], n),
                        static_mask=static.reshape(1, n), topo=[zone, rack], taint_mask=taint.reshape(1, n), taint_prefer=[1],
                        taint_lists=[[0] if int(x) else [] for x in taint])
    ctr = [abi.make_counter(0, rng.integers(0, 40, 20), inc=1, elig_bit=2),           # soft zone constraint, inclusion policies
           abi.make_counter(-1, rng.integers(0, 3, n), inc=1),                        # soft hostname constraint
           abi.make_counter(1, rng.integers(-50, 50, 200), inc=-3),                   # pod (anti-)affinity weights per rack
           abi.make_counter(-1, rng.integers(-5, 20, n), inc=7)]                      # ... and per node
    t = abi.default_template(300, 256 << 20)
    t.n_spts = 2
    t.spts_ignored_bit = -1 if system_default else 0
    t.spts[0].counter, t.spts[0].max_skew, t.spts[0].hostname, t.spts[0].has_key_bit = 0, 5, 0, -1
    t.spts[1].counter, t.spts[1].max_skew, t.spts[1].hostname, t.spts[1].has_key_bit = 1, 3, 1, 1
    t.n_ipa_score = 2
    t.ipa_score_counter[0], t.ipa_score_counter[1] = 2, 3
    img = np.where(rng.random(n) < 0.3, rng.integers(1, 101, n), 0).astype(np.uint8)
    t._keep_img = img
    t.image_score = img.ctypes.data_as(abi.C.POINTER(abi.C.c_uint8))
    return snap, [t], ctr


def reason_text(r, taint_dict, scalar_names):
    if r < abi.R_FIXED_COUNT:
        return abi.REASON_TEXT[r]
    if r < abi.R_TAINT0:
        return "Insufficient %s" % scalar_names[r - abi.R_SCALAR0]
    t = taint_dict[r - abi.R_TAINT0]
    return "node(s) had untolerated taint {%s: %s}" % (t["key"], t["value"])


def stop_reason_from_result(res, n, max_pods, taint_dict, scalar_names, preemption_never=False):
    if res.stop_code == abi.STOP_LIMIT_REACHED:
        return "LimitReached: Maximum number of pods simulated: %d" % max_pods
    hist = {i: int(c) for i, c in enumerate(res.reason_hist) if c}
    msg = abi.fit_error_message(n, hist, res.preempt_no_victims, res.preempt_not_helpful, lambda r: reason_text(r, taint_dict, scalar_names))
    if preemption_never:
        msg = msg.split(" preemption: ")[0] + " preemption: not eligible due to preemptionPolicy=Never."
    return "Unschedulable: " + msg


# ---- object-level scenarios ------------------------------------------------------------------------------------------
def make_node(name, cpu="4", mem="8Gi", pods="20", labels=None, taints=None, unschedulable=False, extra_alloc=None):
    alloc = {"cpu": cpu, "memory": mem, "pods": pods, "ephemeral-storage": "100Gi"}
    alloc.update(extra_alloc or {})
    lab = {"kubernetes.io/hostname": name}
    lab.update(labels or {})
    n = {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": lab}, "spec": {}, "status": {"allocatable": alloc}}
    if taints:
        n["spec"]["taints"] = taints
    if unschedulable:
        n["spec"]["unschedulable"] = True
    return n


def make_pod(name, cpu=None, mem=None, node=None, labels=None, ns="default", phase="Running", **spec_extra):
    req = {}
    if cpu:
        req["cpu"] = cpu
    if mem:
        req["memory"] = mem
    p = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": ns, "labels": labels or {}},
         "spec": {"containers": [{"name": "c", "image": "img", "resources": {"requests": req}}]}, "status": {"phase": phase}}
    if node:
        p["spec"]["nodeName"] = node
    p["spec"].update(spec_extra)
    return p


def random_cluster(seed, n_nodes=40, n_pods=60, zones=3):
    rng = random.Random(seed)
    nodes, pods = [], []
    for i in range(n_nodes):
        labels = {}
        if rng.random() < 0.9:
            labels["topology.kubernetes.io/zone"] = "z%d" % rng.randrange(zones)
            labels["topology.kubernetes.io/region"] = "r%d" % rng.randrange(2)
        if rng.random() < 0.6:
            labels["disk"] = rng.choice(["ssd", "hdd"])
        if rng.random() < 0.5:
            labels["rank"] = str(rng.randrange(10))
        taints = []
        if rng.random() < 0.2:
            taints.append({"key": "dedicated", "value": rng.choice(["a", "b"]), "effect": "NoSchedule"})
        if rng.random() < 0.15:
            taints.append({"key": "flaky", "effect": "PreferNoSchedule"})
        if rng.random() < 0.1:
            taints.append({"key": "gpu", "value": "true", "effect": "NoExecute"})
        extra = {"example.com/foo": str(rng.randrange(0, 6))} if rng.random() < 0.5 else None
        nodes.append(make_node("node-%02d" % i, cpu=rng.choice(["2", "4", "8", "3500m"]), mem=rng.choice(["4Gi", "8Gi", "16Gi", "6000Mi"]),
                               pods=str(rng.choice([5, 8, 12, 110])), labels=labels, taints=taints,
                               unschedulable=rng.random() < 0.05, extra_alloc=extra))
        images = []
        if rng.random() < 0.3:
            images.append({"names": ["img:latest", "registry.local/img@sha256:0123"], "sizeBytes": rng.choice([120, 300, 700]) * 1024 * 1024})
        if rng.random() < 0.2:
            images.append({"names": ["y:latest"], "sizeBytes": 900 * 1024 * 1024})
        if images:
            nodes[-1]["status"]["images"] = images
    for j in range(n_pods):
        node = "node-%02d" % rng.randrange(n_nodes) if rng.random() < 0.92 else None
        labels = {"app": rng.choice(["web", "db", "sim"])}
        extra = {}
        if rng.random() < 0.15:
            extra["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
                {"labelSelector": {"matchLabels": {"app": rng.choice(["sim", "db"])}}, "topologyKey": rng.choice(["kubernetes.io/hostname", "topology.kubernetes.io/zone"])}]}}
        r = rng.random()
        if r < 0.08:      # scored through hardPodAffinityWeight when it matches the incoming pod
            extra.setdefault("affinity", {})["podAffinity"] = {"requiredDuringSchedulingIgnoredDuringExecution": [
                {"labelSelector": {"matchLabels": {"app": rng.choice(["sim", "web"])}}, "topologyKey": "topology.kubernetes.io/zone"}]}
        elif r < 0.16:
            extra.setdefault("affinity", {})["podAffinity"] = {"preferredDuringSchedulingIgnoredDuringExecution": [
                {"weight": rng.choice([10, 35]), "podAffinityTerm": {"labelSelector": {"matchExpressions": [{"key": "app", "operator": "In", "values": ["sim", "web"]}]},
                                                                    "topologyKey": rng.choice(["topology.kubernetes.io/zone", "disk"])}}]}
        elif r < 0.24:
            aa = extra.setdefault("affinity", {}).setdefault("podAntiAffinity", {})
            aa["preferredDuringSchedulingIgnoredDuringExecution"] = [
                {"weight": rng.choice([5, 60]), "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": "kubernetes.io/hostname"}}]
        p = make_pod("pod-%03d" % j, cpu=rng.choice([None, "100m", "250m", "1"]), mem=rng.choice([None, "64Mi", "256Mi", "1Gi"]),
                     node=node, labels=labels, phase=rng.choice(["Running"] * 8 + ["Succeeded", "Pending"]), **extra)
        if rng.random() < 0.2:
            p["spec"]["containers"][0]["ports"] = [{"containerPort": 80, "hostPort": rng.choice([8080, 9090]), "protocol": "TCP"}]
        if rng.random() < 0.15:
            p["spec"]["initContainers"] = [{"name": "init", "image": "img", "resources": {"requests": {"cpu": "500m", "memory": "32Mi"}}}]
        if rng.random() < 0.1:
            p["spec"]["overhead"] = {"cpu": "10m", "memory": "8Mi"}
        if rng.random() < 0.3:
            p["spec"]["containers"][0]["resources"]["requests"]["example.com/foo"] = "1"
        pods.append(p)
    return nodes, pods


TEMPLATE_VARIANTS = ["plain", "selector", "tolerations", "affinity_terms", "hostports", "spread_zone", "spread_two", "anti_hostname",
                     "anti_zone", "affinity_zone", "extended", "best_effort", "init_overhead", "never_preempt", "gt_lt", "name_in", "pref_affinity", "pref_and_required",
                     "soft_spread", "soft_and_hard", "pref_pod_affinity", "svc_default_spread", "owner_default_spread", "spread_everything"]


def workloads_for(variant):
    """Services / controllers synced next to the nodes and pods (only the *_default_spread variants need them)."""
    svc = lambda name, sel, ns="default": {"apiVersion": "v1", "kind": "Service", "metadata": {"name": name, "namespace": ns}, "spec": {"selector": sel}}
    if variant == "svc_default_spread":
        return {"services": [svc("sim", {"app": "sim"}), svc("other-ns", {"app": "sim", "x": "y"}, ns="kube-system"), svc("web", {"app": "web"}),
                             {"apiVersion": "v1", "kind": "Service", "metadata": {"name": "headless", "namespace": "default"}, "spec": {}}]}
    if variant == "owner_default_spread":
        return {"services": [svc("web", {"app": "web"})],
                "replica_sets": [{"apiVersion": "apps/v1", "kind": "ReplicaSet", "metadata": {"name": "sim-rs", "namespace": "default"},
                                  "spec": {"selector": {"matchExpressions": [{"key": "app", "operator": "In", "values": ["sim", "db"]}]}}}]}
    return {}


def list_client(fw, nodes, pods, variant=None, namespaces=()):
    return fw.ListClient(nodes, pods, namespaces, **workloads_for(variant))


def objref_sync(sim, nodes, pods, variant=None, namespaces=()):
    w = workloads_for(variant)
    sim.sync(nodes, pods, namespaces, services=w.get("services", ()), rcs=w.get("replication_controllers", ()),
             replicasets=w.get("replica_sets", ()), statefulsets=w.get("stateful_sets", ()))


def template(variant, seed=0):
    del seed   # variants are deterministic; the parameter keeps the call sites symmetrical with random_cluster
    p = make_pod("small-pod", cpu="150m", mem="100Mi", labels={"app": "sim"})
    s = p["spec"]
    if variant == "selector":
        s["nodeSelector"] = {"disk": "ssd"}
    elif variant == "tolerations":
        s["tolerations"] = [{"key": "dedicated", "operator": "Equal", "value": "a", "effect": "NoSchedule"}, {"key": "gpu", "operator": "Exists"},
                            {"key": "flaky", "operator": "Exists", "effect": "PreferNoSchedule"}]
    elif variant == "affinity_terms":
        s["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
            {"matchExpressions": [{"key": "disk", "operator": "In", "values": ["ssd"]}, {"key": "rank", "operator": "Exists"}]},
            {"matchExpressions": [{"key": "topology.kubernetes.io/zone", "operator": "NotIn", "values": ["z0"]}, {"key": "disk", "operator": "DoesNotExist"}]}]}}}
    elif variant == "gt_lt":
        s["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
            {"matchExpressions": [{"key": "rank", "operator": "Gt", "values": ["3"]}, {"key": "rank", "operator": "Lt", "values": ["8"]}]}]}}}
    elif variant == "name_in":
        s["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
            {"matchFields": [{"key": "metadata.name", "operator": "In", "values": ["node-03"]}]},
            {"matchFields": [{"key": "metadata.name", "operator": "In", "values": ["node-07"]}]}]}}}
    elif variant == "pref_affinity":
        s["affinity"] = {"nodeAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
            {"weight": 50, "preference": {"matchExpressions": [{"key": "disk", "operator": "In", "values": ["ssd"]}]}},
            {"weight": 20, "preference": {"matchExpressions": [{"key": "topology.kubernetes.io/zone", "operator": "In", "values": ["z1", "z2"]}]}},
            {"weight": 0, "preference": {"matchExpressions": [{"key": "rank", "operator": "Exists"}]}},
            {"weight": 7, "preference": {"matchExpressions": [{"key": "rank", "operator": "Gt", "values": ["4"]}]}}]}}
        s["tolerations"] = [{"key": "dedicated", "operator": "Exists"}]
    elif variant == "pref_and_required":
        s["affinity"] = {"nodeAffinity": {
            "requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [{"matchExpressions": [{"key": "disk", "operator": "Exists"}]}]},
            "preferredDuringSchedulingIgnoredDuringExecution": [
                {"weight": 100, "preference": {"matchExpressions": [{"key": "disk", "operator": "In", "values": ["hdd"]}]}},
                {"weight": 1, "preference": {"matchFields": [{"key": "metadata.name", "operator": "In", "values": ["node-05"]}]}}]}}
    elif variant == "soft_spread":
        s["topologySpreadConstraints"] = [
            {"maxSkew": 2, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "ScheduleAnyway", "labelSelector": {"matchLabels": {"app": "sim"}}},
            {"maxSkew": 1, "topologyKey": "kubernetes.io/hostname", "whenUnsatisfiable": "ScheduleAnyway",
             "labelSelector": {"matchExpressions": [{"key": "app", "operator": "In", "values": ["sim", "web"]}]}}]
    elif variant == "soft_and_hard":
        s["topologySpreadConstraints"] = [
            {"maxSkew": 3, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule", "labelSelector": {"matchLabels": {"app": "sim"}}},
            {"maxSkew": 1, "topologyKey": "topology.kubernetes.io/region", "whenUnsatisfiable": "ScheduleAnyway", "labelSelector": {"matchLabels": {"app": "sim"}},
             "nodeTaintsPolicy": "Honor"},
            {"maxSkew": 4, "topologyKey": "disk", "whenUnsatisfiable": "ScheduleAnyway", "labelSelector": {"matchLabels": {"app": "db"}}, "nodeAffinityPolicy": "Ignore"}]
    elif variant == "pref_pod_affinity":
        s["affinity"] = {"podAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
            {"weight": 40, "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "db"}}, "topologyKey": "topology.kubernetes.io/zone"}},
            {"weight": 15, "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": "disk"}}]},
            "podAntiAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
                {"weight": 25, "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": "kubernetes.io/hostname"}}]}}
    elif variant == "owner_default_spread":
        p["metadata"]["ownerReferences"] = [{"apiVersion": "apps/v1", "kind": "ReplicaSet", "name": "sim-rs", "controller": True, "uid": "u"}]
    elif variant == "hostports":
        s["containers"][0]["ports"] = [{"containerPort": 80, "hostPort": 8080}]
    elif variant == "spread_zone":
        s["topologySpreadConstraints"] = [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                                           "labelSelector": {"matchLabels": {"app": "sim"}}}]
    elif variant == "spread_everything":
        # labelSelector {} = Everything: self-matches (filtering.go:341-344) but countPodsMatchSelector returns 0 for an empty
        # selector (common.go:144-147), so the counts never move and the constraint never blocks (skew = 1 - 0)
        s["topologySpreadConstraints"] = [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                                           "labelSelector": {}}]
    elif variant == "spread_two":
        s["topologySpreadConstraints"] = [
            {"maxSkew": 2, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule", "labelSelector": {"matchLabels": {"app": "sim"}}},
            {"maxSkew": 1, "topologyKey": "kubernetes.io/hostname", "whenUnsatisfiable": "DoNotSchedule", "labelSelector": {"matchLabels": {"app": "web"}},
             "minDomains": 2}]
        s["nodeSelector"] = {"disk": "ssd"}
    elif variant == "anti_hostname":
        s["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
            {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": "kubernetes.io/hostname"}]}}
    elif variant == "anti_zone":
        s["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
            {"labelSelector": {"matchExpressions": [{"key": "app", "operator": "In", "values": ["db"]}]}, "topologyKey": "topology.kubernetes.io/zone"}]}}
    elif variant == "affinity_zone":
        s["affinity"] = {"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
            {"labelSelector": {"matchLabels": {"app": "sim"}}, "topologyKey": "topology.kubernetes.io/zone"}]}}
    elif variant == "extended":
        s["containers"][0]["resources"]["requests"]["example.com/foo"] = "2"
        s["containers"][0]["resources"]["requests"]["ephemeral-storage"] = "30Gi"
    elif variant == "best_effort":
        s["containers"][0]["resources"] = {}
    elif variant == "init_overhead":
        s["initContainers"] = [{"name": "i", "image": "x", "resources": {"requests": {"cpu": "1", "memory": "50Mi"}}},
                               {"name": "side", "image": "x", "restartPolicy": "Always", "resources": {"requests": {"cpu": "50m"}}}]
        s["overhead"] = {"cpu": "25m", "memory": "10Mi"}
        s["containers"].append({"name": "c2", "image": "y", "resources": {}})
    elif variant == "never_preempt":
        s["preemptionPolicy"] = "Never"
    return p
