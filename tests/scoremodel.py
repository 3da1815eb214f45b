"""A plain model of the default profile's score plugins, in Go semantics, and of the schedule-one-pod loop for the workloads the
score ladders use (tests/test_score_edges.py). It restates the reference's formulas on its own: no code is shared with the C
oracle or the CUDA kernels, only the flat snapshot / template structs are read.

Go semantics: int64 division truncates toward zero; float64 operations round once each, in the reference's order; int64(x) of a
float truncates. Python ints are exact and Python floats are IEEE float64, so both are restated directly.

exact=True swaps BalancedAllocation for rational arithmetic and the InterPodAffinity normalisation for integer arithmetic. Those
are not what the reference computes: a test runs them only to prove that its inputs sit where the rounding decides the result.
"""
import importlib
from fractions import Fraction

import numpy as np

from oracle.objref import go_log

abi = importlib.import_module("cluster-capacity_b200._abi")

MAX_NODE_SCORE = 100


def go_div(a, b):
    """Go's int64 a / b: truncates toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


# ---- node-local scorers ------------------------------------------------------------------------------------------------
def least_requested(requested, capacity):
    """leastRequestedScore (least_allocated.go:52-61)."""
    if capacity == 0 or requested > capacity:
        return 0
    return go_div((capacity - requested) * MAX_NODE_SCORE, capacity)


def least_allocated(alloc, requested, weights=(1, 1)):
    """leastResourceScorer (least_allocated.go:30-48) over (cpu, memory): requested = NonZeroRequested + the pod's request."""
    score = wsum = 0
    for a, q, w in zip(alloc, requested, weights):
        if a == 0:
            continue
        score += least_requested(q, a) * w
        wsum += w
    return go_div(score, wsum) if wsum else 0


def balanced(alloc, requested, exact=False):
    """balancedResourceScorer (balanced_allocation.go:146-180) over (cpu, memory): requested = Requested + the pod's request."""
    one = Fraction(1) if exact else 1.0
    fr = []
    for a, q in zip(alloc, requested):
        if a == 0:
            continue
        f = Fraction(q, a) if exact else float(q) / float(a)
        fr.append(one if f > 1 else f)
    std = abs((fr[0] - fr[1]) / 2) if len(fr) == 2 else 0 * one
    return int((one - std) * MAX_NODE_SCORE)


# ---- normalisations over the feasible set (numpy arrays of raw scores) ----------------------------------------------------
def taint_norm(raw):
    """TaintToleration NormalizeScore: DefaultNormalizeScore(100, reverse=true) (helper/normalize_score.go:28-56)."""
    mx = int(raw.max()) if len(raw) else 0
    if mx == 0:
        return np.full(len(raw), MAX_NODE_SCORE, np.int64)
    return MAX_NODE_SCORE - MAX_NODE_SCORE * raw // mx


def node_affinity_norm(raw):
    """NodeAffinity NormalizeScore: DefaultNormalizeScore(100, reverse=false); raws are >= 0."""
    mx = int(raw.max()) if len(raw) else 0
    return raw.copy() if mx == 0 else MAX_NODE_SCORE * raw // mx


def go_round(x):
    """math.Round: half away from zero."""
    return np.where(x >= 0, np.floor(x + 0.5), -np.floor(-x + 0.5)).astype(np.int64) if isinstance(x, np.ndarray) else (
        int(np.floor(x + 0.5)) if x >= 0 else -int(np.floor(-x + 0.5)))


def pts_norm(raw):
    """PodTopologySpread NormalizeScore (podtopologyspread/scoring.go:240-265) over the scored nodes: 100 * (max + min - r) / max,
    and 100 for every node when max == 0."""
    if len(raw) == 0:
        return raw.copy()
    mx, mn = int(raw.max()), int(raw.min())
    if mx == 0:
        return np.full(len(raw), MAX_NODE_SCORE, np.int64)
    num = MAX_NODE_SCORE * (mx + mn - raw)
    return np.sign(num) * (np.abs(num) // abs(mx)) * np.sign(mx)      # int64 division, truncating


def ipa_norm(raw, exact=False):
    """InterPodAffinity NormalizeScore (interpodaffinity/scoring.go:258-290): int64(100 * (float64(r - min) / float64(max - min))),
    0 for every node when max == min. exact: integer 100 * (r - min) / (max - min) instead."""
    if len(raw) == 0:
        return raw.copy()
    mx, mn = int(raw.max()), int(raw.min())
    if mx == mn:
        return np.zeros(len(raw), np.int64)
    if exact:
        return MAX_NODE_SCORE * (raw - mn) // (mx - mn)
    return (100.0 * ((raw - mn).astype(np.float64) / float(mx - mn))).astype(np.int64)


# ---- the sequential loop -------------------------------------------------------------------------------------------------
class Result:
    def __init__(self, pod_node, stop_code, reason_hist, ipa_edges):
        self.pod_node = np.asarray(pod_node, np.int32)
        self.placed = len(self.pod_node)
        self.stop_code = stop_code
        self.reason_hist = reason_hist
        self.ipa_edges = ipa_edges      # {(r - min, max - min)}: pairs seen on feasible nodes, for the generator guards


def _check_supported(snap, tmpl, ctr, bound):
    for t in tmpl:
        assert t.n_aff == 0 and t.n_anti == 0 and t.n_pref_terms == 0 and t.nodename_idx < 0, "not modelled"
        assert not (t.flags & (abi.TF_HAS_NODE_SELECTOR | abi.TF_HAS_AFFINITY_TERMS | abi.TF_HAS_HOST_PORTS | abi.TF_PREFILTER_NODES
                               | abi.TF_FIT_ALL_ZERO)), "not modelled"
        assert t.req_eph == 0 and t.least_cpu == t.nz_cpu and t.least_mem == t.nz_mem, "not modelled"
        assert all(int(t.tol_nosched[w]) == 0 and int(t.tol_prefer[w]) == 0 for w in range(snap.taint_words)), "not modelled"
        for c in range(t.n_pts):      # hard spread terms must never bind (skew <= max count + clones + 1): the model has no such filter
            init = np.asarray(ctr[t.pts[c].counter]._keep, np.int64)
            assert t.pts[c].max_skew > int(init.max(initial=0)) + bound + 1, "binding spread term"
        for c in range(t.n_spts):
            assert ctr[t.spts[c].counter].inc == 0 and t.spts[c].hostname and t.spts[c].has_key_bit < 0, "not modelled"
        for k in range(t.n_ipa_score):
            assert ctr[t.ipa_score_counter[k]].inc == 0, "not modelled"
    assert all(int(m) == 0 for m in snap.taint_nosched), "not modelled"


def run(snap, tmpl, ctr=(), max_pods=0, exact=False):
    """The schedule-one-pod-then-update loop (schedule_one.go) over the modelled plugins: NodeResourcesFit (cpu, memory, pods,
    extended resources), PreferNoSchedule taint classes, ImageLocality, and the soft PodTopologySpread (hostname) and
    InterPodAffinity terms over static counters. Pod k is a clone of template k % len(tmpl); the highest total among the feasible
    nodes wins, ties go to the lowest index."""
    n = snap.n
    bound = int(np.maximum(snap.alloc_pods.astype(np.int64) - snap.npods, 0).sum())
    _check_supported(snap, tmpl, ctr, bound)
    a_cpu, a_mem = [int(x) for x in snap.alloc_cpu], [int(x) for x in snap.alloc_mem]
    r_cpu, r_mem = [int(x) for x in snap.req_cpu], [int(x) for x in snap.req_mem]
    z_cpu, z_mem = [int(x) for x in snap.nz_cpu], [int(x) for x in snap.nz_mem]
    free_cpu = snap.alloc_cpu - snap.req_cpu
    free_mem = snap.alloc_mem - snap.req_mem
    free_pods = snap.alloc_pods.astype(np.int64) - snap.npods
    free_sc = [a - r for a, r in snap.scalars]
    prefer = np.zeros(n, np.int64)
    for w in range(snap.taint_words):
        m = snap.taint_mask[w] & np.uint64(snap.taint_prefer[w])
        prefer += np.array([bin(int(x)).count("1") for x in m], np.int64)
    ignored = np.zeros(n, bool)

    def local(t, i):
        s = 0
        if t.score_enable & abi.PL_FIT:
            s += t.w_fit * least_allocated((a_cpu[i], a_mem[i]), (z_cpu[i] + t.least_cpu, z_mem[i] + t.least_mem),
                                           (t.least_w_cpu, t.least_w_mem))
        if (t.score_enable & abi.PL_BALANCED) and not (t.flags & abi.TF_BALANCED_SKIP):
            s += t.w_balanced * balanced((a_cpu[i], a_mem[i]), (r_cpu[i] + t.bal_cpu, r_mem[i] + t.bal_mem), exact)
        return s

    def feasible_mask(t):
        ok = free_pods >= 1
        if t.req_cpu > 0:
            ok &= free_cpu >= t.req_cpu
        if t.req_mem > 0:
            ok &= free_mem >= t.req_mem
        for k, f in enumerate(free_sc):
            if t.req_scalar[k]:
                ok &= f >= t.req_scalar[k]
        return ok

    def reasons(t):
        hist = np.zeros(abi.R_TOTAL, np.int64)
        hist[abi.R_TOO_MANY_PODS] = int((free_pods < 1).sum())
        if t.req_cpu > 0:
            hist[abi.R_INSUFFICIENT_CPU] = int((free_cpu < t.req_cpu).sum())
        if t.req_mem > 0:
            hist[abi.R_INSUFFICIENT_MEMORY] = int((free_mem < t.req_mem).sum())
        for k, f in enumerate(free_sc):
            if t.req_scalar[k]:
                hist[abi.R_SCALAR0 + k] = int((f < t.req_scalar[k]).sum())
        return hist

    live = np.nonzero(free_pods >= 1)[0]          # free pods only shrink: the other nodes are never feasible
    cache = []
    for t in tmpl:
        c = np.zeros(n, np.int64)
        c[live] = [local(t, int(i)) for i in live]
        cache.append(c)
    img = [np.asarray(t._keep_img, np.int64) if getattr(t, "_keep_img", None) is not None and len(t._keep_img) else np.zeros(n, np.int64)
           for t in tmpl]
    ipa_raw, spts_cnt = [], []
    for t in tmpl:
        r = np.zeros(n, np.int64)
        for k in range(t.n_ipa_score):
            c = ctr[t.ipa_score_counter[k]]
            init = np.asarray(c._keep, np.int64)
            if c.topo_col < 0:
                r += init
            else:
                dom = snap.topo[c.topo_col]
                r += np.where(dom >= 0, init[np.maximum(dom, 0)], 0)
        ipa_raw.append(r)
        spts_cnt.append([np.asarray(ctr[t.spts[c].counter]._keep, np.int64) for c in range(t.n_spts)])
        if t.spts_ignored_bit >= 0:
            b = t.spts_ignored_bit
            ignored = ((snap.static_mask[b >> 6] >> np.uint64(b & 63)) & np.uint64(1)).astype(bool)

    pod_node, ipa_edges = [], set()
    k = 0
    while True:
        ti = k % len(tmpl)
        t = tmpl[ti]
        feas = np.nonzero(feasible_mask(t))[0]
        if len(feas) == 0:
            return Result(pod_node, abi.STOP_UNSCHEDULABLE, reasons(t), ipa_edges)
        total = cache[ti][feas].copy()
        if t.score_enable & abi.PL_TAINT_TOLERATION:
            total += t.w_taint * taint_norm(prefer[feas])
        if t.score_enable & abi.PL_IMAGE_LOCALITY:
            total += t.w_image * img[ti][feas]
        if (t.score_enable & abi.PL_POD_TOPOLOGY_SPREAD) and t.n_spts:
            scored = ~ignored[feas]
            size = int(scored.sum())
            raw = np.zeros(len(feas), np.float64)
            for c in range(t.n_spts):      # hostname constraints: one domain per scored node
                raw += spts_cnt[ti][c][feas].astype(np.float64) * go_log(float(size + 2)) + float(t.spts[c].max_skew - 1)
            r = go_round(raw)
            total[scored] += t.w_pts * pts_norm(r[scored])
        if (t.score_enable & abi.PL_INTER_POD_AFFINITY) and t.n_ipa_score:
            r = ipa_raw[ti][feas]
            total += t.w_ipa * ipa_norm(r, exact)
            mn, mx = int(r.min()), int(r.max())
            ipa_edges.update((int(v) - mn, mx - mn) for v in np.unique(r))
        w = int(feas[int(np.argmax(total))])        # argmax: first maximum = lowest index
        pod_node.append(w)
        r_cpu[w] += t.req_cpu
        r_mem[w] += t.req_mem
        z_cpu[w] += t.nz_cpu
        z_mem[w] += t.nz_mem
        free_cpu[w] -= t.req_cpu
        free_mem[w] -= t.req_mem
        free_pods[w] -= 1
        for q, f in enumerate(free_sc):
            f[w] -= t.req_scalar[q]
        for q, tq in enumerate(tmpl):
            cache[q][w] = local(tq, w)
        k += 1
        if max_pods and k >= max_pods:
            return Result(pod_node, abi.STOP_LIMIT_REACHED, np.zeros(abi.R_TOTAL, np.int64), ipa_edges)


# ---- fp32 emulations of the kernels' screens (generator guards only) ----------------------------------------------------------
def fp32_least_estimate(x100, capacity):
    """int64(x100 / capacity) in fp32: both operands rounded to fp32, one fp32 quotient (numpy)."""
    return np.trunc(np.float32(x100) / np.float32(capacity)).astype(np.int64)


def balanced_f64_value(a_cpu, a_mem, q_cpu, q_mem):
    """(1 - std) * 100 before truncation, float64, both allocatables > 0 (numpy)."""
    f0 = np.minimum(np.asarray(q_cpu, np.float64) / np.asarray(a_cpu, np.float64), 1.0)
    f1 = np.minimum(np.asarray(q_mem, np.float64) / np.asarray(a_mem, np.float64), 1.0)
    return (1.0 - np.abs((f0 - f1) / 2.0)) * 100.0


def balanced_exact_int(a_cpu, a_mem, q_cpu, q_mem):
    """floor(100 * (1 - |f0 - f1| / 2)) exactly, both allocatables > 0 (numpy int64; small quantities only)."""
    a0, a1 = np.asarray(a_cpu, np.int64), np.asarray(a_mem, np.int64)
    q0, q1 = np.minimum(np.asarray(q_cpu, np.int64), a0), np.minimum(np.asarray(q_mem, np.int64), a1)
    d = np.abs(q0 * a1 - q1 * a0)
    return 100 + (-50 * d) // (a0 * a1)          # 100 - ceil(50 |d| / (a0 a1))
