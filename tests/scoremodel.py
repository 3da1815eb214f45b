"""A plain model of the default profile's score plugins, in Go semantics, and of the schedule-one-pod loop for the workloads the
score ladders (tests/test_score_edges.py) and the soft-scorer cases (tests/test_soft_scorers.py) use. It restates the reference's
formulas on its own: no code is shared with the C oracle or the CUDA kernels, only the flat snapshot / template structs are read.

Modelled: NodeResourcesFit (filter and LeastAllocated), BalancedAllocation, ImageLocality, TaintToleration's PreferNoSchedule
classes in any taint word (tolerated ones excluded), NodeAffinity preferred terms (node_affinity.go:241-290, normalised with
DefaultNormalizeScore(100, false)), the PodTopologySpread score on any topology column (podtopologyspread/scoring.go:60-265) and
the InterPodAffinity score (interpodaffinity/scoring.go:236-290), with every counter updated per commit: spread counters only when
the winner carries the counter's elig_bit, hostname counters always, InterPodAffinity counters by their signed increment.
The Filter runs every default-profile plugin per node, in the order of apis/config/v1/default_plugins.go:33-47, the first
failing plugin deciding the node's status (framework/runtime/framework.go RunFilterPlugins):
  1. the PreFilterResult node set (schedule_one.go:523-534: nodes outside it are UnschedulableAndUnresolvable);
  2. NodeUnschedulable (nodeunschedulable/node_unschedulable.go:133-150; the node's spec.unschedulable is bit 63 of taint word 0,
     which is no taint);
  3. NodeName (nodename/node_name.go:72-83);
  4. TaintToleration (tainttoleration/taint_toleration.go:111-122): NoSchedule and NoExecute taints in any taint word; the reason
     names the first untolerated taint in node.Spec.Taints order (component-helpers/scheduling/corev1/helpers.go:78-86), the
     lowest taint id when the snapshot carries no taint lists;
  5. NodeAffinity (nodeaffinity/node_affinity.go:206-227): the selector's bits AND the OR of the required terms (zero terms
     match nothing);
  6. NodePorts (nodeports/node_ports.go:157-192): static conflicts, and clones of a conflicting template already on the node;
  7. NodeResourcesFit (noderesources/fit.go:509-533, 564-654): every insufficient resource is a reason, the status is
     UnschedulableAndUnresolvable iff some request exceeds the allocatable itself; "Too many pods" is always Unschedulable;
  8. PodTopologySpread (podtopologyspread/filtering.go:311-356), per constraint in order: a node without the key is
     UnschedulableAndUnresolvable; else cnt + self_match - min > maxSkew is Unschedulable, min being the minimum over the
     present domains [0, n_present) (filtering.go:56-69, 98-137; MaxInt32 without one), 0 when min_zero (fewer domains than
     minDomains). A node whose domain lies outside [0, n_present) reads its counter value, as the flat-struct contract of
     the encoder states; the reference cannot reach that state, since a node that passes every filter has its domain counted,
     and an uncounted domain reads 0 there (filtering.go:347);
  9. InterPodAffinity (interpodaffinity/filtering.go:352-432), in the order of :419-429: the pod's required affinity (every key
     present, every count > 0, or no matching pod in the cluster and the pod matching all its own terms: :382-408;
     UnschedulableAndUnresolvable), its required anti-affinity (a node without the key passes: :367-379; Unschedulable), then
     the existing pods' anti-affinity (:352-364; Unschedulable).
FitError diagnosis (framework/types.go:787-838): the reason histogram over every node, and the preemption split
(preemption/preemption.go:309-331): Unschedulable nodes are the candidates, of which none has a lower-priority victim ("No
preemption victims found"); every other node is "Preemption is not helpful". Every counter moves per commit in exact Python ints,
aff_total included (the pod's own affinity counts move only when it matches all its terms: filtering.go:234-271); the templates
placed on each node are tracked for NodePorts.
Not modelled: reference sampling below 100 %.

PodTopologySpread, per cycle: the scored nodes are the feasible nodes outside IgnoredNodes (spts_ignored_bit; only explicit
constraints ignore nodes, and then exactly the nodes that miss a constraint key). Per constraint w = go_log(size + 2), where size
is the number of scored nodes for a hostname key, else the number of distinct values among the scored nodes, a node without the
label counting as the value "" (only possible under the system defaults). A node's raw score is one math.Round of the float64 sum
over its constraints, in order, of cnt * w + (maxSkew - 1); a node without a constraint's key (has_key_bit for hostname keys)
skips that constraint. Normalised 100 * (max + min - raw) / max over the scored nodes (100 each when max == 0); ignored nodes
score 0.

Go semantics: int64 division truncates toward zero; float64 operations round once each, in the reference's order; int64(x) of a
float truncates. Python ints are exact and Python floats are IEEE float64, so both are restated directly. Counters are exact
Python / int64 values: where the engine's int32 counters could wrap, the model still predicts the reference's result.

exact=True swaps BalancedAllocation for rational arithmetic and the InterPodAffinity normalisation for integer arithmetic. Those
are not what the reference computes: a test runs them only to prove that its inputs sit where the rounding decides the result.
mutate=<name> (one of MUTATIONS or FILTER_MUTATIONS) makes the soft path or the Filter subtly wrong in one named way, for the
same purpose: a test proves that its cases would notice a kernel with that defect.
"""
import importlib
from fractions import Fraction

import numpy as np

from oracle.objref import go_log

abi = importlib.import_module("cluster-capacity_b200._abi")

MAX_NODE_SCORE = 100

MUTATIONS = (
    "domains_all_nodes",       # a constraint's domain count over every non-ignored node instead of the feasible ones
    "empty_not_counted",       # the value "" of nodes without the label not counted under the system defaults
    "empty_counted_explicit",  # ... counted under explicit constraints (from the ignored nodes that miss the key)
    "ignored_in_size",         # ignored feasible nodes counted in size
    "ignored_in_min",          # ignored feasible nodes' raw scores taken into the spread minimum
    "round_per_constraint",    # math.Round applied to each constraint's term instead of once to the sum
    "commits_ignore_elig",     # spread counters incremented on every winner, whatever its elig_bit
    "ipa_inc_dropped",         # InterPodAffinity counters never incremented
)

FILTER_MUTATIONS = (
    "skew_ge",                 # spread skew tested with >= instead of >
    "min_all_domains",         # spread minimum over every domain instead of the present ones
    "min_zero_ignored",        # spread minimum taken over the domains even when fewer than minDomains exist
    "self_match_one",          # spread self_match taken as 1
    "missing_key_as_skew",     # a node without a spread key counted as a skew failure (Unschedulable)
    "aff_bypass_never",        # the first-pod affinity bypass never applies
    "aff_bypass_sticky",       # ... outlives the first clone (aff_total never moves)
    "anti_missing_key_fails",  # anti-affinity fails a node without the term's key
    "taint_bit_order",         # the first untolerated taint in taint-id order instead of Spec order
    "fit_first_reason",        # only the first insufficient resource kept as a reason
    "fit_all_unschedulable",   # every NodeResourcesFit failure Unschedulable
    "ports_after_fit",         # NodePorts checked after NodeResourcesFit
    "ports_cross_template",    # clones of other templates never conflict on a host port
    "hostname_anti_frozen",    # hostname anti-affinity counters never incremented
    "diag_ptsmin_stale",       # the FitError diagnosis reads the spread minimum of the last placing cycle, not the failing one
)

UNSCHEDULABLE, UNRESOLVABLE = 1, 2       # status codes (kube-scheduler framework/interface.go)
MAX_INT32 = 2 ** 31 - 1
U64 = (1 << 64) - 1


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


def pts_norm(raw, mn=None):
    """PodTopologySpread NormalizeScore (podtopologyspread/scoring.go:240-265) over the scored nodes: 100 * (max + min - r) / max,
    and 100 for every node when max == 0. mn: the minimum to use instead of raw's own (mutations only)."""
    if len(raw) == 0:
        return raw.copy()
    mx = int(raw.max())
    mn = int(raw.min()) if mn is None else mn
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


def _edge_kind(raw, mx):
    """Truncation edges of 100 * raw / mx met by a value strictly between 0 and mx: "at" a multiple of mx, or one "below"."""
    out = set()
    for r in np.unique(raw):
        r = int(r)
        if mx > 0 and 0 < r < mx:
            m = (MAX_NODE_SCORE * r) % mx
            if m == 0:
                out.add("at")
            elif m == mx - 1:
                out.add("below")
    return out


# ---- the sequential loop -------------------------------------------------------------------------------------------------
class Result:
    def __init__(self, pod_node, stop_code, reason_hist, ipa_edges, preempt=(0, 0), soft=None, hard=None):
        self.pod_node = np.asarray(pod_node, np.int32)
        self.placed = len(self.pod_node)
        self.stop_code = stop_code
        self.reason_hist = reason_hist
        self.preempt_no_victims, self.preempt_not_helpful = preempt
        self.ipa_edges = ipa_edges      # {(r - min, max - min)}: pairs seen on feasible nodes, for the generator guards
        # what the soft path met, for the generator guards: spread sizes per cycle, truncation edges of the NodeAffinity and
        # PodTopologySpread normalisations ("at" / "below" a multiple of max), cycles where max == 0, cycles without a scored node
        self.soft = soft or {}
        # what the Filter met, for the generator guards: edge name -> number of cycles (or nodes at the terminal cycle) that met it
        self.hard = hard or {}


def _bit(snap, b):
    return ((snap.static_mask[b >> 6] >> np.uint64(b & 63)) & np.uint64(1)).astype(bool)


def _check_supported(snap, tmpl, ctr):
    for t in tmpl:
        assert t.least_cpu == t.nz_cpu and t.least_mem == t.nz_mem, "not modelled"
        if t.spts_ignored_bit >= 0 and t.n_spts:      # explicit constraints: IgnoredNodes are exactly the nodes that miss a key
            missing = np.zeros(snap.n, bool)
            for c in range(t.n_spts):
                sc = t.spts[c]
                if sc.hostname:
                    if sc.has_key_bit >= 0:
                        missing |= ~_bit(snap, sc.has_key_bit)
                else:
                    missing |= snap.topo[ctr[sc.counter].topo_col] < 0
            assert np.array_equal(missing, _bit(snap, t.spts_ignored_bit)), "IgnoredNodes must be the nodes that miss a key"


def _covers(snap, idx, masks):
    """Per node of idx: every bit of masks (one uint64 per static word) is set on the node; a word the snapshot lacks is 0."""
    ok = np.ones(len(idx), bool)
    for w in range(abi.MAX_STATIC_WORDS):
        m = int(masks[w])
        if m:
            ok &= (snap.static_mask[w][idx] & np.uint64(m)) == np.uint64(m) if w < snap.static_words else False
    return ok


def _meets(snap, idx, masks):
    """Per node of idx: some bit of masks is set on the node."""
    hit = np.zeros(len(idx), bool)
    for w in range(snap.static_words):
        if int(masks[w]):
            hit |= (snap.static_mask[w][idx] & np.uint64(int(masks[w]))) != 0
    return hit


def run(snap, tmpl, ctr=(), max_pods=0, exact=False, mutate=None):
    """The schedule-one-pod-then-update loop (schedule_one.go) over the modelled plugins. Pod k is a clone of template k % len(tmpl);
    the highest total among the feasible nodes wins, ties go to the lowest index."""
    assert mutate is None or mutate in MUTATIONS + FILTER_MUTATIONS, mutate
    n = snap.n
    _check_supported(snap, tmpl, ctr)
    a_cpu, a_mem = [int(x) for x in snap.alloc_cpu], [int(x) for x in snap.alloc_mem]
    r_cpu, r_mem = [int(x) for x in snap.req_cpu], [int(x) for x in snap.req_mem]
    z_cpu, z_mem = [int(x) for x in snap.nz_cpu], [int(x) for x in snap.nz_mem]
    free_cpu = snap.alloc_cpu - snap.req_cpu
    free_mem = snap.alloc_mem - snap.req_mem
    free_eph = snap.alloc_eph - snap.req_eph
    free_pods = snap.alloc_pods.astype(np.int64) - snap.npods
    free_sc = [a - r for a, r in snap.scalars]
    cnt = [np.asarray(c._keep, np.int64).copy() for c in ctr]      # exact counts: the reference's are int64
    aff_total = int(tmpl[0].aff_total_init)                        # pods matching the pod's required affinity terms, cluster-wide
    placed = [0] * n                                               # bit q: a clone of template q sits on the node
    ipa_counters = {int(t.ipa_score_counter[k]) for t in tmpl for k in range(t.n_ipa_score)}
    anti_host = {int(t.anti_counter[a]) for t in tmpl for a in range(t.n_anti) if ctr[t.anti_counter[a]].topo_col < 0}

    def local(t, i):
        s = 0
        if t.score_enable & abi.PL_FIT:
            s += t.w_fit * least_allocated((a_cpu[i], a_mem[i]), (z_cpu[i] + t.least_cpu, z_mem[i] + t.least_mem),
                                           (t.least_w_cpu, t.least_w_mem))
        if (t.score_enable & abi.PL_BALANCED) and not (t.flags & abi.TF_BALANCED_SKIP):
            s += t.w_balanced * balanced((a_cpu[i], a_mem[i]), (r_cpu[i] + t.bal_cpu, r_mem[i] + t.bal_mem), exact)
        return s

    # free pods only shrink: while NodeResourcesFit filters, the other nodes are never feasible
    fit_all = all(t.filter_enable & abi.PL_FIT for t in tmpl)
    live = np.nonzero(free_pods >= 1)[0] if fit_all else np.arange(n)

    def domain(j, idx):
        return idx if ctr[j].topo_col < 0 else snap.topo[ctr[j].topo_col][idx]

    def count(j, dom):
        return np.where(dom >= 0, cnt[j][np.maximum(dom, 0)], 0)

    def pts_min(t):
        """Per hard spread constraint: the critical path's count (filtering.go:56-69, 98-137)."""
        out = []
        for c in range(t.n_pts):
            p = t.pts[c]
            if p.min_zero and mutate != "min_zero_ignored":
                out.append(0)
                continue
            hi = ctr[p.counter].n_domains if mutate == "min_all_domains" else ctr[p.counter].n_present
            out.append(int(cnt[p.counter][:hi].min()) if hi > 0 else MAX_INT32)
        return out

    def first_taint(t, i):
        """The first untolerated NoSchedule / NoExecute taint of node i (helpers.go:78-86)."""
        if snap.taint_list_off is not None and mutate != "taint_bit_order":
            for tid in snap.taint_list[snap.taint_list_off[i]:snap.taint_list_off[i + 1]]:
                w, b = int(tid) >> 6, int(tid) & 63
                if (int(snap.taint_nosched[w]) >> b) & 1 and not (int(t.tol_nosched[w]) >> b) & 1:
                    return int(tid)
        for w in range(snap.taint_words):
            m = int(snap.taint_mask[w][i]) & untol_mask(t, w)
            if m:
                return 64 * w + (m & -m).bit_length() - 1
        raise AssertionError("no untolerated taint")

    def untol_mask(t, w):
        m = int(snap.taint_nosched[w]) & ~int(t.tol_nosched[w]) & U64
        return m & ~(1 << abi.TAINT_UNSCHEDULABLE_BIT) if w == 0 else m

    def filt(t, ti, idx, ptsmin, diag=False, seen=None):
        """Status per node of idx (0: passes), first failing plugin wins; with diag also the FitError reasons."""
        st = np.zeros(len(idx), np.int8)
        hist = np.zeros(abi.R_TOTAL, np.int64)
        fe = t.filter_enable

        def fail(bad, status, reason=None):
            bad = bad & (st == 0)
            st[bad] = status
            if reason is not None:
                hist[reason] += int(bad.sum())
            return bad

        def ports():
            if (fe & abi.PL_NODE_PORTS) and (t.flags & abi.TF_HAS_HOST_PORTS):
                conflict = int(t.port_tmpl_conflict) & (1 << ti if mutate == "ports_cross_template" else U64)
                mine = np.array([placed[i] & conflict != 0 for i in idx], bool) if conflict else np.zeros(len(idx), bool)
                fail(_meets(snap, idx, t.port_static_mask) | mine, UNSCHEDULABLE, abi.R_NODE_PORTS)

        if (t.flags & abi.TF_PREFILTER_NODES) and t.prefilter_bit >= 0:
            fail(~_bit(snap, t.prefilter_bit)[idx], UNRESOLVABLE, abi.R_PREFILTER_NODES)
        if (fe & abi.PL_NODE_UNSCHEDULABLE) and not (t.flags & abi.TF_TOLERATES_UNSCHEDULABLE):
            fail((snap.taint_mask[0][idx] >> np.uint64(abi.TAINT_UNSCHEDULABLE_BIT)) & np.uint64(1) != 0, UNRESOLVABLE, abi.R_UNSCHEDULABLE)
        if (fe & abi.PL_NODE_NAME) and t.nodename_idx >= 0:
            fail(idx != t.nodename_idx, UNRESOLVABLE, abi.R_NODE_NAME)
        if fe & abi.PL_TAINT_TOLERATION:
            untol = np.zeros(len(idx), bool)
            for w in range(snap.taint_words):
                untol |= (snap.taint_mask[w][idx] & np.uint64(untol_mask(t, w))) != 0
            bad = fail(untol, UNRESOLVABLE)
            if diag:
                for i in idx[bad]:
                    hist[abi.R_TAINT0 + first_taint(t, int(i))] += 1
        if (fe & abi.PL_NODE_AFFINITY) and (t.flags & (abi.TF_HAS_NODE_SELECTOR | abi.TF_HAS_AFFINITY_TERMS)):
            ok = _covers(snap, idx, t.sel_mask)
            if t.flags & abi.TF_HAS_AFFINITY_TERMS:
                any_term = np.zeros(len(idx), bool)
                for k in range(t.n_aff_terms):
                    any_term |= _covers(snap, idx, t.aff_term_mask[k])
                ok &= any_term
            fail(~ok, UNRESOLVABLE, abi.R_NODE_AFFINITY)
        if mutate != "ports_after_fit":
            ports()
        if fe & abi.PL_FIT:
            rs = [(free_pods[idx] < 1, abi.R_TOO_MANY_PODS, np.zeros(len(idx), bool))]
            for q, free, alloc, r in ((t.req_cpu, free_cpu, snap.alloc_cpu, abi.R_INSUFFICIENT_CPU),
                                      (t.req_mem, free_mem, snap.alloc_mem, abi.R_INSUFFICIENT_MEMORY),
                                      (t.req_eph, free_eph, snap.alloc_eph, abi.R_INSUFFICIENT_EPHEMERAL)):
                if q > 0:
                    rs.append((free[idx] < q, r, alloc[idx] < q))
            for k, f in enumerate(free_sc):
                q = int(t.req_scalar[k])
                if q:
                    rs.append((f[idx] < q, abi.R_SCALAR0 + k, snap.scalars[k][0][idx] < q))
            open_ = st == 0
            bad, unres, first = np.zeros(len(idx), bool), np.zeros(len(idx), bool), np.zeros(len(idx), bool)
            for short, r, beyond in rs:
                counted = short & open_ & ~first if mutate == "fit_first_reason" else short & open_
                hist[r] += int(counted.sum())
                first |= short
                bad |= short
                unres |= short & beyond
            if mutate == "fit_all_unschedulable":
                unres[:] = False
            fail(bad & unres, UNRESOLVABLE)
            fail(bad, UNSCHEDULABLE)
        if mutate == "ports_after_fit":
            ports()
        if fe & abi.PL_POD_TOPOLOGY_SPREAD:
            for c in range(t.n_pts):
                p = t.pts[c]
                dom = domain(p.counter, idx)
                missing = dom < 0
                if seen is not None:
                    seen["missing_key"] += bool((missing & (st == 0)).any())
                if mutate == "missing_key_as_skew":
                    fail(missing, UNSCHEDULABLE, abi.R_PTS_SKEW)
                else:
                    fail(missing, UNRESOLVABLE, abi.R_PTS_MISSING_LABEL)
                skew = count(p.counter, dom) + (1 if mutate == "self_match_one" else p.self_match) - ptsmin[c]
                over = skew >= p.max_skew if mutate == "skew_ge" else skew > p.max_skew
                if seen is not None:
                    open_ = (st == 0) & ~missing
                    seen["skew_at_max"] += bool((open_ & (skew == p.max_skew)).any())
                    seen["skew_one_over"] += bool((open_ & (skew == p.max_skew + 1)).any())
                    seen["outside_present"] += bool((open_ & (dom >= ctr[p.counter].n_present)).any())
                fail(~missing & over, UNSCHEDULABLE, abi.R_PTS_SKEW)
        if fe & abi.PL_INTER_POD_AFFINITY:
            if t.n_aff:
                missing, exist = np.zeros(len(idx), bool), np.ones(len(idx), bool)
                for a in range(t.n_aff):
                    dom = domain(t.aff_counter[a], idx)
                    missing |= dom < 0
                    exist &= count(t.aff_counter[a], dom) > 0
                bypass = aff_total == 0 and bool(t.flags & abi.TF_AFF_SELF_MATCH_ALL) and mutate != "aff_bypass_never"
                if seen is not None and bypass:
                    seen["bypass"] += 1
                fail(missing | (~exist & (not bypass)), UNRESOLVABLE, abi.R_IPA_AFFINITY)
            for a in range(t.n_anti):
                dom = domain(t.anti_counter[a], idx)
                bad = count(t.anti_counter[a], dom) > 0
                if seen is not None:
                    seen["anti_missing_key"] += bool(((dom < 0) & (st == 0)).any())
                fail(bad | (dom < 0) if mutate == "anti_missing_key_fails" else bad, UNSCHEDULABLE, abi.R_IPA_ANTI_AFFINITY)
            fail(_meets(snap, idx, t.existing_anti_mask), UNSCHEDULABLE, abi.R_IPA_EXISTING_ANTI)
        return st, hist

    def reasons(t, ti, ptsmin):
        """FitError histogram over every node, and the preemption split: Unschedulable nodes are preemption candidates without
        lower-priority victims, every other node is "not helpful" (preemption.go:262-277, 309-331)."""
        st, hist = filt(t, ti, np.arange(n), ptsmin, diag=True)
        assert not (st == 0).any()
        unsched = int((st == UNSCHEDULABLE).sum())
        return hist, (unsched, n - unsched)

    cache, img, prefer, na_raw, ignored = [], [], [], [], []
    for t in tmpl:
        c = np.zeros(n, np.int64)
        c[live] = [local(t, int(i)) for i in live]
        cache.append(c)
        img.append(np.asarray(t._keep_img, np.int64) if getattr(t, "_keep_img", None) is not None and len(t._keep_img)
                   else np.zeros(n, np.int64))
        p = np.zeros(n, np.int64)      # intolerable PreferNoSchedule taints (taint_toleration.go:154-182), any taint word
        for w in range(snap.taint_words):
            m = snap.taint_mask[w] & np.uint64(snap.taint_prefer[w]) & ~np.uint64(t.tol_prefer[w])
            p += np.array([bin(int(x)).count("1") for x in m], np.int64)
        prefer.append(p)
        r = np.zeros(n, np.int64)      # matching preferred terms' weights (node_affinity.go:265-290)
        for k in range(t.n_pref_terms):
            m = np.ones(n, bool)
            for w in range(snap.static_words):
                pm = np.uint64(t.pref_mask[k][w])
                m &= (snap.static_mask[w] & pm) == pm
            r += np.where(m, int(t.pref_weight[k]), 0)
        na_raw.append(r)
        ignored.append(_bit(snap, t.spts_ignored_bit) if t.spts_ignored_bit >= 0 else np.zeros(n, bool))

    def domains(col, nodes, missing_counts):
        v = col[nodes]
        return len(np.unique(v[v >= 0])) + (1 if missing_counts and bool((v < 0).any()) else 0)

    def spread(t, ti, feas, soft):
        """Normalised PodTopologySpread scores of the feasible nodes (0 on ignored ones)."""
        ign = ignored[ti][feas]
        nodes, dropped = feas[~ign], feas[ign]
        explicit = t.spts_ignored_bit >= 0
        terms = np.zeros((t.n_spts, len(feas)), np.float64)
        has = np.zeros((t.n_spts, len(feas)), bool)
        sizes = []
        for c in range(t.n_spts):
            sc = t.spts[c]
            j = sc.counter
            if sc.hostname:
                size = len(nodes) + (len(dropped) if mutate == "ignored_in_size" else 0)
                has[c] = _bit(snap, sc.has_key_bit)[feas] if sc.has_key_bit >= 0 else True
                v = cnt[j][feas]
            else:
                col = snap.topo[ctr[j].topo_col]
                pool = nodes
                if mutate == "domains_all_nodes":
                    pool = np.nonzero(~ignored[ti])[0]
                elif mutate == "ignored_in_size":
                    pool = feas
                size = domains(col, pool, not (mutate == "empty_not_counted" and not explicit))
                if mutate == "empty_counted_explicit" and explicit and bool((col[dropped] < 0).any()) and not bool((col[pool] < 0).any()):
                    size += 1
                dom = col[feas]
                has[c] = dom >= 0
                v = np.where(dom >= 0, cnt[j][np.maximum(dom, 0)], 0)
            sizes.append(size)
            w = go_log(float(size + 2))
            terms[c] = v.astype(np.float64) * w + float(sc.max_skew - 1)
        if mutate == "round_per_constraint":
            raw = np.where(has, go_round(terms), 0).sum(axis=0)
        else:
            s = np.zeros(len(feas), np.float64)
            for c in range(t.n_spts):      # float64 sum in constraint order, one Round at the end
                s = s + np.where(has[c], terms[c], 0.0)
            raw = go_round(s)
        out = np.zeros(len(feas), np.int64)
        soft["sizes"].append(tuple(sizes))
        if len(nodes) == 0:
            soft["no_scored"] += 1
            return out
        r = raw[~ign]
        mn = int(raw.min()) if mutate == "ignored_in_min" else None
        out[~ign] = pts_norm(r, mn)
        mx = int(r.max())
        if mx == 0:
            soft["pts_max0"] += 1
        soft["pts_edges"] |= _edge_kind(mx + int(r.min()) - r, mx)
        return out

    soft = {"sizes": [], "no_scored": 0, "pts_max0": 0, "na_max0": 0, "pts_edges": set(), "na_edges": set()}
    hard = dict.fromkeys(("skew_at_max", "skew_one_over", "missing_key", "outside_present", "min_zero_above", "min_moved_last",
                          "bypass", "bypass_ended", "anti_missing_key"), 0)
    pod_node, ipa_edges = [], set()
    k = 0
    last_min = None
    while True:
        ti = k % len(tmpl)
        t = tmpl[ti]
        ptsmin = pts_min(t)
        for c in range(t.n_pts):
            p = t.pts[c]
            hard["min_zero_above"] += bool(p.min_zero and ctr[p.counter].n_present > 0
                                           and int(cnt[p.counter][:ctr[p.counter].n_present].min()) > 0)
        st, _ = filt(t, ti, live, ptsmin, seen=hard)
        feas = live[st == 0]
        if len(feas) == 0:
            hard["min_moved_last"] = int(last_min is not None and last_min != ptsmin)
            hist, preempt = reasons(t, ti, last_min if mutate == "diag_ptsmin_stale" and last_min is not None else ptsmin)
            return Result(pod_node, abi.STOP_UNSCHEDULABLE, hist, ipa_edges, preempt, soft, hard)
        last_min = ptsmin
        total = cache[ti][feas].copy()
        if t.score_enable & abi.PL_TAINT_TOLERATION:
            total += t.w_taint * taint_norm(prefer[ti][feas])
        if t.score_enable & abi.PL_IMAGE_LOCALITY:
            total += t.w_image * img[ti][feas]
        if (t.score_enable & abi.PL_NODE_AFFINITY) and t.n_pref_terms:
            r = na_raw[ti][feas]
            total += t.w_node_affinity * node_affinity_norm(r)
            mx = int(r.max())
            soft["na_max0"] += mx == 0
            soft["na_edges"] |= _edge_kind(r, mx)
        if (t.score_enable & abi.PL_POD_TOPOLOGY_SPREAD) and t.n_spts:
            total += t.w_pts * spread(t, ti, feas, soft)
        if (t.score_enable & abi.PL_INTER_POD_AFFINITY) and t.n_ipa_score:
            r = np.zeros(len(feas), np.int64)
            for q in range(t.n_ipa_score):
                j = t.ipa_score_counter[q]
                if ctr[j].topo_col < 0:
                    r += cnt[j][feas]
                else:
                    dom = snap.topo[ctr[j].topo_col][feas]
                    r += np.where(dom >= 0, cnt[j][np.maximum(dom, 0)], 0)
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
        free_eph[w] -= t.req_eph
        free_pods[w] -= 1
        if free_pods[w] < 1 and fit_all:
            live = live[live != w]
        placed[w] |= 1 << ti
        for q, f in enumerate(free_sc):
            f[w] -= t.req_scalar[q]
        for q, tq in enumerate(tmpl):
            cache[q][w] = local(tq, w)
        aff = {int(t.aff_counter[a]) for a in range(t.n_aff)}
        for j, c in enumerate(ctr):      # the next cycle's PreFilter / PreScore recount sees this clone
            if c.inc == 0 or (mutate == "ipa_inc_dropped" and j in ipa_counters) or (mutate == "hostname_anti_frozen" and j in anti_host):
                continue
            if j in aff and not (t.flags & abi.TF_AFF_SELF_MATCH_ALL):
                continue          # the clone matches its own affinity terms only if it matches all of them (filtering.go:124-130, 187-199)
            if c.elig_bit >= 0 and mutate != "commits_ignore_elig" and not _bit(snap, c.elig_bit)[w]:
                continue
            dom = w if c.topo_col < 0 else int(snap.topo[c.topo_col][w])
            if dom >= 0:
                cnt[j][dom] += c.inc
                if j in aff and mutate != "aff_bypass_sticky":
                    hard["bypass_ended"] += aff_total == 0
                    aff_total += c.inc
        k += 1
        if max_pods and k >= max_pods:
            return Result(pod_node, abi.STOP_LIMIT_REACHED, np.zeros(abi.R_TOTAL, np.int64), ipa_edges, soft=soft, hard=hard)


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
