/*
 * ccsim_oracle.c — CPU ORACLE (test infrastructure, NOT the product path).
 *
 * A plain-C restatement of the reference's schedule-one-pod-then-update loop over the flat snapshot of
 * include/ccsim.h. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this file's shared object; the product (libccsim.so) never does.
 *
 * Parity status: the reference has no golden vectors for instance counts / distributions / messages
 * (SURVEY.md §8c); this oracle is pinned against the reference's own asserted outcomes (TestPrediction fail
 * types, pod_colocation invariants, README 52) and the known-answer vectors KA1-KA5 derived from the cited
 * formulas (tests/test_oracle_known_answers.py, tests/golden/). No Go toolchain exists in the build
 * container, so outputs of a real reference run are NOT available: beyond those vectors parity is "unpinned".
 *
 * Every function cites the reference file:line it follows. Prefixes:
 *   KS: vendor/k8s.io/kubernetes/pkg/scheduler/   PL: KS:framework/plugins/   R: the cluster-capacity repo root
 *
 * Modes:
 *   canonical (0): percentageOfNodesToScore=100 -> every node is filtered each cycle, nextStartNodeIndex stays 0
 *                  (KS:schedule_one.go:538-539,697-723); ties -> first max in scan order, a legal outcome of
 *                  selectHost's reservoir sampling (KS:schedule_one.go:894-941).
 *   faithful  (1): adaptive numFeasibleNodesToFind + rotating start index, sequential scan (a legal interleaving
 *                  of the 16-goroutine filter), ties -> first max in (rotated) scan order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <limits.h>
#include <math.h>
#include <assert.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "../include/ccsim.h"

typedef struct {
  /* mutable copies of the NodeInfo aggregates */
  int64_t *req_cpu, *req_mem, *req_eph, *nz_cpu, *nz_mem;
  int64_t *req_scalar[CCSIM_MAX_SCALARS];
  int32_t *npods;
  uint64_t *placed_mask;
  /* per-counter domain counts */
  int32_t *cnt[CCSIM_MAX_COUNTERS];
  int64_t aff_total;
} ostate;

/* status codes of KF:interface.go (only the two that matter for the preemption suffix) */
#define ST_OK 0
#define ST_UNSCHEDULABLE 1
#define ST_UNRESOLVABLE 2

static inline uint64_t word(const uint64_t *m, int32_t n, int w, int32_t i) { return m[(size_t)w * n + i]; }

/* PL:podtopologyspread/filtering.go:56-69 minMatchNum; :98-137 criticalPaths[0] = global minimum over TpValueToMatchNum */
static int32_t pts_min(const ccsim_counter *c, const int32_t *cnt, const ccsim_pts *p) {
  if (p->min_zero) return 0;
  int32_t m = INT32_MAX; /* newCriticalPaths(): math.MaxInt32 */
  for (int32_t d = 0; d < c->n_present; d++) if (cnt[d] < m) m = cnt[d];
  return m;
}

/*
 * One node through the Filter plugins in default-profile order, first failing plugin wins
 * (KS:framework/runtime/framework.go:897-930; order KS:apis/config/v1/default_plugins.go:33-53).
 * reasons[]: reason ids appended (only NodeResourcesFit can give several, PL:noderesources/fit.go:519-533).
 * Returns the status code.
 */
static int filter_node(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, int ti,
                       const ccsim_counter *ctr, const int32_t *ptsmin, int32_t i,
                       int want_reasons, int *reasons, int *n_reasons) {
  const int32_t n = nd->n_nodes;
  int nr = 0;
  (void)ti;
  /* NodeAffinity PreFilterResult: nodes outside NodeNames never reach any Filter (KS:schedule_one.go:523-534) */
  if ((t->flags & CCSIM_TF_PREFILTER_NODES) && t->prefilter_bit >= 0) {
    int b = t->prefilter_bit;
    if (!((word(nd->static_mask, n, b >> 6, i) >> (b & 63)) & 1)) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_PREFILTER_NODES; *n_reasons = nr; }
      return ST_UNRESOLVABLE;
    }
  }
  /* NodeUnschedulable: PL:nodeunschedulable/node_unschedulable.go:133-150 */
  if (t->filter_enable & CCSIM_PL_NODE_UNSCHEDULABLE) {
    if (((word(nd->taint_mask, n, 0, i) >> CCSIM_TAINT_UNSCHEDULABLE_BIT) & 1) &&
        !(t->flags & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_UNSCHEDULABLE; *n_reasons = nr; }
      return ST_UNRESOLVABLE;
    }
  }
  /* NodeName: PL:nodename/node_name.go:72-83 */
  if (t->filter_enable & CCSIM_PL_NODE_NAME) {
    if (t->nodename_idx >= 0 && t->nodename_idx != i) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_NODE_NAME; *n_reasons = nr; }
      return ST_UNRESOLVABLE;
    }
  }
  /* TaintToleration: PL:tainttoleration/taint_toleration.go:111-122 */
  if (t->filter_enable & CCSIM_PL_TAINT_TOLERATION) {
    int untol = 0;
    for (int w = 0; w < nd->taint_words; w++) {
      uint64_t m = word(nd->taint_mask, n, w, i) & nd->taint_nosched[w] & ~t->tol_nosched[w];
      if (m) untol = 1;
    }
    if (untol) {
      if (want_reasons) {
        /* first untolerated taint in node.Spec.Taints order: CH:scheduling/corev1/helpers.go:78-101 */
        int id = -1;
        if (nd->taint_list_off) {
          for (int32_t k = nd->taint_list_off[i]; k < nd->taint_list_off[i + 1]; k++) {
            int tid = nd->taint_list[k];
            int w = tid >> 6, b = tid & 63;
            if (((nd->taint_nosched[w] >> b) & 1) && !((t->tol_nosched[w] >> b) & 1)) { id = tid; break; }
          }
        }
        if (id < 0) { /* no list given: lowest dictionary id */
          for (int w = 0; w < nd->taint_words && id < 0; w++) {
            uint64_t m = word(nd->taint_mask, n, w, i) & nd->taint_nosched[w] & ~t->tol_nosched[w];
            if (m) id = 64 * w + __builtin_ctzll(m);
          }
        }
        reasons[nr++] = CCSIM_R_TAINT0 + id; *n_reasons = nr;
      }
      return ST_UNRESOLVABLE;
    }
  }
  /* NodeAffinity: PL:nodeaffinity/node_affinity.go:147-155 (Skip), :206-227; CH:.../nodeaffinity.go:323-332 */
  if ((t->filter_enable & CCSIM_PL_NODE_AFFINITY) && (t->flags & (CCSIM_TF_HAS_NODE_SELECTOR | CCSIM_TF_HAS_AFFINITY_TERMS))) {
    int ok = 1;
    for (int w = 0; w < nd->static_words; w++)
      if ((word(nd->static_mask, n, w, i) & t->sel_mask[w]) != t->sel_mask[w]) ok = 0;
    if (ok && (t->flags & CCSIM_TF_HAS_AFFINITY_TERMS)) {
      int any = 0; /* terms are ORed; zero terms match nothing (nodeaffinity.go:84-100) */
      for (int k = 0; k < t->n_aff_terms && !any; k++) {
        int m = 1;
        for (int w = 0; w < nd->static_words; w++)
          if ((word(nd->static_mask, n, w, i) & t->aff_term_mask[k][w]) != t->aff_term_mask[k][w]) m = 0;
        any = m;
      }
      ok = any;
    }
    if (!ok) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_NODE_AFFINITY; *n_reasons = nr; }
      return ST_UNRESOLVABLE;
    }
  }
  /* NodePorts: PL:nodeports/node_ports.go:68-76 (Skip), :157-185 */
  if ((t->filter_enable & CCSIM_PL_NODE_PORTS) && (t->flags & CCSIM_TF_HAS_HOST_PORTS)) {
    int conflict = 0;
    for (int w = 0; w < nd->static_words; w++)
      if (word(nd->static_mask, n, w, i) & t->port_static_mask[w]) conflict = 1;
    if (s->placed_mask && (s->placed_mask[i] & t->port_tmpl_conflict)) conflict = 1;
    if (conflict) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_NODE_PORTS; *n_reasons = nr; }
      return ST_UNSCHEDULABLE;
    }
  }
  /* NodeResourcesFit: PL:noderesources/fit.go:564-660 (fitsRequest), :509-533 (all reasons kept) */
  if (t->filter_enable & CCSIM_PL_FIT) {
    int fail = 0, unres = 0;
    if (s->npods[i] + 1 > nd->alloc_pods[i]) { fail = 1; if (want_reasons) reasons[nr++] = CCSIM_R_TOO_MANY_PODS; }
    if (!(t->flags & CCSIM_TF_FIT_ALL_ZERO)) {
      if (t->req_cpu > 0 && t->req_cpu > nd->alloc_cpu[i] - s->req_cpu[i]) {
        fail = 1; if (t->req_cpu > nd->alloc_cpu[i]) unres = 1;
        if (want_reasons) reasons[nr++] = CCSIM_R_INSUFFICIENT_CPU;
      }
      if (t->req_mem > 0 && t->req_mem > nd->alloc_mem[i] - s->req_mem[i]) {
        fail = 1; if (t->req_mem > nd->alloc_mem[i]) unres = 1;
        if (want_reasons) reasons[nr++] = CCSIM_R_INSUFFICIENT_MEMORY;
      }
      if (t->req_eph > 0 && t->req_eph > nd->alloc_eph[i] - s->req_eph[i]) {
        fail = 1; if (t->req_eph > nd->alloc_eph[i]) unres = 1;
        if (want_reasons) reasons[nr++] = CCSIM_R_INSUFFICIENT_EPHEMERAL;
      }
      for (int k = 0; k < nd->n_scalars; k++) {
        int64_t q = t->req_scalar[k];
        if (q == 0) continue;
        if (q > nd->alloc_scalar[k][i] - s->req_scalar[k][i]) {
          fail = 1; if (q > nd->alloc_scalar[k][i]) unres = 1;
          if (want_reasons) reasons[nr++] = CCSIM_R_SCALAR0 + k;
        }
      }
    }
    if (fail) { if (want_reasons) *n_reasons = nr; return unres ? ST_UNRESOLVABLE : ST_UNSCHEDULABLE; }
  }
  /* PodTopologySpread: PL:podtopologyspread/filtering.go:311-356 */
  if ((t->filter_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD)) {
    for (int c = 0; c < t->n_pts; c++) {
      const ccsim_pts *p = &t->pts[c];
      const ccsim_counter *cc = &ctr[p->counter];
      int32_t dom = cc->topo_col < 0 ? i : nd->topo[cc->topo_col][i];
      if (dom < 0) {
        if (want_reasons) { reasons[nr++] = CCSIM_R_PTS_MISSING_LABEL; *n_reasons = nr; }
        return ST_UNRESOLVABLE;
      }
      int64_t skew = (int64_t)s->cnt[p->counter][dom] + p->self_match - (int64_t)ptsmin[c];
      if (skew > p->max_skew) {
        if (want_reasons) { reasons[nr++] = CCSIM_R_PTS_SKEW; *n_reasons = nr; }
        return ST_UNSCHEDULABLE;
      }
    }
  }
  /* InterPodAffinity: PL:interpodaffinity/filtering.go:352-432 */
  if (t->filter_enable & CCSIM_PL_INTER_POD_AFFINITY) {
    /* satisfyPodAffinity :382-408 */
    int pods_exist = 1, missing = 0;
    for (int a = 0; a < t->n_aff; a++) {
      const ccsim_counter *cc = &ctr[t->aff_counter[a]];
      int32_t dom = cc->topo_col < 0 ? i : nd->topo[cc->topo_col][i];
      if (dom < 0) { missing = 1; break; }
      if (s->cnt[t->aff_counter[a]][dom] <= 0) pods_exist = 0;
    }
    if (missing || (!pods_exist && !(s->aff_total == 0 && (t->flags & CCSIM_TF_AFF_SELF_MATCH_ALL)))) {
      if (want_reasons) { reasons[nr++] = CCSIM_R_IPA_AFFINITY; *n_reasons = nr; }
      return ST_UNRESOLVABLE;
    }
    /* satisfyPodAntiAffinity :367-379 */
    for (int a = 0; a < t->n_anti; a++) {
      const ccsim_counter *cc = &ctr[t->anti_counter[a]];
      int32_t dom = cc->topo_col < 0 ? i : nd->topo[cc->topo_col][i];
      if (dom >= 0 && s->cnt[t->anti_counter[a]][dom] > 0) {
        if (want_reasons) { reasons[nr++] = CCSIM_R_IPA_ANTI_AFFINITY; *n_reasons = nr; }
        return ST_UNSCHEDULABLE;
      }
    }
    /* satisfyExistingPodsAntiAffinity :352-364 (static part; the clones' part coincides with the check above) */
    for (int w = 0; w < nd->static_words; w++)
      if (word(nd->static_mask, n, w, i) & t->existing_anti_mask[w]) {
        if (want_reasons) { reasons[nr++] = CCSIM_R_IPA_EXISTING_ANTI; *n_reasons = nr; }
        return ST_UNSCHEDULABLE;
      }
  }
  if (want_reasons) *n_reasons = 0;
  return ST_OK;
}

/* PL:noderesources/least_allocated.go:52-61 */
static inline int64_t least_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) return 0;
  return ((capacity - requested) * 100) / capacity;
}

/* Fit.Score with LeastAllocated: PL:noderesources/resource_allocation.go:48-114 (NonZeroRequested + pod request),
 * least_allocated.go:30-48 */
static int64_t score_least_v(int64_t alloc_cpu, int64_t alloc_mem, int64_t nz_cpu, int64_t nz_mem, const ccsim_template *t) {
  int64_t node_score = 0, weight_sum = 0;
  int64_t alloc[2] = { alloc_cpu, alloc_mem };
  int64_t req[2] = { nz_cpu + t->least_cpu, nz_mem + t->least_mem };
  int64_t w[2] = { t->least_w_cpu, t->least_w_mem };
  for (int k = 0; k < 2; k++) {
    if (alloc[k] == 0) continue;
    node_score += least_requested_score(req[k], alloc[k]) * w[k];
    weight_sum += w[k];
  }
  if (weight_sum == 0) return 0;
  return node_score / weight_sum;
}

/* BalancedAllocation: PL:noderesources/balanced_allocation.go:146-180 (Requested + pod request, float64) */
static int64_t score_balanced_v(int64_t alloc_cpu, int64_t alloc_mem, int64_t req_cpu, int64_t req_mem, const ccsim_template *t) {
  volatile double f[2]; /* volatile: no contraction / excess precision */
  int nf = 0;
  int64_t alloc[2] = { alloc_cpu, alloc_mem };
  int64_t req[2] = { req_cpu + t->bal_cpu, req_mem + t->bal_mem };
  for (int k = 0; k < 2; k++) {
    if (alloc[k] == 0) continue;
    double fr = (double)req[k] / (double)alloc[k];
    if (fr > 1) fr = 1;
    f[nf++] = fr;
  }
  volatile double std = 0.0;
  if (nf == 2) { volatile double d = f[0] - f[1]; volatile double h = d / 2; std = fabs(h); }
  volatile double one_minus = 1 - std;
  volatile double sc = one_minus * 100.0;
  return (int64_t)sc;
}

static int64_t score_least(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, int32_t i) {
  return score_least_v(nd->alloc_cpu[i], nd->alloc_mem[i], s->nz_cpu[i], s->nz_mem[i], t);
}
static int64_t score_balanced(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, int32_t i) {
  return score_balanced_v(nd->alloc_cpu[i], nd->alloc_mem[i], s->req_cpu[i], s->req_mem[i], t);
}

/* raw TaintToleration score: PL:tainttoleration/taint_toleration.go:154-182 */
static int taint_raw(const ccsim_nodes *nd, const ccsim_template *t, int32_t i) {
  int c = 0;
  for (int w = 0; w < nd->taint_words; w++)
    c += __builtin_popcountll(word(nd->taint_mask, nd->n_nodes, w, i) & nd->taint_prefer[w] & ~t->tol_prefer[w]);
  return c;
}

/* raw NodeAffinity score: PL:nodeaffinity/node_affinity.go:265-290 (sum of the weights of the matching preferred terms) */
static int64_t node_affinity_raw(const ccsim_nodes *nd, const ccsim_template *t, int32_t i) {
  int64_t c = 0;
  for (int k = 0; k < t->n_pref_terms; k++) {
    int m = 1;
    for (int w = 0; w < nd->static_words; w++)
      if ((word(nd->static_mask, nd->n_nodes, w, i) & t->pref_mask[k][w]) != t->pref_mask[k][w]) m = 0;
    if (m) c += t->pref_weight[k];
  }
  return c;
}

static inline int static_bit(const ccsim_nodes *nd, int32_t i, int b) {
  return (int)((word(nd->static_mask, nd->n_nodes, b >> 6, i) >> (b & 63)) & 1ull);
}

/* Go's math.Log on amd64: the pure-Go port of FreeBSD's e_log.c (go/src/math/log.go:80-129; only s390x has an
 * assembly version). No fused multiply-add (GOAMD64=v1), hence -ffp-contract=off. Finite x > 0 only. */
static double go_log(double x) {
  const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10;
  const double L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01, L3 = 2.857142874366239149e-01,
               L4 = 2.222219843214978396e-01, L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01,
               L7 = 1.479819860511658591e-01;
  int ki; double f1 = frexp(x, &ki);
  if (f1 < 0.70710678118654752440 /* Sqrt2/2 */) { f1 *= 2; ki--; }
  const double f = f1 - 1, k = (double)ki;
  const double s = f / (2 + f), s2 = s * s, s4 = s2 * s2;
  const double t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)));
  const double t2 = s4 * (L2 + s4 * (L4 + s4 * L6));
  const double R = t1 + t2, hfsq = 0.5 * f * f;
  return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f);
}

/* PodTopologySpread.Score for one node given the cycle's weights (PL:podtopologyspread/scoring.go:192-224,302-304);
 * the caller has already excluded IgnoredNodes */
static int64_t spts_raw(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, const ccsim_counter *ctr,
                        const double *weight, int32_t i) {
  double score = 0;
  for (int c = 0; c < t->n_spts; c++) {
    const ccsim_spts *sc = &t->spts[c];
    int64_t cnt;
    if (sc->hostname) {
      if (sc->has_key_bit >= 0 && !static_bit(nd, i, sc->has_key_bit)) continue;
      cnt = s->cnt[sc->counter][i];
    } else {
      const int32_t dom = nd->topo[ctr[sc->counter].topo_col][i];
      if (dom < 0) continue;
      cnt = s->cnt[sc->counter][dom];
    }
    score += (double)cnt * weight[c] + (double)(sc->max_skew - 1);
  }
  return (int64_t)round(score);   /* math.Round: half away from zero */
}

/* InterPodAffinity.Score (PL:interpodaffinity/scoring.go:236-256) */
static int64_t ipa_raw(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, const ccsim_counter *ctr, int32_t i) {
  int64_t sc = 0;
  for (int k = 0; k < t->n_ipa_score; k++) {
    const int j = t->ipa_score_counter[k];
    const int32_t dom = ctr[j].topo_col < 0 ? i : nd->topo[ctr[j].topo_col][i];
    if (dom >= 0) sc += s->cnt[j][dom];
  }
  return sc;
}

/* KS:schedule_one.go:697-723 */
static int32_t num_feasible_nodes_to_find(int32_t n, int32_t pct) {
  if (n < 100) return n;
  if (pct == 0) { pct = 50 - n / 125; if (pct < 5) pct = 5; }
  int32_t k = (int32_t)((int64_t)n * pct / 100);
  if (k < 100) return 100;
  return k;
}

/* the part of the node score that does not depend on the feasible set */
static inline int64_t score_rest(const ccsim_nodes *nd, const ostate *s, const ccsim_template *t, int32_t i) {
  int64_t sc = 0;
  if (t->score_enable & CCSIM_PL_FIT) sc += (int64_t)t->w_fit * score_least(nd, s, t, i);
  if ((t->score_enable & CCSIM_PL_BALANCED) && !(t->flags & CCSIM_TF_BALANCED_SKIP))
    sc += (int64_t)t->w_balanced * score_balanced(nd, s, t, i);
  /* ImageLocality: static per node (PL:imagelocality/image_locality.go:54-131); NULL = no node holds an image of the pod */
  if ((t->score_enable & CCSIM_PL_IMAGE_LOCALITY) && t->image_score) sc += (int64_t)t->w_image * t->image_score[i];
  return sc;
}

/* flags bit 0 (CCSIM_ORACLE_MEMO): memoise score_rest per (template, node) and recompute it only after that node was committed.
 * score_rest depends on the node's own Requested / NonZeroRequested and the template only, so the results are identical (a test
 * compares both); it makes full-size parity runs affordable. The timed CPU baseline never sets it: the reference rescores every
 * feasible node in every cycle (KS:schedule_one.go:776-886). */
#define CCSIM_ORACLE_MEMO 1
int ccsim_oracle_run_ex(const ccsim_nodes *nd, int32_t n_templates, const ccsim_template *tmpl,
                        int32_t n_counters, const ccsim_counter *ctr,
                        int64_t max_pods, int32_t mode, int32_t pct_nodes_to_score, int32_t threads, int32_t flags,
                        ccsim_result *out, int32_t *pod_node, int64_t pod_node_cap);
int ccsim_oracle_run(const ccsim_nodes *nd, int32_t n_templates, const ccsim_template *tmpl,
                     int32_t n_counters, const ccsim_counter *ctr,
                     int64_t max_pods, int32_t mode, int32_t pct_nodes_to_score, int32_t threads,
                     ccsim_result *out, int32_t *pod_node, int64_t pod_node_cap) {
  return ccsim_oracle_run_ex(nd, n_templates, tmpl, n_counters, ctr, max_pods, mode, pct_nodes_to_score, threads, 0, out, pod_node, pod_node_cap);
}
int ccsim_oracle_run_ex(const ccsim_nodes *nd, int32_t n_templates, const ccsim_template *tmpl,
                        int32_t n_counters, const ccsim_counter *ctr,
                        int64_t max_pods, int32_t mode, int32_t pct_nodes_to_score, int32_t threads, int32_t flags,
                        ccsim_result *out, int32_t *pod_node, int64_t pod_node_cap) {
  const int32_t n = nd->n_nodes;
  if (n_templates < 1 || n_templates > CCSIM_MAX_TEMPLATES || n_counters > CCSIM_MAX_COUNTERS) return CCSIM_EINVAL;
  if (n_templates > 1 && n_counters > 0) return CCSIM_EUNSUPPORTED;
  for (int j = 0; j < n_counters; j++)
    for (int t = 0; t < n_templates; t++)
      for (int c = 0; c < tmpl[t].n_pts; c++)
        if (tmpl[t].pts[c].counter == j && ctr[j].topo_col < 0) return CCSIM_EUNSUPPORTED;
  /* Preconditions the engine checks too (ccsim_load_nodes / ccsim_set_templates): LeastAllocated's (capacity - requested) * 100
     must not wrap, and no plugin weight is negative (so every feasible node's total is >= 0 > best's initial -1). Resource
     weights in [1, 100]: NodeResourcesFitArgs validation (PL:../apis/config/validation/validation_pluginargs.go). */
  for (int32_t i = 0; i < n; i++)
    if (nd->alloc_cpu[i] > CCSIM_MAX_SCORED_ALLOCATABLE || nd->alloc_mem[i] > CCSIM_MAX_SCORED_ALLOCATABLE) return CCSIM_EUNSUPPORTED;
  for (int t = 0; t < n_templates; t++) {
    const ccsim_template *T = &tmpl[t];
    if (T->w_taint < 0 || T->w_node_affinity < 0 || T->w_fit < 0 || T->w_pts < 0 || T->w_ipa < 0 || T->w_balanced < 0 || T->w_image < 0 ||
        T->least_w_cpu < 1 || T->least_w_cpu > 100 || T->least_w_mem < 1 || T->least_w_mem > 100)
      return CCSIM_EUNSUPPORTED;
  }
  /* The per-domain counters are int32 (s.cnt), the reference's counts int64 (PL:podtopologyspread/scoring.go:192-224,
     PL:interpodaffinity/scoring.go:236-256): refuse a counter that could leave int32 within the run, as the engine does
     (ccsim_prepare). A domain receives at most min(placements, its free pod slots) commits while NodeResourcesFit filters
     (fit.go:567-576), at most `placements` otherwise; placements = min(max_pods, the cluster's free pod slots). */
  {
    int64_t bound = 0;
    int fit_off = 0;
    for (int32_t i = 0; i < n; i++) if (nd->alloc_pods[i] > nd->npods[i]) bound += (int64_t)nd->alloc_pods[i] - nd->npods[i];
    for (int t = 0; t < n_templates; t++) if (!(tmpl[t].filter_enable & CCSIM_PL_FIT)) fit_off = 1;
    if (max_pods > 0 && (max_pods < bound || fit_off)) bound = max_pods;
    for (int j = 0; j < n_counters; j++) {
      const int64_t inc = llabs((long long)ctr[j].inc);
      if (inc == 0 || ctr[j].n_domains <= 0) continue;
      int64_t *slots = (int64_t*)calloc((size_t)ctr[j].n_domains, 8);
      for (int32_t i = 0; i < n; i++) {
        const int32_t d = ctr[j].topo_col < 0 ? i : nd->topo[ctr[j].topo_col][i];
        if (d >= 0 && d < ctr[j].n_domains && nd->alloc_pods[i] > nd->npods[i]) slots[d] += (int64_t)nd->alloc_pods[i] - nd->npods[i];
      }
      int refuse = 0;
      for (int32_t d = 0; d < ctr[j].n_domains && !refuse; d++) {
        const int64_t m = fit_off || slots[d] > bound ? bound : slots[d];
        if (m > 0 && llabs((long long)ctr[j].init[d]) + m * inc > INT32_MAX) refuse = 1;
      }
      free(slots);
      if (refuse) return CCSIM_EUNSUPPORTED;
    }
  }
#ifdef _OPENMP
  if (threads > 0) omp_set_num_threads(threads);
#else
  (void)threads;
#endif
  memset(out, 0, sizeof(*out));
  out->n_nodes = n;

  ostate s; memset(&s, 0, sizeof(s));
  size_t b64 = (size_t)(n > 0 ? n : 1) * sizeof(int64_t);
#define DUP64(dst, src) do { dst = (int64_t*)malloc(b64); if (n) memcpy(dst, src, (size_t)n * 8); } while (0)
  DUP64(s.req_cpu, nd->req_cpu); DUP64(s.req_mem, nd->req_mem); DUP64(s.req_eph, nd->req_eph);
  DUP64(s.nz_cpu, nd->nz_cpu); DUP64(s.nz_mem, nd->nz_mem);
  for (int k = 0; k < nd->n_scalars; k++) DUP64(s.req_scalar[k], nd->req_scalar[k]);
  s.npods = (int32_t*)malloc((size_t)(n > 0 ? n : 1) * 4); if (n) memcpy(s.npods, nd->npods, (size_t)n * 4);
  s.placed_mask = nd->has_placed_mask ? (uint64_t*)calloc((size_t)(n > 0 ? n : 1), 8) : NULL;
  for (int j = 0; j < n_counters; j++) {
    int32_t d = ctr[j].n_domains > 0 ? ctr[j].n_domains : 1;
    s.cnt[j] = (int32_t*)malloc((size_t)d * 4);
    if (ctr[j].n_domains) memcpy(s.cnt[j], ctr[j].init, (size_t)ctr[j].n_domains * 4);
  }
  s.aff_total = tmpl[0].aff_total_init;

  int32_t *memo = NULL;                     /* [n_templates][n] memoised score_rest, -1 = stale */
  if ((flags & CCSIM_ORACLE_MEMO) && mode == 0 && n > 0) {
    memo = (int32_t*)malloc((size_t)n_templates * (size_t)n * 4);
    if (memo) memset(memo, 0xff, (size_t)n_templates * (size_t)n * 4);
  }
  int64_t *key = (int64_t*)malloc(b64);     /* per-node rest score or -1 if infeasible */
  int32_t *raw = (int32_t*)malloc((size_t)(n > 0 ? n : 1) * 4);
  int64_t placed = 0, waves = 0, evals = 0;
  int32_t start = 0;
  int stop = CCSIM_STOP_UNSCHEDULABLE;
  const ccsim_template *tfail = &tmpl[0];
  int32_t ptsmin_fail[CCSIM_MAX_PTS] = {0};

  /* KS:scheduler.go:68 ErrNoNodesAvailable is a host-side message; with n == 0 nothing is placed. */
  for (int64_t k = 0; n > 0; k++) {
    const int ti = (int)(k % n_templates);           /* R:pkg/framework/report.go:160 (i % templatesCount) */
    const ccsim_template *t = &tmpl[ti];
    int32_t ptsmin[CCSIM_MAX_PTS];
    for (int c = 0; c < t->n_pts; c++) ptsmin[c] = pts_min(&ctr[t->pts[c].counter], s.cnt[t->pts[c].counter], &t->pts[c]);

    int32_t examined = n;
    int64_t feasible = 0;
    int32_t maxraw_par = 0;   /* canonical mode: max raw TaintToleration score over the feasible nodes, reduced inside the filter loop */
    if (mode == 0) {
      /* findNodesThatPassFilters, all nodes: KS:schedule_one.go:610-693 */
      int64_t fc = 0;
      int32_t mr = 0;
      #pragma omp parallel for schedule(static) reduction(+:fc) reduction(max:mr) if(n >= 4096)
      for (int32_t i = 0; i < n; i++) {
        int st = filter_node(nd, &s, t, ti, ctr, ptsmin, i, 0, NULL, NULL);
        if (st == ST_OK) {
          if (memo) { int32_t *m = &memo[(size_t)ti * (size_t)n + i]; if (*m < 0) *m = (int32_t)score_rest(nd, &s, t, i); key[i] = *m; }
          else key[i] = score_rest(nd, &s, t, i);
          raw[i] = (t->score_enable & CCSIM_PL_TAINT_TOLERATION) ? taint_raw(nd, t, i) : 0; fc++;
          if (raw[i] > mr) mr = raw[i];
        }
        else key[i] = -1;
      }
      feasible = fc; maxraw_par = mr;
    } else {
      int32_t want = num_feasible_nodes_to_find(n, pct_nodes_to_score);
      examined = 0;
      for (int32_t i = 0; i < n; i++) key[i] = -2; /* not examined */
      for (int32_t q = 0; q < n && feasible < want; q++) {
        int32_t i = (start + q) % n;
        examined++;
        int st = filter_node(nd, &s, t, ti, ctr, ptsmin, i, 0, NULL, NULL);
        if (st == ST_OK) { key[i] = score_rest(nd, &s, t, i); raw[i] = (t->score_enable & CCSIM_PL_TAINT_TOLERATION) ? taint_raw(nd, t, i) : 0; feasible++; }
        else key[i] = -1;
      }
    }
    waves++; evals += examined;
    if (feasible == 0) { stop = CCSIM_STOP_UNSCHEDULABLE; tfail = t; memcpy(ptsmin_fail, ptsmin, sizeof(ptsmin)); break; }

    /* prioritizeNodes + selectHost: KS:schedule_one.go:776-886,894-941; RunScorePlugins KS:framework/runtime/framework.go:1137-1244.
       TaintToleration NormalizeScore: PL:helper/normalize_score.go:28-56 (reverse=true) over the feasible set. */
    int32_t maxraw = 0;
    if (t->score_enable & CCSIM_PL_TAINT_TOLERATION) {
      if (mode == 0) maxraw = maxraw_par;
      else for (int32_t i = 0; i < n; i++) if (key[i] >= 0 && raw[i] > maxraw) maxraw = raw[i];
    }
    /* NodeAffinity preferred terms: PreScore Skip when the pod has none (node_affinity.go:246-249); else
       DefaultNormalizeScore(100, reverse=false) over the feasible nodes (PL:helper/normalize_score.go:28-56) */
    const int na_on = (t->score_enable & CCSIM_PL_NODE_AFFINITY) && t->n_pref_terms > 0;
    int64_t na_max = 0;
    if (na_on)
      for (int32_t i = 0; i < n; i++) if (key[i] >= 0) { int64_t r = node_affinity_raw(nd, t, i); if (r > na_max) na_max = r; }
    /* PodTopologySpread PreScore/Score/NormalizeScore over the feasible nodes (PL:podtopologyspread/scoring.go:60-265) */
    const int spts_on = (t->score_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD) && t->n_spts > 0;
    double spts_w[CCSIM_MAX_PTS]; int64_t spts_min = INT64_MAX, spts_max = 0;
    if (spts_on) {
      int64_t scored = 0;
      for (int32_t i = 0; i < n; i++)
        if (key[i] >= 0 && !(t->spts_ignored_bit >= 0 && static_bit(nd, i, t->spts_ignored_bit))) scored++;
      for (int c = 0; c < t->n_spts; c++) {
        int64_t size = scored;
        if (!t->spts[c].hostname) {   /* distinct values among the scored nodes; a missing key reads as the value "" */
          const ccsim_counter *cc = &ctr[t->spts[c].counter];
          uint8_t *seen = (uint8_t*)calloc((size_t)cc->n_domains + 1, 1);
          size = 0;
          for (int32_t i = 0; i < n; i++) {
            if (key[i] < 0 || (t->spts_ignored_bit >= 0 && static_bit(nd, i, t->spts_ignored_bit))) continue;
            int32_t dom = nd->topo[cc->topo_col][i];
            if (dom < 0) dom = cc->n_domains;
            if (!seen[dom]) { seen[dom] = 1; size++; }
          }
          free(seen);
        }
        spts_w[c] = go_log((double)(size + 2));
      }
      for (int32_t i = 0; i < n; i++) {
        if (key[i] < 0 || (t->spts_ignored_bit >= 0 && static_bit(nd, i, t->spts_ignored_bit))) continue;
        const int64_t r = spts_raw(nd, &s, t, ctr, spts_w, i);
        if (r < spts_min) spts_min = r;
        if (r > spts_max) spts_max = r;
      }
    }
    /* InterPodAffinity NormalizeScore (PL:interpodaffinity/scoring.go:258-290) */
    const int ipa_on = (t->score_enable & CCSIM_PL_INTER_POD_AFFINITY) && t->n_ipa_score > 0;
    int64_t ipa_min = INT64_MAX, ipa_max = INT64_MIN;
    if (ipa_on)
      for (int32_t i = 0; i < n; i++) if (key[i] >= 0) {
        const int64_t r = ipa_raw(nd, &s, t, ctr, i);
        if (r < ipa_min) ipa_min = r;
        if (r > ipa_max) ipa_max = r;
      }
    int64_t best = -1; int32_t besti = -1;
    if (mode == 0 && !na_on && !spts_on && !ipa_on && n >= 4096) {
      /* Same arg-max as the loop below (first maximum in node order), split over the node axis like the reference's own
         16-way parallel score pass (KS:framework/parallelize/parallelism.go:28-78): every thread keeps the first maximum of its
         contiguous block, the blocks are combined in ascending order with a strict '>' */
      const int tt_on = (t->score_enable & CCSIM_PL_TAINT_TOLERATION) != 0;
      int64_t tb[256]; int32_t tbi[256]; int nth = 1;
#ifdef _OPENMP
      const int nthr_want = omp_get_max_threads() < 256 ? omp_get_max_threads() : 256;
#else
      const int nthr_want = 1;
#endif
      (void)nthr_want;
      #pragma omp parallel num_threads(nthr_want)
      {
#ifdef _OPENMP
        const int me = omp_get_thread_num(), nt = omp_get_num_threads();
#else
        const int me = 0, nt = 1;
#endif
        const int32_t per = (n + nt - 1) / nt, lo = me * per < n ? me * per : n, hi = lo + per < n ? lo + per : n;
        int64_t b = -1; int32_t bi = -1;
        for (int32_t i = lo; i < hi; i++) {
          if (key[i] < 0) continue;
          int64_t total = key[i];
          if (tt_on) total += (int64_t)t->w_taint * ((maxraw == 0) ? 100 : 100 - (100 * (int64_t)raw[i] / maxraw));
          if (total > b) { b = total; bi = i; }
        }
        tb[me] = b; tbi[me] = bi;
        if (me == 0) nth = nt;
      }
      for (int q = 0; q < nth; q++) if (tb[q] > best) { best = tb[q]; besti = tbi[q]; }
    } else
    for (int32_t q = 0; q < n; q++) {
      int32_t i = (mode == 0) ? q : (start + q) % n;
      if (key[i] < 0) continue;
      int64_t total = key[i];
      if (t->score_enable & CCSIM_PL_TAINT_TOLERATION) {
        int64_t tt = (maxraw == 0) ? 100 : 100 - (100 * (int64_t)raw[i] / maxraw);
        total += (int64_t)t->w_taint * tt;
      }
      if (na_on) {
        int64_t r = node_affinity_raw(nd, t, i);
        total += (int64_t)t->w_node_affinity * (na_max == 0 ? r : 100 * r / na_max);
      }
      if (spts_on && !(t->spts_ignored_bit >= 0 && static_bit(nd, i, t->spts_ignored_bit))) {
        const int64_t r = spts_raw(nd, &s, t, ctr, spts_w, i);
        total += (int64_t)t->w_pts * (spts_max == 0 ? 100 : 100 * (spts_max + spts_min - r) / spts_max);
      }
      if (ipa_on && ipa_max > ipa_min) {
        const int64_t r = ipa_raw(nd, &s, t, ctr, i);
        const double f = 100.0 * ((double)(r - ipa_min) / (double)(ipa_max - ipa_min));
        total += (int64_t)t->w_ipa * (int64_t)f;
      }
      if (total > best) { best = total; besti = i; }
    }
    if (mode != 0) start = (int32_t)(((int64_t)start + examined) % n); /* KS:schedule_one.go:538-539 */
    assert(besti >= 0);   /* feasible > 0 and every total >= 0 (the weight preconditions above) */

    /* assume -> Cache.AssumePod -> NodeInfo.AddPod -> update(+1): KS:framework/types.go:409-427 */
    const int32_t w = besti;
    s.req_cpu[w] += t->req_cpu; s.req_mem[w] += t->req_mem; s.req_eph[w] += t->req_eph;
    for (int q = 0; q < nd->n_scalars; q++) s.req_scalar[q][w] += t->req_scalar[q];
    s.nz_cpu[w] += t->nz_cpu; s.nz_mem[w] += t->nz_mem;
    s.npods[w] += 1;
    if (memo) for (int q = 0; q < n_templates; q++) memo[(size_t)q * (size_t)n + w] = -1;
    if (s.placed_mask) s.placed_mask[w] |= (1ull << ti);
    /* per-domain counters: the next cycle's PreFilter recount sees this clone
       (PL:podtopologyspread/filtering.go:255-289; PL:interpodaffinity/filtering.go:234-271) */
    for (int j = 0; j < n_counters; j++) {
      if (ctr[j].inc == 0) continue;
      int is_aff = 0;
      for (int a = 0; a < t->n_aff; a++) if (t->aff_counter[a] == j) is_aff = 1;
      if (is_aff && !(t->flags & CCSIM_TF_AFF_SELF_MATCH_ALL)) continue;
      if (ctr[j].elig_bit >= 0 && !static_bit(nd, w, ctr[j].elig_bit)) continue;
      int32_t dom = ctr[j].topo_col < 0 ? w : nd->topo[ctr[j].topo_col][w];
      if (dom < 0) continue;
      s.cnt[j][dom] += ctr[j].inc;
      if (is_aff) s.aff_total += ctr[j].inc;
    }
    /* ClusterCapacityBinder.Bind + postBindHook: R:pkg/framework/plugins/clustercapacitybinder/plugin.go:34-53,
       R:pkg/framework/simulator.go:297-312 */
    if (pod_node && placed < pod_node_cap) pod_node[placed] = w;
    placed++;
    if (max_pods > 0 && placed >= max_pods) { stop = CCSIM_STOP_LIMIT_REACHED; break; }
  }

  out->placed = placed; out->stop_code = stop; out->waves = waves; out->evals = evals; out->examined = evals;
  if (stop == CCSIM_STOP_UNSCHEDULABLE && n > 0) {
    /* FitError histogram: KS:framework/types.go:787-838; preemption suffix: KS:framework/preemption/preemption.go:234-331,
       PL:defaultpreemption/default_preemption.go:218-258 (no lower-priority victims on any node) */
    int ti = (int)(placed % n_templates);
    for (int32_t i = 0; i < n; i++) {
      int rs[8 + CCSIM_MAX_SCALARS], nr = 0;
      int st = filter_node(nd, &s, tfail, ti, ctr, ptsmin_fail, i, 1, rs, &nr);
      for (int q = 0; q < nr; q++) out->reason_hist[rs[q]]++;
      if (st == ST_UNSCHEDULABLE) out->preempt_no_victims++;
      else out->preempt_not_helpful++;
    }
  }
  out->pod_node = pod_node;

  free(key); free(raw); free(memo);
  free(s.req_cpu); free(s.req_mem); free(s.req_eph); free(s.nz_cpu); free(s.nz_mem); free(s.npods); free(s.placed_mask);
  for (int k = 0; k < nd->n_scalars; k++) free(s.req_scalar[k]);
  for (int j = 0; j < n_counters; j++) free(s.cnt[j]);
  return CCSIM_OK;
}

/* Per-node score trajectory helper for known-answer tests (KA1 of SURVEY.md §8c): total score of node i for
 * template t with k clones already committed, all other plugins constant. */
int64_t ccsim_oracle_node_score(const ccsim_nodes *nd, const ccsim_template *t, int32_t i, int32_t clones,
                                int64_t *least_out, int64_t *balanced_out) {
  int64_t rc = nd->req_cpu[i] + clones * t->req_cpu, rm = nd->req_mem[i] + clones * t->req_mem;
  int64_t zc = nd->nz_cpu[i] + clones * t->nz_cpu, zm = nd->nz_mem[i] + clones * t->nz_mem;
  int64_t l = score_least_v(nd->alloc_cpu[i], nd->alloc_mem[i], zc, zm, t);
  int64_t b = score_balanced_v(nd->alloc_cpu[i], nd->alloc_mem[i], rc, rm, t);
  if (least_out) *least_out = l;
  if (balanced_out) *balanced_out = b;
  int64_t total = 0;
  if (t->score_enable & CCSIM_PL_FIT) total += t->w_fit * l;
  if ((t->score_enable & CCSIM_PL_BALANCED) && !(t->flags & CCSIM_TF_BALANCED_SKIP)) total += t->w_balanced * b;
  if (t->score_enable & CCSIM_PL_TAINT_TOLERATION) total += t->w_taint * 100;
  return total;
}
