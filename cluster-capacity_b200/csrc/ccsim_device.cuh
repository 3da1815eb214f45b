// ccsim_device.cuh — device-side data layout and the per-node predicate / score functions (sm_90a).
//
// One predicate-eval = one (pod attempt, node) pair through eval_node(): what checkNode does once in the reference
// (vendor/k8s.io/kubernetes/pkg/scheduler/schedule_one.go:644-666 -> framework/runtime/framework.go:897-930), followed
// for feasible nodes by the node-local part of RunScorePlugins (framework.go:1137-1244).
//
// Integer/indexing work only: int64 compares, one exact int64 quotient in [0,100] per scored resource
// (least_allocated.go:52-61), IEEE float64 for BalancedAllocation (balanced_allocation.go:146-180) with explicit
// round-to-nearest intrinsics so that nothing is contracted into an FMA.
#pragma once
#include <stdint.h>
#include <limits.h>
#include "../../include/ccsim.h"

#define CCSIM_MAX_GRID 160  /* >= SM count of the part (H100 SXM: 132) */
#define SLOT_STRIDE 16      /* 64-bit words per CTA slot: one 128-byte L2 line per CTA (sharing a line between writers costs ~2x) */

struct DevCounter {
  int32_t topo_col;   // -1: node-local column
  int32_t n_domains;
  int32_t n_present;
  int32_t inc;
  int32_t smem_off;   // offset (in int32) into the CTA's shared counter area, or -1: per-CTA replica in global memory
  int32_t is_aff;     // counter belongs to a required pod-affinity key
  int32_t elig_bit;   // static bit a node needs for its commits to count, -1 = every node
  int32_t pad;
  int32_t *init;      // [n_domains] device copy of the initial counts (node-local: snapshot column)
  int32_t *work;      // node-local: working column [n]; replicated-global: base of grid*n_domains replicas
};

struct DevOut {
  int64_t placed;
  int32_t stop_code;
  int32_t error;      // 0 ok, 1 watchdog (a CTA never saw its peers' slots), 2 pod_node overflow
  int64_t waves;
  int64_t evals;
  int64_t examined;                // reference-equivalent nodes examined (== evals unless sampling)
  int32_t ptsmin[CCSIM_MAX_PTS];   // global minima at the terminal cycle (for the diagnosis pass)
  int64_t aff_total;
  unsigned long long reason_hist[CCSIM_R_TOTAL];
  unsigned long long preempt_no_victims;
  unsigned long long n_diag;
  long long phase_cycles[8];       // CTA 0's cycles per phase (multi-commit kernel: always; other kernels: CCSIM_PHASE_TIMERS builds)
  long long stat[4];               // multi-commit kernel: [0] candidates replayed (sum over waves), [1] waves that had to raise the bar T,
                                   // [2] replay rounds, [3] waves replayed in key order (low 32 bits) and waves that selected each
                                   // tile's candidates from the sorted tile (high 32 bits)
};

// DevParams::debug_flags, set from CCSIM_DEBUG_FLAGS (kernel experiments; INTEGRATION.md lists the same values)
constexpr uint32_t DBG_RESCAN_EVERY_MOVE = 1u;    // a multi-commit wave ends at every PTS minimum move
constexpr uint32_t DBG_RECOUNT_EVERY_WAVE = 2u;   // the multi-commit kernel recounts every PTS minimum after every wave
constexpr uint32_t DBG_WAVE_LINES = 4u;           // one line per wave of the multi-commit kernel
constexpr uint32_t DBG_CYCLES = 8u;               // replay / per-CTA cycle summary at the end of a run
constexpr uint32_t DBG_STRICT_ONLY = 16u;         // strict multi-commit waves only (no look-ahead)
constexpr uint32_t DBG_LOOKAHEAD_ALWAYS = 32u;    // look-ahead on every spread term in every wave
constexpr uint32_t DBG_ARGMAX_ROUND = 64u;        // single-use multi-commit waves keep the arg-max replay round instead of key order
constexpr uint32_t DBG_REDUX_SELECT = 128u;       // single-use multi-commit waves select each tile's candidates by REDUX rounds and a merge
constexpr uint32_t DBG_EACH_ONE_PER_CTA = 256u;   // per-analysis runs launch one CTA per analysis however many analyses there are

struct DevParams {
  int32_t n;            // nodes of this shard
  int32_t n_global;     // nodes of the whole cluster
  int32_t node_base;    // global index of local node 0
  int32_t n_scalars, taint_words, static_words, n_topo, n_templates, n_counters, n_classes;
  int32_t grid;         // CTAs of the persistent kernel
  int32_t chunk;        // nodes per CTA (contiguous ownership)
  int32_t rank, world;
  uint32_t epoch;       // run counter (1..255), folded into every exchanged word
  uint32_t debug_flags; // CCSIM_DEBUG_FLAGS (kernel experiments): the DBG_* bits below
  uint32_t xwave0;      // node-sharded runs: exchanges done by earlier runs of this handle; the double-buffer parity of the cross-GPU
                        // buffers continues across runs, so wave 0 of a run never lands in the buffer a lagging peer CTA still reads
  long long sample_k;   // numFeasibleNodesToFind (reference sampling mode)
  // immutable columns
  const int64_t *alloc_cpu, *alloc_mem, *alloc_eph;
  const int32_t *alloc_pods;
  const int64_t *alloc_scalar[CCSIM_MAX_SCALARS];
  const uint64_t *taint_mask, *static_mask;
  const int32_t *topo[CCSIM_MAX_TOPO_COLS];
  // mutable working columns (restored from the snapshot copies before each run)
  int64_t *req_cpu, *req_mem, *req_eph, *nz_cpu, *nz_mem;
  int32_t *npods;
  int64_t *req_scalar[CCSIM_MAX_SCALARS];
  uint64_t *placed_mask;   // nullptr unless a template has hostPorts
  uint8_t *feas;           // per-node feasibility flag of the current wave (multi-phase scoring: normalised soft scorers)
  uint32_t *stamp[CCSIM_MAX_PTS];   // soft PTS constraint c (non-hostname): [n_domains + 1] "a scored node of wave k+1 is in this domain"
  int32_t *score_cache;    // memoised node-local score per node, -1 = stale (streaming mode; resident mode keeps it in the tile)
  int32_t tile_resident;   // 1: the CTA's node tile is staged into shared memory once and stays there for the whole run
  int32_t chunk_pad;       // chunk rounded up to a multiple of 4 (tile column stride)
  int32_t n_local;         // node-local counters (each gets a tile column in resident mode)
  int32_t smem_cnt_ints;   // size of the shared replicated-counter area
  uint64_t taint_nosched[CCSIM_MAX_TAINT_WORDS], taint_prefer[CCSIM_MAX_TAINT_WORDS];
  const ccsim_template *templates;
  DevCounter counters[CCSIM_MAX_COUNTERS];
  int32_t *final_cnt;      // concatenated final replicated counters (written by CTA 0 at exit)
  int32_t final_off[CCSIM_MAX_COUNTERS];
  // exchange: slots[parity][cta][class]
  unsigned long long *slots;
  // cross-GPU exchange (node-sharded run): xslots[parity][rank][SLOT_STRIDE] lives in every rank's memory;
  // xslots_peer[r] is rank r's copy as mapped into this process (CUDA IPC over NVLink), xslots_peer[rank] the local one
  unsigned long long *xslots_peer[CCSIM_MAX_WORLD];
  const int32_t *topo_full[CCSIM_MAX_TOPO_COLS];   // whole-cluster topology columns (sharded runs: winners of other shards)
  int32_t *pod_node;
  int64_t pod_cap;
  int64_t max_pods;
  DevOut *out;
  const int32_t *taint_list_off;
  const uint8_t *taint_list;
  const DevParams *self;   // device-memory copy of this struct, for the out-of-line slow paths
};

// ---- key packing ----------------------------------------------------------------------------------------------
// [63:56] run epoch  [55:44] wave tag (1..4095)  [43:32] score+1 (0 = no feasible node)  [31:0] 0xFFFFFFFF - global node index
// max over keys = highest score, ties -> lowest node index = "first max in scan order" (selectHost, schedule_one.go:894-941).
// The epoch makes words left over from an earlier Run (in particular in the cross-GPU buffers, which cannot be cleared
// without a host barrier) never validate. Scores are < 4095 (checked on the host: sum of weights * 100).
#define KEY_TAG_SHIFT 44
#define KEY_BODY_MASK ((1ull << KEY_TAG_SHIFT) - 1)
__device__ __forceinline__ unsigned long long pack_key(int64_t score, uint32_t gidx) {
  return ((unsigned long long)(score + 1) << 32) | (unsigned long long)(0xFFFFFFFFu - gidx);
}
__device__ __forceinline__ int64_t key_score(unsigned long long k) { return (int64_t)((k & KEY_BODY_MASK) >> 32) - 1; }
__device__ __forceinline__ uint32_t key_index(unsigned long long k) { return 0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFu); }

// ---- exact scorers --------------------------------------------------------------------------------------------
// leastRequestedScore: ((capacity - requested) * 100) / capacity, truncating int64 (least_allocated.go:52-61).
// The quotient is in [0,100]: estimate in fp32, then repair with one exact int64 remainder test (no 64-bit divide).
__device__ __forceinline__ int64_t least_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) return 0;
  const int64_t x100 = (capacity - requested) * 100;
  int64_t q = (int64_t)(__fdividef((float)x100, (float)capacity));
  int64_t r = x100 - q * capacity;
  if (r < 0) { q -= 1; r += capacity; if (r < 0) { q = x100 / capacity; } }
  else if (r >= capacity) { q += 1; r -= capacity; if (r >= capacity) { q = x100 / capacity; } }
  return q;
}

struct ScoreWeights { int32_t w_fit, w_balanced, least_w_cpu, least_w_mem; };

// Fit.Score with LeastAllocated over cpu,mem: resource_allocation.go:48-114 + least_allocated.go:30-48.
// q_* = NonZeroRequested + the pod's non-zero request.
__device__ __forceinline__ int64_t score_least(int64_t a_cpu, int64_t a_mem, int64_t q_cpu, int64_t q_mem,
                                               int32_t w_cpu, int32_t w_mem) {
  int64_t node_score = 0, wsum = 0;
  if (a_cpu != 0) { node_score += least_requested_score(q_cpu, a_cpu) * w_cpu; wsum += w_cpu; }
  if (a_mem != 0) { node_score += least_requested_score(q_mem, a_mem) * w_mem; wsum += w_mem; }
  if (wsum == 0) return 0;
  if (wsum == 2) return node_score >> 1;   // both weights 1 (default): node_score >= 0
  return node_score / wsum;
}

// balancedResourceScorer over cpu,mem (balanced_allocation.go:146-180): float64, one rounding per operation.
// q_* = Requested + the pod's request.
__device__ __noinline__ int64_t score_balanced_f64(int64_t a_cpu, int64_t a_mem, int64_t q_cpu, int64_t q_mem) {
  double f0 = 0.0, f1 = 0.0;
  int nf = 0;
  if (a_cpu != 0) {
    double fr = __ddiv_rn((double)q_cpu, (double)a_cpu);
    if (fr > 1.0) fr = 1.0;
    f0 = fr; nf = 1;
  }
  if (a_mem != 0) {
    double fr = __ddiv_rn((double)q_mem, (double)a_mem);
    if (fr > 1.0) fr = 1.0;
    if (nf == 0) f0 = fr; else f1 = fr;
    nf++;
  }
  double sd = 0.0;
  if (nf == 2) sd = fabs(__dmul_rn(__dsub_rn(f0, f1), 0.5));   // (f0-f1)/2: exact scaling by a power of two
  return (int64_t)__dmul_rn(__dsub_rn(1.0, sd), 100.0);
}
// The float64 result is int64((1-std)*100). An fp32 estimate of (1-std)*100 is within 1e-3 of the float64 value
// (three fp32 roundings + two approximate divides on operands in [0,1]); when the estimate is at least 1/64 away from
// an integer boundary the truncation is decided and the float64 sequence is skipped. Otherwise (ties, f0==f1, clipped
// fractions) the exact float64 path runs. Bit-exactness is therefore never estimated, only the fast path's eligibility.
__device__ __forceinline__ int64_t score_balanced(int64_t a_cpu, int64_t a_mem, int64_t q_cpu, int64_t q_mem) {
  if (a_cpu > 0 && a_mem > 0 && q_cpu >= 0 && q_mem >= 0) {
    const float g0 = fminf(__fdividef((float)q_cpu, (float)a_cpu), 1.0f);
    const float g1 = fminf(__fdividef((float)q_mem, (float)a_mem), 1.0f);
    const float v = (1.0f - fabsf(g0 - g1) * 0.5f) * 100.0f;
    const float fl = floorf(v);
    const float fr = v - fl;
    if (fr > 0.015625f && fr < 0.984375f) return (int64_t)fl;
  }
  return score_balanced_f64(a_cpu, a_mem, q_cpu, q_mem);
}

// ---- per-wave constants of the fused Filter pass (shared memory; rebuilt when the template or a PTS minimum changes) ----
// Everything that depends only on the template is folded into a handful of masks / thresholds so that the per-node
// work is: 7 coalesced loads, ~10 integer ops, plus one (load, shared-memory counter read, compare) per coupled term.
#define CCSIM_X_TAINT_WORDS   (1u << 0)   /* taint dictionary wider than one word                   */
#define CCSIM_X_STATIC_WORDS  (1u << 1)   /* static bits wider than one word / nodeAffinity terms   */
#define CCSIM_X_SCALARS       (1u << 2)   /* extended resources requested                           */
#define CCSIM_X_NODENAME      (1u << 3)
#define CCSIM_X_PREFILTER     (1u << 4)
#define CCSIM_X_PLACED        (1u << 5)   /* hostPorts vs. clones already placed                    */
#define CCSIM_X_EPH           (1u << 6)

struct CoupledTerm {
  const int32_t *col;   // topology column (nullptr: node-local, the counter is indexed by the node itself)
  const int32_t *cnt;   // counter base (shared or global replica, or the node-local working column)
};

struct FilterConsts {
  unsigned long long taint_bad0;   // word 0: untolerated NoSchedule/NoExecute entries | unschedulable bit
  unsigned long long prefer0;      // word 0: PreferNoSchedule entries not tolerated (score classes)
  unsigned long long sel0;         // static word 0: bits that must all be set (nodeSelector)
  unsigned long long forbid0;      // static word 0: bits that must all be clear (port conflicts, existing anti-affinity)
  long long eq_cpu, eq_mem, eq_eph; // effective requests (LLONG_MIN: check disabled)
  int32_t fit_pods;                // 1: npods + 1 > allowedPodNumber rejects
  uint32_t extras;                 // CCSIM_X_*
  int32_t n_pts, n_aff, n_anti, aff_bypass;
  int32_t tmpl_index;
  int32_t pts_lim[CCSIM_MAX_PTS];  // reject when cnt > lim  (lim = maxSkew - selfMatch + globalMin)
  CoupledTerm pts[CCSIM_MAX_PTS], aff[CCSIM_MAX_IPA], anti[CCSIM_MAX_IPA];
};

// Node tile of a CTA. Every pointer is pre-offset so that [i] with the shard-local node index i works, whether the
// tile lives in shared memory (resident mode) or is the global column itself (streaming mode).
// Resident mode keeps the three Fit inputs as differences (free = allocatable - requested: fit.go:585-616 compares the
// pod request against exactly this difference), updated at commit, next to the raw columns the scorers need.
struct Tile {
  const unsigned long long *taint0, *static0;
  const int32_t *alloc_pods;
  int32_t *npods;
  const long long *alloc_cpu, *alloc_mem;
  long long *req_cpu, *req_mem, *nz_cpu, *nz_mem;
  long long *free_cpu, *free_mem;   // resident mode only
  int32_t *free_pods;               // resident mode only: allowedPodNumber - len(Pods)
  int32_t *score;     // memoised node-local score, -1 = stale
};

// one thread: fold template t into FilterConsts. topo_ptr[k] / cnt_ptr[j] are the (pre-offset) bases of topology
// column k and of counter j as this CTA sees them.
// PodTopologySpread's Filter bound for a domain count (filtering.go:341-351): reject when cnt > maxSkew - selfMatch + globalMin
__device__ __forceinline__ int32_t pts_limit(const ccsim_pts &pc, int32_t ptsmin) {
  const long long lim = (long long)pc.max_skew - pc.self_match + (long long)ptsmin;
  return lim > INT32_MAX ? INT32_MAX : (lim < INT32_MIN ? INT32_MIN : (int32_t)lim);
}

// counters: the counter table t's indexes refer to (p.counters, or a per-analysis table of ccsim_run_each)
__device__ void build_filter_consts(const DevParams &p, const DevCounter *counters, const ccsim_template &t, int32_t ti,
                                    const int32_t *const *topo_ptr, int32_t *const *cnt_ptr, const int32_t *ptsmin, long long aff_total,
                                    FilterConsts &fc) {
  const uint32_t fe = t.filter_enable, fl = t.flags;
  fc.tmpl_index = ti;
  unsigned long long tb = 0ull;
  if (fe & CCSIM_PL_TAINT_TOLERATION) tb |= p.taint_nosched[0] & ~t.tol_nosched[0] & ~(1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT);
  if ((fe & CCSIM_PL_NODE_UNSCHEDULABLE) && !(fl & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) tb |= 1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT;
  fc.taint_bad0 = tb;
  fc.prefer0 = (t.score_enable & CCSIM_PL_TAINT_TOLERATION) ? (p.taint_prefer[0] & ~t.tol_prefer[0]) : 0ull;
  const bool aff_on = (fe & CCSIM_PL_NODE_AFFINITY) && (fl & (CCSIM_TF_HAS_NODE_SELECTOR | CCSIM_TF_HAS_AFFINITY_TERMS));
  fc.sel0 = (aff_on && p.static_words > 0) ? t.sel_mask[0] : 0ull;
  unsigned long long fb = 0ull;
  if (p.static_words > 0) {
    if ((fe & CCSIM_PL_NODE_PORTS) && (fl & CCSIM_TF_HAS_HOST_PORTS)) fb |= t.port_static_mask[0];
    if (fe & CCSIM_PL_INTER_POD_AFFINITY) fb |= t.existing_anti_mask[0];
  }
  fc.forbid0 = fb;
  const bool fit = (fe & CCSIM_PL_FIT) != 0, nz = fit && !(fl & CCSIM_TF_FIT_ALL_ZERO);
  fc.fit_pods = fit ? 1 : 0;
  fc.eq_cpu = (nz && t.req_cpu > 0) ? t.req_cpu : LLONG_MIN;
  fc.eq_mem = (nz && t.req_mem > 0) ? t.req_mem : LLONG_MIN;
  fc.eq_eph = (nz && t.req_eph > 0) ? t.req_eph : LLONG_MIN;
  uint32_t x = 0;
  if (p.taint_words > 1) x |= CCSIM_X_TAINT_WORDS;
  if (p.static_words > 1 || (aff_on && (fl & CCSIM_TF_HAS_AFFINITY_TERMS))) x |= CCSIM_X_STATIC_WORDS;
  if (nz) for (int k = 0; k < p.n_scalars; k++) if (t.req_scalar[k] != 0) x |= CCSIM_X_SCALARS;
  if ((fe & CCSIM_PL_NODE_NAME) && t.nodename_idx >= 0) x |= CCSIM_X_NODENAME;
  if (fl & CCSIM_TF_PREFILTER_NODES) x |= CCSIM_X_PREFILTER;
  if ((fe & CCSIM_PL_NODE_PORTS) && (fl & CCSIM_TF_HAS_HOST_PORTS) && p.placed_mask) x |= CCSIM_X_PLACED;
  if (fc.eq_eph != LLONG_MIN) x |= CCSIM_X_EPH;
  fc.extras = x;
  fc.n_pts = (fe & CCSIM_PL_POD_TOPOLOGY_SPREAD) ? t.n_pts : 0;
  for (int c = 0; c < fc.n_pts; c++) {
    const DevCounter &dc = counters[t.pts[c].counter];
    fc.pts[c].col = dc.topo_col < 0 ? nullptr : topo_ptr[dc.topo_col];
    fc.pts[c].cnt = cnt_ptr[t.pts[c].counter];
    fc.pts_lim[c] = pts_limit(t.pts[c], ptsmin[c]);
  }
  const bool ipa = (fe & CCSIM_PL_INTER_POD_AFFINITY) != 0;
  fc.n_aff = ipa ? t.n_aff : 0;
  fc.n_anti = ipa ? t.n_anti : 0;
  for (int a = 0; a < fc.n_aff; a++) {
    const DevCounter &dc = counters[t.aff_counter[a]];
    fc.aff[a].col = dc.topo_col < 0 ? nullptr : topo_ptr[dc.topo_col];
    fc.aff[a].cnt = cnt_ptr[t.aff_counter[a]];
  }
  for (int a = 0; a < fc.n_anti; a++) {
    const DevCounter &dc = counters[t.anti_counter[a]];
    fc.anti[a].col = dc.topo_col < 0 ? nullptr : topo_ptr[dc.topo_col];
    fc.anti[a].cnt = cnt_ptr[t.anti_counter[a]];
  }
  fc.aff_bypass = (aff_total == 0 && (fl & CCSIM_TF_AFF_SELF_MATCH_ALL)) ? 1 : 0;
}
__device__ __forceinline__ void build_filter_consts(const DevParams &p, const ccsim_template &t, int32_t ti, const int32_t *const *topo_ptr,
                                                    int32_t *const *cnt_ptr, const int32_t *ptsmin, long long aff_total, FilterConsts &fc) {
  build_filter_consts(p, p.counters, t, ti, topo_ptr, cnt_ptr, ptsmin, aff_total, fc);
}

// status codes for the diagnosis pass
#define ST_OK 0
#define ST_UNSCHEDULABLE 1
#define ST_UNRESOLVABLE 2

// the uncommon predicates (wide dictionaries, nodeAffinity terms, extended resources, nodeName, hostPorts vs clones)
__device__ __noinline__ bool filter_extras(const DevParams *pp, int32_t ti, uint32_t extras, int32_t i) {
  const DevParams &p = *pp;
  const ccsim_template &t = p.templates[ti];
  const int32_t n = p.n;
  bool ok = true;
  if (extras & CCSIM_X_PREFILTER) {
    const int b = t.prefilter_bit;
    ok &= (bool)((p.static_mask[(size_t)(b >> 6) * n + i] >> (b & 63)) & 1ull);
  }
  if (extras & CCSIM_X_NODENAME) ok &= (t.nodename_idx == p.node_base + i);
  if ((extras & CCSIM_X_TAINT_WORDS) && (t.filter_enable & CCSIM_PL_TAINT_TOLERATION))
    for (int w = 1; w < p.taint_words; w++) ok &= ((p.taint_mask[(size_t)w * n + i] & p.taint_nosched[w] & ~t.tol_nosched[w]) == 0);
  if (extras & CCSIM_X_STATIC_WORDS) {
    uint64_t sw[CCSIM_MAX_STATIC_WORDS];
    for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) sw[w] = (w < p.static_words) ? p.static_mask[(size_t)w * n + i] : 0ull;
    if ((t.filter_enable & CCSIM_PL_NODE_AFFINITY) && (t.flags & (CCSIM_TF_HAS_NODE_SELECTOR | CCSIM_TF_HAS_AFFINITY_TERMS))) {
      bool m = true;
      for (int w = 1; w < CCSIM_MAX_STATIC_WORDS; w++) m &= ((sw[w] & t.sel_mask[w]) == t.sel_mask[w]);
      if (t.flags & CCSIM_TF_HAS_AFFINITY_TERMS) {   // terms are ORed; zero terms match nothing
        bool any = false;
        for (int k = 0; k < t.n_aff_terms; k++) {
          bool tm = true;
          for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) tm &= ((sw[w] & t.aff_term_mask[k][w]) == t.aff_term_mask[k][w]);
          any |= tm;
        }
        m &= any;
      }
      ok &= m;
    }
    uint64_t c = 0;
    if ((t.filter_enable & CCSIM_PL_NODE_PORTS) && (t.flags & CCSIM_TF_HAS_HOST_PORTS))
      for (int w = 1; w < CCSIM_MAX_STATIC_WORDS; w++) c |= sw[w] & t.port_static_mask[w];
    if (t.filter_enable & CCSIM_PL_INTER_POD_AFFINITY)
      for (int w = 1; w < CCSIM_MAX_STATIC_WORDS; w++) c |= sw[w] & t.existing_anti_mask[w];
    ok &= (c == 0);
  }
  if (extras & CCSIM_X_PLACED) ok &= ((p.placed_mask[i] & t.port_tmpl_conflict) == 0);
  if (extras & CCSIM_X_EPH) ok &= !(t.req_eph > p.alloc_eph[i] - p.req_eph[i]);
  if (extras & CCSIM_X_SCALARS)
    for (int k = 0; k < p.n_scalars; k++) {
      const int64_t q = t.req_scalar[k];
      if (q != 0) ok &= !(q > p.alloc_scalar[k][i] - p.req_scalar[k][i]);
    }
  return ok;
}

// untolerated PreferNoSchedule taints of node i in taint words 1.. (word 0's are counted inline): the rest of its TaintToleration
// raw score, i.e. of its normalisation class
__device__ __noinline__ int prefer_count_hi(const DevParams *pp, int32_t ti, int32_t i) {
  const DevParams &p = *pp;
  const ccsim_template &t = p.templates[ti];
  if (!(t.score_enable & CCSIM_PL_TAINT_TOLERATION)) return 0;
  int c = 0;
  for (int w = 1; w < p.taint_words; w++) c += __popcll(p.taint_mask[(size_t)w * p.n + i] & p.taint_prefer[w] & ~t.tol_prefer[w]);
  return c;
}

// register copy of the FilterConsts fields every node needs (hoisted out of the node loop)
struct HotConsts {
  unsigned long long taint_bad0, prefer0, sel0, forbid0;
  long long eq_cpu, eq_mem;
  int32_t fit_pods, pods_need, n_pts, n_aff, n_anti;
  uint32_t extras;
};
__device__ __forceinline__ HotConsts load_hot(const FilterConsts &fc) {
  HotConsts h;
  h.taint_bad0 = fc.taint_bad0; h.prefer0 = fc.prefer0; h.sel0 = fc.sel0; h.forbid0 = fc.forbid0;
  h.eq_cpu = fc.eq_cpu; h.eq_mem = fc.eq_mem; h.fit_pods = fc.fit_pods; h.pods_need = fc.fit_pods ? 1 : INT32_MIN;
  h.n_pts = fc.n_pts; h.n_aff = fc.n_aff; h.n_anti = fc.n_anti; h.extras = fc.extras;
  return h;
}

// The coupled Filter terms of node i, ANDed into ok: PodTopologySpread hard constraints (podtopologyspread/filtering.go:311-356) and
// InterPodAffinity required terms (interpodaffinity/filtering.go:367-432). sel picks the terms: bit c spread constraint c, bit 8 + a
// affinity key a, bit 16 + a anti-affinity key a; ALL: every term, sel unused (filter_node). The affinity test splits exactly over the
// terms: with the bypass every selected key must be present, without it every selected key must also count a pod.
#define COUPLED_AFF_SEL(a) (1u << (8 + (a)))
#define COUPLED_ANTI_SEL(a) (1u << (16 + (a)))
template <bool ALL>
__device__ __forceinline__ void coupled_ok(const FilterConsts &fc, int n_pts, int n_aff, int n_anti, int32_t i, uint32_t sel, bool &ok) {
  for (int c = 0; c < n_pts; c++) {
    if (!ALL && !((sel >> c) & 1u)) continue;
    const int32_t dom = fc.pts[c].col ? fc.pts[c].col[i] : i;
    ok &= (dom >= 0) && !(fc.pts[c].cnt[dom < 0 ? 0 : dom] > fc.pts_lim[c]);
  }
  if (n_aff) {
    bool pods_exist = true, missing = false;
    for (int a = 0; a < n_aff; a++) {
      if (!ALL && !(sel & COUPLED_AFF_SEL(a))) continue;
      const int32_t dom = fc.aff[a].col ? fc.aff[a].col[i] : i;
      missing |= (dom < 0);
      pods_exist &= (dom >= 0) && (fc.aff[a].cnt[dom < 0 ? 0 : dom] > 0);
    }
    ok &= !(missing || (!pods_exist && !fc.aff_bypass));
  }
  for (int a = 0; a < n_anti; a++) {
    if (!ALL && !(sel & COUPLED_ANTI_SEL(a))) continue;
    const int32_t dom = fc.anti[a].col ? fc.anti[a].col[i] : i;
    ok &= !((dom >= 0) && (fc.anti[a].cnt[dom < 0 ? 0 : dom] > 0));
  }
}

// Hot path: the fused Filter pass for node i (shard-local index). One predicate-eval.
// Plugin order does not matter for feasibility (the AND of all enabled plugins); the order only matters for the
// FitError reasons, which the terminal diagnosis kernel reproduces.
template <bool RESIDENT>
__device__ __forceinline__ bool filter_node(const DevParams &p, const HotConsts &hc, const FilterConsts &fc,
                                            const Tile &tl, int32_t i, int &raw) {
  // NodeUnschedulable + TaintToleration (node_unschedulable.go:133-150, taint_toleration.go:111-122)
  const unsigned long long taint0 = tl.taint0[i];
  bool ok = (taint0 & hc.taint_bad0) == 0ull;
  raw = __popcll(taint0 & hc.prefer0);
  // NodeResourcesFit (fit.go:564-660)
  if (RESIDENT) {
    ok &= !(hc.pods_need > tl.free_pods[i]);
    ok &= !(hc.eq_cpu > tl.free_cpu[i]);
    ok &= !(hc.eq_mem > tl.free_mem[i]);
  } else {
    ok &= !(hc.fit_pods && tl.npods[i] + 1 > tl.alloc_pods[i]);
    ok &= !(hc.eq_cpu > tl.alloc_cpu[i] - tl.req_cpu[i]);
    ok &= !(hc.eq_mem > tl.alloc_mem[i] - tl.req_mem[i]);
  }
  // NodeAffinity nodeSelector, NodePorts, existing pods' anti-affinity: static bits
  if (hc.sel0 | hc.forbid0) {
    const unsigned long long sw = tl.static0[i];
    ok &= ((~sw & hc.sel0) | (sw & hc.forbid0)) == 0ull;
  }
  coupled_ok<true>(fc, hc.n_pts, hc.n_aff, hc.n_anti, i, 0u, ok);
  if (hc.extras && ok) ok = filter_extras(p.self, fc.tmpl_index, hc.extras, i);
  if ((hc.extras & CCSIM_X_TAINT_WORDS) && ok) raw += prefer_count_hi(p.self, fc.tmpl_index, i);
  return ok;
}

// node-local score of a feasible node (framework.go:1137-1244: plugin score * weight, summed); depends only on the
// node's own NodeInfo and the template, so it is memoised per node until that node is committed again (the
// reference's snapshot likewise only refreshes NodeInfos whose generation changed: backend/cache/cache.go:194-288).
// lq_* = NonZeroRequested + pod non-zero request (LeastAllocated); bq_* = Requested + pod request (BalancedAllocation).
__device__ __noinline__ int32_t score_node(int64_t a_cpu, int64_t a_mem, int64_t lq_cpu, int64_t lq_mem,
                                           int64_t bq_cpu, int64_t bq_mem, ScoreWeights sw) {
  int64_t sc = 0;
  if (sw.w_fit) sc += (int64_t)sw.w_fit * score_least(a_cpu, a_mem, lq_cpu, lq_mem, sw.least_w_cpu, sw.least_w_mem);
  if (sw.w_balanced) sc += (int64_t)sw.w_balanced * score_balanced(a_cpu, a_mem, bq_cpu, bq_mem);
  return (int32_t)sc;
}

// ------------------------------------------------------------------------------------------------------------------
// slot exchange primitives: relaxed 64-bit accesses that bypass L1 (the tag inside the word carries the ordering)
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_slot(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_slot(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// warp-wide max of a packed 64-bit key with two REDUX.MAX.U32 (high word, then low word among the lanes that tie)
// system-scope variants for words that cross NVLink (peer memory)
__device__ __forceinline__ void st_slot_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_slot_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
  const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
  const unsigned mhi = __reduce_max_sync(0xffffffffu, hi);
  const unsigned mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
  return ((unsigned long long)mhi << 32) | mlo;
}


struct CommitInfo {
  const int32_t *gtopo;   // global topology column (any node)
  const int32_t *ltopo;   // this CTA's view of it (pre-offset tile column in resident mode)
  int32_t inc;            // 0: this template does not touch the counter
  int32_t pts_idx;        // PTS constraint tracking its minimum on this counter, or -1
  int32_t n_present;
  int32_t is_aff;
  int32_t local;          // node-local counter
  int32_t elig_bit;       // static bit the winner must carry, -1 none
};


#ifndef WATCHDOG_SPINS
#define WATCHDOG_SPINS (1u << 24)
#endif
// CTA 0's cycles per phase of the lean and generic kernels; the kernel declares ph[8], tc0 and tc1 in CCSIM_PHASE_TIMERS builds
#ifdef CCSIM_PHASE_TIMERS
#define PH_START() do { if (cta == 0 && tid == 0) tc0 = clock64(); } while (0)
#define PH_MARK(i) do { if (cta == 0 && tid == 0) { tc1 = clock64(); ph[i] += tc1 - tc0; tc0 = tc1; } } while (0)
#else
#define PH_START() do {} while (0)
#define PH_MARK(i) do {} while (0)
#endif

// Second level of the per-wave exchange for node-sharded multi-GPU runs (warp 0 of every CTA, after the intra-GPU gather):
// CTA 0 stores this GPU's class winners, tagged, into EVERY rank's exchange buffer (P2P stores over NVLink; 8-byte stores
// are single transactions, the tag inside the word validates it), then every CTA polls its LOCAL copy for all ranks.
// This is the whole collective: an all-gather of one word per rank fused into the kernel, no NCCL call per wave.
__device__ __forceinline__ bool cross_gpu_exchange(const DevParams &p, long long k, uint32_t tag, int ncls,
                                                   unsigned long long *cbest, int lane, int cta) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  const size_t base = (size_t)((k + p.xwave0) & 1) * CCSIM_MAX_WORLD * SLOT_STRIDE;
  if (cta == 0 && lane < p.world)
    for (int c = 0; c < ncls; c++) st_slot_sys(&p.xslots_peer[lane][base + (size_t)p.rank * SLOT_STRIDE + c], cbest[c] | tagbits);
  const unsigned long long *local = p.xslots_peer[p.rank] + base;
  bool dead = false;
  for (int c = 0; c < ncls; c++) {
    unsigned long long v = tagbits;
    unsigned spins = 0;
    bool pending;
    do {
      if (lane < p.world) v = ld_slot_sys(&local[(size_t)lane * SLOT_STRIDE + c]);
      pending = ((uint32_t)(v >> KEY_TAG_SHIFT) != tag);
      if (++spins > WATCHDOG_SPINS) { dead = true; break; }
    } while (__any_sync(0xffffffffu, pending));
    cbest[c] = warp_max_u64(lane < p.world ? (v & KEY_BODY_MASK) : 0ull);
  }
  return __any_sync(0xffffffffu, dead);
}

// ---- tagged-word gather: the grid-wide half of an intra-GPU exchange --------------------------------------------------
// Each CTA publishes one word, tagged with the wave, in word `word` of its slot line of parity k & 1; warp 0 of every CTA then
// waits here until the word of every CTA carries `tag`. All of a lane's loads are in flight together. On return v[q] holds the
// body of CTA lane + 32 q's word (0 past the grid); the result is true when the watchdog expired first. Every lane leaves the
// loop in the same iteration, but the compiler cannot see that: gather_tagged votes the flag, poll_tagged leaves the vote to
// a caller that schedules it after its own reduction.
#define GATHER_Q (CCSIM_MAX_GRID / 32)
__device__ __forceinline__ bool poll_tagged(const DevParams &p, long long k, uint32_t tag, int word, int lane,
                                            unsigned long long (&v)[GATHER_Q]) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  const unsigned long long *all = p.slots + (size_t)(k & 1) * CCSIM_MAX_GRID * SLOT_STRIDE + word;
  unsigned spins = 0;
  bool pending, dead = false;
  do {
    pending = false;
    #pragma unroll
    for (int q = 0; q < GATHER_Q; q++) { const int b = lane + 32 * q; v[q] = (b < p.grid) ? ld_slot(&all[(size_t)b * SLOT_STRIDE]) : tagbits; }
    #pragma unroll
    for (int q = 0; q < GATHER_Q; q++) pending |= ((uint32_t)(v[q] >> KEY_TAG_SHIFT) != tag);
    if (++spins > WATCHDOG_SPINS) { dead = true; break; }
  } while (__any_sync(0xffffffffu, pending));
  #pragma unroll
  for (int q = 0; q < GATHER_Q; q++) v[q] &= KEY_BODY_MASK;
  return dead;
}
__device__ __forceinline__ bool gather_tagged(const DevParams &p, long long k, uint32_t tag, int word, int lane,
                                              unsigned long long (&v)[GATHER_Q]) {
  return __any_sync(0xffffffffu, poll_tagged(p, k, tag, word, lane, v));
}
// the largest gathered body (keys: the winner; 0 = no CTA had one)
__device__ __forceinline__ unsigned long long gather_max(const unsigned long long (&v)[GATHER_Q]) {
  unsigned long long m = 0ull;
  #pragma unroll
  for (int q = 0; q < GATHER_Q; q++) m = v[q] > m ? v[q] : m;
  return warp_max_u64(m);
}
// the sum of the gathered bodies of the CTAs below `cta`, and of all of them
__device__ __forceinline__ void gather_prefix_total(const unsigned long long (&v)[GATHER_Q], int lane, int cta,
                                                    unsigned long long &prefix, unsigned long long &total) {
  unsigned long long pre = 0, tot = 0;
  #pragma unroll
  for (int q = 0; q < GATHER_Q; q++) {
    tot += v[q];
    if (lane + 32 * q < cta) pre += v[q];
  }
  for (int o = 16; o > 0; o >>= 1) { pre += __shfl_xor_sync(0xffffffffu, pre, o); tot += __shfl_xor_sync(0xffffffffu, tot, o); }
  prefix = pre; total = tot;
}

// Several grid-wide maxima at once: lane q < NV publishes vals[q] (< 2^44, 0 = "nothing") in word word0+q of this CTA's
// slot line; every CTA then gathers all lines. One wait for the slowest CTA, the remaining words are already there.
template <int NV>
__device__ __forceinline__ void exchange_max_n(const DevParams &p, long long k, uint32_t tag, int word0,
                                               unsigned long long (&vals)[NV], int lane, int cta, bool &dead) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  unsigned long long mine = 0ull;
  #pragma unroll
  for (int q = 0; q < NV; q++) if (lane == q) mine = vals[q];
  if (lane < NV) st_slot(p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE + word0 + lane, (mine & KEY_BODY_MASK) | tagbits);
  #pragma unroll
  for (int w = 0; w < NV; w++) {
    const unsigned long long *all = p.slots + (size_t)(k & 1) * CCSIM_MAX_GRID * SLOT_STRIDE + word0 + w;
    unsigned long long v[CCSIM_MAX_GRID / 32];
    unsigned spins = 0;
    bool pending;
    do {
      pending = false;
      #pragma unroll
      for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) { const int b = lane + 32 * q; v[q] = (b < p.grid) ? ld_slot(&all[(size_t)b * SLOT_STRIDE]) : tagbits; }
      #pragma unroll
      for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) pending |= ((uint32_t)(v[q] >> KEY_TAG_SHIFT) != tag);
      if (++spins > WATCHDOG_SPINS) { dead = true; break; }
    } while (__any_sync(0xffffffffu, pending));
    unsigned long long m = 0ull;
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) { const unsigned long long b = v[q] & KEY_BODY_MASK; m = b > m ? b : m; }
    vals[w] = warp_max_u64(m);
  }
  dead = __any_sync(0xffffffffu, dead);
}

// grid-wide prefix and total of one value per CTA (< 2^44 in total) through word `word` of the slot lines: the sum over the
// CTAs below this one, and over all of them. Returns true, on every lane, when the watchdog expired.
__device__ __forceinline__ bool exchange_prefix_total(const DevParams &p, long long k, uint32_t tag, int word, unsigned long long mine,
                                                      int lane, int cta, unsigned long long &prefix, unsigned long long &total) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  if (lane == 0) st_slot(p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE + word, (mine & KEY_BODY_MASK) | tagbits);
  unsigned long long v[GATHER_Q];
  const bool dead = poll_tagged(p, k, tag, word, lane, v);
  gather_prefix_total(v, lane, cta, prefix, total);
  return __any_sync(0xffffffffu, dead);
}

// grid-wide sum of one count per CTA (< 2^44 in total), with release/acquire fences around it: global stores made by the
// CTA before the call (after a __syncthreads) are visible to every CTA's threads after it (and their next __syncthreads)
__device__ __forceinline__ unsigned long long exchange_sum_fenced(const DevParams &p, long long k, uint32_t tag, int word,
                                                                  unsigned long long mine, int lane, int cta, bool &dead) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  __threadfence();
  if (lane == 0) st_slot(p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE + word, (mine & KEY_BODY_MASK) | tagbits);
  const unsigned long long *all = p.slots + (size_t)(k & 1) * CCSIM_MAX_GRID * SLOT_STRIDE + word;
  unsigned long long v[CCSIM_MAX_GRID / 32];
  unsigned spins = 0;
  bool pending;
  do {
    pending = false;
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) { const int b = lane + 32 * q; v[q] = (b < p.grid) ? ld_slot(&all[(size_t)b * SLOT_STRIDE]) : tagbits; }
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) pending |= ((uint32_t)(v[q] >> KEY_TAG_SHIFT) != tag);
    if (++spins > WATCHDOG_SPINS) { dead = true; break; }
  } while (__any_sync(0xffffffffu, pending));
  __threadfence();
  unsigned long long s = 0ull;
  #pragma unroll
  for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) s += v[q] & KEY_BODY_MASK;
  #pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  dead = __any_sync(0xffffffffu, dead);
  return s;
}

// Shared-memory accesses by explicit 32-bit shared address. nvcc otherwise re-derives the CTA's shared window base (S2UR
// SR_CgaCtaId + ULEA, a slow special-register read) in front of accesses that follow a barrier or a divergent region; inside
// latency-bound single-warp loops that costs more than the access itself. pin_u32 keeps the once-computed base from being
// rematerialised.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t pin_u32(uint32_t v) { uint32_t r; asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(v)); return r; }
__device__ __forceinline__ int32_t lds_s32(uint32_t a) { int32_t v; asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts_s32(uint32_t a, int32_t v) { asm volatile("st.shared.s32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }

__device__ __forceinline__ bool static_bit(const DevParams &p, int32_t i, int b) {
  return (p.static_mask[(size_t)(b >> 6) * p.n + i] >> (b & 63)) & 1ull;
}

// Go's math.Log on amd64 = the pure-Go port of FreeBSD's e_log.c (go/src/math/log.go:80-129), every operation rounded on
// its own (no FMA contraction: GOAMD64=v1). x must be a positive normal number (here: an integer >= 2).
__device__ __noinline__ double go_log(double x) {
  const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10;
  const double L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01, L3 = 2.857142874366239149e-01,
               L4 = 2.222219843214978396e-01, L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01,
               L7 = 1.479819860511658591e-01;
  const unsigned long long bits = (unsigned long long)__double_as_longlong(x);
  int ki = (int)((bits >> 52) & 0x7ffull) - 1022;                                   // Frexp: x = f1 * 2^ki, f1 in [0.5, 1)
  double f1 = __longlong_as_double((long long)((bits & 0x800fffffffffffffull) | (1022ull << 52)));
  if (f1 < 0.70710678118654752440) { f1 = __dmul_rn(f1, 2.0); ki--; }
  const double f = __dsub_rn(f1, 1.0), k = (double)ki;
  const double s = __ddiv_rn(f, __dadd_rn(2.0, f)), s2 = __dmul_rn(s, s), s4 = __dmul_rn(s2, s2);
  const double t1 = __dmul_rn(s2, __dadd_rn(L1, __dmul_rn(s4, __dadd_rn(L3, __dmul_rn(s4, __dadd_rn(L5, __dmul_rn(s4, L7)))))));
  const double t2 = __dmul_rn(s4, __dadd_rn(L2, __dmul_rn(s4, __dadd_rn(L4, __dmul_rn(s4, L6)))));
  const double R = __dadd_rn(t1, t2), hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
  // k*Ln2Hi - ((hfsq - (s*(hfsq+R) + k*Ln2Lo)) - f)
  const double inner = __dadd_rn(__dmul_rn(s, __dadd_rn(hfsq, R)), __dmul_rn(k, Ln2Lo));
  return __dsub_rn(__dmul_rn(k, Ln2Hi), __dsub_rn(__dsub_rn(hfsq, inner), f));
}

// raw NodeAffinity score of a node: sum of the weights of the matching preferred terms (node_affinity.go:265-290)
__device__ __forceinline__ int32_t node_affinity_raw(const DevParams &p, const ccsim_template &t, int32_t i) {
  int32_t raw = 0;
  for (int k = 0; k < t.n_pref_terms; k++) {
    bool m = true;
    for (int w = 0; w < p.static_words; w++) m &= ((p.static_mask[(size_t)w * p.n + i] & t.pref_mask[k][w]) == t.pref_mask[k][w]);
    if (m) raw += t.pref_weight[k];
  }
  return raw;
}

// TaintToleration NormalizeScore, reverse (helper/normalize_score.go:28-56)
__device__ __forceinline__ int64_t taint_norm(int raw, int maxraw) {
  if (maxraw == 0) return 100;
  return 100 - (100 * (int64_t)raw / maxraw);
}

// prioritizeNodes + selectHost over the winners of the normalisation classes (schedule_one.go:776-941): class c holds the
// feasible nodes with c untolerated PreferNoSchedule taints, whose TaintToleration NormalizeScore depends only on c and on the
// highest class present. Returns the winner's key with its total score (0: no feasible node).
__device__ __forceinline__ unsigned long long select_host_over_classes(const unsigned long long *cbest, int ncls, const ccsim_template &t) {
  unsigned long long wkey = cbest[0];
  if (ncls > 1 || (t.score_enable & CCSIM_PL_TAINT_TOLERATION)) {
    int maxraw = 0;
    for (int c = 0; c < ncls; c++) if (cbest[c] != 0ull) maxraw = c;
    wkey = 0ull;
    for (int c = 0; c < ncls; c++) {
      if (cbest[c] == 0ull) continue;
      int64_t total = key_score(cbest[c]);
      if (t.score_enable & CCSIM_PL_TAINT_TOLERATION) total += (int64_t)t.w_taint * taint_norm(c, maxraw);
      const unsigned long long kk = pack_key(total, key_index(cbest[c]));
      wkey = kk > wkey ? kk : wkey;
    }
  }
  return wkey;
}

// PodTopologySpread's global minimum (filtering.go:56-69) as a recount: the minimum of cnt[0..n_present) and how many domains
// hold it, over all NT (== blockDim.x) threads of the block. scratch: NT / 32 ints of shared memory. Every thread gets the minimum; the
// multiplicity is valid in thread 0.
template <int NT>
__device__ __forceinline__ int32_t block_min_count(const int32_t *cnt, int32_t n_present, int32_t *scratch, int32_t &num) {
  int32_t m = INT32_MAX;
  for (int d = threadIdx.x; d < n_present; d += blockDim.x) m = min(m, cnt[d]);
  m = __reduce_min_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = m;
  __syncthreads();
  m = INT32_MAX;
  for (int w = 0; w < NT / 32; w++) m = min(m, scratch[w]);
  __syncthreads();
  int32_t s = 0;
  for (int d = threadIdx.x; d < n_present; d += blockDim.x) s += (cnt[d] == m);
  s = __reduce_add_sync(0xffffffffu, s);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = s;
  __syncthreads();
  num = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < NT / 32; w++) num += scratch[w];
  return m;
}
