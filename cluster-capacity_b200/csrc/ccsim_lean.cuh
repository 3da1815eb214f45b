// ccsim_lean.cuh — the lean resident wave kernel: the common case of the hot path, written for latency.
//
// Eligibility (decided on the host, plan_lean): the CTA tiles fit in shared memory, one template, one taint word,
// at most one static word, none of the "extras" predicates (extended resources, nodeAffinity terms, nodeName, hostPort
// clones, ephemeral storage), every per-domain counter replicated in shared memory or node-local.
// Everything else runs on the generic kernel (ccsim_wave_kernel) with identical results.
//
// Per wave (pod k) every node of the tile goes through the fused Filter pass again from its current state:
//   3 x LDS.128 of the node's hot record  [taint0 | static0] [free_cpu | free_mem] [free_pods | score | dom0 | dom1] (+ more dom/count slots)
//   ~20 integer ops for NodeUnschedulable/TaintToleration/NodeAffinity(nodeSelector)/NodePorts/NodeResourcesFit,
//   one (LDS dom, LDS counter, compare) per PodTopologySpread / InterPodAffinity term,
// then REDUX arg-max, the tagged-word exchange through L2, and the commit by the owner CTA.
// The hot record is AoS with a stride of an odd number of 16-byte units: LDS.128 by consecutive threads is then
// bank-conflict free (each quarter-warp's 8 x 16 B requests land on distinct bank groups).
#pragma once
#include "ccsim_device.cuh"

#define LEAN_THREADS 768
#define LEAN_WARPS (LEAN_THREADS / 32)
#define LEAN_MAX_TERMS 16
#define LEAN_MAX_SLOTS 10   /* extra int32 slots per record: domain ids and node-local counters */

#define LT_PTS 0
#define LT_ANTI 1
#define LT_AFF 2

// int32 indices into a node's hot record, after [taint0 | static0] [free_cpu | free_mem] (ints 0..7)
#define LR_FREE_PODS 8
#define LR_SCORE 9          /* memoised node-local score, < 0: stale */
#define LR_SLOT0 10         /* extra slot s (domain id or node-local count) is int LR_SLOT0 + s */
#define LEAN_COLD_BYTES (6 * 8 + 2 * 4)   /* cold SoA columns per node: alloc/req/nz cpu and mem (int64), alloc_pods, npods (int32) */

// One per-domain term of the Filter pass, 16 bytes (one LDS.128). PodTopologySpread and anti-affinity share one form:
//   reject  <=>  (node has the topology key) ? count(domain) > lim : miss_rejects
// (PTS: lim = maxSkew - selfMatch + globalMin, missing key rejects; anti-affinity: lim = 0, missing key passes).
// Required pod-affinity terms (LT_AFF) need the all-terms "pods exist" logic and are evaluated in a second loop.
struct __align__(16) LeanTerm {
  int16_t kind;      // LT_*
  int16_t miss_rejects;
  int32_t slot;      // record int index (LR_SLOT0 + s) holding the node's domain id, or the node-local count itself
  int32_t cnt_off;   // offset of the counter in the shared replicated-counter area, -1: node-local (the slot IS the count)
  int32_t lim;
};

struct LeanParams {
  int32_t stride_u;        // record stride in 16-byte units (odd)
  int32_t n_slots;         // extra int slots used
  int32_t slot_topo[LEAN_MAX_SLOTS];     // slot s mirrors topology column slot_topo[s] (>=0) ...
  int32_t slot_counter[LEAN_MAX_SLOTS];  // ... or node-local counter slot_counter[s] (>=0)
  int32_t counter_slot[CCSIM_MAX_COUNTERS]; // counter j -> slot holding its domain id (topo) or its count (node-local)
  uint32_t rec_off, cold_off, own_off;   // byte offsets in dynamic shared memory (lean_layout)
};

// The tile of the lean, tie-run and multi-commit kernels in dynamic shared memory, one definition for the host (the kernel's
// shared-memory size, lean_smem_bytes) and the kernels (their pointers, lean_tile):
//   [replicated counters, padded to 16 B] [hot records: stride_u x 16 B per node] [cold columns: LEAN_COLD_BYTES per node]
//   [the kernel's own per-node columns]
inline void lean_layout(LeanParams &lp, int32_t cnt_ints, int32_t chunk_pad) {
  int units = (LR_SLOT0 + lp.n_slots + 3) / 4;
  if ((units & 1) == 0) units++;
  lp.stride_u = units;
  lp.rec_off = ((uint32_t)cnt_ints * 4u + 15u) & ~15u;
  lp.cold_off = lp.rec_off + (uint32_t)units * 16u * (uint32_t)chunk_pad;
  lp.own_off = lp.cold_off + (uint32_t)LEAN_COLD_BYTES * (uint32_t)chunk_pad;
}
inline size_t lean_smem_bytes(const LeanParams &lp, int32_t chunk_pad, size_t own_bytes_per_node) {
  return (size_t)lp.own_off + own_bytes_per_node * (size_t)chunk_pad;
}

struct LeanTile {
  int32_t *cnt;                                     // replicated counter cells
  uint4 *rec;                                       // hot records
  long long *acpu, *amem, *rcpu, *rmem, *zcpu, *zmem;
  int32_t *apods, *npods;
  unsigned char *own;                               // the kernel's own columns
  int32_t su;                                       // record stride in 16-byte units
};

__device__ __forceinline__ LeanTile lean_tile(unsigned char *smem, const LeanParams &lp, size_t cp) {
  LeanTile t;
  t.cnt = reinterpret_cast<int32_t *>(smem);
  t.rec = reinterpret_cast<uint4 *>(smem + lp.rec_off);
  t.acpu = reinterpret_cast<long long *>(smem + lp.cold_off);
  t.amem = t.acpu + cp; t.rcpu = t.amem + cp; t.rmem = t.rcpu + cp; t.zcpu = t.rmem + cp; t.zmem = t.zcpu + cp;
  t.apods = reinterpret_cast<int32_t *>(t.zmem + cp);
  t.npods = t.apods + cp;
  t.own = smem + lp.own_off;
  t.su = lp.stride_u;
  return t;
}

__device__ __forceinline__ int32_t *lean_rec4(const LeanTile &t, const LeanParams &lp, int32_t j) {
  return reinterpret_cast<int32_t *>(t.rec + (size_t)j * t.su);
}

// a hot record unpacked
struct LeanRow {
  unsigned long long taint0, static0;
  long long free_cpu, free_mem;
  int32_t free_pods, score;
};
__device__ __forceinline__ LeanRow lean_row(const uint4 *r) {
  const uint4 u0 = r[0], u1 = r[1], u2 = r[2];
  LeanRow w;
  w.taint0 = ((unsigned long long)u0.y << 32) | u0.x;
  w.static0 = ((unsigned long long)u0.w << 32) | u0.z;
  w.free_cpu = (long long)(((unsigned long long)u1.y << 32) | u1.x);
  w.free_mem = (long long)(((unsigned long long)u1.w << 32) | u1.z);
  w.free_pods = (int32_t)u2.x;
  w.score = (int32_t)u2.y;
  return w;
}

struct __align__(16) LeanShared {
  ccsim_template tmpl;
  unsigned long long taint_bad0, prefer0, sel0, forbid0;
  long long eq_cpu, eq_mem;
  int32_t pods_need, n_terms, aff_bypass, has_aff, n_cmp_terms, pad1[3];   // terms[0..n_cmp_terms) are PTS/anti, the rest LT_AFF
  LeanTerm terms[LEAN_MAX_TERMS];
  CommitInfo cinfo[CCSIM_MAX_COUNTERS];
  unsigned long long warp_best[LEAN_WARPS][CCSIM_MAX_CLASSES];
  int32_t ptsmin[CCSIM_MAX_PTS], ptsnum[CCSIM_MAX_PTS];
  long long aff_total;
  ScoreWeights sw;
  int32_t winner, stop, dirty, pad0;
  int32_t scratch[LEAN_WARPS];
  // FAITHFUL sampling state
  long long f_preA, f_preB, f_total, examined, examined_total;
  unsigned long long warp_kth[LEAN_WARPS];
};

__shared__ LeanShared ls;

// the node-local part of the Filter pass: NodeUnschedulable, TaintToleration, NodeAffinity(nodeSelector), NodePorts, existing
// anti-affinity, NodeResourcesFit (the constants are ls's, read by the caller where it wants them in registers)
struct LeanFit {
  unsigned long long taint_bad0, sel0, forbid0;
  long long eq_cpu, eq_mem;
  int32_t pods_need;
};
__device__ __forceinline__ LeanFit lean_fit() {
  LeanFit f;
  f.taint_bad0 = ls.taint_bad0; f.sel0 = ls.sel0; f.forbid0 = ls.forbid0;
  f.eq_cpu = ls.eq_cpu; f.eq_mem = ls.eq_mem; f.pods_need = ls.pods_need;
  return f;
}
__device__ __forceinline__ bool lean_fits(const LeanRow &w, const LeanFit &f) {
  bool ok = ((w.taint0 & f.taint_bad0) | (~w.static0 & f.sel0) | (w.static0 & f.forbid0)) == 0ull;
  ok &= (w.free_cpu >= f.eq_cpu) & (w.free_mem >= f.eq_mem) & (w.free_pods >= f.pods_need);
  return ok;
}

// the count of a per-domain term for the node of record r4, and whether the node has the term's topology key
__device__ __forceinline__ int32_t lean_term_count(const int32_t *r4, const int32_t *cnt, const LeanTerm &lt, bool &has) {
  const int32_t v = r4[lt.slot];                                  // domain id, or the node-local count
  const bool local = lt.cnt_off < 0;
  has = local | (v >= 0);
  return local ? v : cnt[lt.cnt_off + (v < 0 ? 0 : v)];
}

// a stale score memo: the node was committed since its score was last computed; score it again and memoise
__device__ __forceinline__ int32_t lean_rescore(const LeanTile &t, const LeanParams &lp, int32_t j) {
  const ccsim_template &tm = ls.tmpl;
  const int32_t sc = score_node(t.acpu[j], t.amem[j], t.zcpu[j] + tm.least_cpu, t.zmem[j] + tm.least_mem,
                                t.rcpu[j] + tm.bal_cpu, t.rmem[j] + tm.bal_mem, ls.sw);
  lean_rec4(t, lp, j)[LR_SCORE] = sc;
  return sc;
}

// assume -> AssumePod -> NodeInfo.update(+1) for `count` clones on tile node j (schedule_one.go:967-984, types.go:409-427): the
// cold columns, the hot record and (LOCAL_COUNTERS) the node-local counters. `memo`: the node's score after them, or -1 (stale).
// The lean kernel bumps the node-local counters in its counter lanes instead: a loop on its commit lane made every sequential
// cycle ~5 % longer (C4 spread-only, ENGINE_SEQUENTIAL, one H100).
template <bool LOCAL_COUNTERS = true>
__device__ __forceinline__ void lean_commit_row(const DevParams &p, const LeanParams &lp, const LeanTile &t, int32_t j, int32_t count,
                                                int32_t memo) {
  const ccsim_template &tm = ls.tmpl;
  const long long rc = t.rcpu[j] + count * tm.req_cpu, rm = t.rmem[j] + count * tm.req_mem;
  const int32_t np = t.npods[j] + count;
  t.rcpu[j] = rc; t.rmem[j] = rm; t.zcpu[j] += count * tm.nz_cpu; t.zmem[j] += count * tm.nz_mem; t.npods[j] = np;
  int32_t *r4 = lean_rec4(t, lp, j);
  unsigned long long *r8 = reinterpret_cast<unsigned long long *>(r4);
  r8[2] = (unsigned long long)(t.acpu[j] - rc);
  r8[3] = (unsigned long long)(t.amem[j] - rm);
  r4[LR_FREE_PODS] = t.apods[j] - np;
  r4[LR_SCORE] = memo;
  if (LOCAL_COUNTERS)
    for (int c = 0; c < p.n_counters; c++) {
      const CommitInfo &ci = ls.cinfo[c];
      if (ci.inc && ci.local) r4[LR_SLOT0 + lp.counter_slot[c]] += count * ci.inc;
    }
}

// one thread: fold the template into the lean constants (see build_filter_consts for the generic kernel)
__device__ void lean_build_consts(const DevParams &p, const LeanParams &lp) {
  const ccsim_template &t = ls.tmpl;
  const uint32_t fe = t.filter_enable, fl = t.flags;
  unsigned long long tb = 0ull;
  if (fe & CCSIM_PL_TAINT_TOLERATION) tb |= p.taint_nosched[0] & ~t.tol_nosched[0] & ~(1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT);
  if ((fe & CCSIM_PL_NODE_UNSCHEDULABLE) && !(fl & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) tb |= 1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT;
  ls.taint_bad0 = tb;
  ls.prefer0 = (t.score_enable & CCSIM_PL_TAINT_TOLERATION) ? (p.taint_prefer[0] & ~t.tol_prefer[0]) : 0ull;
  const bool aff_on = (fe & CCSIM_PL_NODE_AFFINITY) && (fl & CCSIM_TF_HAS_NODE_SELECTOR);
  ls.sel0 = (aff_on && p.static_words > 0) ? t.sel_mask[0] : 0ull;
  unsigned long long fb = 0ull;
  if (p.static_words > 0) {
    if ((fe & CCSIM_PL_NODE_PORTS) && (fl & CCSIM_TF_HAS_HOST_PORTS)) fb |= t.port_static_mask[0];
    if (fe & CCSIM_PL_INTER_POD_AFFINITY) fb |= t.existing_anti_mask[0];
  }
  ls.forbid0 = fb;
  const bool fit = (fe & CCSIM_PL_FIT) != 0, nz = fit && !(fl & CCSIM_TF_FIT_ALL_ZERO);
  ls.pods_need = fit ? 1 : INT32_MIN;
  ls.eq_cpu = (nz && t.req_cpu > 0) ? t.req_cpu : LLONG_MIN;
  ls.eq_mem = (nz && t.req_mem > 0) ? t.req_mem : LLONG_MIN;
  int nt = 0;
  if (fe & CCSIM_PL_POD_TOPOLOGY_SPREAD)
    for (int c = 0; c < t.n_pts; c++) {
      LeanTerm &lt = ls.terms[nt++];
      const int j = t.pts[c].counter;
      lt.kind = LT_PTS; lt.miss_rejects = 1;
      lt.slot = LR_SLOT0 + lp.counter_slot[j];
      lt.cnt_off = p.counters[j].topo_col < 0 ? -1 : p.counters[j].smem_off;
      const long long lim = (long long)t.pts[c].max_skew - t.pts[c].self_match + (long long)ls.ptsmin[c];
      lt.lim = lim > INT32_MAX ? INT32_MAX : (lim < INT32_MIN ? INT32_MIN : (int32_t)lim);
    }
  ls.has_aff = 0;
  if (fe & CCSIM_PL_INTER_POD_AFFINITY)
    for (int a = 0; a < t.n_anti; a++) {
      LeanTerm &lt = ls.terms[nt++];
      const int j = t.anti_counter[a];
      lt.kind = LT_ANTI; lt.miss_rejects = 0; lt.lim = 0;
      lt.slot = LR_SLOT0 + lp.counter_slot[j];
      lt.cnt_off = p.counters[j].topo_col < 0 ? -1 : p.counters[j].smem_off;
    }
  ls.n_cmp_terms = nt;
  if (fe & CCSIM_PL_INTER_POD_AFFINITY)
    for (int a = 0; a < t.n_aff; a++) {
      LeanTerm &lt = ls.terms[nt++];
      const int j = t.aff_counter[a];
      lt.kind = LT_AFF; lt.miss_rejects = 1; lt.lim = 0;
      lt.slot = LR_SLOT0 + lp.counter_slot[j];
      lt.cnt_off = p.counters[j].topo_col < 0 ? -1 : p.counters[j].smem_off;
      ls.has_aff = 1;
    }
  ls.n_terms = nt;
  ls.aff_bypass = (ls.aff_total == 0 && (fl & CCSIM_TF_AFF_SELF_MATCH_ALL)) ? 1 : 0;
  ls.sw.w_fit = (t.score_enable & CCSIM_PL_FIT) ? t.w_fit : 0;
  ls.sw.w_balanced = ((t.score_enable & CCSIM_PL_BALANCED) && !(fl & CCSIM_TF_BALANCED_SKIP)) ? t.w_balanced : 0;
  ls.sw.least_w_cpu = t.least_w_cpu; ls.sw.least_w_mem = t.least_w_mem;
  for (int j = 0; j < p.n_counters; j++) {
    const DevCounter &dc = p.counters[j];
    CommitInfo &ci = ls.cinfo[j];
    const bool skip = (dc.inc == 0) || (dc.is_aff && !(fl & CCSIM_TF_AFF_SELF_MATCH_ALL));
    ci.inc = skip ? 0 : dc.inc;
    ci.local = dc.topo_col < 0; ci.is_aff = dc.is_aff; ci.n_present = dc.n_present;
    ci.gtopo = dc.topo_col < 0 ? nullptr : p.topo_full[dc.topo_col];
    ci.ltopo = nullptr;
    ci.pts_idx = -1;
    for (int c = 0; c < t.n_pts; c++) if (t.pts[c].counter == j && !t.pts[c].min_zero) ci.pts_idx = c;
  }
}

// minimum and its multiplicity of PTS constraint c over the present domains (all threads)
__device__ void lean_pts_recount(const DevParams &p, const int32_t *smem_cnt, int c) {
  const ccsim_pts &pc = ls.tmpl.pts[c];
  const DevCounter &dc = p.counters[pc.counter];
  int32_t num;
  const int32_t m = block_min_count<LEAN_THREADS>(smem_cnt + dc.smem_off, dc.n_present, ls.scratch, num);
  if (threadIdx.x == 0) {
    ls.ptsmin[c] = pc.min_zero ? 0 : m;
    ls.ptsnum[c] = num;
    ls.dirty = 1;
  }
  __syncthreads();
}

// after a wave: recount every PTS minimum whose last domain at the minimum took a clone (all of them when `force`)
__device__ __forceinline__ void lean_pts_after_wave(const DevParams &p, const int32_t *smem_cnt, bool force) {
  for (int c = 0; c < ls.tmpl.n_pts; c++)
    if (!ls.tmpl.pts[c].min_zero && (ls.ptsnum[c] <= 0 || force) && p.counters[ls.tmpl.pts[c].counter].n_present > 0) lean_pts_recount(p, smem_cnt, c);
}

// Stage the tile (once): hot AoS records and cold SoA columns of tile nodes [0, cnt_nodes) = global [lo, lo + cnt_nodes),
// template 0, the replicated counter cells, ls's run state (all threads, ends after a barrier).
__device__ __forceinline__ void lean_stage(const DevParams &p, const LeanParams &lp, const LeanTile &t, int32_t lo, int32_t cnt_nodes) {
  const int tid = threadIdx.x;
  for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
    const int32_t i = lo + j;
    const long long ac = p.alloc_cpu[i], am = p.alloc_mem[i], rc = p.req_cpu[i], rm = p.req_mem[i];
    const int32_t ap = p.alloc_pods[i], np = p.npods[i];
    int32_t *r4 = lean_rec4(t, lp, j);
    unsigned long long *r8 = reinterpret_cast<unsigned long long *>(r4);
    r8[0] = p.taint_mask[i];
    r8[1] = p.static_words > 0 ? p.static_mask[i] : 0ull;
    r8[2] = (unsigned long long)(ac - rc);
    r8[3] = (unsigned long long)(am - rm);
    r4[LR_FREE_PODS] = ap - np;
    r4[LR_SCORE] = -1;
    for (int s = 0; s < lp.n_slots; s++)
      r4[LR_SLOT0 + s] = lp.slot_topo[s] >= 0 ? p.topo[lp.slot_topo[s]][i] : p.counters[lp.slot_counter[s]].work[i];
    t.acpu[j] = ac; t.amem[j] = am; t.rcpu[j] = rc; t.rmem[j] = rm;
    t.zcpu[j] = p.nz_cpu[i]; t.zmem[j] = p.nz_mem[i];
    t.apods[j] = ap; t.npods[j] = np;
  }
  for (int k = tid; k < (int)(sizeof(ccsim_template) / 8); k += LEAN_THREADS)
    reinterpret_cast<unsigned long long *>(&ls.tmpl)[k] = reinterpret_cast<const unsigned long long *>(&p.templates[0])[k];
  for (int j = 0; j < p.n_counters; j++) {
    const DevCounter &dc = p.counters[j];
    if (dc.topo_col < 0) continue;
    for (int d = tid; d < dc.n_domains; d += LEAN_THREADS) t.cnt[dc.smem_off + d] = dc.init[d];
  }
  if (tid == 0) { ls.aff_total = p.templates[0].aff_total_init; ls.winner = -1; ls.stop = 0; ls.dirty = 1; ls.examined = 0; ls.examined_total = 0; }
  __syncthreads();
}

// After the run: the tile goes back to the global columns once (the mutable columns and the node-local counters: the snapshot
// after the run, read by the terminal diagnosis), and CTA 0 writes the final replicated counters and the result fields the
// lean and multi-commit kernels report. Returns p.out to thread 0 of CTA 0, which fills in the kernel's own fields; nullptr elsewhere.
__device__ __forceinline__ DevOut *lean_finish(const DevParams &p, const LeanParams &lp, const LeanTile &t, int32_t lo, int32_t cnt_nodes,
                                               long long placed, bool limit_hit) {
  const int tid = threadIdx.x;
  for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
    const int32_t i = lo + j;
    p.req_cpu[i] = t.rcpu[j]; p.req_mem[i] = t.rmem[j]; p.nz_cpu[i] = t.zcpu[j]; p.nz_mem[i] = t.zmem[j]; p.npods[i] = t.npods[j];
    const int32_t *r4 = lean_rec4(t, lp, j);
    for (int s = 0; s < lp.n_slots; s++) if (lp.slot_topo[s] < 0) p.counters[lp.slot_counter[s]].work[i] = r4[LR_SLOT0 + s];
  }
  if (blockIdx.x != 0) return nullptr;
  for (int j = 0; j < p.n_counters; j++) {
    const DevCounter &dc = p.counters[j];
    if (dc.topo_col < 0) continue;
    for (int d = tid; d < dc.n_domains; d += LEAN_THREADS) p.final_cnt[p.final_off[j] + d] = t.cnt[dc.smem_off + d];
  }
  if (tid != 0) return nullptr;
  DevOut *o = p.out;
  o->placed = placed;
  o->stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
  o->error = (ls.stop == 3) ? 1 : 0;
  for (int c = 0; c < CCSIM_MAX_PTS; c++) o->ptsmin[c] = c < ls.tmpl.n_pts ? ls.ptsmin[c] : 0;
  o->aff_total = ls.aff_total;
  return o;
}

// FAITHFUL: the reference's default sampling (adaptive numFeasibleNodesToFind + rotating start index,
// schedule_one.go:538-539,644-723) as a deterministic sequential scan: only the first K feasible nodes in rotated order
// compete, ties -> first maximum in rotated order, and the start index advances by the number of nodes examined.
template <bool FAITHFUL>
__global__ void __launch_bounds__(LEAN_THREADS, 1) ccsim_wave_lean_kernel(const DevParams p, const LeanParams lp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const size_t cp = (size_t)p.chunk_pad;
  const LeanTile t = lean_tile(smem_raw, lp, cp);
  int32_t *smem_cnt = t.cnt;
  uint4 *rec = t.rec;   // (the rows below are addressed as rec + j * su: through lean_rec4, lean<true> spilled 24 more bytes)
  int32_t *feas = reinterpret_cast<int32_t *>(t.own);   // FAITHFUL only: feasibility flag and exclusive feasible-rank of every tile node
  int32_t *pre = feas + cp;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int32_t cnt_nodes = hi - lo;
  const int ncls = p.n_classes;
  const int su = lp.stride_u;
  uint32_t start = 0;               // sched.nextStartNodeIndex (FAITHFUL)

  lean_stage(p, lp, t, lo, cnt_nodes);
  for (int c = 0; c < ls.tmpl.n_pts; c++) lean_pts_recount(p, smem_cnt, c);

#ifdef CCSIM_PHASE_TIMERS
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tc0 = 0, tc1 = 0;
#endif
  long long k = 0;
  bool limit_hit = false;   // postBindHook's limit (simulator.go:300-305)
  uint32_t wtag = 1;
  uint32_t tag = (p.epoch << 12) | wtag;
  for (;; k++) {
    PH_START();
    if (p.max_pods > 0 && k >= p.max_pods) { limit_hit = true; break; }   // uniform; no shared write (slower threads may still be reading ls.stop)
    if (k > p.pod_cap) { if (tid == 0) ls.stop = 3; __syncthreads(); break; }   // cannot happen (pod_cap bounds every run): never spin forever
    if (ls.dirty) {   // uniform: set before the last barrier, cleared only after the barrier below (no thread can miss it)
      if (tid == 0) lean_build_consts(p, lp);
      __syncthreads();
      if (tid == 0) ls.dirty = 0;
    }
    // ---- fused Filter pass: one predicate-eval per node of the tile ----
    const LeanFit fit = lean_fit();
    const unsigned long long prefer0 = ls.prefer0;
    const int32_t n_terms = ls.n_terms, n_cmp = ls.n_cmp_terms;
    unsigned long long best = 0ull;      // single class
    unsigned long long bestc[CCSIM_MAX_CLASSES];
    if (ncls > 1) {
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) bestc[c] = 0ull;
    }
    for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
      const uint4 *r = rec + (size_t)j * su;
      const LeanRow w = lean_row(r);
      const unsigned long long taint0 = w.taint0;
      int32_t sc = w.score;
      bool ok = lean_fits(w, fit);
      // PodTopologySpread + anti-affinity terms: reject <=> has ? count > lim : miss_rejects
      if (n_cmp) {
        const int32_t *r4 = reinterpret_cast<const int32_t *>(r);
        #pragma unroll 4
        for (int q = 0; q < n_cmp; q++) {
          const LeanTerm lt = ls.terms[q];
          bool has; const int32_t c = lean_term_count(r4, smem_cnt, lt, has);
          ok &= has ? (c <= lt.lim) : (lt.miss_rejects == 0);
        }
      }
      if (n_terms > n_cmp) {   // required pod affinity (interpodaffinity/filtering.go:382-408)
        const int32_t *r4 = reinterpret_cast<const int32_t *>(r);
        bool aff_exist = true, aff_missing = false;
        for (int q = n_cmp; q < n_terms; q++) {
          const LeanTerm lt = ls.terms[q];
          bool has; const int32_t c = lean_term_count(r4, smem_cnt, lt, has);
          aff_missing |= !has; aff_exist &= has & (c > 0);
        }
        ok &= !(aff_missing | (!aff_exist & !ls.aff_bypass));
      }
      if (FAITHFUL) feas[j] = ok ? 1 : 0;
      if (ok) {
        if (sc < 0) sc = lean_rescore(t, lp, j);
        if (FAITHFUL) continue;     // keys are built after the sampling cut is known
        const unsigned long long key = pack_key(sc, (uint32_t)(p.node_base + lo + j));
        if (ncls == 1) best = key > best ? key : best;
        else {
          const int cls = __popcll(taint0 & prefer0);
          #pragma unroll
          for (int c = 0; c < CCSIM_MAX_CLASSES; c++) if (c == cls) bestc[c] = key > bestc[c] ? key : bestc[c];
        }
      }
    }
    unsigned long long kth = 0ull;    // FAITHFUL: rotated position + 1 of the K-th feasible node, if it is in this thread's nodes
    if (FAITHFUL) {
      __syncthreads();
      // exclusive feasible-rank in node order (each thread owns a contiguous segment), tile total
      const int seg = (cnt_nodes + LEAN_THREADS - 1) / LEAN_THREADS;
      const int b0 = min(cnt_nodes, tid * seg), b1 = min(cnt_nodes, b0 + seg);
      int32_t sfe = 0;
      for (int j = b0; j < b1; j++) sfe += feas[j];
      int32_t incl = sfe;
      for (int o = 1; o < 32; o <<= 1) { const int32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
      if (lane == 31) ls.scratch[warp] = incl;
      __syncthreads();
      int32_t wbase = 0, ctot = 0;
      for (int w = 0; w < LEAN_WARPS; w++) { if (w < warp) wbase += ls.scratch[w]; ctot += ls.scratch[w]; }
      int32_t base = wbase + incl - sfe;
      for (int j = b0; j < b1; j++) { pre[j] = base; base += feas[j]; }
      __syncthreads();
      // boundary of the rotation inside this tile: nodes with global index >= start come first ("part A")
      const long long jb_ll = (long long)start - (long long)(p.node_base + lo);
      const int32_t jb = jb_ll < 0 ? 0 : (jb_ll > cnt_nodes ? cnt_nodes : (int32_t)jb_ll);
      const int32_t cB = jb >= cnt_nodes ? ctot : pre[jb];
      const int32_t cA = ctot - cB;
      if (warp == 0) {   // exchange 1: (cA, cB) of every tile -> feasible-rank offsets of this tile's two parts
        // both counts travel in one word as two 22-bit fields; their sums over the grid stay below 2^22 too (a resident lean tile
        // holds a few thousand nodes at most, the grid at most CCSIM_MAX_GRID tiles), so the packed sums split without a carry.
        // tests/test_gpu_kernel_edges.py::test_sampling_largest_lean_tile runs the largest cluster this kernel takes (267 168 nodes
        // on an H100) and checks that it is below 2^22 nodes
        unsigned long long pre, tot;
        const bool dead = exchange_prefix_total(p, k, tag, CCSIM_MAX_CLASSES + 1, ((unsigned long long)cA << 22) | (unsigned long long)cB, lane, cta, pre, tot);
        const unsigned long long F = (1ull << 22) - 1;
        const unsigned long long preA = pre >> 22, totA = tot >> 22, preB = pre & F, totB = tot & F;
        if (lane == 0) { ls.f_preA = (long long)preA; ls.f_preB = (long long)(totA + preB); ls.f_total = (long long)(totA + totB); if (dead) ls.stop = 3; }
      }
      __syncthreads();
      const long long preA = ls.f_preA, preB = ls.f_preB, K = p.sample_k;
      for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
        if (!feas[j]) continue;
        const long long gr = (j >= jb) ? preA + (pre[j] - cB) : preB + pre[j];
        if (gr >= K) continue;                       // beyond numFeasibleNodesToFind: never examined
        const uint32_t gidx = (uint32_t)(p.node_base + lo + j);
        const uint32_t rot = gidx >= start ? gidx - start : gidx + (uint32_t)p.n_global - start;
        if (gr == K - 1) kth = (unsigned long long)rot + 1ull;
        const int32_t sc = reinterpret_cast<const int32_t *>(rec + (size_t)j * su)[LR_SCORE];
        const unsigned long long key = pack_key(sc, rot);     // ties -> first in rotated order
        if (ncls == 1) best = key > best ? key : best;
        else {
          const unsigned long long taint0 = reinterpret_cast<const unsigned long long *>(rec + (size_t)j * su)[0];
          const int cls = __popcll(taint0 & prefer0);
          #pragma unroll
          for (int c = 0; c < CCSIM_MAX_CLASSES; c++) if (c == cls) bestc[c] = key > bestc[c] ? key : bestc[c];
        }
      }
      const unsigned long long kv = warp_max_u64(kth);
      if (lane == 0) ls.warp_kth[warp] = kv;
    }
    if (ncls == 1) {
      const unsigned long long v = warp_max_u64(best);
      if (lane == 0) ls.warp_best[warp][0] = v;
    } else {
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++)
        if (c < ncls) { const unsigned long long v = warp_max_u64(bestc[c]); if (lane == 0) ls.warp_best[warp][c] = v; }
    }
    PH_MARK(0);
    __syncthreads();                                                    // S1
    PH_MARK(1);

    if (warp == 0) {
      const ccsim_template &tm = ls.tmpl;
      const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
      unsigned long long *myslots = p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE;
      for (int c = 0; c < ncls; c++) {
        const unsigned long long v = warp_max_u64(lane < LEAN_WARPS ? ls.warp_best[lane][c] : 0ull);
        if (lane == 0) st_slot(&myslots[c], v | tagbits);
      }
      if (FAITHFUL) {
        const unsigned long long kv = warp_max_u64(lane < LEAN_WARPS ? ls.warp_kth[lane] : 0ull);
        if (lane == 0) st_slot(&myslots[CCSIM_MAX_CLASSES], kv | tagbits);
      }
      PH_MARK(2);
      unsigned long long cbest[CCSIM_MAX_CLASSES];
      bool dead = false;
      unsigned long long kth_all = 0ull;
      if (FAITHFUL) {
        unsigned long long v[GATHER_Q];
        dead = gather_tagged(p, k, tag, CCSIM_MAX_CLASSES, lane, v);
        kth_all = gather_max(v);
      }
      for (int c = 0; c < ncls; c++) {
        unsigned long long v[GATHER_Q];
        dead |= gather_tagged(p, k, tag, c, lane, v);
        cbest[c] = gather_max(v);
      }
      if (p.world > 1 && !dead) dead = cross_gpu_exchange(p, k, tag, ncls, cbest, lane, cta);
      PH_MARK(3);
      const unsigned long long wkey = select_host_over_classes(cbest, ncls, tm);
      if (lane == 0) {
        if (dead) { ls.stop = 3; ls.winner = -1; }
        else if (wkey == 0ull) { ls.stop = 1; ls.winner = -1; }
        else ls.winner = (int32_t)key_index(wkey);
        if (FAITHFUL) {   // processedNodes of this cycle (schedule_one.go:538-539): up to and including the K-th feasible node
          ls.examined = (ls.f_total >= p.sample_k && kth_all > 0ull) ? (long long)kth_all : (long long)p.n_global;
          if (cta == 0) ls.examined_total += ls.examined;
        }
      }
      // ---- commit: the owner's row (lean_commit_row) and every CTA's replicated counters ----
      if (!dead && wkey != 0ull) {
        const int32_t g = FAITHFUL ? (int32_t)(((unsigned long long)start + key_index(wkey)) % (unsigned long long)p.n_global) : (int32_t)key_index(wkey);
        const int32_t w = g - p.node_base;
        const bool mine = (w >= lo && w < hi);
        const int32_t jw = w - lo;
        if (mine && lane == 31) {
          lean_commit_row<false>(p, lp, t, jw, 1, -1);      // this node's NodeInfo generation changed: its memoised score is stale
          if (k < p.pod_cap) p.pod_node[k] = g; else ls.stop = 3;
        }
        if (p.world > 1 && !mine && cta == 0 && lane == 31) {   // sharded run: every rank keeps the whole pod -> node sequence
          const bool local = (w >= 0 && w < p.n);
          if (!local) { if (k < p.pod_cap) p.pod_node[k] = g; else ls.stop = 3; }
        }
        if (lane < p.n_counters) {
          const int j = lane;
          const CommitInfo ci = ls.cinfo[j];
          if (ci.inc) {
            if (ci.local) {
              if (mine) reinterpret_cast<int32_t *>(rec + (size_t)jw * su)[LR_SLOT0 + lp.counter_slot[j]] += ci.inc;
              if (ci.is_aff) { atomicAdd((unsigned long long *)&ls.aff_total, (unsigned long long)ci.inc); ls.dirty = 1; }
            } else {
              // the winner's domain id: from this CTA's tile if it owns the node, else from the whole-cluster column (L2).
              // (Carrying the ids with the exchanged key instead — as extra words or packed into the key's low bits — lengthens every
              //  CTA's exchange for a lookup only the non-owner CTAs make.)
              const int32_t dom = mine ? reinterpret_cast<const int32_t *>(rec + (size_t)jw * su)[LR_SLOT0 + lp.counter_slot[j]] : ci.gtopo[g];
              if (dom >= 0) {
                int32_t *cnt = smem_cnt + p.counters[j].smem_off;
                const int32_t old = cnt[dom];
                cnt[dom] = old + ci.inc;
                if (ci.is_aff) { atomicAdd((unsigned long long *)&ls.aff_total, (unsigned long long)ci.inc); ls.dirty = 1; }
                if (ci.pts_idx >= 0 && dom < ci.n_present && old == ls.ptsmin[ci.pts_idx]) ls.ptsnum[ci.pts_idx] -= 1;
              }
            }
          }
        }
      }
    }
    PH_MARK(4);
    __syncthreads();                                                    // S2
    PH_MARK(5);
    if (ls.stop) break;
    lean_pts_after_wave(p, smem_cnt, false);
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
    if (FAITHFUL) start = (uint32_t)(((unsigned long long)start + (unsigned long long)ls.examined) % (unsigned long long)p.n_global);
  }

  if (DevOut *o = lean_finish(p, lp, t, lo, cnt_nodes, k, limit_hit)) {
    o->waves = limit_hit ? k : k + 1;
    o->evals = o->waves * (long long)p.n;
    o->examined = FAITHFUL ? ls.examined_total : o->evals;
#ifdef CCSIM_PHASE_TIMERS
    for (int q = 0; q < 8; q++) o->phase_cycles[q] = ph[q];
#endif
  }
}
