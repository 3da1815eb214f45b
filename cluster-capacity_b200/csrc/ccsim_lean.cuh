// ccsim_lean.cuh — the lean resident wave kernel: the common case of the hot path, written for latency.
//
// Eligibility (decided on the host, see ccsim_run): the CTA tiles fit in shared memory, one template, one taint word,
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

// One per-domain term of the Filter pass, 16 bytes (one LDS.128). PodTopologySpread and anti-affinity share one form:
//   reject  <=>  (node has the topology key) ? count(domain) > lim : miss_rejects
// (PTS: lim = maxSkew - selfMatch + globalMin, missing key rejects; anti-affinity: lim = 0, missing key passes).
// Required pod-affinity terms (LT_AFF) need the all-terms "pods exist" logic and are evaluated in a second loop.
struct __align__(16) LeanTerm {
  int16_t kind;      // LT_*
  int16_t miss_rejects;
  int32_t slot;      // record int index (10 + s) holding the node's domain id, or the node-local count itself
  int32_t cnt_off;   // offset of the counter in the shared replicated-counter area, -1: node-local (the slot IS the count)
  int32_t lim;
};

struct LeanParams {
  int32_t stride_u;        // record stride in 16-byte units (odd)
  int32_t n_slots;         // extra int slots used
  int32_t slot_topo[LEAN_MAX_SLOTS];     // slot s mirrors topology column slot_topo[s] (>=0) ...
  int32_t slot_counter[LEAN_MAX_SLOTS];  // ... or node-local counter slot_counter[s] (>=0)
  int32_t counter_slot[CCSIM_MAX_COUNTERS]; // counter j -> slot holding its domain id (topo) or its count (node-local)
  uint32_t rec_bytes_total; // stride * chunk_pad
  uint32_t cold_off;        // byte offset of the cold SoA columns (alloc/req/nz) in dynamic shared memory
  uint32_t cnt_off_bytes;   // byte offset of the replicated counters (0)
};

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
      lt.slot = 10 + lp.counter_slot[j];
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
      lt.slot = 10 + lp.counter_slot[j];
      lt.cnt_off = p.counters[j].topo_col < 0 ? -1 : p.counters[j].smem_off;
    }
  ls.n_cmp_terms = nt;
  if (fe & CCSIM_PL_INTER_POD_AFFINITY)
    for (int a = 0; a < t.n_aff; a++) {
      LeanTerm &lt = ls.terms[nt++];
      const int j = t.aff_counter[a];
      lt.kind = LT_AFF; lt.miss_rejects = 1; lt.lim = 0;
      lt.slot = 10 + lp.counter_slot[j];
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

// FAITHFUL: the reference's default sampling (adaptive numFeasibleNodesToFind + rotating start index,
// schedule_one.go:538-539,644-723) as a deterministic sequential scan: only the first K feasible nodes in rotated order
// compete, ties -> first maximum in rotated order, and the start index advances by the number of nodes examined.
template <bool FAITHFUL>
__global__ void __launch_bounds__(LEAN_THREADS, 1) ccsim_wave_lean_kernel(const DevParams p, const LeanParams lp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t *smem_cnt = reinterpret_cast<int32_t *>(smem_raw);
  const uint32_t cnt_bytes = ((uint32_t)p.smem_cnt_ints * 4u + 15u) & ~15u;
  uint4 *rec = reinterpret_cast<uint4 *>(smem_raw + cnt_bytes);
  const size_t cp = (size_t)p.chunk_pad;
  long long *c_acpu = reinterpret_cast<long long *>(smem_raw + cnt_bytes + lp.rec_bytes_total);
  long long *c_amem = c_acpu + cp, *c_rcpu = c_amem + cp, *c_rmem = c_rcpu + cp, *c_zcpu = c_rmem + cp, *c_zmem = c_zcpu + cp;
  int32_t *c_apods = reinterpret_cast<int32_t *>(c_zmem + cp);
  int32_t *c_npods = c_apods + cp;
  int32_t *feas = c_npods + cp;     // FAITHFUL only: feasibility flag and exclusive feasible-rank of every tile node
  int32_t *pre = feas + cp;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int32_t cnt_nodes = hi - lo;
  const int ncls = p.n_classes;
  const int su = lp.stride_u;
  uint32_t start = 0;               // sched.nextStartNodeIndex (FAITHFUL)

  // ---- stage the tile (once): hot AoS records + cold SoA columns ----
  for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
    const int32_t i = lo + j;
    const long long ac = p.alloc_cpu[i], am = p.alloc_mem[i], rc = p.req_cpu[i], rm = p.req_mem[i];
    const int32_t ap = p.alloc_pods[i], np = p.npods[i];
    unsigned long long *r8 = reinterpret_cast<unsigned long long *>(rec + (size_t)j * su);
    int32_t *r4 = reinterpret_cast<int32_t *>(r8);
    r8[0] = p.taint_mask[i];
    r8[1] = p.static_words > 0 ? p.static_mask[i] : 0ull;
    r8[2] = (unsigned long long)(ac - rc);
    r8[3] = (unsigned long long)(am - rm);
    r4[8] = ap - np;
    r4[9] = -1;
    for (int s = 0; s < lp.n_slots; s++)
      r4[10 + s] = lp.slot_topo[s] >= 0 ? p.topo[lp.slot_topo[s]][i] : p.counters[lp.slot_counter[s]].work[i];
    c_acpu[j] = ac; c_amem[j] = am; c_rcpu[j] = rc; c_rmem[j] = rm;
    c_zcpu[j] = p.nz_cpu[i]; c_zmem[j] = p.nz_mem[i];
    c_apods[j] = ap; c_npods[j] = np;
  }
  for (int k = tid; k < (int)(sizeof(ccsim_template) / 8); k += LEAN_THREADS)
    reinterpret_cast<unsigned long long *>(&ls.tmpl)[k] = reinterpret_cast<const unsigned long long *>(&p.templates[0])[k];
  for (int j = 0; j < p.n_counters; j++) {
    const DevCounter &dc = p.counters[j];
    if (dc.topo_col < 0) continue;
    for (int d = tid; d < dc.n_domains; d += LEAN_THREADS) smem_cnt[dc.smem_off + d] = dc.init[d];
  }
  if (tid == 0) { ls.aff_total = p.templates[0].aff_total_init; ls.winner = -1; ls.stop = 0; ls.dirty = 1; ls.examined = 0; ls.examined_total = 0; }
  __syncthreads();
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
    const unsigned long long taint_bad0 = ls.taint_bad0, prefer0 = ls.prefer0, sel0 = ls.sel0, forbid0 = ls.forbid0;
    const long long eq_cpu = ls.eq_cpu, eq_mem = ls.eq_mem;
    const int32_t pods_need = ls.pods_need, n_terms = ls.n_terms, n_cmp = ls.n_cmp_terms;
    unsigned long long best = 0ull;      // single class
    unsigned long long bestc[CCSIM_MAX_CLASSES];
    if (ncls > 1) {
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) bestc[c] = 0ull;
    }
    for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
      const uint4 *r = rec + (size_t)j * su;
      const uint4 u0 = r[0], u1 = r[1], u2 = r[2];
      const unsigned long long taint0 = ((unsigned long long)u0.y << 32) | u0.x;
      const unsigned long long static0 = ((unsigned long long)u0.w << 32) | u0.z;
      const long long free_cpu = (long long)(((unsigned long long)u1.y << 32) | u1.x);
      const long long free_mem = (long long)(((unsigned long long)u1.w << 32) | u1.z);
      const int32_t free_pods = (int32_t)u2.x;
      int32_t sc = (int32_t)u2.y;
      // NodeUnschedulable, TaintToleration, NodeAffinity(nodeSelector), NodePorts, existing anti-affinity, NodeResourcesFit
      bool ok = ((taint0 & taint_bad0) | (~static0 & sel0) | (static0 & forbid0)) == 0ull;
      ok &= (free_cpu >= eq_cpu) & (free_mem >= eq_mem) & (free_pods >= pods_need);
      // PodTopologySpread + anti-affinity terms: reject <=> has ? count > lim : miss_rejects
      if (n_cmp) {
        const int32_t *r4 = reinterpret_cast<const int32_t *>(r);
        #pragma unroll 4
        for (int q = 0; q < n_cmp; q++) {
          const LeanTerm lt = ls.terms[q];
          const int32_t v = r4[lt.slot];                                  // domain id, or the node-local count
          const bool local = lt.cnt_off < 0;
          const int32_t c = local ? v : smem_cnt[lt.cnt_off + (v < 0 ? 0 : v)];
          const bool has = local | (v >= 0);
          ok &= has ? (c <= lt.lim) : (lt.miss_rejects == 0);
        }
      }
      if (n_terms > n_cmp) {   // required pod affinity (interpodaffinity/filtering.go:382-408)
        const int32_t *r4 = reinterpret_cast<const int32_t *>(r);
        bool aff_exist = true, aff_missing = false;
        for (int q = n_cmp; q < n_terms; q++) {
          const LeanTerm lt = ls.terms[q];
          const int32_t v = r4[lt.slot];
          const bool local = lt.cnt_off < 0;
          const int32_t c = local ? v : smem_cnt[lt.cnt_off + (v < 0 ? 0 : v)];
          const bool has = local | (v >= 0);
          aff_missing |= !has; aff_exist &= has & (c > 0);
        }
        ok &= !(aff_missing | (!aff_exist & !ls.aff_bypass));
      }
      if (FAITHFUL) feas[j] = ok ? 1 : 0;
      if (ok) {
        if (sc < 0) {   // stale memo: this node was committed since its score was last computed
          sc = score_node(c_acpu[j], c_amem[j], c_zcpu[j] + ls.tmpl.least_cpu, c_zmem[j] + ls.tmpl.least_mem,
                          c_rcpu[j] + ls.tmpl.bal_cpu, c_rmem[j] + ls.tmpl.bal_mem, ls.sw);
          reinterpret_cast<int32_t *>(rec + (size_t)j * su)[9] = sc;
        }
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
        const int32_t sc = reinterpret_cast<const int32_t *>(rec + (size_t)j * su)[9];
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
      const ccsim_template &t = ls.tmpl;
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
      const unsigned long long wkey = select_host_over_classes(cbest, ncls, t);
      if (lane == 0) {
        if (dead) { ls.stop = 3; ls.winner = -1; }
        else if (wkey == 0ull) { ls.stop = 1; ls.winner = -1; }
        else ls.winner = (int32_t)key_index(wkey);
        if (FAITHFUL) {   // processedNodes of this cycle (schedule_one.go:538-539): up to and including the K-th feasible node
          ls.examined = (ls.f_total >= p.sample_k && kth_all > 0ull) ? (long long)kth_all : (long long)p.n_global;
          if (cta == 0) ls.examined_total += ls.examined;
        }
      }
      // ---- commit (assume -> AssumePod -> NodeInfo.update(+1): schedule_one.go:967-984, types.go:409-427) ----
      if (!dead && wkey != 0ull) {
        const int32_t g = FAITHFUL ? (int32_t)(((unsigned long long)start + key_index(wkey)) % (unsigned long long)p.n_global) : (int32_t)key_index(wkey);
        const int32_t w = g - p.node_base;
        const bool mine = (w >= lo && w < hi);
        const int32_t jw = w - lo;
        if (mine && lane == 31) {
          const long long rc = c_rcpu[jw] + t.req_cpu, rm = c_rmem[jw] + t.req_mem;
          const long long zc = c_zcpu[jw] + t.nz_cpu, zm = c_zmem[jw] + t.nz_mem;
          const int32_t np = c_npods[jw] + 1;
          c_rcpu[jw] = rc; c_rmem[jw] = rm; c_zcpu[jw] = zc; c_zmem[jw] = zm; c_npods[jw] = np;
          unsigned long long *r8 = reinterpret_cast<unsigned long long *>(rec + (size_t)jw * su);
          int32_t *r4 = reinterpret_cast<int32_t *>(r8);
          r8[2] = (unsigned long long)(c_acpu[jw] - rc);
          r8[3] = (unsigned long long)(c_amem[jw] - rm);
          r4[8] = c_apods[jw] - np;
          r4[9] = -1;            // this node's NodeInfo generation changed: its memoised score is stale
          p.req_cpu[w] = rc; p.req_mem[w] = rm; p.nz_cpu[w] = zc; p.nz_mem[w] = zm; p.npods[w] = np;   // write through
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
              if (mine) {
                int32_t *r4 = reinterpret_cast<int32_t *>(rec + (size_t)jw * su);
                const int32_t nv = r4[10 + lp.counter_slot[j]] + ci.inc;
                r4[10 + lp.counter_slot[j]] = nv;
                p.counters[j].work[w] = nv;
              }
              if (ci.is_aff) { atomicAdd((unsigned long long *)&ls.aff_total, (unsigned long long)ci.inc); ls.dirty = 1; }
            } else {
              // the winner's domain id: from this CTA's tile if it owns the node, else from the whole-cluster column (L2).
              // (Carrying the ids with the exchanged key instead — as extra words or packed into the key's low bits — lengthens every
              //  CTA's exchange for a lookup only the non-owner CTAs make.)
              const int32_t dom = mine ? reinterpret_cast<const int32_t *>(rec + (size_t)jw * su)[10 + lp.counter_slot[j]] : ci.gtopo[g];
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
    for (int c = 0; c < ls.tmpl.n_pts; c++)
      if (!ls.tmpl.pts[c].min_zero && ls.ptsnum[c] <= 0 && p.counters[ls.tmpl.pts[c].counter].n_present > 0) lean_pts_recount(p, smem_cnt, c);
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
    if (FAITHFUL) start = (uint32_t)(((unsigned long long)start + (unsigned long long)ls.examined) % (unsigned long long)p.n_global);
  }

  if (cta == 0) {
    for (int j = 0; j < p.n_counters; j++) {
      const DevCounter &dc = p.counters[j];
      if (dc.topo_col < 0) continue;
      for (int d = tid; d < dc.n_domains; d += LEAN_THREADS) p.final_cnt[p.final_off[j] + d] = smem_cnt[dc.smem_off + d];
    }
    if (tid == 0) {
      DevOut *o = p.out;
      o->placed = k;
      o->stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
      o->error = (ls.stop == 3) ? 1 : 0;
      o->waves = limit_hit ? k : k + 1;
      o->evals = o->waves * (long long)p.n;
      o->examined = FAITHFUL ? ls.examined_total : o->evals;
      for (int c = 0; c < CCSIM_MAX_PTS; c++) o->ptsmin[c] = ls.ptsmin[c];
      o->aff_total = ls.aff_total;
#ifdef CCSIM_PHASE_TIMERS
      for (int q = 0; q < 8; q++) o->phase_cycles[q] = ph[q];
#endif
    }
  }
}
