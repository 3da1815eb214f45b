// ccsim_wave.cuh — the generic wave kernel (ccsim_wave_kernel): every template the lean, tie-run, multi-commit and streaming
// kernels do not take (normalised soft scorers, several templates with counters, the extras predicates, elig_bit counters, tiles
// too large for those kernels), resident or streaming, one winner per wave.
#pragma once
#include "ccsim_device.cuh"

#define BLOCK_THREADS 512
#define MAX_WARPS (BLOCK_THREADS / 32)
#define SMEM_CNT_MAX_INTS 16384      /* 64 KB of replicated counters in shared memory; above that: global replicas */

struct __align__(16) WaveShared {
  ccsim_template tmpl;                              // current template
  FilterConsts fc;                                  // folded per-wave constants of the Filter pass
  unsigned long long warp_best[MAX_WARPS][CCSIM_MAX_CLASSES];
  const int32_t *topo_ptr[CCSIM_MAX_TOPO_COLS];     // topology columns as this CTA indexes them (pre-offset)
  int32_t *cnt_ptr[CCSIM_MAX_COUNTERS];             // counter bases (shared replica / global replica / node-local column)
  int32_t ptsmin[CCSIM_MAX_PTS];
  int32_t ptsnum[CCSIM_MAX_PTS];
  long long aff_total;
  int32_t winner;        // global node index, -1 = none
  int32_t stop;          // 0 continue, 1 unschedulable, 2 limit, 3 error
  int32_t dirty;         // FilterConsts must be rebuilt before the next scan
  // normalised soft scorers (multi-phase waves): extrema of the raw scores over the feasible nodes of this wave
  long long na_max, spts_min, spts_max, ipa_min, ipa_max;
  long long spts_scored;                 // feasible nodes that are not in IgnoredNodes
  double spts_w[CCSIM_MAX_PTS];          // topologyNormalizingWeight per soft constraint
  long long red[MAX_WARPS][6];           // block reductions of the above
  ScoreWeights sw;       // scalar copy of the template's score configuration (passed by value to score_node)
  CommitInfo cinfo[CCSIM_MAX_COUNTERS];   // what a commit does to each counter under the current template
  int32_t scratch[MAX_WARPS];
};

// Statically allocated so that every access is a direct LDS/STS with a compile-time offset (a reference obtained by
// casting the dynamic shared array makes nvcc re-derive the generic window base — S2UR SR_CgaCtaId — at each use).
__shared__ WaveShared ws;

// recount of a PTS constraint's minimum and its multiplicity over the present domains (all threads of the CTA). Not
// block_min_count<BLOCK_THREADS>: inlined at the per-wave call, that spills 8 B in wave<true> (stack frame 64 -> 80 B; nvcc 12.9)
__device__ void pts_recount(const DevParams &p, int c) {
  const ccsim_pts &pc = ws.tmpl.pts[c];
  const DevCounter &dc = p.counters[pc.counter];
  const int32_t *cnt = ws.cnt_ptr[pc.counter];
  int32_t m = INT32_MAX;
  for (int d = threadIdx.x; d < dc.n_present; d += blockDim.x) m = min(m, cnt[d]);
  for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) ws.scratch[threadIdx.x >> 5] = m;
  __syncthreads();
  m = INT32_MAX;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) m = min(m, ws.scratch[w]);
  __syncthreads();
  int32_t num = 0;
  for (int d = threadIdx.x; d < dc.n_present; d += blockDim.x) num += (cnt[d] == m);
  for (int o = 16; o > 0; o >>= 1) num += __shfl_xor_sync(0xffffffffu, num, o);
  if ((threadIdx.x & 31) == 0) ws.scratch[threadIdx.x >> 5] = num;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += ws.scratch[w];
    ws.ptsmin[c] = pc.min_zero ? 0 : m;    // filtering.go:56-69: fewer domains than minDomains -> global minimum 0
    ws.ptsnum[c] = s;
    ws.dirty = 1;
  }
  __syncthreads();
}

// PodTopologySpread.Score of a node that is not in IgnoredNodes, with this wave's weights (scoring.go:192-224,302-304)
__device__ __forceinline__ long long spts_raw(const DevParams &p, const ccsim_template &t, int32_t i) {
  double score = 0.0;
  for (int c = 0; c < t.n_spts; c++) {
    const ccsim_spts sc = t.spts[c];
    long long cnt;
    if (sc.hostname) {
      if (sc.has_key_bit >= 0 && !static_bit(p, i, sc.has_key_bit)) continue;
      cnt = ws.cnt_ptr[sc.counter][i];
    } else {
      const int32_t dom = ws.topo_ptr[p.counters[sc.counter].topo_col][i];
      if (dom < 0) continue;
      cnt = ws.cnt_ptr[sc.counter][dom];
    }
    score = __dadd_rn(score, __dadd_rn(__dmul_rn((double)cnt, ws.spts_w[c]), (double)(sc.max_skew - 1)));
  }
  return __double2ll_rn(round(score)) ;   // math.Round: half away from zero (round() already yields an integer value)
}

// InterPodAffinity.Score (interpodaffinity/scoring.go:236-256)
__device__ __forceinline__ long long ipa_raw(const DevParams &p, const ccsim_template &t, int32_t i) {
  long long sc = 0;
  for (int k = 0; k < t.n_ipa_score; k++) {
    const int j = t.ipa_score_counter[k];
    const int32_t tc = p.counters[j].topo_col;
    const int32_t dom = tc < 0 ? i : ws.topo_ptr[tc][i];
    if (dom >= 0) sc += ws.cnt_ptr[j][dom];
  }
  return sc;
}

// Dynamic shared memory of ccsim_wave_kernel: the counters, then (RESIDENT) the node tile. Must agree with the kernel's carving: per node
// 8 B for taint, static (if any), alloc / req / nz / free cpu and memory; 4 B for free_pods, alloc_pods, npods, score, topology, local counters
static size_t wave_smem_bytes(const DevParams &p, bool resident) {
  const size_t per_node = 8 * (9 + (p.static_words > 0 ? 1 : 0)) + 4 * (4 + p.n_topo + p.n_local);
  return (((size_t)p.smem_cnt_ints * 4 + 15) & ~(size_t)15) + (resident ? per_node * (size_t)p.chunk_pad : 0);
}

// ------------------------------------------------------------------------------------------------------------------
// The persistent wave kernel (sequential engine: one winner per wave; always a valid execution of the reference loop)
//   RESIDENT: the CTA's node tile (every column the Filter/Score pass reads) is staged into shared memory once and
//             stays there for all waves; commits write through to the global columns (read by the diagnosis pass).
//   streaming: tiles too large for shared memory are re-read from global memory (L2) every wave.
// ------------------------------------------------------------------------------------------------------------------
template <bool RESIDENT>
__global__ void __launch_bounds__(BLOCK_THREADS, 1) ccsim_wave_kernel(const DevParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t *smem_cnt = reinterpret_cast<int32_t *>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int ncls = p.n_classes;
  const bool use_cache = (p.n_templates == 1);

  // ---- tile: shared-memory columns (pre-offset by -lo) or the global columns themselves ----
  Tile tl;
  int32_t *tile_topo = nullptr, *tile_local = nullptr;
  if (RESIDENT) {
    const size_t cp = (size_t)p.chunk_pad;
    unsigned char *base = smem_raw + (((size_t)p.smem_cnt_ints * 4 + 15) & ~(size_t)15);
    unsigned long long *q8 = reinterpret_cast<unsigned long long *>(base);
    unsigned long long *s_taint = q8;            q8 += cp;
    unsigned long long *s_static = q8;           if (p.static_words > 0) q8 += cp;
    long long *s_acpu = (long long *)q8;         q8 += cp;
    long long *s_amem = (long long *)q8;         q8 += cp;
    long long *s_rcpu = (long long *)q8;         q8 += cp;
    long long *s_rmem = (long long *)q8;         q8 += cp;
    long long *s_zcpu = (long long *)q8;         q8 += cp;
    long long *s_zmem = (long long *)q8;         q8 += cp;
    long long *s_fcpu = (long long *)q8;         q8 += cp;
    long long *s_fmem = (long long *)q8;         q8 += cp;
    int32_t *q4 = reinterpret_cast<int32_t *>(q8);
    int32_t *s_fpods = q4;                       q4 += cp;
    int32_t *s_apods = q4;                       q4 += cp;
    int32_t *s_npods = q4;                       q4 += cp;
    int32_t *s_score = q4;                       q4 += cp;
    tile_topo = q4;                              q4 += cp * p.n_topo;
    tile_local = q4;
    for (int32_t i = lo + tid; i < hi; i += blockDim.x) {
      const int32_t j = i - lo;
      s_taint[j] = p.taint_mask[i];
      if (p.static_words > 0) s_static[j] = p.static_mask[i];
      s_acpu[j] = p.alloc_cpu[i]; s_amem[j] = p.alloc_mem[i];
      s_rcpu[j] = p.req_cpu[i];   s_rmem[j] = p.req_mem[i];
      s_zcpu[j] = p.nz_cpu[i];    s_zmem[j] = p.nz_mem[i];
      s_apods[j] = p.alloc_pods[i]; s_npods[j] = p.npods[i];
      s_fcpu[j] = s_acpu[j] - s_rcpu[j]; s_fmem[j] = s_amem[j] - s_rmem[j]; s_fpods[j] = s_apods[j] - s_npods[j];
      s_score[j] = -1;
      for (int c = 0; c < p.n_topo; c++) tile_topo[(size_t)c * cp + j] = p.topo[c][i];
    }
    tl.taint0 = s_taint - lo; tl.static0 = s_static - lo;
    tl.alloc_cpu = s_acpu - lo; tl.alloc_mem = s_amem - lo; tl.req_cpu = s_rcpu - lo; tl.req_mem = s_rmem - lo;
    tl.nz_cpu = s_zcpu - lo; tl.nz_mem = s_zmem - lo;
    tl.alloc_pods = s_apods - lo; tl.npods = s_npods - lo; tl.score = s_score - lo;
    tl.free_cpu = s_fcpu - lo; tl.free_mem = s_fmem - lo; tl.free_pods = s_fpods - lo;
  } else {
    tl.taint0 = (const unsigned long long *)p.taint_mask; tl.static0 = (const unsigned long long *)p.static_mask;
    tl.alloc_cpu = (const long long *)p.alloc_cpu; tl.alloc_mem = (const long long *)p.alloc_mem;
    tl.req_cpu = (long long *)p.req_cpu; tl.req_mem = (long long *)p.req_mem;
    tl.nz_cpu = (long long *)p.nz_cpu; tl.nz_mem = (long long *)p.nz_mem;
    tl.alloc_pods = p.alloc_pods; tl.npods = p.npods; tl.score = p.score_cache;
    tl.free_cpu = nullptr; tl.free_mem = nullptr; tl.free_pods = nullptr;
    for (int32_t i = lo + tid; i < hi; i += blockDim.x) p.score_cache[i] = -1;
  }

  // ---- prologue: template 0, replicated counters, pointer tables, PTS minima ----
  for (int k = tid; k < (int)(sizeof(ccsim_template) / 8); k += blockDim.x)
    reinterpret_cast<unsigned long long *>(&ws.tmpl)[k] = reinterpret_cast<const unsigned long long *>(&p.templates[0])[k];
  {
    int nl = 0;
    for (int j = 0; j < p.n_counters; j++) {
      const DevCounter &dc = p.counters[j];
      if (dc.topo_col < 0) {   // node-local column (restored by the host before the launch)
        int32_t *col = dc.work;
        if (RESIDENT) {
          int32_t *sc = tile_local + (size_t)nl * p.chunk_pad;
          for (int32_t i = lo + tid; i < hi; i += blockDim.x) sc[i - lo] = dc.work[i];
          col = sc - lo;
        }
        if (tid == 0) ws.cnt_ptr[j] = col;
        nl++;
        continue;
      }
      int32_t *dst = dc.smem_off >= 0 ? smem_cnt + dc.smem_off : dc.work + (size_t)cta * dc.n_domains;
      for (int d = tid; d < dc.n_domains; d += blockDim.x) dst[d] = dc.init[d];
      if (tid == 0) ws.cnt_ptr[j] = dst;
    }
  }
  if (tid == 0) {
    for (int c = 0; c < p.n_topo; c++) ws.topo_ptr[c] = RESIDENT ? (tile_topo + (size_t)c * p.chunk_pad - lo) : p.topo[c];
    ws.aff_total = p.templates[0].aff_total_init; ws.winner = -1; ws.stop = 0; ws.dirty = 1;
  }
  __syncthreads();
  for (int c = 0; c < ws.tmpl.n_pts; c++) pts_recount(p, c);

#ifdef CCSIM_PHASE_TIMERS
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tc0 = 0, tc1 = 0;
#endif
  long long k = 0;
  bool limit_hit = false;   // postBindHook's limit (simulator.go:300-305)
  uint32_t wtag = 1;         // 1..4095; waves k and k+2 (same parity buffer) always differ
  uint32_t tag = (p.epoch << 12) | wtag;
  int32_t ti = 0;            // template of pod k = k % n_templates (report.go:160)
  for (;; k++) {
    PH_START();
    // postBindHook limit (pkg/framework/simulator.go:300-305): checked after the k-th pod was bound
    if (p.max_pods > 0 && k >= p.max_pods) { limit_hit = true; break; }   // uniform; no shared write (slower threads may still be reading ws.stop)
    if (k > p.pod_cap) { if (tid == 0) ws.stop = 3; __syncthreads(); break; }   // cannot happen (pod_cap bounds every run): never spin forever
    if (p.n_templates > 1) {
      const ccsim_template *src = &p.templates[ti];
      for (int q = tid; q < (int)(sizeof(ccsim_template) / 8); q += blockDim.x)
        reinterpret_cast<unsigned long long *>(&ws.tmpl)[q] = reinterpret_cast<const unsigned long long *>(src)[q];
      if (tid == 0) ws.dirty = 1;
      __syncthreads();
    }
    const ccsim_template &t = ws.tmpl;
    if (ws.dirty) {    // uniform: written before the last barrier
      if (tid == 0) {
        build_filter_consts(p, t, ti, ws.topo_ptr, ws.cnt_ptr, ws.ptsmin, ws.aff_total, ws.fc);
        ws.sw.w_fit = (t.score_enable & CCSIM_PL_FIT) ? t.w_fit : 0;
        ws.sw.w_balanced = ((t.score_enable & CCSIM_PL_BALANCED) && !(t.flags & CCSIM_TF_BALANCED_SKIP)) ? t.w_balanced : 0;
        ws.sw.least_w_cpu = t.least_w_cpu; ws.sw.least_w_mem = t.least_w_mem;
        for (int j = 0; j < p.n_counters; j++) {
          const DevCounter &dc = p.counters[j];
          CommitInfo &ci = ws.cinfo[j];
          const bool skip = (dc.inc == 0) || (dc.is_aff && !(t.flags & CCSIM_TF_AFF_SELF_MATCH_ALL));
          ci.inc = skip ? 0 : dc.inc;
          ci.local = dc.topo_col < 0; ci.is_aff = dc.is_aff; ci.n_present = dc.n_present; ci.elig_bit = dc.elig_bit;
          ci.gtopo = dc.topo_col < 0 ? nullptr : p.topo_full[dc.topo_col];
          ci.ltopo = dc.topo_col < 0 ? nullptr : ws.topo_ptr[dc.topo_col];
          ci.pts_idx = -1;
          for (int c = 0; c < t.n_pts; c++) if (t.pts[c].counter == j && !t.pts[c].min_zero) ci.pts_idx = c;
        }
      }
      __syncthreads();
      if (tid == 0) ws.dirty = 0;    // cleared only after every thread has read it
    }
    const FilterConsts &fc = ws.fc;
    const HotConsts hc = load_hot(fc);

    // ---- fused Filter pass over this CTA's tile (+ memoised node-local score of the feasible nodes) ----
    unsigned long long best[CCSIM_MAX_CLASSES];
    #pragma unroll
    for (int c = 0; c < CCSIM_MAX_CLASSES; c++) best[c] = 0ull;
    // Normalised soft scorers (NodeAffinity preferred terms, PodTopologySpread ScheduleAnyway/system defaults, InterPodAffinity
    // score) need extrema of their raw scores over the FEASIBLE nodes of this cycle before any node's total is known
    // (helper/normalize_score.go:28-56; podtopologyspread/scoring.go:226-265; interpodaffinity/scoring.go:258-290): such
    // templates take up to three passes over the tile with one or two extra grid-wide exchanges per wave.
    const bool na_on = (t.n_pref_terms > 0) && (t.score_enable & CCSIM_PL_NODE_AFFINITY);
    const bool spts_on = (t.n_spts > 0) && (t.score_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD);
    const bool ipa_on = (t.n_ipa_score > 0) && (t.score_enable & CCSIM_PL_INTER_POD_AFFINITY);
    const bool soft = na_on || spts_on || ipa_on;
    const int32_t w_image = ((t.score_enable & CCSIM_PL_IMAGE_LOCALITY) && t.image_score) ? t.w_image : 0;
    const uint32_t stamp_now = (uint32_t)(k + 1);
    long long na_local = 0, ipa_lo = LLONG_MAX, ipa_hi = LLONG_MIN, scored_local = 0;
    for (int32_t i = lo + tid; i < hi; i += blockDim.x) {
      int cls;
      const bool ok = filter_node<RESIDENT>(p, hc, fc, tl, i, cls);
      if (soft) p.feas[i] = ok ? 1 : 0;
      if (ok) {
        int32_t sc = use_cache ? tl.score[i] : -1;
        if (sc < 0) {
          sc = score_node(tl.alloc_cpu[i], tl.alloc_mem[i], tl.nz_cpu[i] + t.least_cpu, tl.nz_mem[i] + t.least_mem,
                          tl.req_cpu[i] + t.bal_cpu, tl.req_mem[i] + t.bal_mem, ws.sw);
          if (w_image) sc += w_image * (int32_t)t.image_score[i];
          if (use_cache || soft) tl.score[i] = sc;
        }
        if (soft) {
          if (na_on) na_local = max(na_local, (long long)node_affinity_raw(p, t, i));
          if (ipa_on) { const long long r = ipa_raw(p, t, i); ipa_lo = min(ipa_lo, r); ipa_hi = max(ipa_hi, r); }
          if (spts_on && !(t.spts_ignored_bit >= 0 && static_bit(p, i, t.spts_ignored_bit))) {
            scored_local++;
            for (int c = 0; c < t.n_spts; c++) {
              if (t.spts[c].hostname) continue;
              const DevCounter &dc = p.counters[t.spts[c].counter];
              const int32_t dom = ws.topo_ptr[dc.topo_col][i];
              __stcg(&p.stamp[c][dom < 0 ? dc.n_domains : dom], stamp_now);   // a missing key reads as the value ""
            }
          }
          continue;
        }
        const unsigned long long key = pack_key(sc, (uint32_t)(p.node_base + i));
        if (ncls == 1) best[0] = key > best[0] ? key : best[0];
        else {
          #pragma unroll
          for (int c = 0; c < CCSIM_MAX_CLASSES; c++) if (c == cls) best[c] = key > best[c] ? key : best[c];
        }
      }
    }
    if (soft) {
      long long spts_lo = LLONG_MAX, spts_hi = 0;
      if (spts_on) {
        // ---- PreScore: sizes of the topologies among the scored nodes -> weights (scoring.go:60-116,294-296) ----
        for (int o = 16; o > 0; o >>= 1) scored_local += __shfl_xor_sync(0xffffffffu, scored_local, o);
        if (lane == 0) ws.red[warp][0] = scored_local;
        __syncthreads();
        if (warp == 0) {
          long long m = (lane < (int)(blockDim.x >> 5)) ? ws.red[lane][0] : 0;
          for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
          bool dead = false;
          const unsigned long long g = exchange_sum_fenced(p, k, tag, CCSIM_MAX_CLASSES, (unsigned long long)m, lane, cta, dead);
          if (lane == 0) { ws.spts_scored = (long long)g; if (dead) ws.stop = 3; }
        }
        __syncthreads();
        for (int c = 0; c < t.n_spts; c++) {
          long long size = ws.spts_scored;
          if (!t.spts[c].hostname) {
            const int nd1 = p.counters[t.spts[c].counter].n_domains + 1;
            int32_t cnt = 0;
            for (int d = tid; d < nd1; d += blockDim.x) cnt += (__ldcg(&p.stamp[c][d]) == stamp_now);
            for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
            if (lane == 0) ws.scratch[warp] = cnt;
            __syncthreads();
            size = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); w++) size += ws.scratch[w];
          }
          if (tid == 0) ws.spts_w[c] = go_log((double)(size + 2));
          __syncthreads();
        }
        for (int32_t i = lo + tid; i < hi; i += blockDim.x) {
          if (!p.feas[i] || (t.spts_ignored_bit >= 0 && static_bit(p, i, t.spts_ignored_bit))) continue;
          const long long r = spts_raw(p, t, i);
          spts_lo = min(spts_lo, r); spts_hi = max(spts_hi, r);
        }
      }
      // ---- extrema over the feasible nodes: block reduction, then one grid-wide exchange of five words ----
      {
        long long v[5] = {na_local, spts_hi, spts_lo == LLONG_MAX ? LLONG_MIN : -spts_lo, ipa_hi, ipa_lo == LLONG_MAX ? LLONG_MIN : -ipa_lo};
        #pragma unroll
        for (int q = 0; q < 5; q++) {
          for (int o = 16; o > 0; o >>= 1) { const long long u = __shfl_xor_sync(0xffffffffu, v[q], o); v[q] = u > v[q] ? u : v[q]; }
          if (lane == 0) ws.red[warp][q] = v[q];
        }
      }
      __syncthreads();
      if (warp == 0) {
        const long long IPA_BIAS = 1ll << 40;
        long long v[5];
        #pragma unroll
        for (int q = 0; q < 5; q++) {
          long long m = (q == 0 || q == 1) ? 0 : LLONG_MIN;
          if (lane < (int)(blockDim.x >> 5)) m = ws.red[lane][q];
          for (int o = 16; o > 0; o >>= 1) { const long long u = __shfl_xor_sync(0xffffffffu, m, o); m = u > m ? u : m; }
          v[q] = m;
        }
        // encode as non-zero unsigned maxima (0 = this CTA has no feasible node)
        unsigned long long e[5];
        e[0] = (unsigned long long)(v[0] + 1);
        e[1] = (v[2] == LLONG_MIN) ? 0ull : (unsigned long long)(v[1] + 1);
        e[2] = (v[2] == LLONG_MIN) ? 0ull : (unsigned long long)((1ll << 43) + v[2]);       // 2^43 - min
        e[3] = (v[4] == LLONG_MIN) ? 0ull : (unsigned long long)(v[3] + IPA_BIAS);
        e[4] = (v[4] == LLONG_MIN) ? 0ull : (unsigned long long)(v[4] + IPA_BIAS);          // bias - min
        bool dead = false;
        exchange_max_n<5>(p, k, tag, CCSIM_MAX_CLASSES + 1, e, lane, cta, dead);
        if (lane == 0) {
          ws.na_max = e[0] ? (long long)e[0] - 1 : 0;
          ws.spts_max = e[1] ? (long long)e[1] - 1 : 0;
          ws.spts_min = e[2] ? (1ll << 43) - (long long)e[2] : LLONG_MAX;
          ws.ipa_max = e[3] ? (long long)e[3] - IPA_BIAS : LLONG_MIN;
          ws.ipa_min = e[4] ? IPA_BIAS - (long long)e[4] : LLONG_MAX;
          if (dead) ws.stop = 3;
        }
      }
      __syncthreads();
      const long long na_max = ws.na_max, pmin = ws.spts_min, pmax = ws.spts_max, imin = ws.ipa_min, imax = ws.ipa_max;
      for (int32_t i = lo + tid; i < hi; i += blockDim.x) {
        if (!p.feas[i]) continue;
        long long total = tl.score[i];
        if (na_on) {
          const long long raw = node_affinity_raw(p, t, i);
          total += (long long)t.w_node_affinity * (na_max == 0 ? raw : 100 * raw / na_max);
        }
        if (spts_on && !(t.spts_ignored_bit >= 0 && static_bit(p, i, t.spts_ignored_bit))) {
          const long long r = spts_raw(p, t, i);
          total += (long long)t.w_pts * (pmax == 0 ? 100 : 100 * (pmax + pmin - r) / pmax);
        }
        if (ipa_on && imax > imin) {
          const long long r = ipa_raw(p, t, i);
          const double f = __dmul_rn(100.0, __ddiv_rn((double)(r - imin), (double)(imax - imin)));
          total += (long long)t.w_ipa * __double2ll_rz(f);
        }
        const unsigned long long key = pack_key(total, (uint32_t)(p.node_base + i));
        if (ncls == 1) best[0] = key > best[0] ? key : best[0];
        else {
          const int cls = __popcll(tl.taint0[i] & hc.prefer0) + ((hc.extras & CCSIM_X_TAINT_WORDS) ? prefer_count_hi(p.self, fc.tmpl_index, i) : 0);
          #pragma unroll
          for (int c = 0; c < CCSIM_MAX_CLASSES; c++) if (c == cls) best[c] = key > best[c] ? key : best[c];
        }
      }
    }
    for (int c = 0; c < ncls; c++) {
      unsigned long long v = 0ull;
      #pragma unroll
      for (int q = 0; q < CCSIM_MAX_CLASSES; q++) if (q == c) v = best[q];
      v = warp_max_u64(v);
      if (lane == 0) ws.warp_best[warp][c] = v;
    }
    PH_MARK(0);
    __syncthreads();                                                    // S1
    PH_MARK(1);

    if (warp == 0) {
      const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
      unsigned long long *myslots = p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE;
      // CTA arg-max per class, published as one tagged word each
      for (int c = 0; c < ncls; c++) {
        unsigned long long v = (lane < (int)(blockDim.x >> 5)) ? ws.warp_best[lane][c] : 0ull;
        v = warp_max_u64(v);
        if (lane == 0) st_slot(&myslots[c], v | tagbits);
      }
      PH_MARK(2);
      // gather every CTA's word: all of a lane's loads are in flight together; retry until every tag is this wave's
      const unsigned long long *all = p.slots + (size_t)(k & 1) * CCSIM_MAX_GRID * SLOT_STRIDE;
      unsigned long long cbest[CCSIM_MAX_CLASSES];
      bool dead = false;
      for (int c = 0; c < ncls; c++) {
        unsigned long long v[CCSIM_MAX_GRID / 32];
        unsigned spins = 0;
        bool pending;
        do {
          pending = false;
          #pragma unroll
          for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) {
            const int b = lane + 32 * q;
            v[q] = (b < p.grid) ? ld_slot(&all[(size_t)b * SLOT_STRIDE + c]) : tagbits;
          }
          #pragma unroll
          for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) pending |= ((uint32_t)(v[q] >> KEY_TAG_SHIFT) != tag);
          if (++spins > WATCHDOG_SPINS) { dead = true; break; }
        } while (__any_sync(0xffffffffu, pending));
        unsigned long long m = 0ull;
        #pragma unroll
        for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) { const unsigned long long b = v[q] & KEY_BODY_MASK; m = b > m ? b : m; }
        cbest[c] = warp_max_u64(m);
      }
      dead = __any_sync(0xffffffffu, dead);
      if (p.world > 1 && !dead) dead = cross_gpu_exchange(p, k, tag, ncls, cbest, lane, cta);
      PH_MARK(3);
      // prioritizeNodes + selectHost over the class winners (schedule_one.go:776-941)
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
      if (lane == 0) {
        if (dead) { ws.stop = 3; ws.winner = -1; }
        else if (wkey == 0ull) { ws.stop = 1; ws.winner = -1; }
        else ws.winner = (int32_t)key_index(wkey);
      }
      // ---- commit (assume -> AssumePod -> NodeInfo.update(+1): schedule_one.go:967-984, types.go:409-427) ----
      if (!dead && wkey != 0ull) {
        const int32_t g = (int32_t)key_index(wkey);
        const int32_t w = g - p.node_base;
        const bool mine = (w >= lo && w < hi);
        if (mine && lane == 31) {
          const long long rc = tl.req_cpu[w] + t.req_cpu, rm = tl.req_mem[w] + t.req_mem;
          const long long zc = tl.nz_cpu[w] + t.nz_cpu, zm = tl.nz_mem[w] + t.nz_mem;
          const int32_t np = tl.npods[w] + 1;
          tl.req_cpu[w] = rc; tl.req_mem[w] = rm; tl.nz_cpu[w] = zc; tl.nz_mem[w] = zm; tl.npods[w] = np;
          tl.score[w] = -1;    // this node's NodeInfo generation changed
          if (RESIDENT) {      // write through: the global columns stay the authoritative snapshot-after-run
            tl.free_cpu[w] = tl.alloc_cpu[w] - rc; tl.free_mem[w] = tl.alloc_mem[w] - rm; tl.free_pods[w] = tl.alloc_pods[w] - np;
            p.req_cpu[w] = rc; p.req_mem[w] = rm; p.nz_cpu[w] = zc; p.nz_mem[w] = zm; p.npods[w] = np;
          }
          if (t.req_eph != 0) p.req_eph[w] += t.req_eph;
          for (int q = 0; q < p.n_scalars; q++) if (t.req_scalar[q] != 0) p.req_scalar[q][w] += t.req_scalar[q];
          if (p.placed_mask) p.placed_mask[w] |= 1ull << ti;
          // ClusterCapacityBinder.Bind + postBindHook: record pod k -> node (plugin.go:34-53; simulator.go:297-312)
          if (k < p.pod_cap) p.pod_node[k] = g; else ws.stop = 3;
        }
        if (p.world > 1 && !mine && cta == 0 && lane == 31) {   // sharded run: every rank keeps the whole pod -> node sequence
          const bool local = (w >= 0 && w < p.n);
          if (!local) { if (k < p.pod_cap) p.pod_node[k] = g; else ws.stop = 3; }
        }
        // per-domain counters: every CTA applies the same update to its own replica, one lane per counter
        // (the next cycle's PreFilter recount would see this clone: podtopologyspread/filtering.go:255-289,
        //  interpodaffinity/filtering.go:234-271)
        if (lane < p.n_counters) {
          const int j = lane;
          const CommitInfo ci = ws.cinfo[j];
          if (ci.inc && !(ci.elig_bit >= 0 && !static_bit(p, w, ci.elig_bit))) {   // elig_bit only exists on single-GPU runs: w is a local index
            if (ci.local) {
              if (mine) {
                const int32_t nv = ws.cnt_ptr[j][w] + ci.inc;
                ws.cnt_ptr[j][w] = nv;
                if (RESIDENT) p.counters[j].work[w] = nv;
              }
              if (ci.is_aff) { atomicAdd((unsigned long long *)&ws.aff_total, (unsigned long long)ci.inc); ws.dirty = 1; }
            } else {
              // the winner's domain id: from this CTA's tile if it owns the node, else from the global column (L2)
              const int32_t dom = mine ? ci.ltopo[w] : ci.gtopo[g];   // gtopo: whole-cluster column, global index
              if (dom >= 0) {
                int32_t *cnt = ws.cnt_ptr[j];
                const int32_t old = cnt[dom];
                cnt[dom] = old + ci.inc;
                if (ci.is_aff) { atomicAdd((unsigned long long *)&ws.aff_total, (unsigned long long)ci.inc); ws.dirty = 1; }
                if (ci.pts_idx >= 0 && dom < ci.n_present && old == ws.ptsmin[ci.pts_idx]) ws.ptsnum[ci.pts_idx] -= 1;
              }
            }
          }
        }
      }
    }
    PH_MARK(4);
    __syncthreads();                                                    // S2
    PH_MARK(5);
    if (ws.stop) break;
    // a PTS minimum whose last domain moved up: recount (rare: once per n_present commits at that level)
    for (int c = 0; c < t.n_pts; c++)
      if (!t.pts[c].min_zero && ws.ptsnum[c] <= 0 && p.counters[t.pts[c].counter].n_present > 0) pts_recount(p, c);
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
    ti = (ti + 1 == p.n_templates) ? 0 : ti + 1;
  }

  // ---- epilogue ----
  if (cta == 0) {
    for (int j = 0; j < p.n_counters; j++) {
      const DevCounter &dc = p.counters[j];
      if (dc.topo_col < 0) continue;
      const int32_t *src = ws.cnt_ptr[j];
      for (int d = tid; d < dc.n_domains; d += blockDim.x) p.final_cnt[p.final_off[j] + d] = src[d];
    }
    if (tid == 0) {
      DevOut *o = p.out;
      o->placed = k;
      o->stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
      o->error = (ws.stop == 3) ? 1 : 0;
      o->waves = limit_hit ? k : k + 1;
      o->evals = o->waves * (long long)p.n;
      for (int c = 0; c < CCSIM_MAX_PTS; c++) o->ptsmin[c] = ws.ptsmin[c];
      o->aff_total = ws.aff_total;
#ifdef CCSIM_PHASE_TIMERS
      for (int q = 0; q < 8; q++) o->phase_cycles[q] = ph[q];
#endif
    }
  }
}
