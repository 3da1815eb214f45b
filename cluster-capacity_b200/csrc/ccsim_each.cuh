// ccsim_each.cuh — per-analysis runs (ccsim_run_each): every template of the handle is analysed on its own against the loaded
// snapshot, one CTA per analysis, all analyses in one launch (DESIGN.md §4.1g).
//
// Only node-local templates run here (no per-domain counters, no normalised soft scorer, no hostPorts): placing a clone on node i
// then changes node i's feasibility and score only, and node i's state after k clones is its snapshot row plus k times the
// template's request. An analysis therefore keeps a clone count k[i] per node and a 32-ary max-tree over per-node keys (pack_key
// body, 0 = infeasible): a placement reads the root, commits the winner, re-evaluates that one node and re-reduces O(log N) entries.
//
// One tree per normalisation class (untolerated PreferNoSchedule taints, static per template and node): the class trees cover a
// stable partition of the nodes by class, and their roots go through select_host_over_classes like the class winners of the wave
// kernels. Level 0 (the leaves) and the upper levels that do not fit in shared memory live in global memory; the host chooses the
// split (EachParams::split).
#pragma once

#define EACH_THREADS 512
#define EACH_MAX_LEVELS 7     /* 32^7 > 2^31 nodes: levels 1..7 above the leaves at most */

struct EachOut {
  long long placed;
  int32_t stop_code;
  int32_t error;        // 1: the sequence buffer would overflow (cannot happen: the host sizes it from the run's bound)
};

struct EachParams {
  int32_t n_levels;     // level of the class roots (0: the leaves are the roots, N == 1)
  int32_t split;        // levels [1, split) in global memory, [split, n_levels] in shared memory
  long long lev_off[EACH_MAX_LEVELS + 1];   // first entry of level l in its region (the analysis's global block / the shared block)
  long long glev_stride;                    // entries of an analysis's global block of upper levels
  long long seq_cap;                        // entries of an analysis's placement sequence
  long long max_pods;
  int32_t *k;                   // [T][N] clones placed on each node
  unsigned long long *leaf;     // [T][N] leaf keys in partition order
  int32_t *pos;                 // [T][N] leaf position of each node; nullptr with one class (position = node index)
  unsigned long long *glev;     // [T][glev_stride]
  int32_t *seq;                 // [T][seq_cap] node of clone k
  EachOut *out;                 // [T]
  // the snapshot rows a node's state is computed from
  const int64_t *s_req_cpu, *s_req_mem, *s_req_eph, *s_nz_cpu, *s_nz_mem;
  const int32_t *s_npods;
  const int64_t *s_req_scalar[CCSIM_MAX_SCALARS];
};

struct __align__(16) EachShared {
  ccsim_template tmpl;
  FilterConsts fc;
  ScoreWeights sw;
  int32_t w_image;
  int32_t wcnt[EACH_THREADS / 32][CCSIM_MAX_CLASSES];   // partition: nodes of each class per warp in the current chunk
  int32_t crun[CCSIM_MAX_CLASSES];                       // partition: next position of each class
  long long coff[EACH_MAX_LEVELS + 1][CCSIM_MAX_CLASSES + 1];   // class c's entries of level l: [coff[l][c], coff[l][c+1])
};
__shared__ EachShared es;

// x + k * r with the wrap of k repeated int64 additions (the wave kernels' commit)
__device__ __forceinline__ long long each_add(int64_t x, uint32_t k, int64_t r) {
  return (long long)((unsigned long long)x + (unsigned long long)k * (unsigned long long)r);
}

// normalisation class of node i (filter_node's raw TaintToleration count): static per template and node
__device__ __forceinline__ int each_class(const DevParams &p, int32_t ti, int32_t i) {
  return __popcll(p.taint_mask[i] & es.fc.prefer0) + (p.taint_words > 1 ? prefer_count_hi(p.self, ti, i) : 0);
}

// leaf key of node i after kk clones of the analysis's template: filter_node's Filter and the wave kernel's score on the computed
// state (snapshot row + kk * request); 0 when infeasible
__device__ unsigned long long each_leaf(const DevParams &p, const EachParams &ep, int32_t ti, int32_t i, uint32_t kk) {
  const ccsim_template &t = es.tmpl;
  const FilterConsts &fc = es.fc;
  bool ok = (p.taint_mask[i] & fc.taint_bad0) == 0ull;
  const long long rc = each_add(ep.s_req_cpu[i], kk, t.req_cpu), rm = each_add(ep.s_req_mem[i], kk, t.req_mem);
  if (fc.fit_pods) ok &= !((int32_t)((uint32_t)ep.s_npods[i] + kk) + 1 > p.alloc_pods[i]);
  ok &= !(fc.eq_cpu > p.alloc_cpu[i] - rc);
  ok &= !(fc.eq_mem > p.alloc_mem[i] - rm);
  if (fc.sel0 | fc.forbid0) {
    const unsigned long long sw = p.static_mask[i];
    ok &= ((~sw & fc.sel0) | (sw & fc.forbid0)) == 0ull;
  }
  // filter_extras reads ephemeral storage and extended resources from the working columns: here they are computed
  if (ok && (fc.extras & CCSIM_X_EPH)) ok = !(t.req_eph > p.alloc_eph[i] - each_add(ep.s_req_eph[i], kk, t.req_eph));
  if (ok && (fc.extras & CCSIM_X_SCALARS))
    for (int q = 0; q < p.n_scalars; q++)
      if (t.req_scalar[q] != 0) ok &= !(t.req_scalar[q] > p.alloc_scalar[q][i] - each_add(ep.s_req_scalar[q][i], kk, t.req_scalar[q]));
  const uint32_t ext = fc.extras & ~(CCSIM_X_EPH | CCSIM_X_SCALARS);
  if (ok && ext) ok = filter_extras(p.self, ti, ext, i);
  if (!ok) return 0ull;
  int32_t sc = score_node(p.alloc_cpu[i], p.alloc_mem[i], each_add(ep.s_nz_cpu[i], kk, t.nz_cpu) + t.least_cpu,
                          each_add(ep.s_nz_mem[i], kk, t.nz_mem) + t.least_mem, rc + t.bal_cpu, rm + t.bal_mem, es.sw);
  if (es.w_image) sc += es.w_image * (int32_t)t.image_score[i];
  return pack_key(sc, (uint32_t)i);
}

// level l of this analysis's trees (level 0: the leaves)
__device__ __forceinline__ unsigned long long *each_level(const EachParams &ep, unsigned long long *leaf, unsigned long long *glev,
                                                          unsigned long long *slev, int l) {
  return l == 0 ? leaf : (l < ep.split ? glev : slev) + ep.lev_off[l];
}

__global__ void __launch_bounds__(EACH_THREADS, 1) ccsim_each_kernel(const DevParams p, const EachParams ep) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long *slev = reinterpret_cast<unsigned long long *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int32_t ti = blockIdx.x, n = p.n;
  const int ncls = p.n_classes, L = ep.n_levels;
  int32_t *kcol = ep.k + (size_t)ti * n;
  unsigned long long *leaf = ep.leaf + (size_t)ti * n;
  int32_t *pos = ep.pos ? ep.pos + (size_t)ti * n : nullptr;
  unsigned long long *glev = ep.glev + (size_t)ti * ep.glev_stride;
  int32_t *seq = ep.seq + (size_t)ti * ep.seq_cap;

  // ---- template, folded Filter constants, score configuration ----
  for (int q = tid; q < (int)(sizeof(ccsim_template) / 8); q += blockDim.x)
    reinterpret_cast<unsigned long long *>(&es.tmpl)[q] = reinterpret_cast<const unsigned long long *>(&p.templates[ti])[q];
  if (tid < CCSIM_MAX_CLASSES) es.crun[tid] = 0;
  __syncthreads();
  if (tid == 0) {
    const ccsim_template &t = es.tmpl;
    const int32_t *no_topo[CCSIM_MAX_TOPO_COLS] = {};
    int32_t *no_cnt[CCSIM_MAX_COUNTERS] = {};
    const int32_t no_min[CCSIM_MAX_PTS] = {};
    build_filter_consts(p, t, ti, no_topo, no_cnt, no_min, t.aff_total_init, es.fc);
    es.sw.w_fit = (t.score_enable & CCSIM_PL_FIT) ? t.w_fit : 0;
    es.sw.w_balanced = ((t.score_enable & CCSIM_PL_BALANCED) && !(t.flags & CCSIM_TF_BALANCED_SKIP)) ? t.w_balanced : 0;
    es.sw.least_w_cpu = t.least_w_cpu; es.sw.least_w_mem = t.least_w_mem;
    es.w_image = ((t.score_enable & CCSIM_PL_IMAGE_LOCALITY) && t.image_score) ? t.w_image : 0;
  }
  __syncthreads();

  // ---- class sizes (several classes only): class c's leaves are positions [coff[0][c], coff[0][c+1]) ----
  if (ncls > 1) {
    int cnt[CCSIM_MAX_CLASSES] = {};
    for (int32_t i = tid; i < n; i += blockDim.x) {
      const int c = each_class(p, ti, i);
      #pragma unroll
      for (int q = 0; q < CCSIM_MAX_CLASSES; q++) cnt[q] += (q == c);
    }
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_CLASSES; q++) {
      const int v = __reduce_add_sync(0xffffffffu, cnt[q]);
      if (lane == 0 && v) atomicAdd(&es.crun[q], v);
    }
  } else if (tid == 0) es.crun[0] = n;
  __syncthreads();
  if (tid == 0) {   // entries per class and level: ceil(size / 32^l); crun becomes the partition's running position
    long long run = 0;
    for (int c = 0; c < ncls; c++) { const long long sz = es.crun[c]; es.crun[c] = (int32_t)run; es.coff[0][c] = run; run += sz; }
    es.coff[0][ncls] = run;
    for (int l = 1; l <= L; l++) {
      long long acc = 0;
      for (int c = 0; c < ncls; c++) {
        const long long sz = es.coff[l - 1][c + 1] - es.coff[l - 1][c];
        es.coff[l][c] = acc; acc += (sz + 31) >> 5;
      }
      es.coff[l][ncls] = acc;
    }
  }
  __syncthreads();

  // ---- leaves: stable partition by class (node order inside a class), every node evaluated with no clone placed ----
  for (int32_t base = 0; base < n; base += blockDim.x) {
    const int32_t i = base + tid;
    int32_t at = i;
    if (ncls > 1) {
      const int c = i < n ? each_class(p, ti, i) : -1;
      int rank = 0;
      for (int q = 0; q < ncls; q++) {
        const unsigned b = __ballot_sync(0xffffffffu, c == q);
        if (c == q) rank = __popc(b & ((1u << lane) - 1u));
        if (lane == 0) es.wcnt[warp][q] = __popc(b);
      }
      __syncthreads();
      if (c >= 0) {
        at = es.crun[c] + rank;
        for (int w = 0; w < warp; w++) at += es.wcnt[w][c];
      }
      __syncthreads();
      if (tid < ncls) { int s = 0; for (int w = 0; w < nw; w++) s += es.wcnt[w][tid]; es.crun[tid] += s; }
      __syncthreads();
    }
    if (i < n) {
      kcol[i] = 0;
      if (pos) pos[i] = at;
      leaf[at] = each_leaf(p, ep, ti, i, 0u);
    }
  }
  __syncthreads();

  // ---- upper levels, bottom up: one warp per entry, its 32 children in one coalesced load ----
  for (int l = 1; l <= L; l++) {
    const unsigned long long *lo = each_level(ep, leaf, glev, slev, l - 1);
    unsigned long long *up = each_level(ep, leaf, glev, slev, l);
    for (long long g = warp; g < es.coff[l][ncls]; g += nw) {
      int c = 0;
      while (g >= es.coff[l][c + 1]) c++;
      const long long child = es.coff[l - 1][c] + 32 * (g - es.coff[l][c]) + lane;
      const unsigned long long v = warp_max_u64(child < es.coff[l - 1][c + 1] ? lo[child] : 0ull);
      if (lane == 0) up[g] = v;
    }
    __syncthreads();
  }

  // ---- placements: warp 0 alone ----
  if (warp != 0) return;
  const ccsim_template &t = es.tmpl;
  unsigned long long *top = each_level(ep, leaf, glev, slev, L);
  unsigned long long *lv1 = L >= 2 ? each_level(ep, leaf, glev, slev, 1) : nullptr;
  long long k = 0;
  bool limit_hit = false;
  int error = 0;
  for (;; k++) {
    if (ep.max_pods > 0 && k >= ep.max_pods) { limit_hit = true; break; }   // postBindHook limit (simulator.go:300-305)
    if (k >= ep.seq_cap) { error = 1; break; }
    // prioritizeNodes + selectHost over the class roots (schedule_one.go:776-941)
    const unsigned long long r = (lane < ncls && es.coff[L][lane + 1] > es.coff[L][lane]) ? top[es.coff[L][lane]] : 0ull;
    unsigned long long cbest[CCSIM_MAX_CLASSES];
    #pragma unroll
    for (int c = 0; c < CCSIM_MAX_CLASSES; c++) cbest[c] = __shfl_sync(0xffffffffu, r, c);
    const unsigned long long wkey = select_host_over_classes(cbest, ncls, t);
    if (wkey == 0ull) break;                                                // Unschedulable
    const int32_t i = (int32_t)key_index(wkey);
    const long long at = pos ? pos[i] : i;
    int c = 0;
    while (at >= es.coff[0][c + 1]) c++;
    // the winner's group of 32 on level 0 and on level 1, loaded while lane 0 re-evaluates the winner
    const long long e0 = at - es.coff[0][c], e1 = e0 >> 5;
    const long long g0 = es.coff[0][c] + (e0 & ~31ll) + lane;
    unsigned long long v0 = g0 < es.coff[0][c + 1] ? leaf[g0] : 0ull, v1 = 0ull;
    if (lv1) { const long long g1 = es.coff[1][c] + (e1 & ~31ll) + lane; v1 = g1 < es.coff[1][c + 1] ? lv1[g1] : 0ull; }
    unsigned long long nv = 0ull;
    if (lane == 0) {
      const uint32_t kk = (uint32_t)kcol[i] + 1u;                          // ClusterCapacityBinder commit: one more clone on i
      kcol[i] = (int32_t)kk;
      seq[k] = i;
      nv = each_leaf(p, ep, ti, i, kk);
    }
    nv = __shfl_sync(0xffffffffu, nv, 0);
    // level l's entry e (within class c's segment) gets nv; its group's maximum becomes level l + 1's entry e >> 5
    long long e = e0;
    for (int l = 0; l < L; l++) {
      unsigned long long *lv = each_level(ep, leaf, glev, slev, l) + es.coff[l][c];
      unsigned long long v;
      if (l == 0) v = v0;
      else if (l == 1) v = v1;
      else { const long long g = (e & ~31ll) + lane; v = g < es.coff[l][c + 1] - es.coff[l][c] ? lv[g] : 0ull; }
      if (lane == (int)(e & 31)) { v = nv; lv[e] = nv; }
      nv = warp_max_u64(v);
      e >>= 5;
    }
    if (lane == 0) top[es.coff[L][c]] = nv;
    __syncwarp();
  }
  if (lane == 0) {
    EachOut o;
    o.placed = k;
    o.stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
    o.error = error;
    ep.out[ti] = o;
  }
}

// Analysis t's final node state into the working columns, for the terminal diagnosis (ccsim_diag_kernel)
__global__ void ccsim_each_scatter_kernel(const DevParams p, const EachParams ep, int32_t ti) {
  const ccsim_template &t = p.templates[ti];
  const int32_t *kcol = ep.k + (size_t)ti * p.n;
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const uint32_t kk = (uint32_t)kcol[i];
    p.req_cpu[i] = each_add(ep.s_req_cpu[i], kk, t.req_cpu);
    p.req_mem[i] = each_add(ep.s_req_mem[i], kk, t.req_mem);
    p.req_eph[i] = each_add(ep.s_req_eph[i], kk, t.req_eph);
    p.nz_cpu[i] = each_add(ep.s_nz_cpu[i], kk, t.nz_cpu);
    p.nz_mem[i] = each_add(ep.s_nz_mem[i], kk, t.nz_mem);
    p.npods[i] = (int32_t)((uint32_t)ep.s_npods[i] + kk);
    for (int q = 0; q < p.n_scalars; q++) p.req_scalar[q][i] = each_add(ep.s_req_scalar[q][i], kk, t.req_scalar[q]);
  }
}
