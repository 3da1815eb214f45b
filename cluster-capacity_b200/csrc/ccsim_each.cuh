// ccsim_each.cuh — per-analysis runs (ccsim_run_each): every template of the handle is analysed on its own against the loaded
// snapshot, one CTA per analysis, all analyses in one launch (DESIGN.md §4.1g).
//
// For a node-local template (no per-domain counters, no normalised soft scorer, no hostPorts) placing a clone on node i changes node
// i's feasibility and score only, and node i's state after k clones is its snapshot row plus k times the template's request. An
// analysis therefore keeps a clone count k[i] per node and a 32-ary max-tree over per-node keys (pack_key body, 0 = infeasible): a
// placement reads the root, commits the winner, re-evaluates that one node and re-reduces O(log N) entries.
//
// One tree segment per normalisation class (untolerated PreferNoSchedule taints, static per template and node): the segments cover a
// stable partition of the nodes by class, made on the host (EachTerms: segment offsets, each node's leaf position), and their roots go
// through select_host_over_classes like the class winners of the wave kernels. Level 0 (the leaves) and the upper levels that do not
// fit in shared memory live in global memory; the host chooses the split (EachParams::split).
//
// Templates with coupled terms (ccsim_set_analyses: hard spread, required pod (anti-)affinity, hostPorts) keep their counters per
// analysis (EachTerms). A term whose domains hold one node each (node-local counters, hostname columns) and the hostPort self-conflict
// (k > 0) depend on the node's own clones only: they fold into the leaf. The other terms split the nodes into domain groups (class,
// domain in each of their columns), also partitioned on the host; each group is a segment, and a placement takes a group's root only
// when the group's domains pass those terms (coupled_ok on one of its nodes, the code filter_node runs). When a leaf-folded term
// changes on every node at once (a folded spread minimum moves, the affinity bypass ends) the leaves and levels are rebuilt.
#pragma once

#define EACH_THREADS 512
#define EACH_MAX_LEVELS 7     /* 32^7 > 2^31 nodes: levels 1..7 above the leaves at most */

struct EachOut {
  long long placed;
  int32_t stop_code;
  int32_t error;        // 1: the sequence buffer would overflow (cannot happen: the host sizes it from the run's bound)
  long long rebuilds;   // leaf and level rebuilds after a folded term changed on every node
};

struct EachTerms {      // one analysis's coupled terms (ccsim_set_analyses), device memory
  DevCounter counters[CCSIM_MAX_COUNTERS];   // work: the analysis's working counts (initialised from init at kernel start)
  const int32_t *topo[CCSIM_MAX_TOPO_COLS];  // the analysis's topology columns
  int32_t n_counters;
  int32_t n_seg;        // tree segments: classes, or domain groups
  int32_t port_self;    // a clone's hostPorts conflict with the next clone's (template bit t, with a placed mask as in ccsim_run)
  uint32_t leaf_sel;    // coupled_ok selection of the terms folded into the leaf
  uint32_t group_sel;   // the terms tested per group
  const long long *cof; // [(L + 1) * (n_seg + 1)]: group s's entries of level l are [cof[l * (n_seg + 1) + s], cof[... + s + 1])
  const int32_t *seg_rep;   // [n_seg] a node of group s (its domains in the group columns are the group's)
  const int32_t *seg_cls;   // [n_seg] the group's normalisation class
  const int32_t *pos;       // [n] leaf position of each node; nullptr when the partition is the identity
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
  unsigned long long *glev;     // [T][glev_stride]
  int32_t *seq;                 // [T][seq_cap] node of clone k
  EachOut *out;                 // [T]
  const EachTerms *terms;       // [T]
  DevOut *diag;                 // [T] the diagnosis's outputs: final spread minima and affinity total
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
  long long coff[EACH_MAX_LEVELS + 1][CCSIM_MAX_CLASSES + 1];   // node-local analyses: class c's entries of level l, the host's cof
  const long long *cof;   // the analysis's segment offsets (EachTerms::cof)
  int32_t cstride, nseg;  // entries per level of cof, segments
  int32_t grouped;        // segments are domain groups: a placement tests each group's terms and takes the maximum per class
  int32_t coupled;        // the analysis has counters or hostPorts
  int32_t port_self;      // a clone's hostPorts conflict with the next clone's
  uint32_t leaf_sel, group_sel;
  const int32_t *topo_ptr[CCSIM_MAX_TOPO_COLS];
  int32_t *cnt_ptr[CCSIM_MAX_COUNTERS];
  CommitInfo cinfo[CCSIM_MAX_COUNTERS];
  int32_t ptsmin[CCSIM_MAX_PTS], ptsnum[CCSIM_MAX_PTS];
  unsigned long long aff_total;
};
__shared__ EachShared es;
// G: some analysis has counters or a hostPort self-conflict (segments from the host's table); else the analyses are node-local, their
// segments are classes and the host's offsets are read from es.coff (the per-placement loads stay plain shared-memory loads)
template <bool G> __device__ __forceinline__ long long cof(int l, int s) {
  return G ? es.cof[(long long)l * es.cstride + s] : es.coff[l][s];
}

// the segment holding entry e of level l: the last s with cof(l, s) <= e
template <bool G> __device__ __forceinline__ int each_seg_of(int l, long long e) {
  if (!G) { int c = 0; while (e >= es.coff[l][c + 1]) c++; return c; }
  int lo = 0, hi = es.nseg;   // cof(l, lo) <= e < cof(l, hi)
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (cof<G>(l, mid) <= e) lo = mid; else hi = mid; }
  return lo;
}

// spread constraint c's global minimum (filtering.go:56-69) and how many domains hold it, recounted by one warp
__device__ void each_pts_recount(int c, int lane) {
  const ccsim_pts &pc = es.tmpl.pts[c];
  const int32_t *cnt = es.cnt_ptr[pc.counter];
  const int32_t np = es.cinfo[pc.counter].n_present;
  int32_t m = INT32_MAX, s = 0;
  for (int d = lane; d < np; d += 32) m = min(m, cnt[d]);
  m = __reduce_min_sync(0xffffffffu, m);
  for (int d = lane; d < np; d += 32) s += (cnt[d] == m);
  s = __reduce_add_sync(0xffffffffu, s);
  if (lane == 0) {
    es.ptsmin[c] = pc.min_zero ? 0 : m;
    es.ptsnum[c] = s;
    es.fc.pts_lim[c] = pts_limit(pc, es.ptsmin[c]);
  }
  __syncwarp();
}

// x + k * r with the wrap of k repeated int64 additions (the wave kernels' commit)
__device__ __forceinline__ long long each_add(int64_t x, uint32_t k, int64_t r) {
  return (long long)((unsigned long long)x + (unsigned long long)k * (unsigned long long)r);
}

// leaf key of node i after kk clones of the analysis's template: filter_node's Filter and the wave kernel's score on the computed
// state (snapshot row + kk * request); 0 when infeasible
template <bool G>
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
  if (G && es.coupled) {   // the terms of the node's own domain: its clones' hostPorts, node-local counters and one-node domains
    ok &= !(es.port_self && kk > 0u);
    if (ok && es.leaf_sel) coupled_ok<false>(fc, fc.n_pts, fc.n_aff, fc.n_anti, i, es.leaf_sel, ok);
  }
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

// every leaf at its node's position, evaluated after its current clones (at kernel start: none), by threads t0, t0 + nt, ...
template <bool G>
__device__ void each_leaves(const DevParams &p, const EachParams &ep, int32_t ti, int32_t *kcol, unsigned long long *leaf,
                            const int32_t *pos, bool start, int t0, int nt) {
  for (int32_t i = t0; i < p.n; i += nt) {
    if (start) kcol[i] = 0;
    leaf[pos ? pos[i] : i] = each_leaf<G>(p, ep, ti, i, start ? 0u : (uint32_t)kcol[i]);
  }
}

// upper levels, bottom up: one warp per entry, its 32 children in one coalesced load. BLOCK: the whole CTA (kernel start), else warp 0
template <bool G, bool BLOCK>
__device__ void each_levels(const EachParams &ep, unsigned long long *leaf, unsigned long long *glev, unsigned long long *slev,
                            int nseg, int w0, int nw, int lane) {
  for (int l = 1; l <= ep.n_levels; l++) {
    const unsigned long long *lo = each_level(ep, leaf, glev, slev, l - 1);
    unsigned long long *up = each_level(ep, leaf, glev, slev, l);
    const long long ne = cof<G>(l, nseg);
    for (long long g = w0; g < ne; g += nw) {
      const int c = each_seg_of<G>(l, g);
      const long long child = cof<G>(l - 1, c) + 32 * (g - cof<G>(l, c)) + lane;
      const unsigned long long v = warp_max_u64(child < cof<G>(l - 1, c + 1) ? lo[child] : 0ull);
      if (lane == 0) up[g] = v;
    }
    if (BLOCK) __syncthreads(); else __syncwarp();
  }
}

// Two instantiations (G above), so that the node-local one is compiled and register-allocated on its own
template <bool G>
__global__ void __launch_bounds__(EACH_THREADS, 1) ccsim_each_kernel(const DevParams p, const EachParams ep) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long *slev = reinterpret_cast<unsigned long long *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int32_t ti = blockIdx.x, n = p.n;
  const int ncls = p.n_classes, L = ep.n_levels;
  const EachTerms *et = ep.terms + ti;
  int32_t *kcol = ep.k + (size_t)ti * n;
  unsigned long long *leaf = ep.leaf + (size_t)ti * n;
  const int32_t *pos = et->pos;
  unsigned long long *glev = ep.glev + (size_t)ti * ep.glev_stride;
  int32_t *seq = ep.seq + (size_t)ti * ep.seq_cap;

  // ---- template, the analysis's working counters, folded Filter constants, score configuration ----
  for (int q = tid; q < (int)(sizeof(ccsim_template) / 8); q += blockDim.x)
    reinterpret_cast<unsigned long long *>(&es.tmpl)[q] = reinterpret_cast<const unsigned long long *>(&p.templates[ti])[q];
  const int ncnt = et->n_counters;
  for (int j = 0; j < ncnt; j++) {
    const DevCounter &dc = et->counters[j];
    for (int d = tid; d < dc.n_domains; d += blockDim.x) dc.work[d] = dc.init[d];
  }
  __syncthreads();
  if (tid == 0) {
    const ccsim_template &t = es.tmpl;
    es.aff_total = (unsigned long long)t.aff_total_init;
    es.leaf_sel = et->leaf_sel; es.group_sel = et->group_sel;
    es.grouped = et->group_sel ? 1 : 0;
    es.port_self = et->port_self;
    es.coupled = ncnt > 0 || es.port_self;
    es.cof = et->cof; es.cstride = et->n_seg + 1; es.nseg = et->n_seg;
    for (int k = 0; k < CCSIM_MAX_TOPO_COLS; k++) es.topo_ptr[k] = et->topo[k];
    for (int j = 0; j < CCSIM_MAX_COUNTERS; j++) es.cnt_ptr[j] = j < ncnt ? et->counters[j].work : nullptr;
    for (int j = 0; j < ncnt; j++) {   // what a commit does to each counter (the generic wave kernel's CommitInfo)
      const DevCounter &dc = et->counters[j];
      CommitInfo &ci = es.cinfo[j];
      const bool skip = (dc.inc == 0) || (dc.is_aff && !(t.flags & CCSIM_TF_AFF_SELF_MATCH_ALL));
      ci.inc = skip ? 0 : dc.inc;
      ci.local = dc.topo_col < 0; ci.is_aff = dc.is_aff; ci.n_present = dc.n_present; ci.elig_bit = dc.elig_bit;
      ci.gtopo = ci.ltopo = dc.topo_col < 0 ? nullptr : et->topo[dc.topo_col];
      ci.pts_idx = -1;
      for (int c = 0; c < t.n_pts; c++) if (t.pts[c].counter == j && !t.pts[c].min_zero) ci.pts_idx = c;
    }
    for (int c = 0; c < CCSIM_MAX_PTS; c++) { es.ptsmin[c] = 0; es.ptsnum[c] = 0; }
  }
  __syncthreads();
  if (tid == 0) {
    const ccsim_template &t = es.tmpl;
    build_filter_consts(p, et->counters, t, ti, es.topo_ptr, es.cnt_ptr, es.ptsmin, (long long)es.aff_total, es.fc);
    es.fc.extras &= ~CCSIM_X_PLACED;   // hostPorts against the analysis's own clones: k > 0 in the leaf
    es.sw.w_fit = (t.score_enable & CCSIM_PL_FIT) ? t.w_fit : 0;
    es.sw.w_balanced = ((t.score_enable & CCSIM_PL_BALANCED) && !(t.flags & CCSIM_TF_BALANCED_SKIP)) ? t.w_balanced : 0;
    es.sw.least_w_cpu = t.least_w_cpu; es.sw.least_w_mem = t.least_w_mem;
    es.w_image = ((t.score_enable & CCSIM_PL_IMAGE_LOCALITY) && t.image_score) ? t.w_image : 0;
  }
  __syncthreads();
  if (warp == 0) for (int c = 0; c < es.fc.n_pts; c++) each_pts_recount(c, lane);   // the spread minima and their limits
  __syncthreads();

  if (!G)   // the host's class offsets into shared memory (classes <= CCSIM_MAX_CLASSES, levels <= EACH_MAX_LEVELS)
    for (int q = tid; q < (L + 1) * (es.nseg + 1); q += blockDim.x) es.coff[q / (es.nseg + 1)][q % (es.nseg + 1)] = et->cof[q];

  // ---- leaves at the host's positions, every node evaluated with no clone placed; then the upper levels ----
  each_leaves<G>(p, ep, ti, kcol, leaf, pos, true, tid, blockDim.x);
  __syncthreads();
  each_levels<G, true>(ep, leaf, glev, slev, es.nseg, warp, nw, lane);

  // ---- placements: warp 0 alone ----
  if (warp != 0) return;
  const ccsim_template &t = es.tmpl;
  unsigned long long *top = each_level(ep, leaf, glev, slev, L);
  unsigned long long *lv1 = L >= 2 ? each_level(ep, leaf, glev, slev, 1) : nullptr;
  long long k = 0, rebuilds = 0;
  bool limit_hit = false;
  int error = 0;
  for (;; k++) {
    if (ep.max_pods > 0 && k >= ep.max_pods) { limit_hit = true; break; }   // postBindHook limit (simulator.go:300-305)
    if (k >= ep.seq_cap) { error = 1; break; }
    // prioritizeNodes + selectHost over the class roots (schedule_one.go:776-941)
    unsigned long long cbest[CCSIM_MAX_CLASSES];
    if (!G || !es.grouped) {   // one segment per class
      const unsigned long long r = (lane < ncls && cof<G>(L, lane + 1) > cof<G>(L, lane)) ? top[cof<G>(L, lane)] : 0ull;
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) cbest[c] = __shfl_sync(0xffffffffu, r, c);
    } else {             // a group's root counts when its domains pass the group terms; the best open group per class
      unsigned long long mine[CCSIM_MAX_CLASSES];
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) mine[c] = 0ull;
      for (int s = lane; s < es.nseg; s += 32) {
        const long long e = cof<G>(L, s);
        if (cof<G>(L, s + 1) == e) continue;
        bool ok = true;
        coupled_ok<false>(es.fc, es.fc.n_pts, es.fc.n_aff, es.fc.n_anti, et->seg_rep[s], es.group_sel, ok);
        if (!ok) continue;
        const unsigned long long v = top[e];
        const int cl = et->seg_cls[s];
        #pragma unroll
        for (int c = 0; c < CCSIM_MAX_CLASSES; c++) if (c == cl && v > mine[c]) mine[c] = v;
      }
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) cbest[c] = c < ncls ? warp_max_u64(mine[c]) : 0ull;
    }
    const unsigned long long wkey = select_host_over_classes(cbest, ncls, t);
    if (wkey == 0ull) break;                                                // Unschedulable
    const int32_t i = (int32_t)key_index(wkey);
    const long long at = pos ? pos[i] : i;
    const int c = each_seg_of<G>(0, at);
    // the winner's group of 32 on level 0 and on level 1, loaded while lane 0 commits the winner
    const long long e0 = at - cof<G>(0, c), e1 = e0 >> 5;
    const long long g0 = cof<G>(0, c) + (e0 & ~31ll) + lane;
    unsigned long long v0 = g0 < cof<G>(0, c + 1) ? leaf[g0] : 0ull, v1 = 0ull;
    if (lv1) { const long long g1 = cof<G>(1, c) + (e1 & ~31ll) + lane; v1 = g1 < cof<G>(1, c + 1) ? lv1[g1] : 0ull; }
    uint32_t kk = 0u;
    if (lane == 0) {
      kk = (uint32_t)kcol[i] + 1u;                                          // ClusterCapacityBinder commit: one more clone on i
      kcol[i] = (int32_t)kk;
      seq[k] = i;
    }
    bool rebuild = false;
    if (G && es.coupled) {
      // the counters of the winner's domains, one lane per counter (the generic wave kernel's commit)
      if (lane < ncnt) {
        const CommitInfo &ci = es.cinfo[lane];
        if (ci.inc && !(ci.elig_bit >= 0 && !static_bit(p, i, ci.elig_bit))) {
          const int32_t dom = ci.local ? i : ci.ltopo[i];
          if (dom >= 0) {
            int32_t *cnt = es.cnt_ptr[lane];
            const int32_t old = cnt[dom];
            cnt[dom] = old + ci.inc;
            if (ci.is_aff) atomicAdd(&es.aff_total, (unsigned long long)(long long)ci.inc);
            if (ci.pts_idx >= 0 && dom < ci.n_present && old == es.ptsmin[ci.pts_idx]) atomicSub(&es.ptsnum[ci.pts_idx], 1);
          }
        }
      }
      __syncwarp();
      // a spread minimum whose last domain moved up: recount; a folded constraint's limit then changed on every node
      for (int q = 0; q < es.fc.n_pts; q++)
        if (!t.pts[q].min_zero && es.ptsnum[q] <= 0 && es.cinfo[t.pts[q].counter].n_present > 0) {
          each_pts_recount(q, lane);
          rebuild |= (es.leaf_sel >> q) & 1u;
        }
      if (es.fc.aff_bypass && es.aff_total != 0ull) {   // the first matching pod ends the bypass (filtering.go:396-405)
        __syncwarp();
        if (lane == 0) es.fc.aff_bypass = 0;
        rebuild = true;
      }
      __syncwarp();
    }
    if (G && rebuild) {   // every leaf and level again, with the code of the kernel start
      each_leaves<G>(p, ep, ti, kcol, leaf, pos, false, lane, 32);
      __syncwarp();
      each_levels<G, false>(ep, leaf, glev, slev, es.nseg, 0, 1, lane);
      rebuilds++;
      continue;
    }
    unsigned long long nv = 0ull;
    if (lane == 0) nv = each_leaf<G>(p, ep, ti, i, kk);
    nv = __shfl_sync(0xffffffffu, nv, 0);
    // level l's entry e (within segment c) gets nv; its group's maximum becomes level l + 1's entry e >> 5
    long long e = e0;
    for (int l = 0; l < L; l++) {
      unsigned long long *lv = each_level(ep, leaf, glev, slev, l) + cof<G>(l, c);
      unsigned long long v;
      if (l == 0) v = v0;
      else if (l == 1) v = v1;
      else { const long long g = (e & ~31ll) + lane; v = g < cof<G>(l, c + 1) - cof<G>(l, c) ? lv[g] : 0ull; }
      if (lane == (int)(e & 31)) { v = nv; lv[e] = nv; }
      nv = warp_max_u64(v);
      e >>= 5;
    }
    if (lane == 0) top[cof<G>(L, c)] = nv;
    __syncwarp();
  }
  if (lane == 0) {
    EachOut o;
    o.placed = k;
    o.stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
    o.error = error;
    o.rebuilds = rebuilds;
    ep.out[ti] = o;
    if (G) {   // what the diagnosis reads besides the counters
      for (int q = 0; q < CCSIM_MAX_PTS; q++) ep.diag[ti].ptsmin[q] = es.ptsmin[q];
      ep.diag[ti].aff_total = (long long)es.aff_total;
    }
  }
}


// Analysis t's final node state into the working columns, for the terminal diagnosis (ccsim_diag_kernel); its counters are read
// where the run left them (EachTerms::counters[].work)
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
    if (p.placed_mask) p.placed_mask[i] = kk > 0u ? 1ull << ti : 0ull;   // hostPorts: the analysis's own clones
  }
}
