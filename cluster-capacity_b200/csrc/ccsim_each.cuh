// ccsim_each.cuh — per-analysis runs (ccsim_run_each): every template of the handle is analysed on its own against the loaded
// snapshot, one CTA per analysis, all analyses in one launch (DESIGN.md §4.1g). Node-local analyses that outnumber the CTAs the device
// holds at once share CTAs instead, one warp's placement loop each (ccsim_each_packed_kernel).
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
#define EACH_MAX_PACK 16      /* analyses per CTA of ccsim_each_packed_kernel: one warp each */

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
  // ccsim_each_packed_kernel: analyses per CTA, shared tree-level entries of each analysis's share
  int32_t pack, n_analyses;
  long long slev_stride;
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
__shared__ EachShared es;   // ccsim_each_kernel: the CTA's analysis (the packed kernel keeps one slot per warp in dynamic shared memory)
// G: some analysis has counters or a hostPort self-conflict (segments from the host's table); else the analyses are node-local, their
// segments are classes and the host's offsets are read from S.coff (the per-placement loads stay plain shared-memory loads)
template <bool G> __device__ __forceinline__ long long cof(const EachShared &S, int l, int s) {
  return G ? S.cof[(long long)l * S.cstride + s] : S.coff[l][s];
}

// the segment holding entry e of level l: the last s with cof(l, s) <= e
template <bool G> __device__ __forceinline__ int each_seg_of(const EachShared &S, int l, long long e) {
  if (!G) { int c = 0; while (e >= S.coff[l][c + 1]) c++; return c; }
  int lo = 0, hi = S.nseg;   // cof(l, lo) <= e < cof(l, hi)
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (cof<G>(S, l, mid) <= e) lo = mid; else hi = mid; }
  return lo;
}

// spread constraint c's global minimum (filtering.go:56-69) and how many domains hold it, recounted by one warp
__device__ void each_pts_recount(EachShared &S, int c, int lane) {
  const ccsim_pts &pc = S.tmpl.pts[c];
  const int32_t *cnt = S.cnt_ptr[pc.counter];
  const int32_t np = S.cinfo[pc.counter].n_present;
  int32_t m = INT32_MAX, s = 0;
  for (int d = lane; d < np; d += 32) m = min(m, cnt[d]);
  m = __reduce_min_sync(0xffffffffu, m);
  for (int d = lane; d < np; d += 32) s += (cnt[d] == m);
  s = __reduce_add_sync(0xffffffffu, s);
  if (lane == 0) {
    S.ptsmin[c] = pc.min_zero ? 0 : m;
    S.ptsnum[c] = s;
    S.fc.pts_lim[c] = pts_limit(pc, S.ptsmin[c]);
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
__device__ unsigned long long each_leaf(const EachShared &S, const DevParams &p, const EachParams &ep, int32_t ti, int32_t i, uint32_t kk) {
  const ccsim_template &t = S.tmpl;
  const FilterConsts &fc = S.fc;
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
  if (G && S.coupled) {   // the terms of the node's own domain: its clones' hostPorts, node-local counters and one-node domains
    ok &= !(S.port_self && kk > 0u);
    if (ok && S.leaf_sel) coupled_ok<false>(fc, fc.n_pts, fc.n_aff, fc.n_anti, i, S.leaf_sel, ok);
  }
  if (!ok) return 0ull;
  int32_t sc = score_node(p.alloc_cpu[i], p.alloc_mem[i], each_add(ep.s_nz_cpu[i], kk, t.nz_cpu) + t.least_cpu,
                          each_add(ep.s_nz_mem[i], kk, t.nz_mem) + t.least_mem, rc + t.bal_cpu, rm + t.bal_mem, S.sw);
  if (S.w_image) sc += S.w_image * (int32_t)t.image_score[i];
  return pack_key(sc, (uint32_t)i);
}

// level l of this analysis's trees (level 0: the leaves)
__device__ __forceinline__ unsigned long long *each_level(const EachParams &ep, unsigned long long *leaf, unsigned long long *glev,
                                                          unsigned long long *slev, int l) {
  return l == 0 ? leaf : (l < ep.split ? glev : slev) + ep.lev_off[l];
}

// every leaf at its node's position, evaluated after its current clones (at kernel start: none), by threads t0, t0 + nt, ...
template <bool G>
__device__ void each_leaves(const EachShared &S, const DevParams &p, const EachParams &ep, int32_t ti, int32_t *kcol,
                                            unsigned long long *leaf, const int32_t *pos, bool start, int t0, int nt) {
  for (int32_t i = t0; i < p.n; i += nt) {
    if (start) kcol[i] = 0;
    leaf[pos ? pos[i] : i] = each_leaf<G>(S, p, ep, ti, i, start ? 0u : (uint32_t)kcol[i]);
  }
}

// upper levels, bottom up: one warp per entry, its 32 children in one coalesced load. BLOCK: the whole CTA (kernel start), else one warp
template <bool G, bool BLOCK>
__device__ void each_levels(const EachShared &S, const EachParams &ep, unsigned long long *leaf, unsigned long long *glev,
                                            unsigned long long *slev, int nseg, int w0, int nw, int lane) {
  for (int l = 1; l <= ep.n_levels; l++) {
    const unsigned long long *lo = each_level(ep, leaf, glev, slev, l - 1);
    unsigned long long *up = each_level(ep, leaf, glev, slev, l);
    const long long ne = cof<G>(S, l, nseg);
    for (long long g = w0; g < ne; g += nw) {
      const int c = each_seg_of<G>(S, l, g);
      const long long child = cof<G>(S, l - 1, c) + 32 * (g - cof<G>(S, l, c)) + lane;
      const unsigned long long v = warp_max_u64(child < cof<G>(S, l - 1, c + 1) ? lo[child] : 0ull);
      if (lane == 0) up[g] = v;
    }
    if (BLOCK) __syncthreads(); else __syncwarp();
  }
}

// The analysis's own state in its slot, by one thread: the terms (after its working counters are initialised), then the folded Filter
// constants and the score configuration
__device__ __forceinline__ void each_slot_terms(EachShared &S, const EachTerms *et, int ncnt) {
  const ccsim_template &t = S.tmpl;
  S.aff_total = (unsigned long long)t.aff_total_init;
  S.leaf_sel = et->leaf_sel; S.group_sel = et->group_sel;
  S.grouped = et->group_sel ? 1 : 0;
  S.port_self = et->port_self;
  S.coupled = ncnt > 0 || S.port_self;
  S.cof = et->cof; S.cstride = et->n_seg + 1; S.nseg = et->n_seg;
  for (int k = 0; k < CCSIM_MAX_TOPO_COLS; k++) S.topo_ptr[k] = et->topo[k];
  for (int j = 0; j < CCSIM_MAX_COUNTERS; j++) S.cnt_ptr[j] = j < ncnt ? et->counters[j].work : nullptr;
  for (int j = 0; j < ncnt; j++) {   // what a commit does to each counter (the generic wave kernel's CommitInfo)
    const DevCounter &dc = et->counters[j];
    CommitInfo &ci = S.cinfo[j];
    const bool skip = (dc.inc == 0) || (dc.is_aff && !(t.flags & CCSIM_TF_AFF_SELF_MATCH_ALL));
    ci.inc = skip ? 0 : dc.inc;
    ci.local = dc.topo_col < 0; ci.is_aff = dc.is_aff; ci.n_present = dc.n_present; ci.elig_bit = dc.elig_bit;
    ci.gtopo = ci.ltopo = dc.topo_col < 0 ? nullptr : et->topo[dc.topo_col];
    ci.pts_idx = -1;
    for (int c = 0; c < t.n_pts; c++) if (t.pts[c].counter == j && !t.pts[c].min_zero) ci.pts_idx = c;
  }
  for (int c = 0; c < CCSIM_MAX_PTS; c++) { S.ptsmin[c] = 0; S.ptsnum[c] = 0; }
}
__device__ __forceinline__ void each_slot_consts(EachShared &S, const DevParams &p, const EachTerms *et, int32_t ti) {
  const ccsim_template &t = S.tmpl;
  build_filter_consts(p, et->counters, t, ti, S.topo_ptr, S.cnt_ptr, S.ptsmin, (long long)S.aff_total, S.fc);
  S.fc.extras &= ~CCSIM_X_PLACED;   // hostPorts against the analysis's own clones: k > 0 in the leaf
  S.sw.w_fit = (t.score_enable & CCSIM_PL_FIT) ? t.w_fit : 0;
  S.sw.w_balanced = ((t.score_enable & CCSIM_PL_BALANCED) && !(t.flags & CCSIM_TF_BALANCED_SKIP)) ? t.w_balanced : 0;
  S.sw.least_w_cpu = t.least_w_cpu; S.sw.least_w_mem = t.least_w_mem;
  S.w_image = ((t.score_enable & CCSIM_PL_IMAGE_LOCALITY) && t.image_score) ? t.w_image : 0;
}

// Analysis ti's placements by one warp, from its built trees (slot S; slev: its shared tree levels; pos: et's), and its EachOut
template <bool G>
__device__ __forceinline__ void each_place(EachShared &S, const DevParams &p, const EachParams &ep, const EachTerms *et, int32_t ti,
                                           const int32_t *pos, int32_t *kcol, unsigned long long *leaf, unsigned long long *glev,
                                           unsigned long long *slev, int32_t *seq, int lane) {
  const int ncls = p.n_classes, L = ep.n_levels, ncnt = et->n_counters;
  const ccsim_template &t = S.tmpl;
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
    if (!G || !S.grouped) {   // one segment per class
      const unsigned long long r = (lane < ncls && cof<G>(S, L, lane + 1) > cof<G>(S, L, lane)) ? top[cof<G>(S, L, lane)] : 0ull;
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) cbest[c] = __shfl_sync(0xffffffffu, r, c);
    } else {             // a group's root counts when its domains pass the group terms; the best open group per class
      unsigned long long mine[CCSIM_MAX_CLASSES];
      #pragma unroll
      for (int c = 0; c < CCSIM_MAX_CLASSES; c++) mine[c] = 0ull;
      for (int s = lane; s < S.nseg; s += 32) {
        const long long e = cof<G>(S, L, s);
        if (cof<G>(S, L, s + 1) == e) continue;
        bool ok = true;
        coupled_ok<false>(S.fc, S.fc.n_pts, S.fc.n_aff, S.fc.n_anti, et->seg_rep[s], S.group_sel, ok);
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
    const int c = each_seg_of<G>(S, 0, at);
    // the winner's group of 32 on level 0 and on level 1, loaded while lane 0 commits the winner
    const long long e0 = at - cof<G>(S, 0, c), e1 = e0 >> 5;
    const long long g0 = cof<G>(S, 0, c) + (e0 & ~31ll) + lane;
    unsigned long long v0 = g0 < cof<G>(S, 0, c + 1) ? leaf[g0] : 0ull, v1 = 0ull;
    if (lv1) { const long long g1 = cof<G>(S, 1, c) + (e1 & ~31ll) + lane; v1 = g1 < cof<G>(S, 1, c + 1) ? lv1[g1] : 0ull; }
    uint32_t kk = 0u;
    if (lane == 0) {
      kk = (uint32_t)kcol[i] + 1u;                                          // ClusterCapacityBinder commit: one more clone on i
      kcol[i] = (int32_t)kk;
      seq[k] = i;
    }
    bool rebuild = false;
    if (G && S.coupled) {
      // the counters of the winner's domains, one lane per counter (the generic wave kernel's commit)
      if (lane < ncnt) {
        const CommitInfo &ci = S.cinfo[lane];
        if (ci.inc && !(ci.elig_bit >= 0 && !static_bit(p, i, ci.elig_bit))) {
          const int32_t dom = ci.local ? i : ci.ltopo[i];
          if (dom >= 0) {
            int32_t *cnt = S.cnt_ptr[lane];
            const int32_t old = cnt[dom];
            cnt[dom] = old + ci.inc;
            if (ci.is_aff) atomicAdd(&S.aff_total, (unsigned long long)(long long)ci.inc);
            if (ci.pts_idx >= 0 && dom < ci.n_present && old == S.ptsmin[ci.pts_idx]) atomicSub(&S.ptsnum[ci.pts_idx], 1);
          }
        }
      }
      __syncwarp();
      // a spread minimum whose last domain moved up: recount; a folded constraint's limit then changed on every node
      for (int q = 0; q < S.fc.n_pts; q++)
        if (!t.pts[q].min_zero && S.ptsnum[q] <= 0 && S.cinfo[t.pts[q].counter].n_present > 0) {
          each_pts_recount(S, q, lane);
          rebuild |= (S.leaf_sel >> q) & 1u;
        }
      if (S.fc.aff_bypass && S.aff_total != 0ull) {   // the first matching pod ends the bypass (filtering.go:396-405)
        __syncwarp();
        if (lane == 0) S.fc.aff_bypass = 0;
        rebuild = true;
      }
      __syncwarp();
    }
    if (G && rebuild) {   // every leaf and level again, with the code of the kernel start
      each_leaves<G>(S, p, ep, ti, kcol, leaf, pos, false, lane, 32);
      __syncwarp();
      each_levels<G, false>(S, ep, leaf, glev, slev, S.nseg, 0, 1, lane);
      rebuilds++;
      continue;
    }
    unsigned long long nv = 0ull;
    if (lane == 0) nv = each_leaf<G>(S, p, ep, ti, i, kk);
    nv = __shfl_sync(0xffffffffu, nv, 0);
    // level l's entry e (within segment c) gets nv; its group's maximum becomes level l + 1's entry e >> 5
    long long e = e0;
    for (int l = 0; l < L; l++) {
      unsigned long long *lv = each_level(ep, leaf, glev, slev, l) + cof<G>(S, l, c);
      unsigned long long v;
      if (l == 0) v = v0;
      else if (l == 1) v = v1;
      else { const long long g = (e & ~31ll) + lane; v = g < cof<G>(S, l, c + 1) - cof<G>(S, l, c) ? lv[g] : 0ull; }
      if (lane == (int)(e & 31)) { v = nv; lv[e] = nv; }
      nv = warp_max_u64(v);
      e >>= 5;
    }
    if (lane == 0) top[cof<G>(S, L, c)] = nv;
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
      for (int q = 0; q < CCSIM_MAX_PTS; q++) ep.diag[ti].ptsmin[q] = S.ptsmin[q];
      ep.diag[ti].aff_total = (long long)S.aff_total;
    }
  }
}

// Two instantiations (G above), so that the node-local one is compiled and register-allocated on its own. One CTA per analysis.
template <bool G>
__global__ void __launch_bounds__(EACH_THREADS, 1) ccsim_each_kernel(const DevParams p, const EachParams ep) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long *slev = reinterpret_cast<unsigned long long *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int32_t ti = blockIdx.x, n = p.n;
  const int L = ep.n_levels;
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
  if (tid == 0) each_slot_terms(es, et, ncnt);
  __syncthreads();
  if (tid == 0) each_slot_consts(es, p, et, ti);
  __syncthreads();
  if (warp == 0) for (int c = 0; c < es.fc.n_pts; c++) each_pts_recount(es, c, lane);   // the spread minima and their limits
  __syncthreads();

  if (!G)   // the host's class offsets into shared memory (classes <= CCSIM_MAX_CLASSES, levels <= EACH_MAX_LEVELS)
    for (int q = tid; q < (L + 1) * (es.nseg + 1); q += blockDim.x) es.coff[q / (es.nseg + 1)][q % (es.nseg + 1)] = et->cof[q];

  // ---- leaves at the host's positions, every node evaluated with no clone placed; then the upper levels ----
  each_leaves<G>(es, p, ep, ti, kcol, leaf, pos, true, tid, blockDim.x);
  __syncthreads();
  each_levels<G, true>(es, ep, leaf, glev, slev, es.nseg, warp, nw, lane);

  // ---- placements: warp 0 alone ----
  if (warp != 0) return;
  each_place<G>(es, p, ep, et, ti, pos, kcol, leaf, glev, slev, seq, lane);
}

// Node-local analyses that outnumber the CTAs the device holds at once: EachParams::pack analyses per CTA (analysis t0 + a in slot a).
// The whole CTA builds each analysis's leaves and levels in turn; then warp a runs analysis t0 + a's placements, the loop warp 0 of
// ccsim_each_kernel<false> runs, with its own slot of shared state and its own share (EachParams::slev_stride entries) of the shared
// tree levels. Dynamic shared memory: pack slots, then pack shares.
__global__ void __launch_bounds__(EACH_THREADS, 1) ccsim_each_packed_kernel(const DevParams p, const EachParams ep) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EachShared *slot = reinterpret_cast<EachShared *>(smem_raw);
  unsigned long long *slev0 = reinterpret_cast<unsigned long long *>(smem_raw + (size_t)ep.pack * sizeof(EachShared));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int32_t t0 = blockIdx.x * ep.pack, na = min(ep.pack, ep.n_analyses - t0), n = p.n;
  const int L = ep.n_levels;
  constexpr int words = (int)(sizeof(ccsim_template) / 8);
  for (int q = tid; q < na * words; q += blockDim.x)
    reinterpret_cast<unsigned long long *>(&slot[q / words].tmpl)[q % words] = reinterpret_cast<const unsigned long long *>(&p.templates[t0 + q / words])[q % words];
  __syncthreads();
  if (tid < na) {   // one thread per analysis (node-local: no counters, no spread minima)
    each_slot_terms(slot[tid], ep.terms + t0 + tid, 0);
    each_slot_consts(slot[tid], p, ep.terms + t0 + tid, t0 + tid);
  }
  __syncthreads();
  for (int a = 0; a < na; a++) {
    EachShared &S = slot[a];
    const int32_t ti = t0 + a;
    const EachTerms *et = ep.terms + ti;
    for (int q = tid; q < (L + 1) * (S.nseg + 1); q += blockDim.x) S.coff[q / (S.nseg + 1)][q % (S.nseg + 1)] = et->cof[q];
    each_leaves<false>(S, p, ep, ti, ep.k + (size_t)ti * n, ep.leaf + (size_t)ti * n, et->pos, true, tid, blockDim.x);
    __syncthreads();
    each_levels<false, true>(S, ep, ep.leaf + (size_t)ti * n, ep.glev + (size_t)ti * ep.glev_stride, slev0 + (size_t)a * ep.slev_stride,
                             S.nseg, warp, nw, lane);
  }
  if (warp >= na) return;
  const int32_t ti = t0 + warp;
  each_place<false>(slot[warp], p, ep, ep.terms + ti, ti, ep.terms[ti].pos, ep.k + (size_t)ti * n, ep.leaf + (size_t)ti * n,
                    ep.glev + (size_t)ti * ep.glev_stride, slev0 + (size_t)warp * ep.slev_stride, ep.seq + (size_t)ti * ep.seq_cap, lane);
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
    if (p.placed_mask) p.placed_mask[i] = kk > 0u ? 1ull << (ti & 63) : 0ull;   // hostPorts: the analysis's own clones, bit t mod 64
  }
}
