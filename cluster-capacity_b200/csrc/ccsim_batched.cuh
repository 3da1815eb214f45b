// ccsim_batched.cuh — batched tie-run waves: many commits per wave, same placement sequence as the sequential loop.
//
// Eligibility (host, ccsim_run): ONE template whose enabled predicates and scorers are all node-local (no
// PodTopologySpread / InterPodAffinity counters, no hostPort-vs-clone conflicts, TaintToleration's normalised score constant
// because no feasible-set normalisation class beyond 0 exists) and a shared-memory resident tile.
// Then every node's total score is a function of its own clone count only, and the reference loop is a k-way merge of N
// independent score trajectories (SURVEY.md §8a design note). With "first maximum in node order" tie-breaking
// (a legal outcome of selectHost, schedule_one.go:894-941) the merge is:
//
//   wave:  S* = max score over feasible nodes                      (one fused Filter pass over all N nodes + exchange)
//          for the nodes tied at S*, in node order: place clones on node i while it stays feasible and its score >= S*
//            (while i's score is > S* it is the unique maximum; when it is == S* it still has the lowest index among the
//             ties; when it drops below S* the next tied node is the maximum)
//          pod indices = exclusive prefix sum of the run lengths in node order  (block scan + one more exchange)
//
// which reproduces the sequential pod -> node sequence exactly (tests compare it with the oracle pod by pod), including
// --max-limit truncation in the middle of a wave. Every wave still pushes all N nodes through the Filter pass from their
// current state; what disappears is one grid-wide exchange per pod.
#pragma once
#include "ccsim_lean.cuh"

struct __align__(16) BatchShared {
  long long cta_prefix, total, remaining;
  int32_t scan_tmp[LEAN_WARPS];
};
__shared__ BatchShared bs;

// tagged exchange of one 44-bit value per CTA through word `word` of the slot line; returns (prefix over lower CTAs, total)
__device__ __forceinline__ bool exchange_totals(const DevParams &p, long long k_parity, uint32_t tag, int word, unsigned long long mine,
                                                int lane, int cta, unsigned long long &prefix, unsigned long long &total) {
  const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
  unsigned long long *myslot = p.slots + ((size_t)(k_parity & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE + word;
  if (lane == 0) st_slot(myslot, (mine & KEY_BODY_MASK) | tagbits);
  const unsigned long long *all = p.slots + (size_t)(k_parity & 1) * CCSIM_MAX_GRID * SLOT_STRIDE + word;
  unsigned long long v[CCSIM_MAX_GRID / 32];
  unsigned spins = 0;
  bool pending, dead = false;
  do {
    pending = false;
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) {
      const int b = lane + 32 * q;
      v[q] = (b < p.grid) ? ld_slot(&all[(size_t)b * SLOT_STRIDE]) : tagbits;
    }
    #pragma unroll
    for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) pending |= ((uint32_t)(v[q] >> KEY_TAG_SHIFT) != tag);
    if (++spins > WATCHDOG_SPINS) { dead = true; break; }
  } while (__any_sync(0xffffffffu, pending));
  unsigned long long pre = 0, tot = 0;
  #pragma unroll
  for (int q = 0; q < CCSIM_MAX_GRID / 32; q++) {
    const int b = lane + 32 * q;
    const unsigned long long x = (b < p.grid) ? (v[q] & KEY_BODY_MASK) : 0ull;
    tot += x;
    if (b < cta) pre += x;
  }
  for (int o = 16; o > 0; o >>= 1) { pre += __shfl_xor_sync(0xffffffffu, pre, o); tot += __shfl_xor_sync(0xffffffffu, tot, o); }
  prefix = pre; total = tot;
  return __any_sync(0xffffffffu, dead);
}

__global__ void __launch_bounds__(LEAN_THREADS, 1) ccsim_wave_batched_kernel(const DevParams p, const LeanParams lp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const uint32_t cnt_bytes = ((uint32_t)p.smem_cnt_ints * 4u + 15u) & ~15u;
  uint4 *rec = reinterpret_cast<uint4 *>(smem_raw + cnt_bytes);
  const size_t cp = (size_t)p.chunk_pad;
  long long *c_acpu = reinterpret_cast<long long *>(smem_raw + cnt_bytes + lp.rec_bytes_total);
  long long *c_amem = c_acpu + cp, *c_rcpu = c_amem + cp, *c_rmem = c_rcpu + cp, *c_zcpu = c_rmem + cp, *c_zmem = c_zcpu + cp;
  int32_t *c_apods = reinterpret_cast<int32_t *>(c_zmem + cp);
  int32_t *c_npods = c_apods + cp;
  int32_t *run = c_npods + cp;        // run length of each node in this wave (0: not tied at S*)
  int32_t *fscore = run + cp;         // memo score after the full run (-1: node ended the run infeasible)
  int32_t *off = fscore + cp;         // exclusive prefix of run[] in node order

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int32_t cnt_nodes = hi - lo;
  const int su = lp.stride_u;

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
    c_acpu[j] = ac; c_amem[j] = am; c_rcpu[j] = rc; c_rmem[j] = rm;
    c_zcpu[j] = p.nz_cpu[i]; c_zmem[j] = p.nz_mem[i];
    c_apods[j] = ap; c_npods[j] = np;
  }
  for (int k = tid; k < (int)(sizeof(ccsim_template) / 8); k += LEAN_THREADS)
    reinterpret_cast<unsigned long long *>(&ls.tmpl)[k] = reinterpret_cast<const unsigned long long *>(&p.templates[0])[k];
  if (tid == 0) { ls.aff_total = 0; ls.winner = -1; ls.stop = 0; ls.dirty = 1; }
  __syncthreads();
  if (tid == 0) { lean_build_consts(p, lp); ls.dirty = 0; }
  __syncthreads();

  const unsigned long long taint_bad0 = ls.taint_bad0, sel0 = ls.sel0, forbid0 = ls.forbid0;
  const long long eq_cpu = ls.eq_cpu, eq_mem = ls.eq_mem;
  const int32_t pods_need = ls.pods_need;
  const ccsim_template &t = ls.tmpl;

  long long k = 0, waves = 0, extra_evals = 0;
  bool limit_hit = false;   // postBindHook's limit (simulator.go:300-305)
  uint32_t wtag = 1;
  uint32_t tag = (p.epoch << 12) | wtag;
  for (;;) {
    if (p.max_pods > 0 && k >= p.max_pods) { limit_hit = true; break; }   // uniform; no shared write (slower threads may still be reading ls.stop)
    if (k > p.pod_cap) { if (tid == 0) ls.stop = 3; __syncthreads(); break; }
    // ---- fused Filter pass over the tile: one predicate-eval per node ----
    unsigned long long best = 0ull;
    for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
      const uint4 *r = rec + (size_t)j * su;
      const uint4 u0 = r[0], u1 = r[1], u2 = r[2];
      const unsigned long long taint0 = ((unsigned long long)u0.y << 32) | u0.x;
      const unsigned long long static0 = ((unsigned long long)u0.w << 32) | u0.z;
      const long long free_cpu = (long long)(((unsigned long long)u1.y << 32) | u1.x);
      const long long free_mem = (long long)(((unsigned long long)u1.w << 32) | u1.z);
      int32_t sc = (int32_t)u2.y;
      bool ok = ((taint0 & taint_bad0) | (~static0 & sel0) | (static0 & forbid0)) == 0ull;
      ok &= (free_cpu >= eq_cpu) & (free_mem >= eq_mem) & ((int32_t)u2.x >= pods_need);
      run[j] = 0;
      if (ok) {
        if (sc < 0) {
          sc = score_node(c_acpu[j], c_amem[j], c_zcpu[j] + t.least_cpu, c_zmem[j] + t.least_mem, c_rcpu[j] + t.bal_cpu, c_rmem[j] + t.bal_mem, ls.sw);
          reinterpret_cast<int32_t *>(rec + (size_t)j * su)[9] = sc;
        }
        const unsigned long long key = pack_key(sc, (uint32_t)(p.node_base + lo + j));
        best = key > best ? key : best;
      } else if (sc >= 0) reinterpret_cast<int32_t *>(rec + (size_t)j * su)[9] = -2 - sc;   // remember: infeasible (memo kept as -2-score)
    }
    { const unsigned long long v = warp_max_u64(best); if (lane == 0) ls.warp_best[warp][0] = v; }
    __syncthreads();                                                    // S1
    if (warp == 0) {
      const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
      unsigned long long *myslots = p.slots + ((size_t)(waves & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE;
      const unsigned long long vb = warp_max_u64(lane < LEAN_WARPS ? ls.warp_best[lane][0] : 0ull);
      if (lane == 0) st_slot(&myslots[0], vb | tagbits);
      unsigned long long v[GATHER_Q];
      bool dead = poll_tagged(p, waves, tag, 0, lane, v);
      const unsigned long long m = gather_max(v);
      dead = __any_sync(0xffffffffu, dead);
      if (lane == 0) {
        if (dead) ls.stop = 3;
        else if (m == 0ull) ls.stop = 1;
        ls.winner = (m == 0ull) ? -1 : (int32_t)key_score(m);      // S*: the node-local part of the maximum total score
        bs.remaining = (p.max_pods > 0) ? (p.max_pods - k) : (long long)0x7fffffffffffLL;
      }
    }
    __syncthreads();                                                    // S2
    waves++;
    if (ls.stop) break;
    const int32_t sstar = ls.winner;
    // ---- runs of the tied nodes: place while feasible and score >= S* ----
    for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
      const int32_t sc = reinterpret_cast<const int32_t *>(rec + (size_t)j * su)[9];
      if (sc != sstar) continue;                                      // infeasible nodes carry a negative memo
      long long rc = c_rcpu[j], rm = c_rmem[j], zc = c_zcpu[j], zm = c_zmem[j];
      const long long ac = c_acpu[j], am = c_amem[j];
      int32_t np = c_npods[j];
      const int32_t ap = c_apods[j];
      int32_t r = 0, cur = sstar;
      bool feasible = true;
      do {
        r++; rc += t.req_cpu; rm += t.req_mem; zc += t.nz_cpu; zm += t.nz_mem; np++;
        feasible = (ac - rc >= eq_cpu) & (am - rm >= eq_mem) & (ap - np >= pods_need);
        if (!feasible) break;
        cur = score_node(ac, am, zc + t.least_cpu, zm + t.least_mem, rc + t.bal_cpu, rm + t.bal_mem, ls.sw);
      } while (cur >= sstar);
      run[j] = r;
      fscore[j] = feasible ? cur : -1;
    }
    __syncthreads();                                                    // S3
    // ---- exclusive prefix of run[] in node order (each thread owns a contiguous segment) ----
    {
      const int seg = (cnt_nodes + LEAN_THREADS - 1) / LEAN_THREADS;
      const int b0 = min(cnt_nodes, tid * seg), b1 = min(cnt_nodes, b0 + seg);
      int32_t s = 0;
      for (int j = b0; j < b1; j++) s += run[j];
      int32_t incl = s;
      for (int o = 1; o < 32; o <<= 1) { const int32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
      if (lane == 31) bs.scan_tmp[warp] = incl;
      __syncthreads();
      int32_t wbase = 0;
      for (int w = 0; w < warp; w++) wbase += bs.scan_tmp[w];
      int32_t base = wbase + incl - s;
      for (int j = b0; j < b1; j++) { off[j] = base; base += run[j]; }
      __syncthreads();
      if (warp == 0) {
        long long T = 0;
        for (int w = 0; w < LEAN_WARPS; w++) T += bs.scan_tmp[w];
        unsigned long long pre, tot;
        const bool dead = exchange_totals(p, waves - 1, tag, 1, (unsigned long long)T, lane, cta, pre, tot);
        if (lane == 0) { bs.cta_prefix = (long long)pre; bs.total = (long long)tot; if (dead) ls.stop = 3; }
      }
    }
    __syncthreads();                                                    // S4
    if (ls.stop) break;
    // ---- commit the runs (NodeInfo.update(+1) per clone: types.go:409-427; bind record: simulator.go:297-312) ----
    const long long remaining = bs.remaining, cta_prefix = bs.cta_prefix;
    for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
      const int32_t r = run[j];
      if (r == 0) continue;
      const long long goff = cta_prefix + off[j];
      long long allowed = remaining - goff;
      allowed = allowed < 0 ? 0 : (allowed > r ? r : allowed);
      if (allowed == 0) continue;
      const int32_t w = lo + j;
      const long long rc = c_rcpu[j] + allowed * t.req_cpu, rm = c_rmem[j] + allowed * t.req_mem;
      const long long zc = c_zcpu[j] + allowed * t.nz_cpu, zm = c_zmem[j] + allowed * t.nz_mem;
      const int32_t np = c_npods[j] + (int32_t)allowed;
      c_rcpu[j] = rc; c_rmem[j] = rm; c_zcpu[j] = zc; c_zmem[j] = zm; c_npods[j] = np;
      unsigned long long *r8 = reinterpret_cast<unsigned long long *>(rec + (size_t)j * su);
      int32_t *r4 = reinterpret_cast<int32_t *>(r8);
      r8[2] = (unsigned long long)(c_acpu[j] - rc);
      r8[3] = (unsigned long long)(c_amem[j] - rm);
      r4[8] = c_apods[j] - np;
      r4[9] = (allowed == r) ? fscore[j] : -1;
      p.req_cpu[w] = rc; p.req_mem[w] = rm; p.nz_cpu[w] = zc; p.nz_mem[w] = zm; p.npods[w] = np;
      const int32_t g = p.node_base + w;
      for (long long q = 0; q < allowed; q++) { const long long kk = k + goff + q; if (kk < p.pod_cap) p.pod_node[kk] = g; }
    }
    {
      const long long placed_now = bs.total < remaining ? bs.total : remaining;
      k += placed_now;
      extra_evals += placed_now;
    }
    __syncthreads();                                                    // S5
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
  }

  if (cta == 0 && tid == 0) {
    DevOut *o = p.out;
    o->placed = k;
    o->stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
    o->error = (ls.stop == 3) ? 1 : 0;
    o->waves = waves;
    o->evals = waves * (long long)p.n + extra_evals;
    o->examined = o->evals;
    for (int c = 0; c < CCSIM_MAX_PTS; c++) o->ptsmin[c] = 0;
    o->aff_total = 0;
  }
}
