// ccsim_batched.cuh — batched tie-run waves: many commits per wave, same placement sequence as the sequential loop.
//
// Eligibility (host, run_prepare): ONE template whose enabled predicates and scorers are all node-local (no
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
  const size_t cp = (size_t)p.chunk_pad;
  const LeanTile t = lean_tile(smem_raw, lp, cp);
  int32_t *run = reinterpret_cast<int32_t *>(t.own);   // run length of each node in this wave (0: not tied at S*)
  int32_t *fscore = run + cp;         // memo score after the full run (-1: node ended the run infeasible)
  int32_t *off = fscore + cp;         // exclusive prefix of run[] in node order

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int32_t cnt_nodes = hi - lo;
  uint4 *rec = t.rec;
  const int su = lp.stride_u;

  lean_stage(p, lp, t, lo, cnt_nodes);
  if (tid == 0) { lean_build_consts(p, lp); ls.dirty = 0; }
  __syncthreads();

  const LeanFit fit = lean_fit();
  const ccsim_template &tm = ls.tmpl;

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
      const LeanRow w = lean_row(r);
      int32_t sc = w.score;
      const bool ok = lean_fits(w, fit);
      run[j] = 0;
      if (ok) {
        if (sc < 0) sc = lean_rescore(t, lp, j);
        const unsigned long long key = pack_key(sc, (uint32_t)(p.node_base + lo + j));
        best = key > best ? key : best;
      } else if (sc >= 0) reinterpret_cast<int32_t *>(rec + (size_t)j * su)[LR_SCORE] = -2 - sc;   // remember: infeasible (memo kept as -2-score)
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
      const int32_t sc = reinterpret_cast<const int32_t *>(rec + (size_t)j * su)[LR_SCORE];
      if (sc != sstar) continue;                                      // infeasible nodes carry a negative memo
      long long rc = t.rcpu[j], rm = t.rmem[j], zc = t.zcpu[j], zm = t.zmem[j];
      const long long ac = t.acpu[j], am = t.amem[j];
      int32_t np = t.npods[j];
      const int32_t ap = t.apods[j];
      int32_t r = 0, cur = sstar;
      bool feasible = true;
      do {
        r++; rc += tm.req_cpu; rm += tm.req_mem; zc += tm.nz_cpu; zm += tm.nz_mem; np++;
        feasible = (ac - rc >= fit.eq_cpu) & (am - rm >= fit.eq_mem) & (ap - np >= fit.pods_need);
        if (!feasible) break;
        cur = score_node(ac, am, zc + tm.least_cpu, zm + tm.least_mem, rc + tm.bal_cpu, rm + tm.bal_mem, ls.sw);
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
      lean_commit_row<false>(p, lp, t, j, (int32_t)allowed, (allowed == r) ? fscore[j] : -1);   // (no counters in this kernel)
      const int32_t w = lo + j;
      p.req_cpu[w] = t.rcpu[j]; p.req_mem[w] = t.rmem[j]; p.nz_cpu[w] = t.zcpu[j]; p.nz_mem[w] = t.zmem[j]; p.npods[w] = t.npods[j];   // write through
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

  // (this kernel writes its commits through instead of using lean_finish: a write-back after the loop, or lean_finish's result
  //  fields, cost it 8 B more stack, 12 B more spill stores and 20 B more spill loads)
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
