// ccsim_stream.cuh — the streaming wave kernel: node-local templates (no per-domain counters) on clusters whose tiles do not
// fit in shared memory, and runs with several templates (BASELINE config C5: 1M nodes x 64 podspecs placed round-robin).
//
// One predicate-eval needs, per node, only what NodeResourcesFit compares (fit.go:564-660) and the node's memoised score:
//   free_cpu, free_mem (int64: allocatable - requested), free_pods (int32), score memo of THIS template (int32)  = 24 B
//   (+ taint / static words, 16 B, only when a template filters on them)
// instead of the 72 B NodeInfo row of SURVEY.md §8(d): the row is read again only for a node whose memo is stale (it was
// committed since that template last scored it; the reference's snapshot likewise refreshes only NodeInfos whose generation
// changed, backend/cache/cache.go:194-288).
//
// Every persistent CTA owns a contiguous chunk of the node axis, stored padded to whole tiles (padding rows have
// free_pods = INT_MIN and never pass the Filter). Per wave the CTA streams its chunk through a ring of shared-memory stages:
// one elected thread arms the stage's mbarrier with the byte count and issues one 1-D bulk-async copy per column
// (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes — the TMA engine, no register staging), the 512
// consumer threads wait on the mbarrier phase, run the fused Filter + arg-max on the tile from shared memory, and the stage
// is re-armed for the tile STREAM_STAGES ahead. Then the usual tagged-word exchange through L2, and the owner CTA commits:
// the winner's row (global columns, write-through for the terminal diagnosis), its free_* entries, and the memo entries of
// ALL templates for that node (-1). Generic-proxy writes are ordered before later bulk-async reads by fence.proxy.async.
#pragma once
#include "ccsim_lean.cuh"

#define STREAM_THREADS 512
#define STREAM_WARPS (STREAM_THREADS / 32)
#define STREAM_WQ 8
#define STREAM_WQ_STOP (-2)
#define STREAM_BLOCK (STREAM_THREADS + 64)   /* + two service warps: the exchange warp, and the memory warp (bulk-copy requests, commit) */
#define STREAM_TILE 1024          /* nodes per stage: 24 KB (40 KB with the mask columns) */
#define STREAM_STAGES 4           /* stages of the ring when every column is streamed */
#define STREAM_STAGES_RES 8       /* ... when only the 4-byte memo column is streamed (resident free_* columns): a whole 1M-node chunk (7 tiles) in flight */

struct StreamTmpl {               // per-template constants of the fused Filter pass + scorer inputs (shared memory table)
  long long eq_cpu, eq_mem;       // effective requests (LLONG_MIN: check disabled)
  unsigned long long taint_bad0, sel0, forbid0;
  long long least_cpu, least_mem, bal_cpu, bal_mem, req_cpu, req_mem, nz_cpu, nz_mem;
  ScoreWeights sw;
  int32_t pods_need, pad[3];
};

struct StreamParams {
  long long *f_cpu, *f_mem;       // [n_pad] allocatable - requested
  int32_t *f_pods;                // [n_pad] allowedPodNumber - len(Pods); INT_MIN on padding rows
  const unsigned long long *m_taint, *m_static;   // [n_pad] or nullptr when no template filters on them
  int32_t *memo;                  // [n_templates][n_pad] memoised node-local score of template t, -1 = stale
  int32_t chunk_pad;              // nodes per CTA, padded to a multiple of STREAM_TILE
  int32_t tiles;                  // chunk_pad / STREAM_TILE
  long long n_pad;                // grid * chunk_pad
  int32_t use_masks;
  int32_t res_rows;               // MODE 2: resident rows per CTA (chunk rounded up to a warp; <= chunk_pad)
};

struct __align__(16) StreamShared {
  StreamTmpl tc[CCSIM_MAX_TEMPLATES];
  unsigned long long full[STREAM_STAGES_RES];  // mbarriers: "the stage's bytes have landed"
  unsigned long long warp_best[STREAM_WARPS];
  int32_t winner, stop, commit_seq, commit_full;   // commit_seq / commit_full: waves whose urgent / whole commit is done (+1)
  int32_t wq[STREAM_WQ];                            // winners handed to the commit warp (ring), STREAM_WQ_STOP ends it
  int32_t w_seq, c_done, pad2[2];                   // winners published / consumed
  long long ph[8], tc0, n_stale;   // CTA 0 / thread 0: clock cycles per phase; stale memo entries re-scored by CTA 0
};

__shared__ StreamShared ss;
#define SPH_START() do { if (cta == 0 && tid == 0) ss.tc0 = clock64(); } while (0)
#define SPH_MARK(i) do { if (cta == 0 && tid == 0) { const long long t1_ = clock64(); ss.ph[i] += t1_ - ss.tc0; ss.tc0 = t1_; } } while (0)

__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// 1-D bulk-async copy global -> shared (TMA engine); size and both addresses are multiples of 16 bytes
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// orders this thread's earlier generic-proxy accesses to GLOBAL memory before later async-proxy (bulk copy) accesses
__device__ __forceinline__ void bar_sync_n(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ int32_t ld_vol_s32(const int32_t *p) { return *reinterpret_cast<const volatile int32_t *>(p); }
__device__ __forceinline__ void st_vol_s32(int32_t *p, int32_t v) { *reinterpret_cast<volatile int32_t *>(p) = v; }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// fills the padded streaming columns from the snapshot's working columns (once per run)
__global__ void ccsim_stream_prep_kernel(const DevParams p, const StreamParams sp) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < sp.n_pad; q += (long long)gridDim.x * blockDim.x) {
    const int cta = (int)(q / sp.chunk_pad), off = (int)(q - (long long)cta * sp.chunk_pad);
    const long long i = (long long)cta * p.chunk + off;
    const bool real = off < p.chunk && i < p.n;
    sp.f_cpu[q] = real ? p.alloc_cpu[i] - p.req_cpu[i] : 0;
    sp.f_mem[q] = real ? p.alloc_mem[i] - p.req_mem[i] : 0;
    sp.f_pods[q] = real ? p.alloc_pods[i] - p.npods[i] : INT_MIN;
    if (sp.use_masks) {
      const_cast<unsigned long long *>(sp.m_taint)[q] = real ? p.taint_mask[i] : 0ull;
      const_cast<unsigned long long *>(sp.m_static)[q] = (real && p.static_words > 0) ? p.static_mask[i] : 0ull;
    }
  }
}

// Dynamic shared memory of ccsim_wave_stream_kernel<mode> as it carves it: NST stages of STAGE_BYTES, mode 2's 24-B rows, 128 B spare
constexpr size_t stream_smem_bytes(int mode, size_t res_rows) {
  return mode == 2 ? (size_t)STREAM_STAGES_RES * STREAM_TILE * 4 + res_rows * 24 + 128
                   : (size_t)STREAM_STAGES * STREAM_TILE * (mode == 1 ? 40 : 24) + 128;
}

// MODE 0: everything streamed (24 B per node and wave); 1: + taint/static words (40 B); 2: the free_* columns of the CTA's chunk stay in
// shared memory for the whole run (24 B per node, sized by the chunk rather than its tile padding: 1M nodes fit in the 132 SMs' shared
// memory of an H100) and only the score memo column of the wave's template is streamed (4 B per node and wave)
template <int MODE>
__global__ void __launch_bounds__(STREAM_BLOCK, 1) ccsim_wave_stream_kernel(const DevParams p, const StreamParams sp) {
  constexpr bool MASKS = MODE == 1, RESF = MODE == 2;
  constexpr int NST = RESF ? STREAM_STAGES_RES : STREAM_STAGES;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // stage s: [f_cpu TILE x 8][f_mem TILE x 8][f_pods TILE x 4][memo TILE x 4]([taint TILE x 8][static TILE x 8])
  constexpr uint32_t STAGE_BYTES = STREAM_TILE * (MASKS ? 40u : (RESF ? 4u : 24u));
  constexpr uint32_t MEMO_OFF = RESF ? 0u : STREAM_TILE * 20u;      // the memo tile inside a stage
  // RESF: resident columns behind the stage ring
  // RESF: per node {free_cpu, free_mem} (16 B: one LDS.128) and {free_pods, generation} (8 B: one LDS.64)
  longlong2 *r_free = reinterpret_cast<longlong2 *>(smem_raw + NST * STAGE_BYTES);
  // A generation number per node instead of invalidating 64 memo entries at every commit: a memo entry is (generation << 12 |
  // score + 1) and is valid only while the node's generation stands (NodeInfo.Generation, framework/types.go:409-427).
  int2 *r_pg = reinterpret_cast<int2 *>(r_free + sp.res_rows);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const long long base = (long long)cta * sp.chunk_pad;           // this CTA's first padded row
  const int T = p.n_templates;

  // ---- per-template constants (folded like lean_build_consts) ----
  for (int t = tid; t < T; t += STREAM_THREADS) {
    const ccsim_template &tp = p.templates[t];
    StreamTmpl &c = ss.tc[t];
    const uint32_t fe = tp.filter_enable, fl = tp.flags;
    unsigned long long tb = 0ull;
    if (fe & CCSIM_PL_TAINT_TOLERATION) tb |= p.taint_nosched[0] & ~tp.tol_nosched[0] & ~(1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT);
    if ((fe & CCSIM_PL_NODE_UNSCHEDULABLE) && !(fl & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) tb |= 1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT;
    c.taint_bad0 = tb;
    const bool aff_on = (fe & CCSIM_PL_NODE_AFFINITY) && (fl & CCSIM_TF_HAS_NODE_SELECTOR);
    c.sel0 = (aff_on && p.static_words > 0) ? tp.sel_mask[0] : 0ull;
    unsigned long long fb = 0ull;
    if (p.static_words > 0) {
      if ((fe & CCSIM_PL_NODE_PORTS) && (fl & CCSIM_TF_HAS_HOST_PORTS)) fb |= tp.port_static_mask[0];
      if (fe & CCSIM_PL_INTER_POD_AFFINITY) fb |= tp.existing_anti_mask[0];
    }
    c.forbid0 = fb;
    const bool fit = (fe & CCSIM_PL_FIT) != 0, nz = fit && !(fl & CCSIM_TF_FIT_ALL_ZERO);
    c.pods_need = fit ? 1 : INT32_MIN + 1;       // (padding rows carry INT_MIN: they fail even when NodeResourcesFit is disabled)
    c.eq_cpu = (nz && tp.req_cpu > 0) ? tp.req_cpu : LLONG_MIN;
    c.eq_mem = (nz && tp.req_mem > 0) ? tp.req_mem : LLONG_MIN;
    c.least_cpu = tp.least_cpu; c.least_mem = tp.least_mem; c.bal_cpu = tp.bal_cpu; c.bal_mem = tp.bal_mem;
    c.req_cpu = tp.req_cpu; c.req_mem = tp.req_mem; c.nz_cpu = tp.nz_cpu; c.nz_mem = tp.nz_mem;
    c.sw.w_fit = (tp.score_enable & CCSIM_PL_FIT) ? tp.w_fit : 0;
    c.sw.w_balanced = ((tp.score_enable & CCSIM_PL_BALANCED) && !(fl & CCSIM_TF_BALANCED_SKIP)) ? tp.w_balanced : 0;
    c.sw.least_w_cpu = tp.least_w_cpu; c.sw.least_w_mem = tp.least_w_mem;
  }
  if (RESF)
    for (int j = threadIdx.x; j < sp.res_rows; j += STREAM_BLOCK) {
      r_free[j] = make_longlong2(sp.f_cpu[(long long)blockIdx.x * sp.chunk_pad + j], sp.f_mem[(long long)blockIdx.x * sp.chunk_pad + j]);
      r_pg[j] = make_int2(sp.f_pods[(long long)blockIdx.x * sp.chunk_pad + j], 0);
    }
  if (tid == 0) {
    for (int s = 0; s < NST; s++) mbar_init(&ss.full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    ss.winner = -1; ss.stop = 0; ss.commit_seq = 0; ss.commit_full = 0; ss.w_seq = 0; ss.c_done = 0;
    for (int q = 0; q < 8; q++) ss.ph[q] = 0;
    ss.n_stale = 0;
  }
  __syncthreads();

  // thread 0: arm stage `s` and issue the bulk copies of tile `tile` of template t's pass
  auto issue = [&](int tile, int s, int t) {
    unsigned char *st = smem_raw + (size_t)s * STAGE_BYTES;
    const long long row = base + (long long)tile * STREAM_TILE;
    mbar_expect_tx(&ss.full[s], STAGE_BYTES);
    if (!RESF) {
      bulk_g2s(st, sp.f_cpu + row, STREAM_TILE * 8, &ss.full[s]);
      bulk_g2s(st + STREAM_TILE * 8, sp.f_mem + row, STREAM_TILE * 8, &ss.full[s]);
      bulk_g2s(st + STREAM_TILE * 16, sp.f_pods + row, STREAM_TILE * 4, &ss.full[s]);
    }
    bulk_g2s(st + MEMO_OFF, sp.memo + (size_t)t * sp.n_pad + row, STREAM_TILE * 4, &ss.full[s]);
    if (MASKS) {
      bulk_g2s(st + STREAM_TILE * 24, sp.m_taint + row, STREAM_TILE * 8, &ss.full[s]);
      bulk_g2s(st + STREAM_TILE * 32, sp.m_static + row, STREAM_TILE * 8, &ss.full[s]);
    }
  };

  long long k = 0;
  bool limit_hit = false;
  long long dbg_t = 0, dbg_wait = 0, dbg_scan = 0, dbg_xchg = 0, dbg_rest = 0;    // DBG_CYCLES: this CTA's cycle split (thread 0)
  const bool dbg = (p.debug_flags & DBG_CYCLES) != 0u && tid == 0;
  // Warp specialisation. Warps 0..15 SCAN. Warp 16, the EXCHANGE warp, publishes the CTA's key, requests the next wave's bulk
  // copies and polls: a wave's critical path is scan -> barrier A -> publish / poll (one L2 round trip) -> barrier B -> next scan.
  // Warp 17, the COMMIT warp, is decoupled from those barriers: it takes the winners from a small ring in shared memory and, when
  // the node is this CTA's, commits it in two parts — URGENT: row columns from L2, the resident copy, the new generation, the score
  // of the NEXT wave's template patched into the landed memo column (then `commit_seq` releases the one scanning thread that
  // looks at this node); LAZY: write-through of the global columns, the re-scores of the other 63 templates, their memo stores,
  // the proxy fence. A stale memo entry read by a bulk copy that overtook the lazy part is caught by the generation check.
  // Before this split the owner CTA's next key — which every other CTA waits for — came one whole commit (several thousand
  // cycles) late, every wave.
  const bool xwarp = warp == STREAM_WARPS, service = warp == STREAM_WARPS + 1, scanner = warp < STREAM_WARPS;
  constexpr int SYNC_N = STREAM_THREADS + 32;      // scanning warps + exchange warp: the participants of barriers A and B
  int pend_off = -1;                 // owner CTA: chunk offset of the node whose commit may still be under way when this pass starts
  bool prefetched = false;           // the first tiles of the coming wave were requested at the end of the last one
  long long pf_wave = 0;             // ... the wave they were requested for
  uint32_t uses = 0;                 // tiles consumed so far by this CTA (all waves): stage = uses % STAGES, parity = (uses / STAGES) & 1
  uint32_t wtag = 1;
  uint32_t tag = (p.epoch << 12) | wtag;
  const int tiles = sp.tiles;
  const bool all_in_flight = tiles <= NST;     // the whole chunk fits in the ring: no stage is reused within a pass
  // RESF: the whole memo column of a wave lands on ONE mbarrier (full[0]); otherwise one barrier per stage
  auto request_first_tiles = [&](uint32_t ubase_, int t_) {
    fence_proxy_async();              // generic-proxy stores (commits, scorers) before the engine reads them
    if (RESF) {
      mbar_expect_tx(&ss.full[0], (uint32_t)tiles * STAGE_BYTES);
      for (int q = 0; q < tiles; q++)
        bulk_g2s(smem_raw + (size_t)q * STAGE_BYTES, sp.memo + (size_t)t_ * sp.n_pad + base + (long long)q * STREAM_TILE, STREAM_TILE * 4, &ss.full[0]);
    } else {
      for (int q = 0; q < NST && q < tiles; q++) issue(q, (int)((ubase_ + q) % NST), t_);
    }
  };
  if (!service)
  for (;; k++) {
    if (p.max_pods > 0 && k >= p.max_pods) { limit_hit = true; break; }
    if (k > p.pod_cap) { if (tid == 0) ss.stop = 3; break; }
    const int t = (int)(k % T);
    const StreamTmpl &c = ss.tc[t];
    const uint32_t ubase = uses;
    if (xwarp && lane == 0 && !prefetched) request_first_tiles(ubase, t);
    SPH_START();
    if (dbg) { const long long c0 = clock64(); if (dbg_t) dbg_rest += c0 - dbg_t; dbg_t = c0; }
    if (scanner) {
      const long long eq_cpu = c.eq_cpu, eq_mem = c.eq_mem;
      const int32_t pods_need = c.pods_need;
      unsigned long long best = 0ull;
      bool wrote = false;
      if (RESF) {
        // ---- resident columns: the whole chunk's memo column is in flight (tile q in stage q), so the pass is ONE flat loop over the
        //      chunk with a 32-bit local key (score + 1 : 12 | ~offset : 20 — same order as pack_key inside a CTA: highest score, then
        //      lowest index). In the owner CTA of the last commit it starts behind the winner's tile, so that the commit — running
        //      in the service warp meanwhile — is over long before anybody needs that node. ----
        while (!mbar_try_wait(&ss.full[0], (uint32_t)(k & 1))) { }
        if (dbg) { const long long c0 = clock64(); dbg_wait += c0 - dbg_t; dbg_t = c0; }
        const int32_t *memo_s = reinterpret_cast<const int32_t *>(smem_raw);      // stage q = tile q: contiguous
        const int cpad = sp.res_rows;     // rows behind it are padding (free_pods = INT_MIN): never feasible
        uint32_t best32 = 0u;
        auto node = [&](int off, bool check) {
          if (check && off == pend_off) {  // the node committed a moment ago: wait for the urgent part of its commit
            while (ld_vol_s32(&ss.commit_seq) != (int32_t)k) { }
            __threadfence_block();
          }
          const longlong2 fr = r_free[off];
          const int2 pg = r_pg[off];
          int32_t enc = memo_s[off];
          if ((fr.x >= eq_cpu) & (fr.y >= eq_mem) & (pg.x >= pods_need)) {
            if ((enc >> 12) != pg.y) {     // never scored by this template (the run's first T waves); the owner re-scores at commit
              const long long i = (long long)cta * p.chunk + off;
              const int32_t sc = score_node(p.alloc_cpu[i], p.alloc_mem[i], p.nz_cpu[i] + c.least_cpu, p.nz_mem[i] + c.least_mem,
                                            p.req_cpu[i] + c.bal_cpu, p.req_mem[i] + c.bal_mem, c.sw);
              enc = (pg.y << 12) | (sc + 1);
              sp.memo[(size_t)t * sp.n_pad + base + off] = enc;
              if (cta == 0) atomicAdd((unsigned long long *)&ss.n_stale, 1ull);
              wrote = true;                // fenced once after the pass (a later bulk-async read of this column must see the store)
            }
            best32 = max(best32, ((uint32_t)enc << 20) | (0xfffffu - (uint32_t)off));     // (enc << 20 keeps exactly the 12 score bits)
          }
        };
        // order: the tiles behind the pending node's tile, the tiles before it, that tile last (only there the node is looked for)
        const int pt = (pend_off >= 0 ? pend_off / STREAM_TILE : tiles - 1) * STREAM_TILE;
        #pragma unroll 2
        for (int off = pt + STREAM_TILE + tid; off < cpad; off += STREAM_THREADS) node(off, false);
        #pragma unroll 2
        for (int off = tid; off < pt; off += STREAM_THREADS) node(off, false);
        #pragma unroll
        for (int off = pt + tid; off < min(pt + STREAM_TILE, cpad); off += STREAM_THREADS) node(off, true);
        if (best32) {
          const int boff = (int)(0xfffffu - (best32 & 0xfffffu));
          best = pack_key((int32_t)(best32 >> 20) - 1, (uint32_t)(p.node_base + (long long)cta * p.chunk + boff));
        }
      } else {
        const unsigned long long taint_bad0 = c.taint_bad0, sel0 = c.sel0, forbid0 = c.forbid0;
        // (streamed rows: tiles requested during this pass read the global columns — thread 0, which requests them, waits for the
        //  WHOLE commit of the last wave first)
        if (tid == 0 && pend_off >= 0) { while (ld_vol_s32(&ss.commit_full) != (int32_t)k) { } __threadfence_block(); }
        for (int tile = 0; tile < tiles; tile++) {
          const uint32_t use = ubase + (uint32_t)tile;
          const int s = (int)(use % NST);
          while (!mbar_try_wait(&ss.full[s], (use / NST) & 1u)) { }
          const unsigned char *st = smem_raw + (size_t)s * STAGE_BYTES;
          const long long *s_fcpu = reinterpret_cast<const long long *>(st);
          const long long *s_fmem = reinterpret_cast<const long long *>(st + STREAM_TILE * 8);
          const int32_t *s_fpods = reinterpret_cast<const int32_t *>(st + STREAM_TILE * 16);
          const int32_t *s_memo = reinterpret_cast<const int32_t *>(st + MEMO_OFF);
          #pragma unroll
          for (int j = tid; j < STREAM_TILE; j += STREAM_THREADS) {
            const int off = tile * STREAM_TILE + j;
            if (off == pend_off) {
              while (ld_vol_s32(&ss.commit_full) != (int32_t)k) { }
              __threadfence_block();
            }
            // NodeResourcesFit (+ NodeUnschedulable / TaintToleration / nodeSelector / NodePorts / existing anti-affinity bits)
            bool ok = (s_fcpu[j] >= eq_cpu) & (s_fmem[j] >= eq_mem) & (s_fpods[j] >= pods_need);
            if (MASKS) {
              const unsigned long long taint0 = reinterpret_cast<const unsigned long long *>(st + STREAM_TILE * 24)[j];
              const unsigned long long static0 = reinterpret_cast<const unsigned long long *>(st + STREAM_TILE * 32)[j];
              ok &= ((taint0 & taint_bad0) | (~static0 & sel0) | (static0 & forbid0)) == 0ull;
            }
            if (ok) {
              const long long i = (long long)cta * p.chunk + off;        // shard-local node index
              int32_t sc = s_memo[j];
              if (sc < 0) {   // stale: this node was committed since template t last scored it (or never scored)
                sc = score_node(p.alloc_cpu[i], p.alloc_mem[i], p.nz_cpu[i] + c.least_cpu, p.nz_mem[i] + c.least_mem,
                                p.req_cpu[i] + c.bal_cpu, p.req_mem[i] + c.bal_mem, c.sw);
                sp.memo[(size_t)t * sp.n_pad + base + off] = sc;
                if (cta == 0) atomicAdd((unsigned long long *)&ss.n_stale, 1ull);
                wrote = true;
              }
              const unsigned long long key = pack_key(sc, (uint32_t)(p.node_base + i));
              best = key > best ? key : best;
            }
          }
          if (!all_in_flight) {
            bar_sync_n(3, STREAM_THREADS);   // the scanning warps are done with stage s
            // (no proxy fence here: the rows of a later tile were last written in an earlier wave)
            if (tid == 0 && tile + NST < tiles) issue(tile + NST, s, t);
          }
        }
      }
      if (wrote) fence_proxy_async();
      if (dbg) { const long long c0 = clock64(); dbg_scan += c0 - dbg_t; dbg_t = c0; }
      const unsigned long long v = warp_max_u64(best);
      if (lane == 0) ss.warp_best[warp] = v;
    }
    SPH_MARK(0);                           // scan: mbarrier wait + Filter/arg-max over the chunk
    bar_sync_n(1, SYNC_N);                 // A: the pass is over — warp maxima visible, stages free
    SPH_MARK(1);                           // barrier A
    if (dbg) { const long long c0 = clock64(); dbg_rest += c0 - dbg_t; dbg_t = c0; }
    uses = ubase + (RESF ? (uint32_t)NST : (uint32_t)tiles);
    const uint32_t uses_next = uses;           // the next wave's tile q lands in stage (uses_next + q) % STAGES
    prefetched = !(p.max_pods > 0 && k + 1 >= p.max_pods);
    if (prefetched) pf_wave = k + 1;
    if (xwarp) {
      const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
      const unsigned long long mine = warp_max_u64(lane < STREAM_WARPS ? ss.warp_best[lane] : 0ull);
      if (lane == 0) st_slot(p.slots + ((size_t)(k & 1) * CCSIM_MAX_GRID + cta) * SLOT_STRIDE, (mine & KEY_BODY_MASK) | tagbits);
      if (lane == 0 && prefetched) request_first_tiles(uses_next, (int)((k + 1) % T));    // the next wave's memo column, while the keys travel
      bool dead = false;
      unsigned long long wkey = 0ull;
      {
        unsigned long long v[GATHER_Q];
        dead = gather_tagged(p, k, tag, 0, lane, v);
        wkey = gather_max(v);
      }
      if (p.world > 1 && !dead) { unsigned long long cb[1] = {wkey}; dead = cross_gpu_exchange(p, k, tag, 1, cb, lane, cta); wkey = cb[0]; }   // node shards: winners of all ranks
      if (lane == 0) {
        if (dead) { ss.stop = 3; ss.winner = -1; }
        else if (wkey == 0ull) { ss.stop = 1; ss.winner = -1; }
        else { ss.winner = (int32_t)key_index(wkey); if (k >= p.pod_cap) ss.stop = 3; }     // (no room to record the placement)
        // hand the winner to the commit warp (ring of STREAM_WQ: it may lag behind, but never by more than the ring)
        while (ld_vol_s32(&ss.c_done) + STREAM_WQ <= (int32_t)k) { }
        ss.wq[k & (STREAM_WQ - 1)] = ss.stop ? STREAM_WQ_STOP : ss.winner;
        __threadfence_block();
        st_vol_s32(&ss.w_seq, (int32_t)k + 1);
      }
    }
    bar_sync_n(2, SYNC_N);                 // B: the winner is known to every scanning thread
    SPH_MARK(2);                           // exchange: publish, poll every CTA's key (one L2 round trip + the slowest CTA)
    if (dbg) { const long long c0 = clock64(); dbg_xchg += c0 - dbg_t; dbg_t = c0; }
    if (ss.stop) break;
    pend_off = -1;
    {
      const int32_t w = ss.winner - p.node_base;
      if (w >= 0 && w < p.n && w / p.chunk == cta) pend_off = w - cta * p.chunk;
    }
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
  }
  else {
    // ---- the commit warp (assume -> AssumePod -> NodeInfo.update(+1): schedule_one.go:967-984, types.go:409-427) ----
    for (long long kc = 0;; kc++) {
      if (p.max_pods > 0 && kc >= p.max_pods) break;
      if (kc > p.pod_cap) break;
      while (ld_vol_s32(&ss.w_seq) <= (int32_t)kc) { }
      __threadfence_block();
      const int32_t wn = ss.wq[kc & (STREAM_WQ - 1)];
      if (wn == STREAM_WQ_STOP) break;
      const StreamTmpl &c = ss.tc[(int)(kc % T)];
      const int32_t w = wn - p.node_base;
      const bool local = w >= 0 && w < p.n;
      const int oc = local ? w / p.chunk : -1;
      if (!local && cta == 0 && lane == 0) p.pod_node[kc] = wn;      // sharded run: every rank keeps the whole pod -> node sequence
      if (oc == cta) {
        const int roff = w - oc * p.chunk;
        const long long q = base + roff;
        const bool pf = !(p.max_pods > 0 && kc + 1 >= p.max_pods);        // the next wave's first tiles were requested before this commit
        const int tn = (int)((kc + 1) % T);
        // URGENT: every lane reads the row columns (one L2 round trip, broadcast); lanes 1..5 write one column each through to global
        // memory at once — a scanning thread of THIS CTA that meets a not-yet-refreshed memo entry of the node re-scores it from
        // those columns, so they must be current before `commit_seq` says so (same SM: the L1 sees the stores)
        const long long a_cpu = p.alloc_cpu[w], a_mem = p.alloc_mem[w];
        const long long n_rcpu = p.req_cpu[w] + c.req_cpu, n_rmem = p.req_mem[w] + c.req_mem;
        const long long n_zcpu = p.nz_cpu[w] + c.nz_cpu, n_zmem = p.nz_mem[w] + c.nz_mem;
        const int32_t n_pods = p.npods[w] + 1;
        const int tw = roff / STREAM_TILE, j = roff - tw * STREAM_TILE;
        if (lane == 0) p.pod_node[kc] = w + p.node_base;
        else if (lane == 1) p.req_cpu[w] = n_rcpu;
        else if (lane == 2) p.req_mem[w] = n_rmem;
        else if (lane == 3) p.nz_cpu[w] = n_zcpu;
        else if (lane == 4) p.nz_mem[w] = n_zmem;
        else if (lane == 5) p.npods[w] = n_pods;
        __threadfence_block();
        __syncwarp();
        int32_t newgen = 0;
        if (RESF) {
          // resident copy + generation, and the next wave's memo entry of this node patched into the landed column
          const StreamTmpl &cn = ss.tc[tn];
          const int32_t scn = score_node(a_cpu, a_mem, n_zcpu + cn.least_cpu, n_zmem + cn.least_mem, n_rcpu + cn.bal_cpu, n_rmem + cn.bal_mem, cn.sw);
          if (lane == 0) {
            longlong2 fr = r_free[roff]; fr.x -= c.req_cpu; fr.y -= c.req_mem; r_free[roff] = fr;
            const int2 pg = r_pg[roff]; newgen = (pg.y + 1) & 0x7ffff; r_pg[roff] = make_int2(pg.x - 1, newgen);
            if (pf) {
              while (!mbar_try_wait(&ss.full[0], (uint32_t)((kc + 1) & 1))) { }
              reinterpret_cast<int32_t *>(smem_raw)[roff] = (newgen << 12) | (scn + 1);
            }
            __threadfence_block();
            st_vol_s32(&ss.commit_seq, (int32_t)kc + 1);
          }
          newgen = __shfl_sync(0xffffffffu, newgen, 0);
        } else if (lane == 0) { sp.f_cpu[q] -= c.req_cpu; sp.f_mem[q] -= c.req_mem; sp.f_pods[q] -= 1; }
        // LAZY: the other templates' memo entries
        if (RESF) {
          // every template's memo entry of this node, re-scored under the new generation (two templates per lane): a stale entry met by
          // a scan costs that CTA an L2 round trip plus the score's divisions in the middle of its pass
          for (int tt = lane; tt < T; tt += 32) {
            const StreamTmpl &ct = ss.tc[tt];
            const int32_t sc = score_node(a_cpu, a_mem, n_zcpu + ct.least_cpu, n_zmem + ct.least_mem, n_rcpu + ct.bal_cpu, n_rmem + ct.bal_mem, ct.sw);
            sp.memo[(size_t)tt * sp.n_pad + q] = (newgen << 12) | (sc + 1);
          }
          fence_proxy_async();             // these generic-proxy stores, before the bulk-async reads of later waves
        } else {
          for (int tt = lane; tt < T; tt += 32) sp.memo[(size_t)tt * sp.n_pad + q] = -1;      // this node's NodeInfo generation changed
          fence_proxy_async();
          // the winner's row may already sit, pre-commit, in a stage requested for the next wave: wait for that copy, then patch it
          if (pf && tw < NST && tw < tiles && lane == 0) {
            const uint32_t u = (uint32_t)(kc + 1) * (uint32_t)tiles + (uint32_t)tw;
            const int s = (int)(u % NST);
            while (!mbar_try_wait(&ss.full[s], (u / NST) & 1u)) { }
            unsigned char *st = smem_raw + (size_t)s * STAGE_BYTES;
            reinterpret_cast<long long *>(st)[j] = sp.f_cpu[q];
            reinterpret_cast<long long *>(st + STREAM_TILE * 8)[j] = sp.f_mem[q];
            reinterpret_cast<int32_t *>(st + STREAM_TILE * 16)[j] = sp.f_pods[q];
            reinterpret_cast<int32_t *>(st + MEMO_OFF)[j] = -1;
          }
        }
        __threadfence_block();
        __syncwarp();                      // the lanes' stores, before lane 0 announces the whole commit
        if (lane == 0) st_vol_s32(&ss.commit_full, (int32_t)kc + 1);
      }
      __syncwarp();
      if (lane == 0) st_vol_s32(&ss.c_done, (int32_t)kc + 1);
    }
  }
  if (prefetched && xwarp && lane == 0) {         // copies requested for a wave that never ran: let them land before the CTA exits
    if (RESF) { while (!mbar_try_wait(&ss.full[0], (uint32_t)(pf_wave & 1))) { } }
    else
      for (int q = 0; q < NST && q < tiles; q++) {
        const uint32_t u = uses + (uint32_t)q;
        while (!mbar_try_wait(&ss.full[u % NST], (u / NST) & 1u)) { }
      }
  }
  __syncthreads();
  if (dbg && p.world == 1) {          // per-CTA cycle split into the (unused at world 1) cross-GPU line buffer: the host prints min / mean / max
    unsigned long long *d = p.xslots_peer[p.rank] + XLINES_OFF + (size_t)cta * 4;
    d[0] = (unsigned long long)dbg_wait; d[1] = (unsigned long long)dbg_scan; d[2] = (unsigned long long)dbg_xchg; d[3] = (unsigned long long)dbg_rest;
  }
  if (cta == 0 && tid == 0) {
    DevOut *o = p.out;
    o->placed = k;
    o->stop_code = limit_hit ? CCSIM_STOP_LIMIT_REACHED : CCSIM_STOP_UNSCHEDULABLE;
    o->error = (ss.stop == 3) ? 1 : 0;
    o->waves = limit_hit ? k : k + 1;
    o->evals = o->waves * (long long)p.n;
    o->examined = o->evals;
    o->aff_total = 0;
    for (int q = 0; q < 8; q++) o->phase_cycles[q] = ss.ph[q];
    o->stat[0] = ss.n_stale; o->stat[1] = 0; o->stat[2] = 0;
  }
}
