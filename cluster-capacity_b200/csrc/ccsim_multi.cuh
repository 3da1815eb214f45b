// ccsim_multi.cuh — multi-commit waves for templates coupled through per-domain counters (PodTopologySpread DoNotSchedule,
// required pod anti-affinity): several reference scheduling cycles per grid-wide exchange, identical pod -> node sequence,
// on one GPU or over node shards on several GPUs (the exchange then crosses NVLink inside the same kernel).
//
// Why it is legal. Within a stretch of cycles in which no PodTopologySpread global minimum changes, a node's feasibility
// depends on its own row and on the match counts of its topology domains only, and it is MONOTONE: counts only grow
// (inc >= 0), so a feasible node can become infeasible but never the reverse; a node's score changes only when the node
// itself is committed. The winner of each cycle is therefore the highest-keyed node that is still feasible under the
// counts as updated so far (podtopologyspread/filtering.go:311-356, interpodaffinity/filtering.go:352-432;
// schedule_one.go:894-941 with the canonical first-max tie rule). Every CTA publishes its M best feasible nodes (the exact
// top-M of its tile: keys are unique) with the domain ids their feasibility depends on; every CTA of every rank then
// replays those cycles redundantly and deterministically from the same published data.
//
// Which published candidates may be replayed. A CTA with more than M feasible nodes has UNSEEN nodes, all keyed below its
// M-th (last) published key. T = the largest such last key over all lists is a wave-wide bar: a candidate keyed >= T
// outranks every unseen node of every tile, a candidate keyed below T might not. The replay therefore works on the
// candidates keyed >= T only (compacted into shared memory) and ends when the best live key falls below T, when
//   (a) a PTS minimum moves (limits change, rejected nodes may come back: rescan),
//   (b) the pod limit is reached (simulator.go:300-305),
//   (c) a node wins for the second time (see below).
// A committed node may win again inside the wave with its new score, which is in nobody's list (a randomized differential
// test, tests/test_gpu_stress.py, found this hole in the first version: spread-only templates). Every published candidate
// therefore carries, next to its domain ids, its key after one more clone (node-local Filter part + score recomputed by the
// publisher; 0 = it would not fit). The winner comes back into the replay once with that key ("second life"); when a node
// wins for the second time in a wave its third key is unknown and the wave ends after that commit.
// The best candidate of a wave is always >= T and feasible, so every wave makes progress; a wave without candidates is the
// Unschedulable stop. Node-local terms (hostname anti-affinity, ...) need no re-check: a node appears once per wave.
//
// Exchange: two 128-byte lines per CTA = M (key, payload) pairs (keys in line 0, payloads in line 1), each word tagged
//   (self-validating, no fences).
//   lines live in the handle's slot buffer (L2), st/ld.relaxed.gpu; every CTA compacts the candidates of all lines.
//   node shards: the lines stay on their GPU; after that compaction ONE CTA of every rank stores a summary of the rank's candidates
//                into every peer's line buffer (CUDA IPC mappings, st.relaxed.sys over NVLink), and every CTA compacts the
//                summaries in rank order the same way.
// Replay: ONE warp, no barrier inside: <= 8 candidates per lane in registers; a round is arg-max (REDUX) -> commit (lane q =
//   counter term q: cell += inc, over-limit test, PTS-minimum tracking, all from registers) -> kill the candidates sitting in
//   a cell that just filled (SWAR field test against the OR-reduced filled cells). Measured on C4 (one H100 80GB HBM3,
//   CCSIM_DEBUG_FLAGS=8: replay cycles minus set-up over rounds, so minimum moves, wake-ups and the hand-off after the loop are
//   included): ~827 cycles per reference cycle with one-pass minimum moves (700 W power limit); ~890 before them and ~1 310 before
//   the round was cut down to its dependent chain (three REDUX, one LDS/STS; 400 W power limit) — against ~2000 for a block-wide
//   round (two barriers over 24 warps). The other 23 warps wait at the barrier that ends the wave. -DMULTI_ROUND_PROFILE splits
//   those cycles (scripts/round_profile.sh). Work around the round stays on this warp: moved onto the whole block (the set-up
//   between G1 and G2, the look-ahead decision after R) it measured slower on C4, whose terms have 8 and 64 domains.
//   Row updates of the winners are done by each node's own thread after that barrier (a thread owns its node).
// Key order (single-use templates: no second lives): the compaction stores the wave's candidates in key order, and the replay
//   warp holds them in rows of 32 in key order; a round is ballot(live) -> the lowest live lane -> one SHFL of its payload -> the same
//   commit -> the kill test on each lane's one slot. A row is judged by a full cell test when the replay reaches it; a wake-up goes
//   back to row 0 (see "the round in key order" below). C4: 778 -> 515 profiled cycles per round, kernel time 21.67-21.72 ->
//   20.87-21.01 ms (one H100 80GB HBM3, 700 W power limit). CCSIM_DEBUG_FLAGS bit 6 keeps the arg-max round.
// Sorted tile (single-use templates): a live node's key does not change during a launch (its row changes only when it wins, and
//   then it is infeasible for the rest of the run; the replicated counters change feasibility, not scores). So the tile is ranked
//   by key once per launch, and the tile's top 16 are its first 16 feasible ranks: one ballot per warp, a barrier and a prefix
//   count instead of up to 16 REDUX rounds per warp and warp 0's 24-way merge. The lines are word for word the same. C4: CTA 0's
//   scan + barrier + merge/publish 4 480 -> 2 880 cycles per wave, kernel time 18.75-18.78 -> 17.54-17.56 ms (one H100 80GB HBM3,
//   700 W power limit). Everything but the replicated counter cells is fixed between constants builds too (the node-local Filter
//   verdict: a winner fails it for good; the payload: static), so each rank has a record {key or 0, payload}, rebuilt at every
//   constants build, and the scan is thread t testing the cells of rank t's record: one barrier before the publish instead of two.
//   C4: those three phases 2 870 -> 1 940 cycles per wave, kernel time 17.47-17.59 -> 16.80-16.91 ms (same H100, 700 W). The host
//   picks the instantiation (template parameter SORTED): the ones without it are the REDUX selection alone, compiled as before
//   this selection existed (every sorted-tile statement sits behind `if constexpr`), for templates with second lives and
//   CCSIM_DEBUG_FLAGS bit 7.
// Look-ahead waves: a PodTopologySpread minimum move that REOPENS closed domains would end the wave (the reopened nodes were
//   rejected by the scan and are in nobody's list). When a term's limit is about to move, the scan publishes the nodes of its
//   closed cells too; they sit in the replay as dormant candidates (key 0: set-up reads the look-ahead terms' cells) and are
//   rebuilt from the wave's candidate arrays when the move comes — see "dormant candidates" in the replay. C4: 3654 -> 2260 waves
//   (scripts/wave_sim.py models the wave structure on the CPU and was used to choose the rule).
#pragma once
#include "ccsim_lean.cuh"

#define MULTI_M 16                /* candidates per CTA and wave: 16 keys in one 128-byte slot line, their 16 payloads in a second */
#define MULTI_LINE_WORDS (2 * SLOT_STRIDE)   /* 64-bit words per CTA in the slot buffer: its two lines (one writer per line) */
#define MULTI_EPT 3               /* gather: entries per thread (grid x MULTI_M <= MULTI_EPT x LEAN_THREADS, host-checked; node shards:
                                     the ranks' summaries, static_assert below) */
#define SLOTS_WORDS (2 * CCSIM_MAX_GRID * MULTI_LINE_WORDS)   /* the handle's slot buffer, sized for this kernel's [parity][CTA][2 lines];
                                                                 the other kernels use [parity][CTA][1 line], its first half */
#define MULTI_PAY_BITS 27         /* payload bits for domain ids (dom+1 per topology slot, each field followed by a zero guard bit) */
#define MULTI_NEXT_SHIFT 27       /* 12 bits: (score + 1) of the node after one more clone, 0 = it would not fit any more */
#define MULTI_MORE_BIT 32         /* key word of the last entry: the tile has more feasible nodes than it published */
#define MULTI_MAX_ACC 64          /* commits one wave may decide */
#define MULTI_GT 6                /* Filter terms on replicated counters a template may have in this kernel */
#ifndef MULTI_CPT
#define MULTI_CPT 8               /* candidates per replay lane */
#endif
#define MULTI_CAP (32 * MULTI_CPT)
#define MULTI_LEVELS 4            /* compaction: score levels below the best key it ranks (one 16-bit count per level in a 64-bit word) */
#define MULTI_GROUPS (MULTI_EPT * LEAN_WARPS)   /* compaction: groups of 32 gathered entries (two lists), one count word each */
#define MULTI_RELAX_K 8           /* look-ahead on a PTS term when at most this many of its domains still sit at the global minimum ... */
#define MULTI_RELAX_R 3           /* ... nodes in cells up to this far over the limit are published as dormant candidates */
static_assert(CCSIM_MAX_WORLD * MULTI_CAP <= MULTI_EPT * LEAN_THREADS, "node shards: the ranks' summaries fit the gather's entries");
static_assert(MULTI_GROUPS <= 96 && MULTI_EPT * LEAN_THREADS < 65536, "compaction: three count words per lane, a count fits 16 bits");
static_assert(MULTI_CPT <= 32, "key order: one won bit per row");
static_assert(MULTI_M == SLOT_STRIDE, "the keys of a CTA's list fill exactly one slot line");
static_assert(4 + 2 * MULTI_CAP <= CCSIM_MAX_GRID * SLOT_STRIDE, "node shards: a rank's summary fits its region of the line buffer");

// Round profile (profiling builds only: -DMULTI_ROUND_PROFILE; the hooks expand to nothing otherwise, and the shipped library's
// SASS is the same with and without them). CTA 0's replay warp adds up, over the run, the cycles of: the set-up's candidate load,
// the common round (arg-max -> commit -> kill), the minimum-move handling of each term, the wake-up rebuilds, and what follows the
// loop (in total, and its parts: the hand-off of the winners to their threads, the look-ahead decision; the rest is barrier R); and
// the events: rounds, minimum moves per term, rebuilds, rounds that kill. The kernel prints the table when the run ends
// (scripts/round_profile.sh).
#define RP_ROUND 0
#define RP_REBUILD 1
#define RP_AFTER 2
#define RP_KILL 3                 /* (event count only) */
#define RP_LOAD 4                 /* set-up: the candidates and the term constants into registers */
#define RP_HANDOFF 5              /* after the loop: winners -> ms.mult */
#define RP_DECIDE 6               /* after the loop: the next wave's look-ahead decision */
#define RP_MINMOVE 7              /* + term q */
#define RP_KROUND (RP_MINMOVE + MULTI_GT)   /* key order: the common round (ballot -> commit -> kill) */
#define RP_ADVANCE (RP_KROUND + 1)  /* key order: moving on to the next row (loads + full cell test), per row loaded */
#define RP_N (RP_KROUND + 2)
#ifdef MULTI_ROUND_PROFILE
#define RPROF(...) __VA_ARGS__
#define RP_ADD(i, cyc, n) do { if (cta == 0 && lane == 0) { ms.rp_cyc[i] += (cyc); ms.rp_cnt[i] += (n); } } while (0)
#else
#define RPROF(...)
#define RP_ADD(i, cyc, n) do { } while (0)
#endif

// Gather profile (profiling builds only: -DMULTI_GATHER_PROFILE; the hooks expand to nothing otherwise). CTA 0 adds up, per wave:
// the cycles from its own publish to the poll round in which the last of its entries was valid (the latest of its threads), and
// the number of poll rounds (the most any thread took); from there to the point where the CTA may read every entry (G1); the
// compaction in key order up to the barrier after its stores (G3), and how often the level clamp raised the bar (node shards: both
// gather levels). Every CTA
// also writes its %globaltimer at publish into gp_pub_ns[wave][CTA]; the host reports the skew of the publishes, latest minus CTA
// 0's, per wave. scripts/gather_profile.sh prints both.
#define GP_POLL 0
#define GP_SYNC 1
#define GP_COMPACT 2
#define GP_CLAMP 3                /* (event count only) */
#define GP_ROUNDS 4               /* (event count only) */
#define GP_N 5
#define GP_MAX_WAVES 4096         /* waves with a publish time */
#ifdef MULTI_GATHER_PROFILE
#define GPROF(...) __VA_ARGS__
__device__ long long gp_pub_ns[GP_MAX_WAVES * CCSIM_MAX_GRID];
__device__ __forceinline__ long long globaltimer_ns() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#else
#define GPROF(...)
#endif

// cross-GPU line buffers inside every rank's exchange allocation (64-bit words): [parity][source rank][CTA][16]
#define XLEAN_WORDS (2 * CCSIM_MAX_WORLD * SLOT_STRIDE)
#define XLINES_OFF XLEAN_WORDS
#define XLINES_WORDS (2 * CCSIM_MAX_WORLD * CCSIM_MAX_GRID * SLOT_STRIDE)
#define XSLOTS_TOTAL_WORDS (XLEAN_WORDS + XLINES_WORDS)

struct __align__(16) MultiShared {
  uint32_t wtop[LEAN_WARPS][MULTI_M];               // per-warp top-M (compact) keys of this wave
  int32_t gt_c1[MULTI_GT][4];                       // per replicated-counter term: {limit, payload shift, payload mask, domains of the counter}
  int32_t gt_commit[MULTI_GT][4];                   // ... {counter base, inc, PTS constraint tracked or -1, n_present}
  uint32_t ckey[MULTI_CAP], cdom[MULTI_CAP], cnext[MULTI_CAP];   // the wave's candidates keyed >= T, in key order: key, domain
                                                                 // payload, second-life key
  unsigned long long gcnt[MULTI_GROUPS];            // compaction: per group of 32 gathered entries, its candidates per level (16 bits each)
  uint32_t red[LEAN_WARPS], red2[LEAN_WARPS];       // block reductions (T, best key)
  int32_t wfeas[LEAN_WARPS];
  int32_t gt_term[MULTI_GT];                        // indices of the Filter terms that read a replicated (non node-local) counter
  int32_t acc_node[MULTI_MAX_ACC];                  // replay: nodes accepted in this wave, in order
  int32_t mult[LEAN_THREADS];                       // replay -> row updates: times tile node j was accepted in this wave (its thread resets it)
  int32_t n_gt, accepted, dead, stopb;
  int32_t single_use;
  int32_t xcount[CCSIM_MAX_WORLD];                  // node shards: candidates in each rank's summary (this rank's: its own)
  uint32_t xglob[4];                                // node shards: best key, T_list, bar over all ranks
  uint32_t delta, st_tile_sel;                      // ..., CTA 0 / thread 0: waves that selected from the sorted tile
  int32_t relax[LEAN_MAX_TERMS];                    // per Filter term: this wave's look-ahead over the limit (0: strict), see "dormant candidates"
  int32_t force_strict, st_relaxed, st_empty, tile_sorted;
  long long ph[8], tc0, st_cand, st_overflow, st_rounds, st_key_order;   // CTA 0 / thread 0: clock cycles per phase, replay statistics
#ifdef MULTI_ROUND_PROFILE
  long long rp_cyc[RP_N], rp_cnt[RP_N], rp_t;                  // CTA 0's replay warp: cycles and events per part of the replay
#endif
#ifdef MULTI_GATHER_PROFILE
  unsigned long long gp_valid, gp_spins;                       // CTA 0, this wave: latest clock at which a thread's entries were all valid, most poll rounds
  long long gp_pub, gp_cyc[GP_N], gp_cnt[GP_N];                // CTA 0: its publish clock; cycles and events per part of the gather
#endif
};

__shared__ MultiShared ms;
static_assert(LEAN_THREADS % 2 == 0 && LEAN_THREADS <= 65536, "sorted tile: 16-byte loads of two records, 16-bit ranks");
// sorted tile: tile node j's rank in key order (once per launch), and the node record of every rank: {the node's key, 0 when the
// node fails a node-local part of the Filter pass; its payload} (at every constants build). Only the sorted instantiation references
// them, so only its static shared memory holds them (WAVE_KERNELS in ccsim_engine.cu adds them there)
__shared__ uint16_t multi_tile_rank[LEAN_THREADS];
__shared__ __align__(16) uint2 multi_tile_rec[LEAN_THREADS];
// sorted tile: the scan's constants of replicated-counter term q (q < ms.n_gt): {counter base, payload shift, payload mask, limit +
// look-ahead}, written by the constants build and by the replay warp for the next wave
__shared__ int4 multi_scan_term[MULTI_GT];
#define MULTI_SORTED_SMEM ((sizeof(uint16_t) + sizeof(uint2)) * LEAN_THREADS + sizeof(int4) * MULTI_GT)

// the position of entry r (0 = best) of a CTA's list in its key line: the best key and the last key share the line's first 16 bytes
__device__ __forceinline__ int multi_kpos(int r) { return r == 0 ? 0 : (r == MULTI_M - 1 ? 1 : r + 1); }

struct MultiParams {
  uint32_t pay_shift[LEAN_MAX_SLOTS];   // record slot s (a topology column) -> bit position of its dom+1 field in the payload
  uint32_t pay_mask[LEAN_MAX_SLOTS];    // field mask (0: the slot is a node-local counter, not carried)
};

// 32-bit keys for everything inside this kernel: (score+1) in bits 20..31, (2^20-1 - global index) below (needs N < 2^20 and
// score+1 < 4096, both host-checked). Same order as pack_key (highest score, then lowest index); one REDUX per arg-max.
#define MULTI_IDX_BITS 20
#define MULTI_IDX_MASK ((1u << MULTI_IDX_BITS) - 1u)
__device__ __forceinline__ uint32_t ckey(int32_t score, uint32_t gidx) { return ((uint32_t)(score + 1) << MULTI_IDX_BITS) | (MULTI_IDX_MASK - gidx); }
__device__ __forceinline__ int32_t ckey_index(uint32_t ck) { return (int32_t)(MULTI_IDX_MASK - (ck & MULTI_IDX_MASK)); }

template <bool XGPU> __device__ __forceinline__ void ld_line2(const unsigned long long *p, unsigned long long &a, unsigned long long &b) {
  if (XGPU) asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
  else asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_line2_sys(unsigned long long *p, unsigned long long a, unsigned long long b) {
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}

// position of the g-th (0-based, g < 4) set bit of m, or -1
__device__ __forceinline__ int nth_set_lane(unsigned m, int g) {
  #pragma unroll
  for (int i = 0; i < 3; i++) if (i < g) m &= m - 1;
  return m ? __ffs(m) - 1 : -1;
}

// ---- the gathered entries keyed >= T go into shared memory in key order, straight to their ranks (every thread of the block calls
//      this, with the same T and kbest). Entry u of thread tid is entry e = tid + u * LEAN_THREADS of a concatenation that is in key
//      order within every score level: ea[u] holds its key (0: none), eb[u] its payload. An entry's level is its score's distance below
//      the best key's score. Entry u of warp w's threads lies in group g = w + LEAN_WARPS * u of 32 entries, in lane order. So a
//      candidate's rank is
//        #(candidates on higher levels) + #(candidates on its level in groups < g) + #(candidates on its level in lanes < its lane),
//      exact because keys are unique. Per-level ballots give the last term and the group's counts, one barrier publishes the
//      counts (one 64-bit word per group), and every warp sums what it needs of them itself.
//      At most MULTI_LEVELS levels are ranked: when the candidates span more, the bar goes up to the lowest key of the lowest
//      level ranked. More than MULTI_CAP candidates: the bar is the key of rank MULTI_CAP - 1. Either bar is above T, and any bar
//      above T is valid: the best candidate is still in, and a strict wave places it. Returns the candidates stored (<= MULTI_CAP),
//      sets T to the bar and `over` when there were more than MULTI_CAP (block-uniform; left as it was otherwise, so that the
//      two gather levels of a node-shard wave raise one flag). The candidate arrays are written after the first barrier only. ----
__device__ __forceinline__ int multi_compact(const unsigned long long (&ea)[MULTI_EPT], const unsigned long long (&eb)[MULTI_EPT], uint32_t &T,
                                             const uint32_t kbest, const int cta, bool &over) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  GPROF(const long long gp_t = clock64();)
  const uint32_t kbl = kbest >> MULTI_IDX_BITS;
  int rk[MULTI_EPT];                       // the entry's level << 8 | its place among the group's candidates on that level; -1: none
  bool beyond = false;                     // a candidate more than MULTI_LEVELS - 1 levels below the best key
  #pragma unroll
  for (int u = 0; u < MULTI_EPT; u++) {
    const uint32_t ck = (uint32_t)ea[u];   // (0 beyond the entries)
    const bool q = ck != 0u && ck >= T;
    const uint32_t lv = kbl - (ck >> MULTI_IDX_BITS);
    beyond |= q && lv >= MULTI_LEVELS;
    unsigned long long wc = 0ull;
    int pos = 0;
    #pragma unroll
    for (int v = 0; v < MULTI_LEVELS; v++) {
      const unsigned b = __ballot_sync(0xffffffffu, q && lv == (uint32_t)v);
      wc |= (unsigned long long)__popc(b) << (16 * v);
      if (lv == (uint32_t)v) pos = __popc(b & ((1u << lane) - 1u));
    }
    rk[u] = (q && lv < MULTI_LEVELS) ? (int)(lv << 8) | pos : -1;
    if (lane == 0) ms.gcnt[warp + LEAN_WARPS * u] = wc;
  }
  const bool clamp = __syncthreads_or(beyond);                      // G2
  // lane l sums groups l, l + 32, l + 64: all of them (the candidates per level), and those before each of this warp's groups
  const unsigned long long g0 = ms.gcnt[lane], g1 = ms.gcnt[lane + 32], g2 = lane + 64 < MULTI_GROUPS ? ms.gcnt[lane + 64] : 0ull;
  const unsigned long long gs = g0 + g1 + g2;
  const unsigned long long S = ((unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)(gs >> 32)) << 32) | __reduce_add_sync(0xffffffffu, (uint32_t)gs);
  const unsigned long long Sabove = S * 0x0001000100010000ull;    // field v: the candidates on levels < v
  const int total = (int)((S * 0x0001000100010001ull) >> 48);
  #pragma unroll
  for (int u = 0; u < MULTI_EPT; u++) {
    const int g = warp + LEAN_WARPS * u;
    const unsigned long long ps = (lane < g ? g0 : 0ull) + (lane + 32 < g ? g1 : 0ull) + (lane + 64 < g ? g2 : 0ull);
    const unsigned long long P = ((unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)(ps >> 32)) << 32) | __reduce_add_sync(0xffffffffu, (uint32_t)ps);
    if (rk[u] >= 0) {
      const int r = (int)(((Sabove + P) >> (16 * (rk[u] >> 8))) & 0xffffu) + (rk[u] & 0xff);
      if (r < MULTI_CAP) {
        ms.ckey[r] = (uint32_t)ea[u];
        ms.cdom[r] = (uint32_t)eb[u] & ((1u << MULTI_PAY_BITS) - 1u);
        ms.cnext[r] = (uint32_t)(eb[u] >> MULTI_NEXT_SHIFT) & 0xfffu;
      }
    }
  }
  if (clamp) T = (kbl - (MULTI_LEVELS - 1)) << MULTI_IDX_BITS;
  if (total > MULTI_CAP) over = true;
  __syncthreads();                                                  // G3
  if (total > MULTI_CAP) T = ms.ckey[MULTI_CAP - 1];
  GPROF(if (cta == 0 && tid == 0) { ms.gp_cyc[GP_COMPACT] += clock64() - gp_t; ms.gp_cnt[GP_CLAMP] += clamp; })
  return min(total, MULTI_CAP);
}

// node shards: wait until the N (2 or 3) words at src — part of a peer's summary, written into this GPU's memory over NVLink — carry
// this wave's tag; after WATCHDOG_SPINS polls the exchange is dead (ms.dead) and the words read as zeros
template <int N>
__device__ __forceinline__ void multi_poll_sys(const unsigned long long *src, uint32_t tag, unsigned long long (&w)[N]) {
  static_assert(N == 2 || N == 3, "one 16-byte load, and one more word");
  unsigned spins = 0;
  for (;;) {
    ld_line2<true>(src, w[0], w[1]);
    if (N == 3) w[N - 1] = ld_slot_sys(src + 2);
    bool ok = true;
    #pragma unroll
    for (int i = 0; i < N; i++) ok = ok && (uint32_t)(w[i] >> KEY_TAG_SHIFT) == tag;
    if (ok) break;
    if (++spins > WATCHDOG_SPINS) { ms.dead = 1; for (int i = 0; i < N; i++) w[i] = 0ull; break; }
  }
}

// phase timers live in shared memory (thread 0 of CTA 0 only): registers are what this kernel is short of
#define MPH_START() do { if (cta == 0 && tid == 0) ms.tc0 = clock64(); } while (0)
#define MPH_MARK(i) do { if (cta == 0 && tid == 0) { const long long tc1_ = clock64(); ms.ph[i] += tc1_ - ms.tc0; ms.tc0 = tc1_; } } while (0)

// ---- end of the run (the CTA that writes the output): the tables of the profiling builds; nothing in the shipped build ----
__device__ __forceinline__ void multi_report(long long waves) {
#ifdef MULTI_ROUND_PROFILE
  {
    const double w = (double)(waves), nr = (double)(ms.st_rounds > 0 ? ms.st_rounds : 1);
    printf("round profile (CTA 0): waves %.0f rounds %lld | replay %.0f cycles/wave, set-up %.0f\n", w, ms.st_rounds, ms.ph[4] / w, ms.ph[6] / w);
    printf("round profile: common round %lld events, %.0f cycles/round, %.0f cycles/wave\n", ms.rp_cnt[RP_ROUND], ms.rp_cyc[RP_ROUND] / nr, ms.rp_cyc[RP_ROUND] / w);
    printf("round profile: wake-up rebuilds %lld, %.0f cycles each, %.0f cycles/wave\n", ms.rp_cnt[RP_REBUILD],
           ms.rp_cyc[RP_REBUILD] / (double)(ms.rp_cnt[RP_REBUILD] > 0 ? ms.rp_cnt[RP_REBUILD] : 1), ms.rp_cyc[RP_REBUILD] / w);
    printf("round profile: set-up: candidate load %.0f cycles/wave\n", ms.rp_cyc[RP_LOAD] / w);
    printf("round profile: after the loop %lld waves, %.0f cycles/wave (hand-off %.0f, look-ahead decision %.0f)\n", ms.rp_cnt[RP_AFTER],
           ms.rp_cyc[RP_AFTER] / w, ms.rp_cyc[RP_HANDOFF] / w, ms.rp_cyc[RP_DECIDE] / w);
    printf("round profile: rounds with a non-zero kill mask %lld\n", ms.rp_cnt[RP_KILL]);
    printf("round profile: key order %lld waves | common round %lld events, %.0f cycles/round, %.0f cycles/wave"
           " | row advances %lld, %.0f cycles each, %.0f cycles/wave\n", ms.st_key_order,
           ms.rp_cnt[RP_KROUND], ms.rp_cyc[RP_KROUND] / (double)(ms.rp_cnt[RP_KROUND] > 0 ? ms.rp_cnt[RP_KROUND] : 1), ms.rp_cyc[RP_KROUND] / w,
           ms.rp_cnt[RP_ADVANCE], ms.rp_cyc[RP_ADVANCE] / (double)(ms.rp_cnt[RP_ADVANCE] > 0 ? ms.rp_cnt[RP_ADVANCE] : 1), ms.rp_cyc[RP_ADVANCE] / w);
    for (int q = 0; q < MULTI_GT; q++)
      if (ms.rp_cnt[RP_MINMOVE + q])
        printf("round profile: term %d minimum moves %lld, %.0f cycles each, %.0f cycles/wave\n", q, ms.rp_cnt[RP_MINMOVE + q],
               ms.rp_cyc[RP_MINMOVE + q] / (double)ms.rp_cnt[RP_MINMOVE + q], ms.rp_cyc[RP_MINMOVE + q] / w);
  }
#endif
#ifdef MULTI_GATHER_PROFILE
  {
    const double w = (double)(waves);
    printf("gather profile (CTA 0): waves %.0f | publish -> all own entries valid %.0f cycles/wave, %.1f poll rounds/wave | -> entries readable (G1) %.0f"
           " | compaction in key order %.0f | bar over %d levels raised in %lld waves\n", w, ms.gp_cyc[GP_POLL] / w, ms.gp_cnt[GP_ROUNDS] / w,
           ms.gp_cyc[GP_SYNC] / w, ms.gp_cyc[GP_COMPACT] / w, MULTI_LEVELS, ms.gp_cnt[GP_CLAMP]);
  }
#endif
}

// SORTED: the host chose the selection from the sorted tile (a single-use template: see plan_multi); the instantiations without it
// are the REDUX selection alone, for templates with second lives and CCSIM_DEBUG_FLAGS bit 7
template <bool XGPU, bool SORTED>
__global__ void __launch_bounds__(LEAN_THREADS, 1) ccsim_wave_multi_kernel(const DevParams p, const LeanParams lp, const MultiParams mp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const size_t cp = (size_t)p.chunk_pad;
  const LeanTile t = lean_tile(smem_raw, lp, cp);
  int32_t *smem_cnt = t.cnt;
  unsigned long long *c_pay = reinterpret_cast<unsigned long long *>(t.own);   // each node's payload (the 16 bytes after it are not read)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = blockIdx.x;
  const int32_t lo = min(p.n, cta * p.chunk), hi = min(p.n, lo + p.chunk);
  const int32_t cnt_nodes = hi - lo;      // <= LEAN_THREADS (host-checked): one node per thread
  const uint32_t cnt_sa = pin_u32(smem_u32(smem_cnt)), ms_sa = pin_u32(smem_u32(&ms));   // shared bases for the replay's explicit-address accesses
#define MS_SA(field) (ms_sa + (uint32_t)offsetof(MultiShared, field))
  const int nlists = p.grid;                            // lines of this GPU (node shards: every rank launches the same grid, sized from the largest shard)
  const int tot = nlists * MULTI_M;

  if (tid == 0) { ms.accepted = 0; ms.dead = 0; ms.stopb = 0; ms.n_gt = 0; ms.delta = 1u << MULTI_IDX_BITS; ms.force_strict = 0; ms.st_relaxed = 0; ms.st_empty = 0;
                  if (SORTED) { ms.tile_sorted = 0; ms.st_tile_sel = 0; }
                  for (int q = 0; q < LEAN_MAX_TERMS; q++) ms.relax[q] = 0;
                  for (int q = 0; q < 8; q++) ms.ph[q] = 0; ms.tc0 = 0; ms.st_cand = 0; ms.st_overflow = 0; ms.st_rounds = 0; ms.st_key_order = 0;
                  RPROF(for (int q = 0; q < RP_N; q++) ms.rp_cyc[q] = ms.rp_cnt[q] = 0; ms.rp_t = 0;)
                  GPROF(for (int q = 0; q < GP_N; q++) ms.gp_cyc[q] = ms.gp_cnt[q] = 0; ms.gp_valid = ms.gp_spins = 0ull; ms.gp_pub = 0;) }
  ms.mult[tid] = 0;
  lean_stage(p, lp, t, lo, cnt_nodes);
  for (int c = 0; c < ls.tmpl.n_pts; c++) lean_pts_recount(p, smem_cnt, c);
  // the node's payload for the candidate exchange: domain id + 1 of every topology slot (static: labels do not change)
  for (int32_t j = tid; j < cnt_nodes; j += LEAN_THREADS) {
    const int32_t *r4 = lean_rec4(t, lp, j);
    unsigned long long py = 0ull;
    for (int s = 0; s < lp.n_slots; s++)
      if (mp.pay_mask[s]) py |= (unsigned long long)((uint32_t)(r4[LR_SLOT0 + s] + 1) & mp.pay_mask[s]) << mp.pay_shift[s];
    c_pay[j] = py;
  }

  long long k = 0, wv = 0;
  uint32_t delta = 1u << MULTI_IDX_BITS;     // bar distance below the best key: starts at one score level
  bool limit_hit = false;   // postBindHook's limit (simulator.go:300-305)
  uint32_t wtag = 1;
  uint32_t tag = (p.epoch << 12) | wtag;
  for (;; wv++) {
    MPH_START();
    if (p.max_pods > 0 && k >= p.max_pods) { limit_hit = true; break; }   // uniform; no shared write (slower threads may still be reading ls.stop)
    if (k > p.pod_cap) { if (tid == 0) ls.stop = 3; __syncthreads(); break; }
    if (ls.dirty) {
      if (tid == 0) {
        lean_build_consts(p, lp);
        int g = 0;
        for (int q = 0; q < ls.n_cmp_terms; q++)
          if (ls.terms[q].cnt_off >= 0 && g < MULTI_GT) {
            const int sl = ls.terms[q].slot - LR_SLOT0;
            ms.gt_c1[g][0] = ls.terms[q].lim; ms.gt_c1[g][1] = (int32_t)mp.pay_shift[sl]; ms.gt_c1[g][2] = (int32_t)mp.pay_mask[sl]; ms.gt_c1[g][3] = 0;
            ms.gt_commit[g][0] = ls.terms[q].cnt_off; ms.gt_commit[g][1] = 0; ms.gt_commit[g][2] = -1; ms.gt_commit[g][3] = 0;
            for (int j = 0; j < p.n_counters; j++)
              if (p.counters[j].topo_col >= 0 && p.counters[j].smem_off == ls.terms[q].cnt_off) {
                ms.gt_commit[g][1] = ls.cinfo[j].inc; ms.gt_commit[g][2] = ls.cinfo[j].pts_idx; ms.gt_commit[g][3] = ls.cinfo[j].n_present;
                ms.gt_c1[g][3] = p.counters[j].n_domains;
              }
            if constexpr (SORTED) multi_scan_term[g] = make_int4(ls.terms[q].cnt_off, ms.gt_c1[g][1], ms.gt_c1[g][2], ls.terms[q].lim + ms.relax[q]);
            ms.gt_term[g++] = q;
          }
        ms.n_gt = g;
        int su1 = 0;   // a self-matching required anti-affinity term on a node-local counter: count 0 -> inc > limit 0 after one clone
        for (int q = 0; q < ls.n_cmp_terms; q++)
          if (ls.terms[q].cnt_off < 0 && ls.terms[q].kind == LT_ANTI)
            for (int j = 0; j < p.n_counters; j++)
              if (p.counters[j].topo_col < 0 && LR_SLOT0 + lp.counter_slot[j] == ls.terms[q].slot && ls.cinfo[j].inc > 0) su1 = 1;
        ms.single_use = su1;
      }
      __syncthreads();
      // ---- single-use templates: the tile in key order, once per launch. A live node's key does not change during the launch: its
      //      row changes only when it wins, and then it never passes the Filter pass again; the replicated counters decide
      //      feasibility, not scores. Rank = the number of greater keys (keys are unique: the index bits), counted by the node's own
      //      thread over the keys staged in the records. Then, at every constants build (the node-local limits move only here), the
      //      node's record at its rank: its key if it passes every node-local part of the Filter pass (taints, selector, resources,
      //      pods, node-local counter terms; a missing topology key where that rejects), else 0, and its payload. The scan below
      //      tests only the replicated counter cells of the records; a winner's record dies in the hand-off before barrier R. ----
      if (SORTED && ms.single_use) {     // (device-checked: otherwise this instantiation runs the REDUX selection)
        uint32_t mine = 0u;
        bool ok = false;
        if (tid < cnt_nodes) {
          const int32_t *r4 = lean_rec4(t, lp, tid);
          const LeanRow w = lean_row(reinterpret_cast<const uint4 *>(r4));
          ok = lean_fits(w, lean_fit());
          for (int q = 0; q < ls.n_cmp_terms; q++) {
            const LeanTerm lt = ls.terms[q];
            const int32_t v = r4[lt.slot];                     // node-local count, or domain id (< 0: no topology key)
            ok &= lt.cnt_off < 0 ? v <= lt.lim : (v >= 0 || lt.miss_rejects == 0);
          }
          int32_t sc = w.score;
          if (sc < 0) sc = lean_rescore(t, lp, tid);
          mine = ckey(sc, (uint32_t)(p.node_base + lo + tid));
          if (wv == 0) multi_tile_rec[tid].x = mine;
        }
        if (wv == 0) {
          __syncthreads();
          if (tid < cnt_nodes) {
            int r = 0, i = 0;
            #pragma unroll 2
            for (; i + 2 <= cnt_nodes; i += 2) {
              const uint4 v = *reinterpret_cast<const uint4 *>(&multi_tile_rec[i]);
              r += (int)(v.x > mine) + (int)(v.z > mine);
            }
            if (i < cnt_nodes) r += (int)(multi_tile_rec[i].x > mine);
            multi_tile_rank[tid] = (uint16_t)r;
          }
          if (tid == 0) ms.tile_sorted = 1;
          __syncthreads();
        }
        if (tid < cnt_nodes) multi_tile_rec[multi_tile_rank[tid]] = make_uint2(ok ? mine : 0u, (uint32_t)c_pay[tid]);
        __syncthreads();
      }
      if (tid == 0) ls.dirty = 0;
    }
    const bool tile_sel = SORTED && ms.tile_sorted != 0;     // (block-uniform)
    uint32_t key = 0u, kpay = 0u;        // (kpay: sorted tile only, the payload of rank tid)
    if constexpr (SORTED) {
      if (tile_sel) {
        // ---- sorted tile: thread t takes the record of rank t and tests the replicated counter cells of its node, the rest of the
        //      Filter pass is in the record (see the constants build) ----
        const uint2 rc = tid < cnt_nodes ? multi_tile_rec[tid] : make_uint2(0u, 0u);
        const int n_gt = ms.n_gt;
        bool bad = false;
        #pragma unroll
        for (int q = 0; q < MULTI_GT; q++)
          if (q < n_gt) {
            const int4 tc = multi_scan_term[q];
            const uint32_t f = (rc.y >> tc.y) & (uint32_t)tc.z;                 // dom + 1 (0: no domain; cell 0 is read and ignored)
            bad |= (f != 0u) & (smem_cnt[tc.x + max((int32_t)f - 1, 0)] > tc.w);
          }
        key = bad ? 0u : rc.x;
        kpay = rc.y;
      }
    }
    // ---- fused Filter pass: this thread's node ----
    if (tid < cnt_nodes && !(SORTED && tile_sel)) {
      const int32_t j = tid;
      const int32_t *r4 = lean_rec4(t, lp, j);
      const LeanRow w = lean_row(reinterpret_cast<const uint4 *>(r4));
      int32_t sc = w.score;
      bool ok = lean_fits(w, lean_fit());
      const int32_t n_cmp = ls.n_cmp_terms;
      #pragma unroll 4
      for (int q = 0; q < n_cmp; q++) {
        const LeanTerm lt = ls.terms[q];
        bool has;
        const int32_t c = lean_term_count(r4, smem_cnt, lt, has);
        ok &= has ? (c <= lt.lim + ms.relax[q]) : (lt.miss_rejects == 0);     // (relax > 0: closed cells close to reopening publish their nodes as dormant candidates)
      }
      if (ok) {
        if (sc < 0) sc = lean_rescore(t, lp, j);
        key = ckey(sc, (uint32_t)(p.node_base + lo + j));
      }
    }
    // ---- the warp's M best keys (REDUX rounds; keys are unique, 0 = none). Sorted tile (single-use templates): none here, thread t
    //      holds rank t, and the warp's count of feasible ranks goes to ms.wfeas for the selection below (its instantiation keeps
    //      this loop for a device that finds the template is not single use; "sorted" goes into the ballot, not into a branch
    //      around the loop: a trip count from a ballot is warp-uniform to the compiler, which then puts no divergence check in
    //      front of every REDUX) ----
    const unsigned fm = __ballot_sync(0xffffffffu, key != 0u);
    {
      uint32_t rem = key;
      bool has = key != 0u;
      if constexpr (SORTED) has = has && !tile_sel;
      const int nf = __popc(SORTED ? __ballot_sync(0xffffffffu, has) : fm);
      if (lane == 0) ms.wfeas[warp] = __popc(fm);
      if (lane >= nf && lane < MULTI_M) ms.wtop[warp][lane] = 0u;
      // (warp-uniform trip count: no REDUX rounds for entries that do not exist; not unrolled — sixteen predicated REDUX
      //  in a row run out of uniform registers and spill)
      const int nr = min(nf, MULTI_M);
      #pragma unroll 1
      for (int r = 0; r < nr; r++) {
        const uint32_t v = __reduce_max_sync(0xffffffffu, rem);
        if (rem == v) rem = 0u;
        if (lane == 0) ms.wtop[warp][r] = v;
      }
    }
    MPH_MARK(0);
    __syncthreads();                                                    // S1
    MPH_MARK(1);
    const unsigned long long tagbits = (unsigned long long)tag << KEY_TAG_SHIFT;
    const int par = (int)(wv & 1);
    // two lines of 16 tagged words: line 0 [0] key 0  [1] key 15 | more-bit  [2..15] keys 1..14, line 1 [0..15] payloads 0..15 —
    // a poller reads words 0-1 of line 0 in one 16-byte load: the list's best key and its last key (with "this tile has more
    // feasible nodes"). (Node shards too: the lines stay on this GPU; what crosses NVLink is one summary per rank, below.)
    bool merge = warp == 0;
    if constexpr (SORTED) {
      if (tile_sel) {
        // ---- the CTA's M best from the sorted tile: its first M non-zero keys in rank order. Thread t holds rank t; its rank among
        //      the feasible nodes is the feasible nodes of the warps before it plus those of the lanes before it (one count per warp,
        //      barrier S1). The threads of ranks < M write their entries, threads tid < M past the last one the empty entries: the
        //      same words as the merge below. ----
        const int32_t nfw = lane < LEAN_WARPS ? ms.wfeas[lane] : 0;
        const int32_t total = __reduce_add_sync(0xffffffffu, nfw);
        const int r = __reduce_add_sync(0xffffffffu, lane < warp ? nfw : 0) + __popc(fm & ((1u << lane) - 1u));
        unsigned long long *myslots = p.slots + ((size_t)par * CCSIM_MAX_GRID + cta) * MULTI_LINE_WORDS;
        if (key != 0u && r < MULTI_M) {
          unsigned long long kw = (unsigned long long)key;
          if (r == MULTI_M - 1 && total > MULTI_M) kw |= 1ull << MULTI_MORE_BIT;
          st_slot(&myslots[multi_kpos(r)], kw | tagbits);
          st_slot(&myslots[SLOT_STRIDE + r], (unsigned long long)kpay | tagbits);
        }
        if (tid < MULTI_M && tid >= total) {
          st_slot(&myslots[multi_kpos(tid)], tagbits);
          st_slot(&myslots[SLOT_STRIDE + tid], tagbits);
        }
        if (cta == 0 && tid == 0) ms.st_tile_sel++;
      }
      merge = merge && !tile_sel;
    }
    if (merge) {
      // ---- the CTA's M best: merge of the 24 sorted warp lists (lane w walks warp w's list), then publish the pairs ----
      int32_t total = lane < LEAN_WARPS ? ms.wfeas[lane] : 0;
      total = __reduce_add_sync(0xffffffffu, total);
      int ptr = 0, L = 0;
      uint32_t mykey = 0u;
      uint32_t head = lane < LEAN_WARPS ? ms.wtop[lane][0] : 0u;
      uint32_t nxt = lane < LEAN_WARPS ? ms.wtop[lane][1] : 0u;     // (prefetched: the shared-memory load stays off the REDUX chain)
      for (int r = 0; r < MULTI_M; r++) {
        const uint32_t g = __reduce_max_sync(0xffffffffu, head);
        if (g == 0u) break;                    // uniform
        if (head == g) { ptr++; head = nxt; nxt = ptr + 1 < MULTI_M ? ms.wtop[lane][ptr + 1] : 0u; }
        if (lane == r) mykey = g;
        L = r + 1;
      }
      unsigned long long pay = 0ull;
      if (lane < L) {
        const int32_t jj = ckey_index(mykey) - (p.node_base + lo);
        pay = c_pay[jj];
        // The node's key after one more clone ("second life" in the replay): the node-local part of the Filter pass and the
        // score again, on the row as it would be after this commit (types.go:409-427). Per-domain terms are re-checked by
        // the replay itself. 0 = the node would not take another clone.
        if (!ms.single_use) {    // (a clone that blocks its own node — hostname anti-affinity — never has a second life)
        const int32_t *r4 = lean_rec4(t, lp, jj);
        const LeanRow w = lean_row(reinterpret_cast<const uint4 *>(r4));
        bool ok2 = (w.free_cpu - ls.tmpl.req_cpu >= ls.eq_cpu) & (w.free_mem - ls.tmpl.req_mem >= ls.eq_mem) & (w.free_pods - 1 >= ls.pods_need);
        for (int q = 0; q < ls.n_cmp_terms; q++) {
          const LeanTerm lt = ls.terms[q];
          if (lt.cnt_off >= 0) continue;                       // replicated counters: the replay's business
          int inc = 0;
          for (int j = 0; j < p.n_counters; j++) if (p.counters[j].topo_col < 0 && LR_SLOT0 + lp.counter_slot[j] == lt.slot) inc = ls.cinfo[j].inc;
          ok2 &= (r4[lt.slot] + inc <= lt.lim);
        }
        if (ok2) {
          const int32_t sc2 = score_node(t.acpu[jj], t.amem[jj], t.zcpu[jj] + ls.tmpl.nz_cpu + ls.tmpl.least_cpu, t.zmem[jj] + ls.tmpl.nz_mem + ls.tmpl.least_mem,
                                         t.rcpu[jj] + ls.tmpl.req_cpu + ls.tmpl.bal_cpu, t.rmem[jj] + ls.tmpl.req_mem + ls.tmpl.bal_mem, ls.sw);
          pay |= (unsigned long long)(uint32_t)(sc2 + 1) << MULTI_NEXT_SHIFT;
        }
        }
      }
      unsigned long long kw = (unsigned long long)mykey;
      if (lane == MULTI_M - 1 && total > L) kw |= 1ull << MULTI_MORE_BIT;
      const int kpos = multi_kpos(lane);
      {
        unsigned long long *myslots = p.slots + ((size_t)par * CCSIM_MAX_GRID + cta) * MULTI_LINE_WORDS;
        if (lane < MULTI_M) {
          st_slot(&myslots[kpos], kw | tagbits);
          st_slot(&myslots[SLOT_STRIDE + lane], pay | tagbits);
        }
      }
    }
    GPROF(if (tid == 0) { if (cta == 0) ms.gp_pub = clock64(); if (wv < GP_MAX_WAVES) gp_pub_ns[wv * CCSIM_MAX_GRID + cta] = globaltimer_ns(); })
    MPH_MARK(2);
    // ---- gather, level 1: the lines of THIS GPU's CTAs. Every thread waits for its own (<= MULTI_EPT) entries — key word and payload
    //      word — so that the bar and the entries cost ONE L2 round trip after the slowest CTA's lines land ----
    const unsigned long long *lbase = p.slots + (size_t)par * CCSIM_MAX_GRID * MULTI_LINE_WORDS;
    uint32_t tloc = 0u, kloc = 0u;
    unsigned long long ea[MULTI_EPT], eb[MULTI_EPT];
    {
      unsigned need = 0u;                      // bit u: entry u of this thread has not arrived yet
      #pragma unroll
      for (int u = 0; u < MULTI_EPT; u++) { ea[u] = eb[u] = 0ull; need |= (unsigned)(tid + u * LEAN_THREADS < tot) << u; }
      unsigned spins = 0;
      while (need) {
        #pragma unroll
        for (int u = 0; u < MULTI_EPT; u++)
          if ((need >> u) & 1u) {
            const int e = tid + u * LEAN_THREADS, ee = e & (MULTI_M - 1);
            const unsigned long long *ln = lbase + (size_t)(e / MULTI_M) * MULTI_LINE_WORDS;
            ea[u] = ld_slot(ln + (ee == 0 ? 0 : (ee == MULTI_M - 1 ? 1 : ee + 1)));
            eb[u] = ld_slot(ln + SLOT_STRIDE + ee);
          }
        #pragma unroll
        for (int u = 0; u < MULTI_EPT; u++)
          if ((uint32_t)(ea[u] >> KEY_TAG_SHIFT) == tag && (uint32_t)(eb[u] >> KEY_TAG_SHIFT) == tag) need &= ~(1u << u);
        if (++spins > WATCHDOG_SPINS) {
          ms.dead = 1;
          #pragma unroll
          for (int u = 0; u < MULTI_EPT; u++) if ((need >> u) & 1u) ea[u] = eb[u] = 0ull;
          break;
        }
      }
      GPROF(if (cta == 0) { atomicMax(&ms.gp_valid, (unsigned long long)clock64()); atomicMax(&ms.gp_spins, (unsigned long long)spins); })
      #pragma unroll
      for (int u = 0; u < MULTI_EPT; u++) {
        const int e = tid + u * LEAN_THREADS, ee = e & (MULTI_M - 1);
        if (e < tot) {
          if (ee == 0) kloc = max(kloc, (uint32_t)ea[u]);
          if (ee == MULTI_M - 1 && ((ea[u] >> MULTI_MORE_BIT) & 1ull)) tloc = max(tloc, (uint32_t)ea[u]);
        }
      }
    }
    tloc = __reduce_max_sync(0xffffffffu, tloc);
    kloc = __reduce_max_sync(0xffffffffu, kloc);
    if (lane == 0) { ms.red[warp] = tloc; ms.red2[warp] = kloc; }
    __syncthreads();                                                    // G1 (also: ms.dead)
    uint32_t Tlist = __reduce_max_sync(0xffffffffu, lane < LEAN_WARPS ? ms.red[lane] : 0u);
    uint32_t kbest = __reduce_max_sync(0xffffffffu, lane < LEAN_WARPS ? ms.red2[lane] : 0u);
    bool dead = ms.dead != 0;
    GPROF(if (cta == 0 && tid == 0) {
            ms.gp_cyc[GP_POLL] += (long long)ms.gp_valid - ms.gp_pub; ms.gp_cyc[GP_SYNC] += clock64() - (long long)ms.gp_valid;
            ms.gp_cnt[GP_ROUNDS] += (long long)ms.gp_spins; ms.gp_valid = ms.gp_spins = 0ull;
          })
    // The replay bar: T = the largest "last key" of a list whose tile has unseen feasible nodes is the lowest VALID bar; any
    // higher bar is valid too, just more conservative. The replay holds MULTI_CAP candidates, and it rarely needs more than the
    // best few dozen before a PTS minimum moves, so the bar is set `delta` below the best key (never below T); delta follows the
    // previous waves (doubled when the replay ran out of candidates above an artificial bar, shrunk when too many qualified).
    // Every CTA of every rank computes the same sequence from the same exchanged data.
    uint32_t T = max(Tlist, kbest > delta ? kbest - delta : 0u);
    // ---- the entries keyed >= T into shared memory in key order. Every list is sorted (keys descending, then zeros), and list l is
    //      tile l: a lower list holds lower node indices, which rank higher at the same score. So the concatenated lists are in key
    //      order within every score level ----
    int C = 0;
    bool over = false;        // a gather level had more than MULTI_CAP candidates: the wave counts once in bar_raised_waves
    if (!dead) C = multi_compact(ea, eb, T, kbest, cta, over);
    if (XGPU) {
      // ---- gather, level 2 (node shards): every rank now holds ITS candidates keyed >= its bar T_r (<= MULTI_CAP of them, the same in
      //      all of its CTAs). One summary per (source, destination) pair crosses NVLink — {best key, count, T_r, T_list_r, the
      //      candidates} written by ONE CTA of the source as a few 128-byte stores — instead of every CTA's line going to every
      //      rank and world x grid lines being polled by every CTA. The global bar max(max_r T_r, best - delta) is at least every
      //      rank's own bar, so the union of the summaries holds every node keyed above it: same candidates as one GPU would see.
      //      The summaries concatenated in rank order are in key order within every score level, as the lists are at level 1: each
      //      summary is in key order, and rank r holds the nodes [per * r, per * (r + 1)), which rank higher than rank r + 1's at the
      //      same score. So the same compaction ranks their union. ----
      const int xpar = (int)((wv + p.xwave0) & 1);
      if (!dead)
        for (int d = cta; d < p.world; d += p.grid) {            // CTA d of the source writes the copy for rank d
          if (d == p.rank) continue;
          unsigned long long *dst = p.xslots_peer[d] + XLINES_OFF + ((size_t)xpar * CCSIM_MAX_WORLD + p.rank) * CCSIM_MAX_GRID * SLOT_STRIDE;
          if (tid < 4 + 2 * C) {
            unsigned long long v;
            if (tid == 0) v = (unsigned long long)kbest | ((unsigned long long)C << 32);
            else if (tid == 1) v = T;
            else if (tid == 2) v = Tlist;
            else if (tid == 3) v = 0ull;
            else { const int ci = (tid - 4) >> 1; v = (tid & 1) ? ((unsigned long long)ms.cdom[ci] | ((unsigned long long)ms.cnext[ci] << MULTI_NEXT_SHIFT)) : (unsigned long long)ms.ckey[ci]; }
            st_slot_sys(dst + tid, v | tagbits);
          }
        }
      uint32_t xkb = kbest, xtl = Tlist, xbar = T;
      if (tid < p.world) {
        int cr = C;
        if (tid != p.rank && !dead) {
          unsigned long long h[3];
          multi_poll_sys(p.xslots_peer[p.rank] + XLINES_OFF + ((size_t)xpar * CCSIM_MAX_WORLD + tid) * CCSIM_MAX_GRID * SLOT_STRIDE, tag, h);
          xkb = (uint32_t)h[0]; cr = (int)((h[0] >> 32) & 0xfffu); xbar = (uint32_t)h[1]; xtl = (uint32_t)h[2];
          if (cr > MULTI_CAP) cr = MULTI_CAP;
        }
        ms.xcount[tid] = cr;
      }
      if (warp == 0) {       // (world <= 32: the pollers are lanes of warp 0; the other lanes carry this rank's own values)
        xkb = __reduce_max_sync(0xffffffffu, xkb); xtl = __reduce_max_sync(0xffffffffu, xtl); xbar = __reduce_max_sync(0xffffffffu, xbar);
        if (lane == 0) { ms.xglob[0] = xkb; ms.xglob[1] = xtl; ms.xglob[2] = xbar; }
      }
      __syncthreads();                                                  // X1
      dead = ms.dead != 0;
      kbest = ms.xglob[0]; Tlist = ms.xglob[1];
      T = max(ms.xglob[2], kbest > delta ? kbest - delta : 0u);
      C = 0;
      if (!dead) {
        // entry e of the concatenated summaries -> (rank, index). This rank's own segment comes from the candidate arrays, which the
        // compaction stores over after its first barrier only.
        #pragma unroll
        for (int u = 0; u < MULTI_EPT; u++) {
          ea[u] = eb[u] = 0ull;
          int e = tid + u * LEAN_THREADS, r = 0;
          while (r < p.world && e >= ms.xcount[r]) { e -= ms.xcount[r]; r++; }
          if (r == p.rank) {
            ea[u] = ms.ckey[e];
            eb[u] = (unsigned long long)ms.cdom[e] | ((unsigned long long)ms.cnext[e] << MULTI_NEXT_SHIFT);
          } else if (r < p.world) {
            unsigned long long w[2];
            multi_poll_sys(p.xslots_peer[p.rank] + XLINES_OFF + ((size_t)xpar * CCSIM_MAX_WORLD + r) * CCSIM_MAX_GRID * SLOT_STRIDE + 4 + 2 * e, tag, w);
            ea[u] = w[0]; eb[u] = w[1];
          }
        }
        C = multi_compact(ea, eb, T, kbest, cta, over);
      }
      dead = dead || ms.dead != 0;
    }
    const bool overflowed = T > max(Tlist, kbest > delta ? kbest - delta : 0u);
    if (cta == 0 && tid == 0) { ms.st_cand += C; if (over) ms.st_overflow++; }
    MPH_MARK(3);
    // ---- key order (single-use templates): no candidate comes back after it wins, so its key stands for the whole wave and the
    //      winner of every round is the first live candidate in key order, the order the compaction stored them in.
    //      CCSIM_DEBUG_FLAGS bit 6 keeps the arg-max round. ----
    const bool key_order = ms.single_use != 0 && !(p.debug_flags & DBG_ARGMAX_ROUND) && !dead;     // (block-uniform)
    // ---- replay: the reference cycles k, k+1, ... this wave can decide; every CTA does the same, in ONE warp and without a
    //      barrier: MULTI_CPT candidates per lane in registers, lane q < n_gt also owns counter term q (its constants, and the
    //      minimum / multiplicity of the PTS constraint it tracks, stay in registers for the whole wave) ----
    if (warp == 0) {
      int32_t acc = 0;
      bool ran_dry = false, any_relax = false;
      if (!dead && !ms.dead) {
        const int n_gt = ms.n_gt;
        uint32_t ck[MULTI_CPT], cd[MULTI_CPT];
        uint32_t second = 0u;
        #pragma unroll
        for (int j = 0; j < MULTI_CPT; j++) {
          const int idx = j * 32 + lane;
          ck[j] = 0u; cd[j] = 0u;
          if (idx < C && !key_order) { ck[j] = ms.ckey[idx]; cd[j] = ms.cdom[idx]; }
        }
        int4 gc = make_int4(0, 0, -1, 0), c1 = make_int4(0, 0, 0, 0);
        int32_t my_min = 0, my_num = 0;
        if (lane < n_gt) {
          gc = *reinterpret_cast<const int4 *>(&ms.gt_commit[lane][0]);   // {cnt_off, inc, pts_idx, n_present}
          c1 = *reinterpret_cast<const int4 *>(&ms.gt_c1[lane][0]);       // {lim, shift, mask, n_domains}
          if (gc.z >= 0) { my_min = ls.ptsmin[gc.z]; my_num = ls.ptsnum[gc.z]; }
        }
        // the kill test's constants: the lowest bit of every term's payload field, and the guard bit right above it (the host
        // leaves it zero in every payload)
        uint32_t flsb = 0u, fguard = 0u;
        #pragma unroll
        for (int q = 0; q < MULTI_GT; q++)
          if (q < n_gt) { flsb |= 1u << ms.gt_c1[q][1]; fguard |= ((uint32_t)ms.gt_c1[q][2] + 1u) << ms.gt_c1[q][1]; }
        RPROF(__syncwarp(); RP_ADD(RP_LOAD, clock64() - ms.tc0, 1);)
        const int32_t lim_off = c1.x - my_min;       // PTS: maxSkew - selfMatch (the limit follows the global minimum)
        bool lim_moved = false;
        const bool single_use = ms.single_use != 0;
        // commits this wave may still decide: --max-limit (simulator.go:300-305), the output capacity, MULTI_MAX_ACC
        long long room = p.pod_cap - k;
        if (p.max_pods > 0 && p.max_pods - k < room) room = p.max_pods - k;
        // (pinned: recomputing it from the kernel parameters inside the round costs two constant loads and a 64-bit compare)
        const int32_t acc_limit = (int32_t)pin_u32(room < MULTI_MAX_ACC ? (uint32_t)room : (uint32_t)MULTI_MAX_ACC);
        bool ended_by_rescan = false;
        // the round's per-lane constants: this lane's term field in the payload, in place, and its guard bit; whether the term
        // tracks a PTS minimum; the lowest key that may still win (0 never does)
        const uint32_t fmask = (uint32_t)c1.z << c1.y, fglane = ((uint32_t)c1.z + 1u) << c1.y;
        const bool trk = (gc.y != 0) & (gc.z >= 0);
        const uint32_t Tr = T > 1u ? T : 1u;
        const uint32_t cnext_sa = pin_u32(MS_SA(cnext) + 4u * (uint32_t)lane);   // this lane's column of the second-life keys
        // ---- dormant candidates. A PTS term whose limit is about to move (few domains left at the global minimum) was scanned with
        //      a look-ahead (ms.relax): nodes in cells up to MULTI_RELAX_R over the limit are in the lists too. They cannot win while
        //      their cell is over the limit (dormant: key 0 in ck[], like a dead candidate) and wake up when a minimum move lifts the
        //      limit over their cell — the wave then goes on instead of ending for a rescan. It still has to end when the limit
        //      reaches a cell that was NOT published: `unpub_min` = the smallest count above limit + look-ahead at the start of the
        //      wave (such cells are closed, so their counts stand for the whole wave).
        //      The dormant candidates of a look-ahead wave are found at set-up by reading the look-ahead terms' cells only: the scan
        //      held every other term to its limit, and no commit has happened since. The round loop itself is unchanged: a candidate
        //      whose cell fills is zeroed as before. Waking is a REBUILD (after a minimum move of a look-ahead term): every slot's key
        //      is read again from the wave's candidate arrays — first-life key, or second-life key when bit j of `second` says the
        //      slot has won already (single-use templates: gone) — and zeroed when one of its cells is over the limit as counters and
        //      limits stand now. ----
        int32_t rlx = 0, unpub_min = INT32_MAX;
        if (lane < n_gt) rlx = lds_s32(MS_SA(relax) + 4u * (uint32_t)lds_s32(MS_SA(gt_term) + 4u * (uint32_t)lane));
        any_relax = __any_sync(0xffffffffu, rlx > 0);
        bool need_rebuild = false;
        if (any_relax) {
          for (unsigned nm = __ballot_sync(0xffffffffu, rlx > 0); nm; nm &= nm - 1) {
            const int q = __ffs(nm) - 1;
            const int32_t off = __shfl_sync(0xffffffffu, gc.x, q), ndom = __shfl_sync(0xffffffffu, c1.w, q), lim = __shfl_sync(0xffffffffu, c1.x, q);
            const uint32_t sh = (uint32_t)__shfl_sync(0xffffffffu, c1.y, q), mk = (uint32_t)__shfl_sync(0xffffffffu, c1.z, q);
            const int32_t publim = __shfl_sync(0xffffffffu, c1.x + rlx, q);
            const uint32_t ca = cnt_sa + 4u * (uint32_t)off;
            int32_t m = INT32_MAX;
            #pragma unroll 1
            for (int d = lane; d < ndom; d += 32) { const int32_t c = lds_s32(ca + 4u * d); if (c > publim) m = min(m, c); }
            // this term's dormant candidates (key order: the full cell test of each row when it is loaded finds them)
            #pragma unroll
            for (int j = 0; j < MULTI_CPT; j++) if (!key_order) {
              const uint32_t f = (cd[j] >> sh) & mk;           // dom + 1 (0: no domain; cell 0 is read and ignored)
              const int32_t c = lds_s32(ca + 4u * (uint32_t)max((int32_t)f - 1, 0));
              if ((f != 0u) & (c > lim)) ck[j] = 0u;
            }
            m = __reduce_min_sync(0xffffffffu, m);
            if (lane == q) unpub_min = m;
          }
          if (cta == 0 && lane == 0) ms.st_relaxed++;
        }
        // ---- commit pod k+acc, whose node's payload is `pay` (assume -> AssumePod -> NodeInfo.update(+1): schedule_one.go:967-984,
        //      types.go:409-427). Only what the next round depends on happens here: the counter cells of the winner's domains (lane
        //      q = term q; the host guarantees one term per incremented replicated counter), whether a cell went over its limit,
        //      whether a PTS minimum moved. The winner's row (NodeInfo.update, node-local counters) is brought up to date by its own
        //      thread after the wave. Returns the OR of the filled cells, with "a minimum moved" in bit 31. ----
        auto commit = [&](const uint32_t pay, bool &rescan, bool &woke RPROF(, long long &rp_mm)) -> uint32_t {
          // (lanes >= n_gt have a zero field mask: no domain, nothing written)
          const uint32_t fpay = pay & fmask;                     // the winner's field of this lane's term, in place
          const bool has = fpay != 0u;
          const uint32_t ca = cnt_sa + 4u * (uint32_t)(gc.x + max((int32_t)(fpay >> c1.y) - 1, 0));
          const int32_t old = lds_s32(ca), nv = old + gc.y;
          if (has) sts_s32(ca, nv);
          // candidates in a cell that went over its limit are dead from now on: its field, with the field's guard bit
          const uint32_t fullf = (has & (nv > c1.x)) ? (fpay | fglane) : 0u;
          const bool atmin = has & trk & ((int32_t)(fpay >> c1.y) - 1 < gc.w) & (old == my_min);   // a domain leaves the global minimum ...
          my_num -= (int32_t)atmin;
          const bool minchg = atmin & (my_num <= 0);                                                  // ... the last one: the minimum moves
          // one OR-reduction carries the filled cells (the fields of different terms are disjoint bit ranges) and, in bit 31, that
          // some term's minimum moved
          const uint32_t F = __reduce_or_sync(0xffffffffu, fullf | ((uint32_t)minchg << 31));
          // A PTS minimum moved (filtering.go:56-69: minMatchNum): recount it and move the term's limit. The wave goes on unless
          // the move changes some node's feasibility: that takes a domain whose count lies in (old limit, new limit] — nodes there
          // were rejected by the scan (or killed earlier in this wave) and pass now. Without such a domain every verdict so far
          // stands (the 8-region constraint of C4 moves its minimum every 8 placements and never binds).
          const unsigned mc = (F >> 31) ? __ballot_sync(0xffffffffu, minchg) : 0u;
          for (unsigned nm = mc; nm; nm &= nm - 1) {
            RPROF(const long long rp_m0 = clock64();)
            const int q = __ffs(nm) - 1;
            const int32_t off = __shfl_sync(0xffffffffu, gc.x, q), npres = __shfl_sync(0xffffffffu, gc.w, q), ndom = __shfl_sync(0xffffffffu, c1.w, q);
            const int32_t lim_old = __shfl_sync(0xffffffffu, c1.x, q), loff = __shfl_sync(0xffffffffu, lim_off, q);
            const uint32_t ca = cnt_sa + 4u * (uint32_t)off;
            // one pass over the cells (one per lane for a term of <= 32 domains): this lane's minimum over the present domains and
            // how many sit at it, and its lowest count over the old limit — the move changes verdicts iff that one is <= the new limit
            int32_t mn = INT32_MAX, num = 0, up = INT32_MAX;
            #pragma unroll 1
            for (int d = lane; d < ndom; d += 32) {
              const int32_t c = lds_s32(ca + 4u * d);
              if (c > lim_old) up = min(up, c);
              if (d < npres) { num = c < mn ? 0 : num; mn = min(mn, c); num += c == mn; }
            }
            const int32_t lmn = mn;
            mn = __reduce_min_sync(0xffffffffu, mn);
            up = __reduce_min_sync(0xffffffffu, up);
            num = __reduce_add_sync(0xffffffffu, lmn == mn ? num : 0);
            const long long liml = (long long)loff + (long long)mn;
            const int32_t lim_new = liml > INT32_MAX ? INT32_MAX : (liml < INT32_MIN ? INT32_MIN : (int32_t)liml);
            const bool hit = up <= lim_new;
            // a term scanned with look-ahead published the nodes of its closed cells: the move only matters when the new limit
            // reaches a cell that was not published; the cells in (old limit, new limit] wake their candidates up instead
            const bool rq = __shfl_sync(0xffffffffu, rlx, q) > 0;
            if (rq) { rescan |= (lim_new >= __shfl_sync(0xffffffffu, unpub_min, q)) | (p.debug_flags & DBG_RESCAN_EVERY_MOVE); woke = true; }
            else rescan |= hit | (p.debug_flags & DBG_RESCAN_EVERY_MOVE);
            if (lane == q) { my_min = mn; my_num = num; c1.x = lim_new; lim_moved = true; sts_s32(MS_SA(gt_c1) + 16u * (uint32_t)q, lim_new); }
            RPROF(__syncwarp(); const long long rp_m1 = clock64(); RP_ADD(RP_MINMOVE + q, rp_m1 - rp_m0, 1); rp_mm += rp_m1 - rp_m0;)
          }
          return F;
        };
        if (cta == 0 && lane == 0) ms.ph[6] += clock64() - ms.tc0;      // replay set-up
        // ---- the round in key order (single-use waves). Lane l holds the candidate of rank 32 * row + l: its payload, its key, and
        //      whether it is live. At the start of every round a candidate is live iff it has not won in this wave and, for every
        //      term with a field in its payload, its cell count is <= the term's current limit: the scan held every term but the
        //      look-ahead ones to its limit, counts only grow, a kill follows every cell that goes over, a minimum move that does
        //      not end the wave leaves no cell in (old limit, new limit] unless it wakes candidates up, and a won candidate never
        //      comes back (single use). So a row is judged when the replay reaches it, by one full cell test against the counters
        //      and limits as they stand; a wake-up sends the replay back to row 0 (rows above may hold revived candidates; the won
        //      bits keep winners out). The winner is the lowest live lane of the first row that has one: a ballot instead of the
        //      arg-max, one shuffle for its payload, a kill test on one slot. Every compacted candidate is keyed >= T, so "no live
        //      candidate left" is the arg-max round's `g < Tr`. ----
        if (key_order) {
          const int nrows = (C + 31) >> 5;
          int row = 0;
          uint32_t won = 0u;                   // bit r: this lane's candidate of row r has won
          uint32_t kd = 0u, kk = 0u;           // its payload and key
          bool live = false;
          auto load_row = [&]() {
            __syncwarp();                      // the counter cells / limits written by the term lanes, before every lane reads them
            const int idx = row * 32 + lane;
            const bool present = idx < C;
            kk = present ? (uint32_t)lds_s32(MS_SA(ckey) + 4u * (uint32_t)idx) : 0u;
            kd = present ? (uint32_t)lds_s32(MS_SA(cdom) + 4u * (uint32_t)idx) : 0u;   // (0: no field, every cell read is cell 0 of its counter)
            // the full cell test. The term constants come from the term lanes' registers (lane q holds term q's current limit;
            // lanes >= n_gt hold zeros: no field, cell 0 of the first counter), so nothing here branches and every load is
            // issued before its first use.
            uint32_t f[MULTI_GT];
            int32_t cv[MULTI_GT], lim[MULTI_GT];
            #pragma unroll
            for (int q = 0; q < MULTI_GT; q++) {
              const int32_t off = __shfl_sync(0xffffffffu, gc.x, q);
              const uint32_t sh = (uint32_t)__shfl_sync(0xffffffffu, c1.y, q), mk = (uint32_t)__shfl_sync(0xffffffffu, c1.z, q);
              lim[q] = __shfl_sync(0xffffffffu, c1.x, q);
              f[q] = (kd >> sh) & mk;                                                  // dom + 1 (0: no domain; cell 0 is read and ignored)
              cv[q] = lds_s32(cnt_sa + 4u * (uint32_t)(off + max((int32_t)f[q] - 1, 0)));
            }
            bool bad = false;
            #pragma unroll
            for (int q = 0; q < MULTI_GT; q++) bad |= (f[q] != 0u) & (cv[q] > lim[q]);
            live = present & !bad & !((won >> row) & 1u);
          };
          load_row();
          if (cta == 0 && lane == 0) ms.st_key_order++;
          for (;;) {
            RPROF(long long rp_t0 = clock64(), rp_mm = 0;)
            unsigned lv = __ballot_sync(0xffffffffu, live);
            if (lv == 0u) {                    // the row is used up: the next one, judged as counters and limits stand now
              RPROF(int rp_n = 0;)
              while (lv == 0u && ++row < nrows) { load_row(); lv = __ballot_sync(0xffffffffu, live); RPROF(rp_n++;) }
              RPROF(const long long rp_a1 = clock64(); RP_ADD(RP_ADVANCE, rp_a1 - rp_t0, rp_n); rp_t0 = rp_a1;)
              if (lv == 0u) { ran_dry = true; RP_ADD(RP_KROUND, clock64() - rp_t0, 1); break; }
            }
            const int w = __ffs(lv) - 1;
            const uint32_t pay = __shfl_sync(0xffffffffu, kd, w);
            if (lane == w) { live = false; won |= 1u << row; sts_s32(MS_SA(acc_node) + 4u * (uint32_t)acc, ckey_index(kk)); }
            acc++;
            bool rescan = false, woke = false;
            const uint32_t F = commit(pay, rescan, woke RPROF(, rp_mm));
            if (rescan | (acc >= acc_limit)) { ended_by_rescan = rescan; RP_ADD(RP_KROUND, clock64() - rp_t0 - rp_mm, 1); break; }
            if (woke) {
              RPROF(const long long rp_w0 = clock64();)
              row = 0;
              load_row();
              RPROF(const long long rp_w1 = clock64(); RP_ADD(RP_REBUILD, rp_w1 - rp_w0, 1); rp_mm += rp_w1 - rp_w0;)
            } else {
              // the single-slot form of the SWAR kill test below (only this row can hold live candidates)
              const uint32_t Fc = F & ((1u << MULTI_PAY_BITS) - 1u);
              if (Fc) {
                const uint32_t fv = Fc & ~fguard, fg = Fc & fguard;
                if (~(((kd ^ fv) | fguard) - flsb) & fg) live = false;
                RP_ADD(RP_KILL, 0, 1);
              }
            }
            RP_ADD(RP_KROUND, clock64() - rp_t0 - rp_mm, 1);
          }
        } else for (;;) {                      // ---- the arg-max round: second lives, and CCSIM_DEBUG_FLAGS bit 6 ----
          RPROF(long long rp_t0 = clock64(), rp_mm = 0;)
          if (need_rebuild) {       // (one call site, off the round's critical path; see "dormant candidates")
            need_rebuild = false;
            __syncwarp();           // the counter cells / limits written by the term lanes, before every lane reads them
            // (every load of a pass is issued before its first use, and none sits behind a branch: the loads overlap)
            uint32_t badm = 0u;
            #pragma unroll 1
            for (int q = 0; q < n_gt; q++) {
              const int4 tg = *reinterpret_cast<const int4 *>(&ms.gt_commit[q][0]);   // {cnt_off, inc, pts_idx, n_present}
              const int4 tc = *reinterpret_cast<const int4 *>(&ms.gt_c1[q][0]);       // {lim (kept current by lane q), shift, mask, n_domains}
              int32_t cv[MULTI_CPT];
              #pragma unroll
              for (int j = 0; j < MULTI_CPT; j++) {
                const int32_t v = (int32_t)((cd[j] >> tc.y) & (uint32_t)tc.z) - 1;   // (-1: no domain; cell 0 is read and ignored)
                cv[j] = lds_s32(cnt_sa + 4u * (uint32_t)(tg.x + max(v, 0)));
              }
              #pragma unroll
              for (int j = 0; j < MULTI_CPT; j++) {
                const bool has = ((cd[j] >> tc.y) & (uint32_t)tc.z) != 0u;
                badm |= (uint32_t)(has & (cv[j] > tc.x)) << j;
              }
            }
            uint32_t k0[MULTI_CPT], k1[MULTI_CPT];
            #pragma unroll
            for (int j = 0; j < MULTI_CPT; j++) {   // (j * 32 + lane < MULTI_CAP: in bounds; slots >= C are ignored below)
              k0[j] = (uint32_t)lds_s32(MS_SA(ckey) + 4u * (uint32_t)(j * 32 + lane));
              k1[j] = (uint32_t)lds_s32(MS_SA(cnext) + 4u * (uint32_t)(j * 32 + lane));
            }
            #pragma unroll
            for (int j = 0; j < MULTI_CPT; j++) {
              const uint32_t life2 = (single_use || k1[j] == 0u) ? 0u : ((k1[j] << MULTI_IDX_BITS) | (k0[j] & MULTI_IDX_MASK));
              const uint32_t base = ((second >> j) & 1u) ? life2 : k0[j];
              ck[j] = (j * 32 + lane < C && !((badm >> j) & 1u)) ? base : 0u;
            }
            RPROF(const long long rp_t1 = clock64(); RP_ADD(RP_REBUILD, rp_t1 - rp_t0, 1); rp_t0 = rp_t1;)
          }
          // ---- the round: only its dependent chain — arg-max (REDUX) -> owner's payload (REDUX) -> counter cells (LDS/STS) -> filled
          //      cells and "a minimum moved" (REDUX) -> kill. No branch is divergent on the common path: every lane runs the same code
          //      and predication selects; the work that does not depend on the arg-max (the lane's best slot, its payload, its
          //      next-life key) overlaps the REDUX. ----
          uint32_t m = ck[0];
          #pragma unroll
          for (int j = 1; j < MULTI_CPT; j++) m = max(m, ck[j]);
          const uint32_t g = __reduce_max_sync(0xffffffffu, m);     // (issued first: what follows up to the test of g fills its latency)
          // this lane's best slot: its payload, with the slot index in bits 27..29 and "this slot has won before" in bit 31 (keys are
          // unique, so when m != 0 exactly one slot matches; when m == 0 the lane is not the owner and the value is not used)
          uint32_t pm = 0u;
          #pragma unroll
          for (int j = 0; j < MULTI_CPT; j++)
            pm |= (ck[j] == m) ? (cd[j] | ((uint32_t)j << MULTI_PAY_BITS) | (((second >> j) & 1u) << 31)) : 0u;
          const uint32_t ns = (uint32_t)lds_s32(cnext_sa + 128u * ((pm >> MULTI_PAY_BITS) & 7u));   // (read ahead: used after the next REDUX)
          if (g < Tr) { ran_dry = true; RP_ADD(RP_ROUND, clock64() - rp_t0, 1); break; }      // nothing left (g == 0), or an unseen node could rank above g
          // ---- commit pod k+acc (assume -> AssumePod -> NodeInfo.update(+1): schedule_one.go:967-984, types.go:409-427) ----
          // the owner lane contributes the winner's payload (keys are unique: exactly one lane and slot match)
          const uint32_t pay = __reduce_or_sync(0xffffffffu, m == g ? pm : 0u);
          // the key the winning slot has after the win: its second life, or 0 (single-use template, second win, or the node takes
          // no further clone)
          const uint32_t nk = (single_use | (ns == 0u) | (pm >> 31)) ? 0u : ((ns << MULTI_IDX_BITS) | (m & MULTI_IDX_MASK));
          // the winner comes back once with the key it has after this clone (if it still fits); when a node wins for the second
          // time in a wave its third key is unknown: the wave ends after that commit (bit 31 of pay). A single-use clone blocks
          // its own node (hostname anti-affinity): the winner just leaves. Bit j of `second`: slot j has won.
          #pragma unroll
          for (int j = 0; j < MULTI_CPT; j++) ck[j] = (ck[j] == g) ? nk : ck[j];
          second |= (uint32_t)(m == g) << ((pm >> MULTI_PAY_BITS) & 7u);
          if (lane == 0) sts_s32(MS_SA(acc_node) + 4u * (uint32_t)acc, ckey_index(g));
          acc++;
          bool rescan = false, woke = false;
          const uint32_t F = commit(pay, rescan, woke RPROF(, rp_mm));
          need_rebuild = woke & !rescan;
          // (no statistics, special registers or kernel parameters are touched inside the round loop: one S2R on this dependent
          //  chain costs as much as ten ALU instructions)
          if ((pay >> 31) | rescan | (acc >= acc_limit)) { ended_by_rescan = rescan; RP_ADD(RP_ROUND, clock64() - rp_t0 - rp_mm, 1); break; }
          // only the candidates sitting in a counter cell that this commit pushed over its limit die (monotone: for the rest of
          // the wave) (the rebuild at the top of the next round sets every candidate as counters and limits stand by then —
          // `fullf` was taken against the limits before the move)
          const uint32_t Fc = woke ? 0u : (F & ((1u << MULTI_PAY_BITS) - 1u));
          if (Fc) {
            // One SWAR test per candidate instead of a compare per term: x = cd ^ (filled cells) is zero in a field exactly where
            // the candidate sits in the filled cell of that term. With every guard bit set, subtracting the fields' lowest bits
            // borrows a guard bit away exactly in the zero fields, and the guard stops the borrow there.
            const uint32_t fv = pin_u32(Fc & ~fguard), fg = Fc & fguard;
            #pragma unroll
            for (int j = 0; j < MULTI_CPT; j++)
              if (~(((cd[j] ^ fv) | fguard) - flsb) & fg) ck[j] = 0u;    // (dead — in a look-ahead wave: dormant, a rebuild may bring it back)
            RP_ADD(RP_KILL, 0, 1);
          }
          RP_ADD(RP_ROUND, clock64() - rp_t0 - rp_mm, 1);
        }
        RPROF(if (cta == 0 && lane == 0) ms.rp_t = clock64();)
        if (cta == 0 && lane == 0) { ms.st_rounds += acc + (int)ran_dry; if (ended_by_rescan) ms.ph[7] += 1; }      // (ph[7]: waves ended by a minimum move that changes verdicts)
        // the winners of this CTA's tile, handed to their threads for the row updates after barrier R (a node may be accepted
        // twice: second life). Sorted tile: a winner's record dies here, before R — no barrier separates the row updates after R
        // from the next scan, which reads the records only
        __syncwarp();
        // (read again here: `tile_sel` kept live across the replay loop changed its register allocation and cost C4 ~1 200 cycles a wave)
        const bool kill_rec = SORTED && ms.tile_sorted != 0;
        for (int i = lane; i < acc; i += 32) {
          const int32_t jw = lds_s32(MS_SA(acc_node) + 4u * (uint32_t)i) - (p.node_base + lo);
          if (jw >= 0 && jw < cnt_nodes) {
            atomicAdd(&ms.mult[jw], 1);
            if constexpr (SORTED) { if (kill_rec) multi_tile_rec[multi_tile_rank[jw]].x = 0u; }
          }
        }
        RPROF(__syncwarp(); const long long rp_h1 = clock64(); RP_ADD(RP_HANDOFF, rp_h1 - ms.rp_t, 1);)
        // ---- the next wave's look-ahead, per PTS term on a replicated counter: its limit is about to move (<= MULTI_RELAX_K present
        //      domains left at the minimum) and the closed domains are not the majority (their nodes would crowd the live ones out of
        //      the tiles' top-M lists). A look-ahead wave that could not place anything is repeated strictly. Every CTA of every rank
        //      decides alike (same counters, same replay). ----
        {
          const bool strict_next = (acc == 0 && any_relax) || (p.debug_flags & DBG_STRICT_ONLY);
          const bool elig = lane < n_gt && gc.z >= 0 && gc.y > 0 && my_num <= MULTI_RELAX_K && c1.x < INT32_MAX - 2 * MULTI_RELAX_R && !strict_next;
          int32_t nrl = 0;
          for (unsigned nm = __ballot_sync(0xffffffffu, elig); nm; nm &= nm - 1) {
            const int q = __ffs(nm) - 1;
            const int32_t off = __shfl_sync(0xffffffffu, gc.x, q), npres = __shfl_sync(0xffffffffu, gc.w, q), lim = __shfl_sync(0xffffffffu, c1.x, q);
            const uint32_t ca = cnt_sa + 4u * (uint32_t)off;
            int32_t closed = 0;
            #pragma unroll 1
            for (int d = lane; d < npres; d += 32) closed += lds_s32(ca + 4u * d) > lim;
            closed = __reduce_add_sync(0xffffffffu, closed);
            if (lane == q && 2 * closed <= npres) nrl = MULTI_RELAX_R;
          }
          if (p.debug_flags & DBG_LOOKAHEAD_ALWAYS) nrl = (lane < n_gt && gc.z >= 0 && gc.y > 0 && c1.x < INT32_MAX - 2 * MULTI_RELAX_R && !strict_next) ? MULTI_RELAX_R : 0;   // tests: look-ahead on every PTS term, every wave
          if (lane < n_gt) sts_s32(MS_SA(relax) + 4u * (uint32_t)lds_s32(MS_SA(gt_term) + 4u * (uint32_t)lane), nrl);
          // (sorted tile: the next scan's constants of this lane's term — its limit as the replay left it, and the look-ahead)
          if constexpr (SORTED) { if (lane < n_gt) multi_scan_term[lane] = make_int4(gc.x, c1.y, c1.z, c1.x + nrl); }
          if (cta == 0 && lane == 0 && acc == 0 && any_relax) ms.st_empty++;
          RPROF(__syncwarp(); RP_ADD(RP_DECIDE, clock64() - rp_h1, 1);)
        }
        // the limits that moved go back to the Filter constants of the next scan
        if (lim_moved) { ls.terms[ms.gt_term[lane]].lim = c1.x; ms.gt_c1[lane][0] = c1.x; }
        if (lane < n_gt && gc.z >= 0) { ls.ptsmin[gc.z] = my_min; ls.ptsnum[gc.z] = my_num; }
      }
      if (lane == 0 && cta == 0 && (p.debug_flags & DBG_WAVE_LINES))
        printf("wave %lld k=%lld acc=%d C=%d T=%08x Tlist=%08x kbest=%08x delta=%08x ran_dry=%d look_ahead=%d first=%d last=%d\n", wv, k, acc, C, T, Tlist, kbest, delta,
               (int)ran_dry, (int)any_relax, acc ? ms.acc_node[0] : -1, acc ? ms.acc_node[acc - 1] : -1);
      if (lane == 0) {
        ms.accepted = acc;
        // next wave's bar distance: the replay ran out of candidates above a bar that was higher than it had to be -> look further
        // down next time; far more candidates than a wave uses -> look less far
        uint32_t nd = delta;
        if (ran_dry && T > Tlist) nd = delta < (1u << 30) ? delta * 2u : delta;
        else if (overflowed) nd = max(delta / 2u, 1u << 8);
        else if (!ran_dry && C > MULTI_CAP / 2) nd = max(delta - delta / 8u, 1u << 8);
        ms.delta = nd;
        if (dead || ms.dead) ls.stop = 3;
        else if (acc == 0 && !any_relax) ls.stop = 1;          // no feasible node anywhere: the pod is unschedulable (after a look-ahead wave: rescan strictly first)
      }
    }
    __syncthreads();                                                    // R: the accepted list, counters, limits
    RPROF(if (cta == 0 && tid == 0 && ms.rp_t) { ms.rp_cyc[RP_AFTER] += clock64() - ms.rp_t; ms.rp_cnt[RP_AFTER]++; ms.rp_t = 0; })
    MPH_MARK(4);
    const int32_t acc = ms.accepted;
    // ClusterCapacityBinder.Bind + postBindHook: pod k+i -> node (plugin.go:34-53; simulator.go:297-312). Every CTA knows the
    // whole list; CTA 0 (of every rank: each keeps the whole sequence) records it.
    if (cta == 0 && tid < acc && k + tid < p.pod_cap) p.pod_node[k + tid] = ms.acc_node[tid];
    // ---- the winners' rows: the replay warp counted this thread's node among the winners (ms.mult). Only this thread reads the
    //      row before the next S1. ----
    if (tid < cnt_nodes && acc) {
      const int mult = ms.mult[tid];
      if (mult) {
        ms.mult[tid] = 0;
        lean_commit_row(p, lp, t, tid, mult, -1);     // this node's NodeInfo generation changed: its memoised score is stale
      }
    }
    MPH_MARK(5);
    k += acc;
    delta = ms.delta;
    if (ls.stop) break;
    lean_pts_after_wave(p, smem_cnt, p.debug_flags & DBG_RECOUNT_EVERY_WAVE);
    wtag = (wtag == 4095u) ? 1u : wtag + 1u;
    tag = (p.epoch << 12) | wtag;
  }

  if (DevOut *o = lean_finish(p, lp, t, lo, cnt_nodes, k, limit_hit)) {
    o->waves = limit_hit ? wv : wv + 1;
    o->evals = o->waves * (long long)p.n;
    o->examined = o->evals;
    for (int q = 0; q < 8; q++) o->phase_cycles[q] = ms.ph[q];
    o->stat[0] = ms.st_cand; o->stat[1] = ms.st_overflow; o->stat[2] = ms.st_rounds; o->stat[3] = SORTED ? (ms.st_key_order | ((long long)ms.st_tile_sel << 32)) : ms.st_key_order;
    // (CCSIM_DEBUG_FLAGS bit 3's summary stays in the kernel body: a printf inlined from a helper puts its argument buffer ahead
    //  of the MultiParams copy in the stack frame, which then grows from 136 to 192 bytes and takes a register more)
    if (p.debug_flags & DBG_CYCLES)
      printf("multi-commit replay: waves %lld rounds %lld look-ahead waves %d (without a placement: %d) | cycles: replay %lld set-up %lld, per round %.0f\n",
             limit_hit ? wv : wv + 1, ms.st_rounds, ms.st_relaxed, ms.st_empty, ms.ph[4], ms.ph[6],
             (double)(ms.ph[4] - ms.ph[6]) / (double)(ms.st_rounds > 0 ? ms.st_rounds : 1));
    multi_report(limit_hit ? wv : wv + 1);
  }
}
