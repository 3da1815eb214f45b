// ccsim_engine.cu — libccsim.so: the H100 cluster-capacity hot path behind the C-ABI of include/ccsim.h.
//
// Replaces the reference's sequential schedule-one-pod-then-update loop
// (pkg/framework/simulator.go:356-381 driving vendor/k8s.io/kubernetes/pkg/scheduler/schedule_one.go:66-148) by ONE
// persistent cooperative kernel per Run:
//
//   wave k (pod k, template k % M):
//     every CTA owns a contiguous tile of nodes and pushes each through the fused Filter+Score pass (eval_node),
//     warp-shuffle + shared-memory arg-max over packed (score, ~index) keys,
//     all-to-all exchange of one 64-bit tagged key per CTA (and per normalisation class) through L2 — this is the
//     only grid-wide synchronisation of the wave (no atomics, no fences: the tag makes each word self-validating),
//     every CTA redundantly reduces the keys of all CTAs (one per SM), the owner CTA commits the winner row (NodeInfo.update,
//     framework/types.go:409-427), every CTA updates its replica of the per-domain counters.
//
// The node state is mutated in place in HBM/L2; only the owner CTA ever reads or writes a given row, so no
// inter-CTA ordering is needed beyond the key exchange.
#include <cuda_runtime.h>
#include <algorithm>
#include <climits>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdarg.h>
#include <dlfcn.h>
#include <map>
#include <string>
#include <vector>
#include "ccsim_device.cuh"
#include "ccsim_lean.cuh"
#include "ccsim_batched.cuh"
#include "ccsim_multi.cuh"
#include "ccsim_stream.cuh"
#include "ccsim_each.cuh"
#include "ccsim_wave.cuh"

// ------------------------------------------------------------------------------------------------------------------
// Terminal diagnosis: FitError histogram of the pod that did not fit (framework/types.go:787-838) and the status codes
// the DefaultPreemption PostFilter groups nodes by (preemption/preemption.go:309-331). Runs once per Run.
// ------------------------------------------------------------------------------------------------------------------
__global__ void ccsim_diag_kernel(const DevParams p, int tmpl_index) {
  const ccsim_template &t = p.templates[tmpl_index];
  DevOut *o = p.out;
  const int32_t n = p.n;
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int st = ST_OK;
    int reasons[8 + CCSIM_MAX_SCALARS]; int nr = 0;
    const uint64_t taint0 = p.taint_mask[i];
    do {
      if ((t.flags & CCSIM_TF_PREFILTER_NODES) && t.prefilter_bit >= 0) {
        const int b = t.prefilter_bit;
        if (!((p.static_mask[(size_t)(b >> 6) * n + i] >> (b & 63)) & 1ull)) { reasons[nr++] = CCSIM_R_PREFILTER_NODES; st = ST_UNRESOLVABLE; break; }
      }
      if ((t.filter_enable & CCSIM_PL_NODE_UNSCHEDULABLE) && ((taint0 >> CCSIM_TAINT_UNSCHEDULABLE_BIT) & 1ull) &&
          !(t.flags & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) { reasons[nr++] = CCSIM_R_UNSCHEDULABLE; st = ST_UNRESOLVABLE; break; }
      if ((t.filter_enable & CCSIM_PL_NODE_NAME) && t.nodename_idx >= 0 && t.nodename_idx != p.node_base + i) {
        reasons[nr++] = CCSIM_R_NODE_NAME; st = ST_UNRESOLVABLE; break; }
      if (t.filter_enable & CCSIM_PL_TAINT_TOLERATION) {
        uint64_t untol_any = 0; int low = -1;
        for (int w = 0; w < p.taint_words; w++) {
          const uint64_t m = p.taint_mask[(size_t)w * n + i] & p.taint_nosched[w] & ~t.tol_nosched[w];
          if (m && low < 0) low = 64 * w + __ffsll((long long)m) - 1;
          untol_any |= m;
        }
        if (untol_any) {
          int id = -1;
          if (p.taint_list_off) {   // first untolerated taint in node.Spec.Taints order (corev1/helpers.go:78-101)
            for (int32_t q = p.taint_list_off[i]; q < p.taint_list_off[i + 1]; q++) {
              const int tid = p.taint_list[q];
              if (((p.taint_nosched[tid >> 6] >> (tid & 63)) & 1ull) && !((t.tol_nosched[tid >> 6] >> (tid & 63)) & 1ull)) { id = tid; break; }
            }
          }
          if (id < 0) id = low;
          reasons[nr++] = CCSIM_R_TAINT0 + id; st = ST_UNRESOLVABLE; break;
        }
      }
      uint64_t sw[CCSIM_MAX_STATIC_WORDS];
      for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) sw[w] = (w < p.static_words) ? p.static_mask[(size_t)w * n + i] : 0ull;
      if ((t.filter_enable & CCSIM_PL_NODE_AFFINITY) && (t.flags & (CCSIM_TF_HAS_NODE_SELECTOR | CCSIM_TF_HAS_AFFINITY_TERMS))) {
        bool m = true;
        for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) m &= ((sw[w] & t.sel_mask[w]) == t.sel_mask[w]);
        if (m && (t.flags & CCSIM_TF_HAS_AFFINITY_TERMS)) {
          bool any = false;
          for (int k = 0; k < t.n_aff_terms; k++) {
            bool tm = true;
            for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) tm &= ((sw[w] & t.aff_term_mask[k][w]) == t.aff_term_mask[k][w]);
            any |= tm;
          }
          m = any;
        }
        if (!m) { reasons[nr++] = CCSIM_R_NODE_AFFINITY; st = ST_UNRESOLVABLE; break; }
      }
      if ((t.filter_enable & CCSIM_PL_NODE_PORTS) && (t.flags & CCSIM_TF_HAS_HOST_PORTS)) {
        uint64_t c = 0;
        for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) c |= sw[w] & t.port_static_mask[w];
        if (p.placed_mask && (p.placed_mask[i] & t.port_tmpl_conflict)) c = 1;
        if (c) { reasons[nr++] = CCSIM_R_NODE_PORTS; st = ST_UNSCHEDULABLE; break; }
      }
      if (t.filter_enable & CCSIM_PL_FIT) {
        bool fail = false, unres = false;
        if (p.npods[i] + 1 > p.alloc_pods[i]) { fail = true; reasons[nr++] = CCSIM_R_TOO_MANY_PODS; }
        if (!(t.flags & CCSIM_TF_FIT_ALL_ZERO)) {
          if (t.req_cpu > 0 && t.req_cpu > p.alloc_cpu[i] - p.req_cpu[i]) { fail = true; unres |= t.req_cpu > p.alloc_cpu[i]; reasons[nr++] = CCSIM_R_INSUFFICIENT_CPU; }
          if (t.req_mem > 0 && t.req_mem > p.alloc_mem[i] - p.req_mem[i]) { fail = true; unres |= t.req_mem > p.alloc_mem[i]; reasons[nr++] = CCSIM_R_INSUFFICIENT_MEMORY; }
          if (t.req_eph > 0 && t.req_eph > p.alloc_eph[i] - p.req_eph[i]) { fail = true; unres |= t.req_eph > p.alloc_eph[i]; reasons[nr++] = CCSIM_R_INSUFFICIENT_EPHEMERAL; }
          for (int k = 0; k < p.n_scalars; k++) {
            const int64_t q = t.req_scalar[k];
            if (q == 0) continue;
            if (q > p.alloc_scalar[k][i] - p.req_scalar[k][i]) { fail = true; unres |= q > p.alloc_scalar[k][i]; reasons[nr++] = CCSIM_R_SCALAR0 + k; }
          }
        }
        if (fail) { st = unres ? ST_UNRESOLVABLE : ST_UNSCHEDULABLE; break; }
      }
      if (t.filter_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD) {
        bool done = false;
        for (int c = 0; c < t.n_pts && !done; c++) {
          const ccsim_pts &pc = t.pts[c];
          const DevCounter &dc = p.counters[pc.counter];
          const int32_t dom = dc.topo_col < 0 ? i : p.topo[dc.topo_col][i];
          if (dom < 0) { reasons[nr++] = CCSIM_R_PTS_MISSING_LABEL; st = ST_UNRESOLVABLE; done = true; break; }
          const int32_t cv = dc.topo_col < 0 ? dc.work[i] : p.final_cnt[p.final_off[pc.counter] + dom];
          const long long skew = (long long)cv + pc.self_match - (long long)o->ptsmin[c];
          if (skew > pc.max_skew) { reasons[nr++] = CCSIM_R_PTS_SKEW; st = ST_UNSCHEDULABLE; done = true; }
        }
        if (done) break;
      }
      if (t.filter_enable & CCSIM_PL_INTER_POD_AFFINITY) {
        bool pods_exist = true, missing = false;
        for (int a = 0; a < t.n_aff; a++) {
          const DevCounter &dc = p.counters[t.aff_counter[a]];
          const int32_t dom = dc.topo_col < 0 ? i : p.topo[dc.topo_col][i];
          if (dom < 0) { missing = true; break; }
          const int32_t cv = dc.topo_col < 0 ? dc.work[i] : p.final_cnt[p.final_off[t.aff_counter[a]] + dom];
          if (cv <= 0) pods_exist = false;
        }
        if (t.n_aff > 0 && (missing || (!pods_exist && !(o->aff_total == 0 && (t.flags & CCSIM_TF_AFF_SELF_MATCH_ALL))))) {
          reasons[nr++] = CCSIM_R_IPA_AFFINITY; st = ST_UNRESOLVABLE; break; }
        bool anti = false;
        for (int a = 0; a < t.n_anti; a++) {
          const DevCounter &dc = p.counters[t.anti_counter[a]];
          const int32_t dom = dc.topo_col < 0 ? i : p.topo[dc.topo_col][i];
          if (dom < 0) continue;
          const int32_t cv = dc.topo_col < 0 ? dc.work[i] : p.final_cnt[p.final_off[t.anti_counter[a]] + dom];
          if (cv > 0) anti = true;
        }
        if (anti) { reasons[nr++] = CCSIM_R_IPA_ANTI_AFFINITY; st = ST_UNSCHEDULABLE; break; }
        uint64_t c = 0;
        for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) c |= sw[w] & t.existing_anti_mask[w];
        if (c) { reasons[nr++] = CCSIM_R_IPA_EXISTING_ANTI; st = ST_UNSCHEDULABLE; break; }
      }
    } while (0);
    for (int q = 0; q < nr; q++) atomicAdd(&o->reason_hist[reasons[q]], 1ull);
    if (st == ST_UNSCHEDULABLE) atomicAdd(&o->preempt_no_victims, 1ull);
    atomicAdd(&o->n_diag, 1ull);
  }
}

// per-node replica counts of template t and first-placement index (report.go:146-180 without the O(P*nodes) scan)
__global__ void ccsim_count_kernel(const int32_t *pod_node, long long placed, int n_templates, int t,
                                   int32_t *counts, unsigned long long *first) {
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < placed; k += (long long)gridDim.x * blockDim.x) {
    if ((int)(k % n_templates) != t) continue;
    const int32_t w = pod_node[k];
    atomicAdd(&counts[w], 1);
    atomicMin(&first[w], (unsigned long long)k);
  }
}

__global__ void ccsim_flush_kernel(unsigned long long *buf, size_t n, unsigned long long v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) buf[i] = v + i;
}

// ------------------------------------------------------------------------------------------------------------------
// host side of the C-ABI
// ------------------------------------------------------------------------------------------------------------------
// Every wave-kernel instantiation run_prepare may pick, in the order of the WK_* indices, and what the host knows about it
enum EngineCode { ENG_GENERIC, ENG_LEAN, ENG_TIE_RUN, ENG_MULTI, ENG_STREAM, ENG_EACH };   // ccsim_run_stats[0]
struct WaveKernel {
  const void *fn;
  const char *name;        // ccsim_kernel_name
  EngineCode engine;
  int block;
  size_t static_smem;      // its __shared__ structs
  size_t fixed_dyn_smem;   // its dynamic shared-memory limit if fixed; 0: what the opt-in limit leaves (take_if_fits)
};
static const WaveKernel WAVE_KERNELS[] = {
  {(const void *)ccsim_wave_kernel<true>, "wave<true>", ENG_GENERIC, BLOCK_THREADS, sizeof(WaveShared), 0},
  {(const void *)ccsim_wave_kernel<false>, "wave<false>", ENG_GENERIC, BLOCK_THREADS, sizeof(WaveShared), SMEM_CNT_MAX_INTS * sizeof(int32_t) + 16},
  {(const void *)ccsim_wave_lean_kernel<false>, "lean<false>", ENG_LEAN, LEAN_THREADS, sizeof(LeanShared), 0},
  {(const void *)ccsim_wave_lean_kernel<true>, "lean<true>", ENG_LEAN, LEAN_THREADS, sizeof(LeanShared), 0},
  {(const void *)ccsim_wave_batched_kernel, "batched", ENG_TIE_RUN, LEAN_THREADS, sizeof(LeanShared) + sizeof(BatchShared), 0},
  {(const void *)ccsim_wave_multi_kernel<false, false>, "multi<false>", ENG_MULTI, LEAN_THREADS, sizeof(LeanShared) + sizeof(MultiShared), 0},
  {(const void *)ccsim_wave_multi_kernel<true, false>, "multi<true>", ENG_MULTI, LEAN_THREADS, sizeof(LeanShared) + sizeof(MultiShared), 0},
  // (the same kernels with the selection from the sorted tile: named alike, ccsim_sorted_tile_waves tells them apart)
  {(const void *)ccsim_wave_multi_kernel<false, true>, "multi<false>", ENG_MULTI, LEAN_THREADS, sizeof(LeanShared) + sizeof(MultiShared) + MULTI_SORTED_SMEM, 0},
  {(const void *)ccsim_wave_multi_kernel<true, true>, "multi<true>", ENG_MULTI, LEAN_THREADS, sizeof(LeanShared) + sizeof(MultiShared) + MULTI_SORTED_SMEM, 0},
  {(const void *)ccsim_wave_stream_kernel<0>, "stream<0>", ENG_STREAM, STREAM_BLOCK, sizeof(StreamShared), stream_smem_bytes(0, 0)},
  {(const void *)ccsim_wave_stream_kernel<1>, "stream<1>", ENG_STREAM, STREAM_BLOCK, sizeof(StreamShared), stream_smem_bytes(1, 0)},
  {(const void *)ccsim_wave_stream_kernel<2>, "stream<2>", ENG_STREAM, STREAM_BLOCK, sizeof(StreamShared), 0},
  {(const void *)ccsim_each_kernel<false>, "each", ENG_EACH, EACH_THREADS, sizeof(EachShared), 0},   // ccsim_run_each: node-local analyses
  {(const void *)ccsim_each_kernel<true>, "each", ENG_EACH, EACH_THREADS, sizeof(EachShared), 0},    // ... some with counters or hostPorts
  {(const void *)ccsim_each_packed_kernel, "each<packed>", ENG_EACH, EACH_THREADS, 0, 0},            // ... node-local, more than the CTAs that fit
};
enum { WK_WAVE, WK_WAVE_STREAMED, WK_LEAN, WK_LEAN_SAMPLING, WK_BATCHED, WK_MULTI, WK_MULTI_SHARDED, WK_MULTI_SORTED, WK_MULTI_SHARDED_SORTED,
       WK_STREAM /* + mode */,
       WK_EACH = WK_STREAM + 3, WK_EACH_TERMS, WK_EACH_PACKED };
static_assert(sizeof(WAVE_KERNELS) / sizeof(WAVE_KERNELS[0]) == WK_EACH_PACKED + 1, "one WAVE_KERNELS entry per WK_* index");

struct RunPlan {      // what run_prepare decided, consumed by the launch
  bool valid = false, empty = false;
  int64_t max_pods = 0;
  DevParams p; LeanParams lp; MultiParams mp; StreamParams sp;
  const WaveKernel *kern = nullptr; size_t smem = 0;   // kern: ccsim_kernel_name, outlives the launch, which clears `valid`
};

// Template facts of the engine choice (ccsim_set_templates): a template without NodeResourcesFit's Filter (no "Too many pods" bound);
// normalised soft scorers; the lean and streaming kernels cover every template (no soft scorer, ImageLocality or needs_extras; one taint word, <= 1 static word)
struct TemplateFacts { bool fit_off, has_soft, lean_filter; };

// the most placements after which every domain of a counter is still exact, with NodeResourcesFit bounding each domain by its free
// pod slots (lim_fit) or not (lim_any), and the domain that sets each bound
struct CounterRange { int64_t lim_fit, lim_any; int32_t dom_fit, dom_any, init_fit, init_any; };

// ccsim_run_each: one analysis's terms and tree segments as the host keeps them
struct AnalysisState {
  EachTerms terms;                            // its device copy is d_terms[t]
  int32_t n_topo = 0;
  int32_t final_off[CCSIM_MAX_COUNTERS] = {};  // counter j's working counts: terms.counters[j].work = work + final_off[j]
  int32_t *work = nullptr;
  CounterRange range[CCSIM_MAX_COUNTERS];
  std::vector<int64_t> dom_slots[CCSIM_MAX_TOPO_COLS];
};

struct ccsim_handle {
  ccsim_config cfg;
  int sm_count = 0;
  size_t l2_bytes = 0;
  size_t smem_optin = 0;
  std::vector<void *> stream_allocs;                    // padded streaming columns + per-template score memo (ccsim_stream.cuh)
  uint64_t taint_or0 = 0;                               // OR over the nodes of taint word 0
  std::vector<std::pair<void *, size_t>> block_cache;   // freed device blocks kept for reuse (exact size match)
  std::map<void *, size_t> block_bytes;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::string err;
  int64_t launches = 0;
  // snapshot
  bool have_nodes = false, have_templates = false;
  int32_t n = 0, n_global = 0, node_base = 0;
  ccsim_nodes meta;            // scalar members only
  std::vector<void *> allocs;  // every device allocation, freed in destroy / reload
  std::vector<void *> tmpl_allocs;
  // device columns: snapshot copies and working copies of the mutable ones
  int64_t *d_alloc_cpu = nullptr, *d_alloc_mem = nullptr, *d_alloc_eph = nullptr;
  int32_t *d_alloc_pods = nullptr;
  int64_t *d_alloc_scalar[CCSIM_MAX_SCALARS] = {};
  uint64_t *d_taint = nullptr, *d_static = nullptr;
  int32_t *d_topo[CCSIM_MAX_TOPO_COLS] = {};
  int64_t *s_req_cpu = nullptr, *s_req_mem = nullptr, *s_req_eph = nullptr, *s_nz_cpu = nullptr, *s_nz_mem = nullptr;
  int32_t *s_npods = nullptr;
  int64_t *s_req_scalar[CCSIM_MAX_SCALARS] = {};
  int64_t *w_req_cpu = nullptr, *w_req_mem = nullptr, *w_req_eph = nullptr, *w_nz_cpu = nullptr, *w_nz_mem = nullptr;
  int32_t *w_npods = nullptr;
  int64_t *w_req_scalar[CCSIM_MAX_SCALARS] = {};
  uint64_t *w_placed = nullptr;
  int32_t *w_score = nullptr;
  uint8_t *w_feas = nullptr;
  uint32_t *d_stamp[CCSIM_MAX_PTS] = {nullptr};
  size_t stamp_len[CCSIM_MAX_PTS] = {0};
  int32_t *d_taint_off = nullptr; uint8_t *d_taint_list = nullptr;
  int64_t pod_bound = 0;       // sum over nodes of max(0, alloc_pods - npods): no run can place more
  int max_prefer_pop = 0;      // max over nodes of popcount(taint & prefer): number of normalisation classes - 1
  // templates
  int32_t n_templates = 0, n_counters = 0;
  std::vector<ccsim_template> h_templates;
  TemplateFacts tf = {};
  ccsim_template *d_templates = nullptr;
  DevCounter counters[CCSIM_MAX_COUNTERS];
  int32_t *d_final_cnt = nullptr; int32_t final_off[CCSIM_MAX_COUNTERS] = {}; int32_t final_total = 0;
  // int32 range of the counters (check_run_bounds): free pod slots of every node and of every domain of each topology column over the
  // whole cluster (ccsim_load_nodes), and per counter the most placements after which all its domains are still exact
  // (ccsim_set_templates), with NodeResourcesFit bounding each domain by its slots (lim_fit) or not (lim_any)
  std::vector<int32_t> node_slots;
  std::vector<int64_t> dom_slots[CCSIM_MAX_TOPO_COLS];
  CounterRange cnt_range[CCSIM_MAX_COUNTERS];
  int32_t smem_cnt_ints = 0;
  // run state
  int grid = 0;
  unsigned long long *d_slots = nullptr;
  unsigned long long *d_xslots = nullptr;                 // cross-GPU exchange buffer (exported over CUDA IPC)
  unsigned long long *x_peer[CCSIM_MAX_WORLD] = {};       // every rank's buffer as mapped here
  bool peers_ready = false;
  bool peers_local = false;                               // peers are plain pointers of this process (nothing to close)
  uint32_t epoch = 0;
  uint32_t xwave0 = 0;                                    // exchanges of earlier sharded runs (buffer parity continues across runs)
  int64_t last_stat[16] = {};                             // ccsim_run_stats
  int64_t last_key_order_waves = 0;                       // ccsim_key_order_waves
  int64_t last_sorted_tile_waves = 0;                     // ccsim_sorted_tile_waves
  RunPlan plan;
  int32_t *d_topo_full[CCSIM_MAX_TOPO_COLS] = {};
  int32_t *d_pod_node = nullptr; int64_t pod_cap = 0;
  std::vector<int32_t> h_pod_node;
  DevOut *d_out = nullptr;
  DevParams *d_params = nullptr;
  int64_t last_placed = 0;
  void *d_flush = nullptr; size_t flush_bytes = 0;
  // ccsim_run_each: per-analysis state, sequences and results of the last per-analysis run (each_ran until the next ccsim_run / prepare)
  std::vector<void *> each_allocs;
  bool each_ran = false;
  int32_t *d_each_seq = nullptr; int64_t each_seq_cap = 0;
  std::vector<int64_t> each_placed;
  std::vector<std::vector<int32_t>> each_seq;
  // ccsim_run_each: every analysis's own counters, columns and tree segments, made by ccsim_set_analyses or, for the node-local
  // templates of ccsim_set_templates, by the first ccsim_run_each (until the next ccsim_set_templates / set_analyses / load_nodes)
  bool analyses = false;                      // the templates came from ccsim_set_analyses
  std::vector<AnalysisState> an;
  EachTerms *d_terms = nullptr;
  std::vector<uint64_t> h_taint;              // the loaded taint masks (word-major): the normalisation class of each node
};

static thread_local std::string g_create_err;   // ccsim_create's error, per thread: several host threads may create engines at once

static int fail(ccsim_handle *h, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  if (h) h->err = buf; else g_create_err = buf;
  return code;
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(h, CCSIM_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// Device blocks are recycled per handle: ccsim_load_nodes / ccsim_set_templates are called once per analysis by the host side,
// usually with the same shapes as the last time, and cudaMalloc/cudaFree are slow, synchronising driver calls.
template <typename T> static int dev_alloc(ccsim_handle *h, std::vector<void *> &pool, T **out, size_t count) {
  void *p = nullptr;
  size_t bytes = (count ? count : 1) * sizeof(T);
  for (size_t i = 0; i < h->block_cache.size(); i++)
    if (h->block_cache[i].second == bytes) { p = h->block_cache[i].first; h->block_cache.erase(h->block_cache.begin() + i); break; }
  if (!p) {
    // stream-ordered allocation: no device-wide synchronisation (a host that drives several ranks from one process may have a
    // peer's persistent kernel running, waiting for this rank's kernel to start)
    cudaError_t e = cudaMallocAsync(&p, bytes, h->stream);
    if (e != cudaSuccess) return fail(h, CCSIM_ENOMEM, "cudaMallocAsync(%zu): %s", bytes, cudaGetErrorString(e));
  }
  pool.push_back(p);
  h->block_bytes[p] = bytes;
  *out = (T *)p;
  return 0;
}
template <typename T> static int dev_upload(ccsim_handle *h, std::vector<void *> &pool, T **out, const T *src, size_t count) {
  int rc = dev_alloc(h, pool, out, count);
  if (rc) return rc;
  if (count) CK(cudaMemcpyAsync(*out, src, count * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  return 0;
}
// blocks of a pool go back to the handle's cache (the stream is drained first: they may still be in use)
static void free_pool(ccsim_handle *h, std::vector<void *> &pool) {
  if (pool.empty()) return;
  cudaStreamSynchronize(h->stream);
  size_t cached = 0;
  for (auto &b : h->block_cache) cached += b.second;
  for (void *p : pool) {
    const size_t bytes = h->block_bytes[p];
    if (cached + bytes <= ((size_t)1 << 31)) { h->block_cache.push_back({p, bytes}); cached += bytes; }   // keep at most 2 GiB around
    else { cudaFreeAsync(p, h->stream); h->block_bytes.erase(p); }
  }
  pool.clear();
}
static void drop_cache(ccsim_handle *h) {
  for (auto &b : h->block_cache) cudaFreeAsync(b.first, h->stream);
  cudaStreamSynchronize(h->stream);
  h->block_cache.clear(); h->block_bytes.clear();
}

extern "C" int ccsim_abi_version(void) { return CCSIM_ABI_VERSION; }

extern "C" const char *ccsim_last_error(const ccsim_handle *h) { return h ? h->err.c_str() : g_create_err.c_str(); }

extern "C" int ccsim_create(const ccsim_config *cfg, ccsim_handle **out) {
  ccsim_handle *h = nullptr;
  if (!cfg || !out) return fail(h, CCSIM_EINVAL, "null argument");
  if (cfg->abi_version != CCSIM_ABI_VERSION) return fail(h, CCSIM_EINVAL, "abi_version %d != %d", cfg->abi_version, CCSIM_ABI_VERSION);
  if (cfg->world < 1 || cfg->world > CCSIM_MAX_WORLD || cfg->rank < 0 || cfg->rank >= cfg->world) return fail(h, CCSIM_EINVAL, "bad rank/world");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(h, CCSIM_ECUDA, "no CUDA device: %s (libccsim has no CPU fallback)", cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(h, CCSIM_EINVAL, "device %d out of range (%d)", cfg->device, ndev);
  h = new ccsim_handle();
  h->cfg = *cfg;
  cudaDeviceProp prop;
  if ((e = cudaSetDevice(cfg->device)) != cudaSuccess || (e = cudaGetDeviceProperties(&prop, cfg->device)) != cudaSuccess) {
    fail(nullptr, CCSIM_ECUDA, "cudaSetDevice/GetDeviceProperties: %s", cudaGetErrorString(e));
    delete h; return CCSIM_ECUDA;
  }
  if (!prop.cooperativeLaunch) { fail(nullptr, CCSIM_EUNSUPPORTED, "device lacks cooperative launch"); delete h; return CCSIM_EUNSUPPORTED; }
  h->sm_count = prop.multiProcessorCount;
  h->l2_bytes = (size_t)prop.l2CacheSize;
  {   // the stream-ordered allocator keeps what it has mapped (default: everything goes back to the driver at the next synchronize,
      // and every analysis would map its snapshot's memory again)
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, cfg->device) == cudaSuccess) { uint64_t keep = UINT64_MAX; cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep); }
  }
  cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  cudaMalloc((void **)&h->d_out, sizeof(DevOut));
  cudaMalloc((void **)&h->d_params, sizeof(DevParams));
  cudaMalloc((void **)&h->d_slots, sizeof(unsigned long long) * SLOTS_WORDS);
  cudaMalloc((void **)&h->d_xslots, sizeof(unsigned long long) * XSLOTS_TOTAL_WORDS);     // winner words (lean kernel) + candidate lines (multi-commit)
  cudaMemset(h->d_xslots, 0, sizeof(unsigned long long) * XSLOTS_TOTAL_WORDS);
  h->x_peer[cfg->rank] = h->d_xslots;
  h->smem_optin = (size_t)prop.sharedMemPerBlockOptin;
  for (const WaveKernel &k : WAVE_KERNELS)   // a fixed size, or what the opt-in limit leaves (take_if_fits)
    cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)(k.fixed_dyn_smem ? k.fixed_dyn_smem : h->smem_optin - k.static_smem - 1024));
  *out = h;
  return CCSIM_OK;
}

extern "C" void ccsim_destroy(ccsim_handle *h) {
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  cudaStreamSynchronize(h->stream);
  free_pool(h, h->allocs); free_pool(h, h->tmpl_allocs); free_pool(h, h->stream_allocs); free_pool(h, h->each_allocs); drop_cache(h);
  for (int r = 0; r < CCSIM_MAX_WORLD; r++) if (h->x_peer[r] && r != h->cfg.rank && !h->peers_local) cudaIpcCloseMemHandle(h->x_peer[r]);
  cudaFree(h->d_xslots);
  if (h->d_pod_node) { cudaFreeAsync(h->d_pod_node, h->stream); cudaStreamSynchronize(h->stream); }
  cudaFree(h->d_out); cudaFree(h->d_params); cudaFree(h->d_slots); cudaFree(h->d_flush);
  cudaEventDestroy(h->ev0); cudaEventDestroy(h->ev1);
  cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" int ccsim_load_nodes(ccsim_handle *h, const ccsim_nodes *nd) {
  if (!h || !nd) return fail(h, CCSIM_EINVAL, "null argument");
  if (nd->n_nodes < 0 || nd->n_scalars < 0 || nd->n_scalars > CCSIM_MAX_SCALARS || nd->taint_words < 1 ||
      nd->taint_words > CCSIM_MAX_TAINT_WORDS || nd->static_words < 0 || nd->static_words > CCSIM_MAX_STATIC_WORDS ||
      nd->n_topo_cols < 0 || nd->n_topo_cols > CCSIM_MAX_TOPO_COLS)
    return fail(h, CCSIM_EINVAL, "ccsim_nodes dimensions out of range");
  CK(cudaSetDevice(h->cfg.device));
  free_pool(h, h->allocs);
  h->have_nodes = false; h->have_templates = false; h->plan.valid = false; h->an.clear();
  const int32_t N = nd->n_nodes;
  // node-axis shard of this rank (SURVEY.md §8e): contiguous block of the nodeTree order
  const int32_t per = (N + h->cfg.world - 1) / h->cfg.world;
  const int32_t lo = std::min<int64_t>((int64_t)per * h->cfg.rank, N), hi = std::min<int64_t>((int64_t)lo + per, N);
  const int32_t n = hi - lo;
  // every rank of a sharded run takes part in the per-wave exchange: a rank without nodes would never launch the kernel and its
  // peers would wait for its words forever
  if (h->cfg.world > 1 && N > 0 && (int64_t)per * (h->cfg.world - 1) >= N)
    return fail(h, CCSIM_EUNSUPPORTED, "sharded run: %d nodes over %d ranks leaves a rank without nodes (use fewer ranks)", N, h->cfg.world);
  h->n = n; h->n_global = N; h->node_base = lo;
  h->meta = *nd;
  int rc;
#define UP(dst, src, T) if ((rc = dev_upload<T>(h, h->allocs, &h->dst, (src) ? (src) + lo : (const T *)nullptr, (src) ? (size_t)n : 0))) return rc
  if (N > 0 && (!nd->alloc_cpu || !nd->alloc_mem || !nd->alloc_eph || !nd->alloc_pods || !nd->req_cpu || !nd->req_mem ||
                !nd->req_eph || !nd->npods || !nd->nz_cpu || !nd->nz_mem || !nd->taint_mask))
    return fail(h, CCSIM_EINVAL, "null core column");
  // LeastAllocated's (capacity - requested) * 100 must not wrap: a wrapped score leaves [0, 100] and runs into the key's tag bits
  for (int32_t i = 0; i < N; i++) {
    if (nd->alloc_cpu[i] > CCSIM_MAX_SCORED_ALLOCATABLE)
      return fail(h, CCSIM_EUNSUPPORTED, "node %d: cpu allocatable %lld exceeds %lld", i, (long long)nd->alloc_cpu[i], (long long)CCSIM_MAX_SCORED_ALLOCATABLE);
    if (nd->alloc_mem[i] > CCSIM_MAX_SCORED_ALLOCATABLE)
      return fail(h, CCSIM_EUNSUPPORTED, "node %d: memory allocatable %lld exceeds %lld", i, (long long)nd->alloc_mem[i], (long long)CCSIM_MAX_SCORED_ALLOCATABLE);
  }
  UP(d_alloc_cpu, nd->alloc_cpu, int64_t); UP(d_alloc_mem, nd->alloc_mem, int64_t); UP(d_alloc_eph, nd->alloc_eph, int64_t);
  UP(d_alloc_pods, nd->alloc_pods, int32_t);
  UP(s_req_cpu, nd->req_cpu, int64_t); UP(s_req_mem, nd->req_mem, int64_t); UP(s_req_eph, nd->req_eph, int64_t);
  UP(s_nz_cpu, nd->nz_cpu, int64_t); UP(s_nz_mem, nd->nz_mem, int64_t); UP(s_npods, nd->npods, int32_t);
  for (int k = 0; k < nd->n_scalars; k++) {
    if (!nd->alloc_scalar[k] || !nd->req_scalar[k]) return fail(h, CCSIM_EINVAL, "null scalar column %d", k);
    UP(d_alloc_scalar[k], nd->alloc_scalar[k], int64_t); UP(s_req_scalar[k], nd->req_scalar[k], int64_t);
  }
#undef UP
  // word-major bitmask columns: copy the shard slice of each word
  if ((rc = dev_alloc(h, h->allocs, &h->d_taint, (size_t)nd->taint_words * n))) return rc;
  for (int w = 0; w < nd->taint_words && n; w++)
    CK(cudaMemcpyAsync(h->d_taint + (size_t)w * n, nd->taint_mask + (size_t)w * N + lo, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
  if ((rc = dev_alloc(h, h->allocs, &h->d_static, (size_t)nd->static_words * n))) return rc;
  if (nd->static_words && N > 0 && !nd->static_mask) return fail(h, CCSIM_EINVAL, "null static_mask");
  for (int w = 0; w < nd->static_words && n; w++)
    CK(cudaMemcpyAsync(h->d_static + (size_t)w * n, nd->static_mask + (size_t)w * N + lo, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
  for (int k = 0; k < nd->n_topo_cols; k++) {
    if (!nd->topo[k] && N > 0) return fail(h, CCSIM_EINVAL, "null topo column %d", k);
    if ((rc = dev_upload<int32_t>(h, h->allocs, &h->d_topo[k], nd->topo[k] ? nd->topo[k] + lo : nullptr, (size_t)n))) return rc;
    h->d_topo_full[k] = h->d_topo[k];
    if (h->cfg.world > 1)   // winners of other shards: their domain ids are looked up in the whole-cluster column
      if ((rc = dev_upload<int32_t>(h, h->allocs, &h->d_topo_full[k], nd->topo[k], (size_t)N))) return rc;
  }
  // working copies
#define WK(dst, T) if ((rc = dev_alloc<T>(h, h->allocs, &h->dst, (size_t)n))) return rc
  WK(w_req_cpu, int64_t); WK(w_req_mem, int64_t); WK(w_req_eph, int64_t); WK(w_nz_cpu, int64_t); WK(w_nz_mem, int64_t); WK(w_npods, int32_t);
  for (int k = 0; k < nd->n_scalars; k++) WK(w_req_scalar[k], int64_t);
  h->w_placed = nullptr;
  if (nd->has_placed_mask) WK(w_placed, uint64_t);
  WK(w_score, int32_t);
  WK(w_feas, uint8_t);
#undef WK
  h->d_taint_off = nullptr; h->d_taint_list = nullptr;
  if (nd->taint_list_off && nd->taint_list && n > 0) {
    std::vector<int32_t> off(n + 1);
    const int32_t base = nd->taint_list_off[lo];
    for (int32_t i = 0; i <= n; i++) off[i] = nd->taint_list_off[lo + i] - base;
    if ((rc = dev_upload<int32_t>(h, h->allocs, &h->d_taint_off, off.data(), (size_t)n + 1))) return rc;
    if ((rc = dev_upload<uint8_t>(h, h->allocs, &h->d_taint_list, nd->taint_list + base, (size_t)off[n]))) return rc;
    CK(cudaStreamSynchronize(h->stream));   // off[] is a local
  }
  // host-side bounds used to size outputs / classes
  int64_t bound = 0; int maxpop = 0;
  for (int32_t i = 0; i < N; i++) {
    const int64_t free_pods = (int64_t)nd->alloc_pods[i] - nd->npods[i];
    if (free_pods > 0) bound += free_pods;
    int pc = 0;
    for (int w = 0; w < nd->taint_words; w++) pc += __builtin_popcountll(nd->taint_mask[(size_t)w * N + i] & nd->taint_prefer[w]);
    if (pc > maxpop) maxpop = pc;
  }
  h->pod_bound = bound; h->max_prefer_pop = maxpop;
  h->node_slots.assign(N, 0);
  for (int32_t i = 0; i < N; i++) h->node_slots[i] = std::max<int32_t>(0, nd->alloc_pods[i] - nd->npods[i]);
  for (int c = 0; c < CCSIM_MAX_TOPO_COLS; c++) h->dom_slots[c].clear();
  for (int c = 0; c < nd->n_topo_cols; c++)
    for (int32_t i = 0; i < N; i++) {
      const int32_t d = nd->topo[c][i];
      if (d < 0) continue;
      if ((size_t)d >= h->dom_slots[c].size()) h->dom_slots[c].resize((size_t)d + 1, 0);
      h->dom_slots[c][d] += h->node_slots[i];
    }
  h->taint_or0 = 0;
  for (int32_t i = 0; i < N; i++) h->taint_or0 |= nd->taint_mask[i];
  h->h_taint.assign(nd->taint_mask, nd->taint_mask + (size_t)nd->taint_words * N);
  CK(cudaStreamSynchronize(h->stream));
  h->have_nodes = true;
  return CCSIM_OK;
}

// A template that needs one of the uncommon predicates the lean and streaming kernels leave out (filter_extras: ephemeral storage,
// extended resources, nodeAffinity terms, nodeName, PreFilter node sets, hostPorts against clones already placed).
static bool needs_extras(const ccsim_handle *h, const ccsim_template &T) {
  const bool nzfit = (T.filter_enable & CCSIM_PL_FIT) && !(T.flags & CCSIM_TF_FIT_ALL_ZERO);
  if (nzfit && T.req_eph > 0) return true;
  if (nzfit) for (int k = 0; k < h->meta.n_scalars; k++) if (T.req_scalar[k] != 0) return true;
  if ((T.filter_enable & CCSIM_PL_NODE_AFFINITY) && (T.flags & CCSIM_TF_HAS_AFFINITY_TERMS)) return true;
  if ((T.filter_enable & CCSIM_PL_NODE_NAME) && T.nodename_idx >= 0) return true;
  if (T.flags & CCSIM_TF_PREFILTER_NODES) return true;
  if ((T.filter_enable & CCSIM_PL_NODE_PORTS) && (T.flags & CCSIM_TF_HAS_HOST_PORTS) && h->w_placed) return true;
  return false;
}

// One template's index ranges against its counter table, and the counters' eligibility bits (CCSIM_EINVAL; `who` prefixes the
// counter messages)
static int check_template(ccsim_handle *h, int t, const ccsim_template &T, int32_t n_counters, const ccsim_counter *counters, const char *who) {
  const ccsim_nodes &nd = h->meta;
  if (T.n_pref_terms < 0 || T.n_pref_terms > CCSIM_MAX_AFF_TERMS) return fail(h, CCSIM_EINVAL, "template %d: n_pref_terms", t);
  if (T.n_pts < 0 || T.n_pts > CCSIM_MAX_PTS || T.n_aff < 0 || T.n_aff > CCSIM_MAX_IPA || T.n_anti < 0 || T.n_anti > CCSIM_MAX_IPA ||
      T.n_aff_terms < 0 || T.n_aff_terms > CCSIM_MAX_AFF_TERMS)
    return fail(h, CCSIM_EINVAL, "template %d: term counts out of range", t);
  for (int c = 0; c < T.n_pts; c++) {
    if (T.pts[c].counter < 0 || T.pts[c].counter >= n_counters) return fail(h, CCSIM_EINVAL, "template %d: pts counter index", t);
    if (counters[T.pts[c].counter].topo_col < 0)
      return fail(h, CCSIM_EUNSUPPORTED, "topology spread over a node-local (hostname) domain is not supported yet");
  }
  for (int a = 0; a < T.n_aff; a++) if (T.aff_counter[a] < 0 || T.aff_counter[a] >= n_counters) return fail(h, CCSIM_EINVAL, "aff counter index");
  for (int a = 0; a < T.n_anti; a++) if (T.anti_counter[a] < 0 || T.anti_counter[a] >= n_counters) return fail(h, CCSIM_EINVAL, "anti counter index");
  if ((T.flags & CCSIM_TF_PREFILTER_NODES) && (T.prefilter_bit < 0 || T.prefilter_bit >= 64 * nd.static_words))
    return fail(h, CCSIM_EINVAL, "template %d: prefilter_bit", t);
  if (T.n_spts < 0 || T.n_spts > CCSIM_MAX_PTS || T.n_ipa_score < 0 || T.n_ipa_score > CCSIM_MAX_IPA)
    return fail(h, CCSIM_EINVAL, "template %d: soft term counts out of range", t);
  if (T.spts_ignored_bit >= 64 * nd.static_words) return fail(h, CCSIM_EINVAL, "template %d: spts_ignored_bit", t);
  for (int c = 0; c < T.n_spts; c++) {
    const ccsim_spts &sc = T.spts[c];
    if (sc.counter < 0 || sc.counter >= n_counters) return fail(h, CCSIM_EINVAL, "template %d: spts counter index", t);
    if ((sc.hostname != 0) != (counters[sc.counter].topo_col < 0)) return fail(h, CCSIM_EINVAL, "template %d: spts %d: hostname constraints use node-local counters (and only they)", t, c);
    if (sc.has_key_bit >= 64 * nd.static_words) return fail(h, CCSIM_EINVAL, "template %d: spts has_key_bit", t);
  }
  for (int a = 0; a < T.n_ipa_score; a++) if (T.ipa_score_counter[a] < 0 || T.ipa_score_counter[a] >= n_counters) return fail(h, CCSIM_EINVAL, "ipa score counter index");
  for (int j = 0; j < n_counters; j++) if (counters[j].elig_bit >= 64 * nd.static_words) return fail(h, CCSIM_EINVAL, "%scounter %d: elig_bit", who, j);
  return CCSIM_OK;
}

static int check_weights(ccsim_handle *h, int t, const ccsim_template &T) {
  // a negative weight can make a total negative, and score + 1 <= 0 sets the key's tag bits; the reference's plugin weights
  // are never negative (framework.go:487-497) and its resource weights are validated to [1, 100] (validation_pluginargs.go)
  const int32_t w[7] = {T.w_taint, T.w_node_affinity, T.w_fit, T.w_pts, T.w_ipa, T.w_balanced, T.w_image};
  const char *wname[7] = {"TaintToleration", "NodeAffinity", "NodeResourcesFit", "PodTopologySpread", "InterPodAffinity",
                          "NodeResourcesBalancedAllocation", "ImageLocality"};
  for (int q = 0; q < 7; q++)
    if (w[q] < 0) return fail(h, CCSIM_EUNSUPPORTED, "template %d: %s score weight %d is negative", t, wname[q], w[q]);
  if (T.least_w_cpu < 1 || T.least_w_cpu > 100 || T.least_w_mem < 1 || T.least_w_mem > 100)
    return fail(h, CCSIM_EUNSUPPORTED, "template %d: NodeResourcesFit resource weights cpu %d / memory %d outside [1, 100]", t, T.least_w_cpu, T.least_w_mem);
  long long wsum = 0;
  for (int q = 0; q < 7; q++) wsum += w[q];
  if (wsum * 100 >= 4095) return fail(h, CCSIM_EUNSUPPORTED, "template %d: sum of score weights %lld too large for the packed key", t, wsum);
  return CCSIM_OK;
}

// Counter c's int32 range (check_run_bounds). dom_slots: the free pod slots of each domain of its column (nullptr: node-local)
static CounterRange counter_range(const ccsim_handle *h, const ccsim_counter &c, const std::vector<int64_t> *dom_slots) {
  // domain d stays exact for m placements into it while |init_d| + m * |inc| <= INT32_MAX, i.e. m <= room_d; it receives at
  // most min(placements, its free slots) of them while NodeResourcesFit filters, at most `placements` otherwise
  CounterRange r;
  r.lim_fit = r.lim_any = INT64_MAX; r.dom_fit = r.dom_any = -1; r.init_fit = r.init_any = 0;
  const int64_t inc = std::llabs((long long)c.inc);
  for (int32_t d = 0; inc > 0 && d < c.n_domains; d++) {
    const int64_t room = std::max<int64_t>(0, ((int64_t)INT32_MAX - std::llabs((long long)c.init[d])) / inc);
    const int64_t slots = !dom_slots ? (d < (int32_t)h->node_slots.size() ? h->node_slots[d] : 0)
                                     : ((size_t)d < dom_slots->size() ? (*dom_slots)[d] : 0);
    if (room < r.lim_any) { r.lim_any = room; r.dom_any = d; r.init_any = c.init[d]; }
    if (slots > room && room < r.lim_fit) { r.lim_fit = room; r.dom_fit = d; r.init_fit = c.init[d]; }
  }
  return r;
}

// What both setters do first: the state and count checks (at most max_templates), then the handle's templates, counters and analyses
// dropped
static int begin_templates(ccsim_handle *h, int32_t n_templates, int32_t max_templates) {
  if (!h->have_nodes) return fail(h, CCSIM_ESTATE, "ccsim_load_nodes must come first");
  if (n_templates < 1 || n_templates > max_templates) return fail(h, CCSIM_EINVAL, "n_templates out of range");
  CK(cudaSetDevice(h->cfg.device));
  free_pool(h, h->tmpl_allocs);
  h->have_templates = false; h->plan.valid = false; h->each_ran = false; h->analyses = false; h->an.clear();
  return CCSIM_OK;
}

// The score weights and the class limit checked, then the facts and the device copy of the templates (ImageLocality columns: this
// shard's slice goes to the device, the device copy of the template points at it)
static int upload_templates(ccsim_handle *h, int32_t n_templates, const ccsim_template *templates, int32_t n_counters, const ccsim_counter *counters) {
  const ccsim_nodes &nd = h->meta;
  int rc;
  for (int t = 0; t < n_templates; t++) if ((rc = check_weights(h, t, templates[t]))) return rc;
  if (h->max_prefer_pop + 1 > CCSIM_MAX_CLASSES)
    return fail(h, CCSIM_EUNSUPPORTED, "a node carries %d PreferNoSchedule taints (max %d)", h->max_prefer_pop, CCSIM_MAX_CLASSES - 1);
  h->h_templates.assign(templates, templates + n_templates);
  TemplateFacts &tf = h->tf;
  tf = TemplateFacts{false, false, nd.taint_words == 1 && nd.static_words <= 1};
  for (const ccsim_template &T : h->h_templates) {
    if (!(T.filter_enable & CCSIM_PL_FIT)) tf.fit_off = true;
    if (T.n_pref_terms > 0 && (T.score_enable & CCSIM_PL_NODE_AFFINITY)) tf.has_soft = true;
    if (T.n_spts > 0 && (T.score_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD)) tf.has_soft = true;
    if (T.n_ipa_score > 0 && (T.score_enable & CCSIM_PL_INTER_POD_AFFINITY)) tf.has_soft = true;
    if ((T.image_score && (T.score_enable & CCSIM_PL_IMAGE_LOCALITY)) || needs_extras(h, T)) tf.lean_filter = false;
  }
  for (int j = 0; j < n_counters; j++) if (counters[j].elig_bit >= 0) tf.has_soft = true;
  if (tf.has_soft) tf.lean_filter = false;
  std::vector<ccsim_template> dev_t(templates, templates + n_templates);
  for (int t = 0; t < n_templates; t++)
    if (templates[t].image_score) {
      uint8_t *d = nullptr;
      if ((rc = dev_upload<uint8_t>(h, h->tmpl_allocs, &d, templates[t].image_score + h->node_base, (size_t)h->n))) return rc;
      dev_t[t].image_score = d;
    }
  if ((rc = dev_upload<ccsim_template>(h, h->tmpl_allocs, &h->d_templates, dev_t.data(), (size_t)n_templates))) return rc;
  CK(cudaStreamSynchronize(h->stream));   // dev_t is about to go out of scope
  return CCSIM_OK;
}

// Counter j of template T on the device, without its columns (init, work) and its place (smem_off)
static DevCounter dev_counter(const ccsim_counter &c, const ccsim_template &T, int j) {
  DevCounter d;
  memset(&d, 0, sizeof(d));
  d.topo_col = c.topo_col; d.n_domains = c.n_domains; d.n_present = c.n_present; d.inc = c.inc; d.smem_off = -1; d.elig_bit = c.elig_bit;
  for (int a = 0; a < T.n_aff; a++) if (T.aff_counter[a] == j) d.is_aff = 1;
  return d;
}

extern "C" int ccsim_set_templates(ccsim_handle *h, int32_t n_templates, const ccsim_template *templates,
                                   int32_t n_counters, const ccsim_counter *counters) {
  if (!h || !templates) return fail(h, CCSIM_EINVAL, "null argument");
  int rc;
  if ((rc = begin_templates(h, n_templates, CCSIM_MAX_TEMPLATES))) return rc;
  if (n_counters < 0 || n_counters > CCSIM_MAX_COUNTERS || (n_counters && !counters)) return fail(h, CCSIM_EINVAL, "n_counters out of range");
  if (n_templates > 1 && n_counters > 0)
    return fail(h, CCSIM_EUNSUPPORTED, "PodTopologySpread/InterPodAffinity templates are single-template only");
  const ccsim_nodes &nd = h->meta;
  for (int t = 0; t < n_templates; t++) if ((rc = check_template(h, t, templates[t], n_counters, counters, ""))) return rc;
  if ((rc = upload_templates(h, n_templates, templates, n_counters, counters))) return rc;
  for (int c = 0; c < CCSIM_MAX_PTS; c++) { h->d_stamp[c] = nullptr; h->stamp_len[c] = 0; }
  for (int c = 0; c < templates[0].n_spts; c++)
    if (!templates[0].spts[c].hostname) {
      h->stamp_len[c] = (size_t)counters[templates[0].spts[c].counter].n_domains + 1;
      if ((rc = dev_alloc<uint32_t>(h, h->tmpl_allocs, &h->d_stamp[c], h->stamp_len[c]))) return rc;
    }
  // counters: small domain sets live replicated in shared memory, large ones as per-CTA replicas in global memory
  h->smem_cnt_ints = 0; h->final_total = 0;
  const int grid_max = std::min(h->sm_count, CCSIM_MAX_GRID);
  for (int j = 0; j < n_counters; j++) {
    const ccsim_counter &c = counters[j];
    DevCounter &d = h->counters[j];
    d = dev_counter(c, templates[0], j);
    if (c.topo_col >= nd.n_topo_cols) return fail(h, CCSIM_EINVAL, "counter %d: topo_col", j);
    h->cnt_range[j] = counter_range(h, c, c.topo_col < 0 ? nullptr : &h->dom_slots[c.topo_col]);
    if (c.topo_col < 0) {
      // node-local: init is a whole-cluster column; keep this shard's slice
      if (c.n_domains != h->n_global) return fail(h, CCSIM_EINVAL, "counter %d: node-local counter needs n_domains == n_nodes", j);
      d.n_domains = h->n;
      if ((rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d.init, c.init + h->node_base, (size_t)h->n))) return rc;
      if ((rc = dev_alloc<int32_t>(h, h->tmpl_allocs, &d.work, (size_t)h->n))) return rc;
    } else {
      if (c.n_domains < 0 || c.n_present < 0 || c.n_present > c.n_domains) return fail(h, CCSIM_EINVAL, "counter %d: domains", j);
      if ((rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d.init, c.init, (size_t)c.n_domains))) return rc;
      if (h->smem_cnt_ints + c.n_domains <= SMEM_CNT_MAX_INTS) { d.smem_off = h->smem_cnt_ints; h->smem_cnt_ints += c.n_domains; }
      else if ((rc = dev_alloc<int32_t>(h, h->tmpl_allocs, &d.work, (size_t)grid_max * c.n_domains))) return rc;
      h->final_off[j] = h->final_total; h->final_total += c.n_domains;
    }
  }
  if ((rc = dev_alloc<int32_t>(h, h->tmpl_allocs, &h->d_final_cnt, (size_t)h->final_total))) return rc;
  h->n_templates = n_templates; h->n_counters = n_counters;
  CK(cudaStreamSynchronize(h->stream));
  h->have_templates = true;
  return CCSIM_OK;
}

// Tree levels of the per-analysis kernel: roots on level L, 32^L >= n
static int each_tree_levels(int32_t n) {
  int L = 0;
  while (n > 0 && (1ll << (5 * L)) < n) L++;
  return L;
}

// Analysis t's device state: its counters and columns, and its tree segments. The segments cover a stable partition of the nodes by
// normalisation class (TaintToleration's raw count of untolerated PreferNoSchedule taints), then by domain in each column of a term
// tested per group. Without such terms segment c is class c (possibly empty), and the partition is a counting one.
static int build_analysis(ccsim_handle *h, int t, const ccsim_template &T, const ccsim_analysis_terms &A, AnalysisState &S) {
  const ccsim_nodes &nd = h->meta;
  const int32_t n = h->n;
  const int ncls = h->max_prefer_pop + 1, L = each_tree_levels(n);
  int rc;
  EachTerms &E = S.terms;
  memset(&E, 0, sizeof(E));
  S.n_topo = A.n_topo_cols;
  // the columns, and whether a column's domains hold one node each
  bool single[CCSIM_MAX_TOPO_COLS] = {};
  for (int k = 0; k < A.n_topo_cols; k++) {
    int32_t *d = nullptr;
    if ((rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d, A.topo[k], (size_t)n))) return rc;
    E.topo[k] = d;
    std::vector<int64_t> &slots = S.dom_slots[k];
    std::vector<int32_t> members;
    for (int32_t i = 0; i < n; i++) {
      const int32_t dd = A.topo[k][i];
      if (dd < 0) continue;
      if ((size_t)dd >= slots.size()) { slots.resize((size_t)dd + 1, 0); members.resize((size_t)dd + 1, 0); }
      slots[dd] += h->node_slots[i];
      members[dd]++;
    }
    single[k] = std::all_of(members.begin(), members.end(), [](int32_t m) { return m <= 1; });
  }
  // the counters: their initial counts, one block of working counts, the int32 range of each
  int32_t total = 0;
  for (int j = 0; j < A.n_counters; j++) { S.final_off[j] = total; total += A.counters[j].n_domains; }
  if ((rc = dev_alloc<int32_t>(h, h->tmpl_allocs, &S.work, (size_t)std::max(total, 1)))) return rc;
  E.n_counters = A.n_counters;
  for (int j = 0; j < A.n_counters; j++) {
    const ccsim_counter &c = A.counters[j];
    DevCounter &d = E.counters[j];
    d = dev_counter(c, T, j);
    int32_t *init = nullptr;
    if ((rc = dev_upload<int32_t>(h, h->tmpl_allocs, &init, c.init, (size_t)c.n_domains))) return rc;
    d.init = init; d.work = S.work + S.final_off[j];
    S.range[j] = counter_range(h, c, c.topo_col < 0 ? nullptr : &S.dom_slots[c.topo_col]);
  }
  // the terms: folded into the leaf when their domains hold one node each, else tested per domain group
  const uint32_t fe = T.filter_enable;
  bool group_col[CCSIM_MAX_TOPO_COLS] = {};
  auto place = [&](int counter, uint32_t bit) {
    const int32_t col = A.counters[counter].topo_col;
    if (col < 0 || single[col]) E.leaf_sel |= bit;
    else { E.group_sel |= bit; group_col[col] = true; }
  };
  if (fe & CCSIM_PL_POD_TOPOLOGY_SPREAD) for (int c = 0; c < T.n_pts; c++) place(T.pts[c].counter, 1u << c);
  if (fe & CCSIM_PL_INTER_POD_AFFINITY) {
    for (int a = 0; a < T.n_aff; a++) place(T.aff_counter[a], COUPLED_AFF_SEL(a));
    for (int a = 0; a < T.n_anti; a++) place(T.anti_counter[a], COUPLED_ANTI_SEL(a));
  }
  // every node in class 0 when no node carries a PreferNoSchedule taint or TaintToleration does not score: no per-node pass then
  const bool one_class = ncls == 1 || !(T.score_enable & CCSIM_PL_TAINT_TOLERATION);
  std::vector<int32_t> cls(one_class ? 0 : (size_t)n, 0);
  if (!one_class)
    for (int32_t i = 0; i < n; i++)
      for (int w = 0; w < nd.taint_words; w++) cls[i] += __builtin_popcountll(h->h_taint[(size_t)w * n + i] & nd.taint_prefer[w] & ~T.tol_prefer[w]);
  std::vector<int32_t> pos, rep, seg_cls;   // pos empty: every node at its own index
  std::vector<long long> start;
  if (!E.group_sel && one_class) {
    for (int c = 0; c < ncls; c++) { start.push_back(c ? n : 0); rep.push_back(0); seg_cls.push_back(c); }
  } else if (!E.group_sel) {   // segment c = class c (possibly empty), as many as the cluster has classes
    pos.resize((size_t)n);
    std::vector<long long> at((size_t)ncls + 1, 0);
    for (int32_t i = 0; i < n; i++) at[cls[i] + 1]++;
    for (int c = 0; c < ncls; c++) { at[c + 1] += at[c]; start.push_back(at[c]); rep.push_back(0); seg_cls.push_back(c); }
    for (int32_t i = 0; i < n; i++) pos[i] = (int32_t)at[cls[i]]++;
  } else {              // one group per (class, domain in each group column)
    std::vector<int32_t> gcols;
    for (int k = 0; k < A.n_topo_cols; k++) if (group_col[k]) gcols.push_back(k);
    const size_t kw = 1 + gcols.size();
    std::vector<int32_t> key((size_t)n * kw);
    pos.resize((size_t)n);
    for (int32_t i = 0; i < n; i++) {
      key[(size_t)i * kw] = one_class ? 0 : cls[i];
      for (size_t q = 0; q < gcols.size(); q++) key[(size_t)i * kw + 1 + q] = A.topo[gcols[q]][i];
    }
    std::vector<int32_t> order((size_t)n);
    for (int32_t i = 0; i < n; i++) order[i] = i;
    auto less = [&](int32_t x, int32_t y) {
      return std::lexicographical_compare(&key[(size_t)x * kw], &key[(size_t)x * kw + kw], &key[(size_t)y * kw], &key[(size_t)y * kw + kw]);
    };
    std::stable_sort(order.begin(), order.end(), less);
    for (int32_t r = 0; r < n; r++) {
      const int32_t i = order[r];
      pos[i] = r;
      if (r == 0 || less(order[r - 1], i)) { start.push_back(r); rep.push_back(i); seg_cls.push_back(one_class ? 0 : cls[i]); }
    }
  }
  const int32_t G = (int32_t)start.size();
  if (G > CCSIM_EACH_MAX_GROUPS)
    return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: analysis %d has %d domain groups (max %d)", t, G, CCSIM_EACH_MAX_GROUPS);
  std::vector<long long> cof((size_t)(L + 1) * (G + 1));
  for (int g = 0; g < G; g++) cof[g] = start[g];
  cof[G] = n;
  for (int l = 1; l <= L; l++) {
    long long acc = 0;
    for (int g = 0; g < G; g++) {
      const long long sz = cof[(size_t)(l - 1) * (G + 1) + g + 1] - cof[(size_t)(l - 1) * (G + 1) + g];
      cof[(size_t)l * (G + 1) + g] = acc; acc += (sz + 31) >> 5;
    }
    cof[(size_t)l * (G + 1) + G] = acc;
  }
  E.n_seg = G;
  // the analysis's own bit of port_tmpl_conflict: t mod 64 (one analysis at a time is diagnosed, so the bits of analyses 64 apart never meet)
  E.port_self = h->w_placed && (T.filter_enable & CCSIM_PL_NODE_PORTS) && (T.flags & CCSIM_TF_HAS_HOST_PORTS) && ((T.port_tmpl_conflict >> (t & 63)) & 1ull);
  bool identity = true;   // then the kernel reads a node's position as its index
  for (int32_t i = 0; i < (int32_t)pos.size() && identity; i++) identity = pos[i] == i;
  long long *d_cof = nullptr; int32_t *d_rep = nullptr, *d_cls = nullptr, *d_pos = nullptr;
  if ((rc = dev_upload<long long>(h, h->tmpl_allocs, &d_cof, cof.data(), cof.size())) ||
      (rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d_rep, rep.data(), rep.size())) ||
      (rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d_cls, seg_cls.data(), seg_cls.size())) ||
      (!identity && (rc = dev_upload<int32_t>(h, h->tmpl_allocs, &d_pos, pos.data(), pos.size()))))
    return rc;
  E.cof = d_cof; E.seg_rep = d_rep; E.seg_cls = d_cls; E.pos = d_pos;
  CK(cudaStreamSynchronize(h->stream));   // the host vectors go out of scope
  return CCSIM_OK;
}

// Every analysis's state (terms: nullptr, the node-local templates of ccsim_set_templates), and its device copy d_terms
static int build_analyses(ccsim_handle *h, const ccsim_analysis_terms *terms) {
  const ccsim_analysis_terms none = {};
  std::vector<AnalysisState> an((size_t)h->n_templates);
  std::vector<EachTerms> dev_terms;
  int rc;
  for (int t = 0; t < h->n_templates; t++) {
    if ((rc = build_analysis(h, t, h->h_templates[t], terms ? terms[t] : none, an[t]))) return rc;
    dev_terms.push_back(an[t].terms);
  }
  if ((rc = dev_upload<EachTerms>(h, h->tmpl_allocs, &h->d_terms, dev_terms.data(), dev_terms.size()))) return rc;
  CK(cudaStreamSynchronize(h->stream));   // dev_terms goes out of scope
  h->an.swap(an);
  return CCSIM_OK;
}

extern "C" int ccsim_set_analyses(ccsim_handle *h, int32_t n_templates, const ccsim_template *templates, const ccsim_analysis_terms *terms) {
  if (!h || !templates || !terms) return fail(h, CCSIM_EINVAL, "null argument");
  int rc;
  if ((rc = begin_templates(h, n_templates, CCSIM_EACH_MAX_ANALYSES))) return rc;
  const int32_t n = h->n;
  if (h->cfg.world > 1) return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: node-sharded runs (world %d) are not supported", h->cfg.world);
  for (int t = 0; t < n_templates; t++) {   // every analysis validated as ccsim_set_templates validates its template alone
    const ccsim_analysis_terms &A = terms[t];
    if (A.n_counters < 0 || A.n_counters > CCSIM_MAX_COUNTERS || (A.n_counters && !A.counters))
      return fail(h, CCSIM_EINVAL, "analysis %d: n_counters out of range", t);
    if (A.n_topo_cols < 0 || A.n_topo_cols > CCSIM_MAX_TOPO_COLS) return fail(h, CCSIM_EINVAL, "analysis %d: n_topo_cols out of range", t);
    for (int k = 0; k < A.n_topo_cols; k++) if (!A.topo[k] && n > 0) return fail(h, CCSIM_EINVAL, "analysis %d: null topo column %d", t, k);
    char who[32]; snprintf(who, sizeof(who), "analysis %d: ", t);
    if ((rc = check_template(h, t, templates[t], A.n_counters, A.counters, who))) return rc;
    for (int j = 0; j < A.n_counters; j++) {
      const ccsim_counter &c = A.counters[j];
      if (c.topo_col >= A.n_topo_cols) return fail(h, CCSIM_EINVAL, "analysis %d: counter %d: topo_col", t, j);
      if (c.topo_col < 0 ? c.n_domains != n : (c.n_domains < 0 || c.n_present < 0 || c.n_present > c.n_domains))
        return fail(h, CCSIM_EINVAL, "analysis %d: counter %d: domains", t, j);
      if (c.n_domains > 0 && !c.init) return fail(h, CCSIM_EINVAL, "analysis %d: counter %d: null init", t, j);
      if (c.topo_col >= 0)
        for (int32_t i = 0; i < n; i++)
          if (A.topo[c.topo_col][i] >= c.n_domains) return fail(h, CCSIM_EINVAL, "analysis %d: counter %d: node %d's domain out of range", t, j, i);
    }
  }
  if ((rc = upload_templates(h, n_templates, templates, 0, nullptr))) return rc;
  h->n_templates = n_templates; h->n_counters = 0; h->final_total = 0;
  if ((rc = build_analyses(h, terms))) return rc;
  h->analyses = true;
  h->have_templates = true;
  return CCSIM_OK;
}

// Counters are int32 here and in the oracle; the reference counts in int64 (podtopologyspread/scoring.go,
// interpodaffinity/scoring.go). A counter that could leave int32 during the run is refused, never left to wrap: a domain that
// receives m placements holds init + m' * inc with m' <= m, so |init| + m * |inc| <= INT32_MAX keeps every value exact, and m is
// at most min(placements, the domain's free pod slots) while NodeResourcesFit filters. `who` prefixes the message.
static int check_counter_bounds(ccsim_handle *h, int64_t max_pods, bool fit_off, int n_counters, const DevCounter *counters,
                                const CounterRange *ranges, const std::vector<int64_t> *dom_slots, const char *who) {
  int64_t placements = h->pod_bound;
  if (max_pods > 0 && (max_pods < placements || fit_off)) placements = max_pods;
  for (int j = 0; j < n_counters; j++) {
    const CounterRange &r = ranges[j];
    const int64_t lim = fit_off ? r.lim_any : r.lim_fit;
    const int32_t d = fit_off ? r.dom_any : r.dom_fit;
    if (placements > lim) {
      const int32_t tc = counters[j].topo_col;
      const int64_t m = fit_off ? placements : std::min(placements, tc < 0 ? (int64_t)h->node_slots[d] : dom_slots[tc][d]);
      return fail(h, CCSIM_EUNSUPPORTED, "%scounter %d, domain %d: |initial count| %lld + %lld placements x |increment| %d can leave int32",
                  who, j, d, std::llabs((long long)(fit_off ? r.init_any : r.init_fit)), (long long)m, std::abs(counters[j].inc));
    }
  }
  return CCSIM_OK;
}

// The output capacity of a run, since no run can place more than sum(max(0, alloc_pods - npods)) pods (fit.go:567-576), or
// max_pods. False: nothing bounds the run ("Too many pods" bounds a run only while NodeResourcesFit filters: with the plugin disabled
// through --default-config an unlimited run never ends in the reference either)
static bool run_cap(const ccsim_handle *h, int64_t max_pods, bool fit_off, int64_t &cap) {
  if (max_pods <= 0 && fit_off) return false;
  cap = h->pod_bound + 1;
  if (max_pods > 0 && (max_pods < cap || fit_off)) cap = max_pods;
  return true;
}

// The refusals a run meets before it touches anything: a run that nothing bounds, and counters that could leave int32. `cap`: the
// output capacity (run_cap)
static int check_run_bounds(ccsim_handle *h, int64_t max_pods, int64_t &cap) {
  const bool fit_off = h->tf.fit_off;
  if (!run_cap(h, max_pods, fit_off, cap))
    return fail(h, CCSIM_EUNSUPPORTED, "NodeResourcesFit is disabled for a template: the run is unbounded, --max-limit is required");
  return check_counter_bounds(h, max_pods, fit_off, h->n_counters, h->counters, h->cnt_range, h->dom_slots, "");
}

// The pod -> node buffer grown to `cap`; the working columns restored from the snapshot (a Run never changes the snapshot)
static int restore_run_state(ccsim_handle *h, int64_t cap) {
  if (cap > h->pod_cap) {
    if (h->d_pod_node) cudaFreeAsync(h->d_pod_node, h->stream);
    h->d_pod_node = nullptr; h->pod_cap = 0;
    CK(cudaMallocAsync((void **)&h->d_pod_node, (size_t)cap * sizeof(int32_t), h->stream));
    h->pod_cap = cap;
  }
  const int32_t n = h->n; cudaStream_t s = h->stream;
  if (n) {
    CK(cudaMemcpyAsync(h->w_req_cpu, h->s_req_cpu, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(h->w_req_mem, h->s_req_mem, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(h->w_req_eph, h->s_req_eph, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(h->w_nz_cpu, h->s_nz_cpu, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(h->w_nz_mem, h->s_nz_mem, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(h->w_npods, h->s_npods, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    for (int k = 0; k < h->meta.n_scalars; k++)
      CK(cudaMemcpyAsync(h->w_req_scalar[k], h->s_req_scalar[k], (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    if (h->w_placed) CK(cudaMemsetAsync(h->w_placed, 0, (size_t)n * 8, s));
    for (int j = 0; j < h->n_counters; j++)
      if (h->counters[j].topo_col < 0)
        CK(cudaMemcpyAsync(h->counters[j].work, h->counters[j].init, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  }
  for (int c = 0; c < CCSIM_MAX_PTS; c++) if (h->d_stamp[c]) CK(cudaMemsetAsync(h->d_stamp[c], 0, h->stamp_len[c] * 4, s));
  CK(cudaMemsetAsync(h->d_out, 0, sizeof(DevOut), s));
  CK(cudaMemsetAsync(h->d_slots, 0, sizeof(unsigned long long) * SLOTS_WORDS, s));
  // (the cross-GPU buffer is NOT cleared here: peers may already be writing wave 0 of this run; stale words are
  //  harmless because runs advance a per-handle epoch that is folded into the tag)
  return CCSIM_OK;
}

// The persistent grid and every kernel's parameters; advances the epoch (every rank of a sharded run prepares alike, refused or not)
static void fill_params(ccsim_handle *h, DevParams &p, int64_t max_pods) {
  memset(&p, 0, sizeof(p));
  const ccsim_nodes &nd = h->meta;
  // grid: one persistent CTA per SM (fewer for tiny clusters: the exchange cost grows with the CTA count)
  // (node-sharded runs: every rank sizes the grid from the largest shard, so that all ranks launch the same grid and every
  //  rank knows how many candidate lines its peers publish)
  const int32_t n_grid = h->cfg.world > 1 ? (h->n_global + h->cfg.world - 1) / h->cfg.world : h->n;
  p.grid = std::max(1, std::min({h->sm_count, CCSIM_MAX_GRID, (n_grid + BLOCK_THREADS - 1) / BLOCK_THREADS}));
  h->grid = p.grid;
  p.n = h->n; p.n_global = h->n_global; p.node_base = h->node_base;
  p.chunk = (p.n + p.grid - 1) / p.grid;
  p.chunk_pad = (p.chunk + 3) & ~3;
  p.n_scalars = nd.n_scalars; p.taint_words = nd.taint_words; p.static_words = nd.static_words; p.n_topo = nd.n_topo_cols;
  p.n_templates = h->n_templates; p.n_counters = h->n_counters;
  for (int j = 0; j < h->n_counters; j++) if (h->counters[j].topo_col < 0) p.n_local++;
  p.smem_cnt_ints = h->smem_cnt_ints;
  p.n_classes = h->max_prefer_pop + 1;
  p.rank = h->cfg.rank; p.world = h->cfg.world;
  h->epoch = (h->epoch % 255u) + 1u;
  p.epoch = h->epoch;
  p.xwave0 = h->xwave0;
  p.debug_flags = getenv("CCSIM_DEBUG_FLAGS") ? (uint32_t)atoi(getenv("CCSIM_DEBUG_FLAGS")) : 0u;
  {   // reference sampling mode (ccsim_config.sampling): numFeasibleNodesToFind (schedule_one.go:697-723)
    const long long N = h->n_global;
    long long pct = h->cfg.pct_nodes_to_score, kf = N;
    if (N >= 100) {
      if (pct == 0) { pct = 50 - N / 125; if (pct < 5) pct = 5; }
      kf = N * pct / 100;
      if (kf < 100) kf = 100;
    }
    p.sample_k = kf;
  }
  p.alloc_cpu = h->d_alloc_cpu; p.alloc_mem = h->d_alloc_mem; p.alloc_eph = h->d_alloc_eph; p.alloc_pods = h->d_alloc_pods;
  for (int k = 0; k < nd.n_scalars; k++) { p.alloc_scalar[k] = h->d_alloc_scalar[k]; p.req_scalar[k] = h->w_req_scalar[k]; }
  p.taint_mask = h->d_taint; p.static_mask = h->d_static;
  for (int k = 0; k < nd.n_topo_cols; k++) { p.topo[k] = h->d_topo[k]; p.topo_full[k] = h->d_topo_full[k]; }
  for (int r = 0; r < CCSIM_MAX_WORLD; r++) p.xslots_peer[r] = h->x_peer[r];
  p.req_cpu = h->w_req_cpu; p.req_mem = h->w_req_mem; p.req_eph = h->w_req_eph; p.nz_cpu = h->w_nz_cpu; p.nz_mem = h->w_nz_mem;
  p.npods = h->w_npods; p.placed_mask = h->w_placed; p.score_cache = h->w_score; p.feas = h->w_feas;
  for (int c = 0; c < CCSIM_MAX_PTS; c++) p.stamp[c] = h->d_stamp[c];
  for (int w = 0; w < CCSIM_MAX_TAINT_WORDS; w++) { p.taint_nosched[w] = nd.taint_nosched[w]; p.taint_prefer[w] = nd.taint_prefer[w]; }
  p.templates = h->d_templates;
  for (int j = 0; j < h->n_counters; j++) { p.counters[j] = h->counters[j]; p.final_off[j] = h->final_off[j]; }
  p.final_cnt = h->d_final_cnt;
  p.slots = h->d_slots;
  p.pod_node = h->d_pod_node; p.pod_cap = h->pod_cap; p.max_pods = max_pods;
  p.out = h->d_out;
  p.taint_list_off = h->d_taint_off; p.taint_list = h->d_taint_list;
  p.self = h->d_params;
}

// Takes kernel `e` with `dyn` bytes of dynamic shared memory if they fit next to its static structs, with 1 KB to spare
static bool take_if_fits(const ccsim_handle *h, RunPlan &pl, const WaveKernel *&k, const WaveKernel &e, size_t dyn) {
  if (dyn + e.static_smem + 1024 > h->smem_optin) return false;
  k = &e; pl.smem = dyn;
  return true;
}

// The lean resident kernel (ccsim_lean.cuh: eligibility): a record slot per topology column and node-local counter, the tile layout
static bool plan_lean(const ccsim_handle *h, RunPlan &pl, bool faithful, const WaveKernel *&k) {
  if (!h->tf.lean_filter || h->n_templates != 1) return false;
  const ccsim_template &T = h->h_templates[0];
  if (T.n_pts + T.n_aff + T.n_anti > LEAN_MAX_TERMS) return false;
  LeanParams &lp = pl.lp;
  int ns = 0;
  for (int j = 0; j < h->n_counters; j++) {
    const DevCounter &dc = h->counters[j];
    if (dc.topo_col >= 0 && dc.smem_off < 0) return false;
    int slot = -1;
    if (dc.topo_col >= 0) for (int q = 0; q < ns; q++) if (lp.slot_topo[q] == dc.topo_col) slot = q;
    if (slot < 0) {
      if (ns >= LEAN_MAX_SLOTS) return false;
      slot = ns++;
      lp.slot_topo[slot] = dc.topo_col >= 0 ? dc.topo_col : -1;
      lp.slot_counter[slot] = dc.topo_col >= 0 ? -1 : j;
    }
    lp.counter_slot[j] = slot;
  }
  lp.n_slots = ns;
  lean_layout(lp, h->smem_cnt_ints, pl.p.chunk_pad);
  return take_if_fits(h, pl, k, WAVE_KERNELS[faithful ? WK_LEAN_SAMPLING : WK_LEAN],
                      lean_smem_bytes(lp, pl.p.chunk_pad, faithful ? 8 : 0));     // + the sampling pass's feasibility and rank
}

// Multi-commit waves (ccsim_multi.cuh) on the lean tile: one template coupled through per-domain counters, one node per thread
static void plan_multi(const ccsim_handle *h, RunPlan &pl, const WaveKernel *&k) {
  const ccsim_template &T = h->h_templates[0];
  const DevParams &p = pl.p;
  if (h->n_counters == 0 || h->max_prefer_pop != 0 || h->cfg.engine != CCSIM_ENGINE_AUTO || T.n_aff != 0 ||
      p.chunk > LEAN_THREADS || h->n_global >= (1 << MULTI_IDX_BITS) || p.grid * MULTI_M > MULTI_EPT * LEAN_THREADS)
    return;
  int refs[CCSIM_MAX_COUNTERS] = {}, gt = 0;      // Filter terms reading each counter; those reading a replicated one
  if (T.filter_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD) for (int c = 0; c < T.n_pts; c++) refs[T.pts[c].counter]++;
  if (T.filter_enable & CCSIM_PL_INTER_POD_AFFINITY) for (int a = 0; a < T.n_anti; a++) refs[T.anti_counter[a]]++;
  for (int j = 0; j < h->n_counters; j++) {
    const DevCounter &dc = h->counters[j];
    if (dc.inc < 0) return;                         // feasibility must be monotone within a wave
    if (dc.topo_col >= 0) gt += refs[j];
    // (a committed node may win again inside a wave: every candidate carries its key after one more clone, MULTI_NEXT_SHIFT)
    // the replay updates counters term by term: every incremented replicated counter must be read by exactly one Filter term
    if (dc.topo_col >= 0 && dc.inc != 0 && refs[j] != 1) return;
  }
  if (gt > MULTI_GT) return;
  const LeanParams &lp = pl.lp; MultiParams &mp = pl.mp;
  uint32_t shift = 0;
  for (int sl = 0; sl < lp.n_slots; sl++) {
    if (lp.slot_topo[sl] < 0) continue;
    int maxd = 1;
    for (int j = 0; j < h->n_counters; j++) if (lp.counter_slot[j] == sl && h->counters[j].topo_col >= 0) maxd = std::max(maxd, h->counters[j].n_domains);
    uint32_t bits = 0; while ((1u << bits) <= (uint32_t)maxd) bits++;        // values 0..maxd (dom + 1)
    if (shift + bits + 1 > MULTI_PAY_BITS) return;
    mp.pay_shift[sl] = shift; mp.pay_mask[sl] = (1u << bits) - 1u; shift += bits + 1;   // + a zero guard bit (the replay's SWAR kill test)
  }
  // + the per-node payload column, and 16 bytes that nothing reads: kept so that the kernel's shared-memory size, which
  //   run_stats() reports, stays what it has been
  const size_t dyn = lean_smem_bytes(lp, p.chunk_pad, 8) + 16;
  // Single-use template (a self-matching required anti-affinity on a node-local counter: a node takes one clone, so no winner comes
  // back in its wave): each tile's candidates come from the tile sorted by key, in the instantiation that has that selection and
  // its rank array — unless CCSIM_DEBUG_FLAGS bit 7 asks for the REDUX selection, or the rank array does not fit next to the tile.
  // The kernel checks the same condition itself (ccsim_multi.cuh: ms.single_use) and runs the REDUX selection when it fails.
  bool single_use = false;
  if (T.filter_enable & CCSIM_PL_INTER_POD_AFFINITY)
    for (int a = 0; a < T.n_anti; a++) {
      const DevCounter &dc = h->counters[T.anti_counter[a]];
      single_use |= dc.topo_col < 0 && dc.inc > 0 && !(dc.is_aff && !(T.flags & CCSIM_TF_AFF_SELF_MATCH_ALL));
    }
  const bool sharded = h->cfg.world > 1;
  if (single_use && !(p.debug_flags & DBG_REDUX_SELECT) &&
      take_if_fits(h, pl, k, WAVE_KERNELS[sharded ? WK_MULTI_SHARDED_SORTED : WK_MULTI_SORTED], dyn))
    return;
  take_if_fits(h, pl, k, WAVE_KERNELS[sharded ? WK_MULTI_SHARDED : WK_MULTI], dyn);
}

// Streaming waves (ccsim_stream.cuh: TMA-staged tiles, per-template score memo) when the lean tile is not taken; fills its padded columns
static int plan_stream(ccsim_handle *h, RunPlan &pl, const WaveKernel *&k) {
  if (!h->tf.lean_filter || h->n_counters != 0 || h->max_prefer_pop != 0) return CCSIM_OK;
  const DevParams &p = pl.p; StreamParams &sp = pl.sp;
  free_pool(h, h->stream_allocs);
  bool masks = false;
  for (const ccsim_template &T : h->h_templates) {
    uint64_t tb = 0;
    if (T.filter_enable & CCSIM_PL_TAINT_TOLERATION) tb |= h->meta.taint_nosched[0] & ~T.tol_nosched[0] & ~(1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT);
    if ((T.filter_enable & CCSIM_PL_NODE_UNSCHEDULABLE) && !(T.flags & CCSIM_TF_TOLERATES_UNSCHEDULABLE)) tb |= 1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT;
    if (tb & h->taint_or0) masks = true;
    if (h->meta.static_words > 0) {
      if ((T.filter_enable & CCSIM_PL_NODE_AFFINITY) && (T.flags & CCSIM_TF_HAS_NODE_SELECTOR) && T.sel_mask[0]) masks = true;
      if ((T.filter_enable & CCSIM_PL_NODE_PORTS) && (T.flags & CCSIM_TF_HAS_HOST_PORTS) && T.port_static_mask[0]) masks = true;
      if ((T.filter_enable & CCSIM_PL_INTER_POD_AFFINITY) && T.existing_anti_mask[0]) masks = true;
    }
  }
  sp.use_masks = masks ? 1 : 0;
  sp.chunk_pad = ((p.chunk + STREAM_TILE - 1) / STREAM_TILE) * STREAM_TILE;
  sp.tiles = sp.chunk_pad / STREAM_TILE;
  sp.n_pad = (long long)p.grid * sp.chunk_pad;
  int rc;
  unsigned long long *mt = nullptr, *mst = nullptr;
  if ((rc = dev_alloc<long long>(h, h->stream_allocs, &sp.f_cpu, (size_t)sp.n_pad))) return rc;
  if ((rc = dev_alloc<long long>(h, h->stream_allocs, &sp.f_mem, (size_t)sp.n_pad))) return rc;
  if ((rc = dev_alloc<int32_t>(h, h->stream_allocs, &sp.f_pods, (size_t)sp.n_pad))) return rc;
  if (masks) {
    if ((rc = dev_alloc<unsigned long long>(h, h->stream_allocs, &mt, (size_t)sp.n_pad))) return rc;
    if ((rc = dev_alloc<unsigned long long>(h, h->stream_allocs, &mst, (size_t)sp.n_pad))) return rc;
  }
  sp.m_taint = mt; sp.m_static = mst;
  if ((rc = dev_alloc<int32_t>(h, h->stream_allocs, &sp.memo, (size_t)sp.n_pad * h->n_templates))) return rc;
  CK(cudaMemsetAsync(sp.memo, 0xFF, (size_t)sp.n_pad * h->n_templates * 4, h->stream));
  ccsim_stream_prep_kernel<<<std::min<long long>(8LL * h->sm_count, (sp.n_pad + 255) / 256), 256, 0, h->stream>>>(p, sp);
  h->launches++;
  CK(cudaGetLastError());
  // resident free_* columns when the chunk fits next to the memo ring (24 B per node: up to ~7.8k nodes per SM)
  sp.res_rows = (p.chunk + 31) & ~31;
  k = &WAVE_KERNELS[WK_STREAM + (masks ? 1 : 0)]; pl.smem = stream_smem_bytes(masks ? 1 : 0, 0);
  if (!masks && sp.tiles <= STREAM_STAGES_RES && !getenv("CCSIM_STREAM_ALL"))
    take_if_fits(h, pl, k, WAVE_KERNELS[WK_STREAM + 2], stream_smem_bytes(2, sp.res_rows));
  return CCSIM_OK;
}

// Everything a Run does before the wave kernel starts: output / streaming buffers, restoring the working columns, choosing the
// kernel, uploading the parameters. Kept apart from the launch (ccsim_prepare) for hosts that drive several ranks from one
// process: every rank must be past its allocations before any rank's persistent kernel starts waiting for its peers.
static int run_prepare(ccsim_handle *h, int64_t max_pods) {
  if (!h->have_nodes || !h->have_templates) return fail(h, CCSIM_ESTATE, "load_nodes and set_templates must come first");
  if (h->analyses) return fail(h, CCSIM_ESTATE, "templates set by ccsim_set_analyses run with ccsim_run_each only");
  if (h->cfg.world > 1 && !h->peers_ready) return fail(h, CCSIM_ESTATE, "sharded run: ccsim_peer_import must come first");
  CK(cudaSetDevice(h->cfg.device));
  RunPlan &pl = h->plan;
  pl = RunPlan();                         // no kernel name until a kernel is chosen; the parameter blocks zeroed
  h->each_ran = false;
  pl.max_pods = max_pods;
  int64_t cap = 0; int rc;
  if ((rc = check_run_bounds(h, max_pods, cap)) || (rc = restore_run_state(h, cap))) return rc;
  if (h->n == 0) {   // ErrNoNodesAvailable (scheduler.go:68): nothing to evaluate; the host formats the message
    CK(cudaStreamSynchronize(h->stream));
    pl.empty = true; pl.valid = true;
    return CCSIM_OK;
  }
  DevParams &p = pl.p;
  fill_params(h, p, max_pods);
  // 1. the generic kernel, its tile resident in shared memory if it fits (the order of DESIGN.md §4; each refusal at its point)
  const WaveKernel *k = &WAVE_KERNELS[WK_WAVE_STREAMED];
  pl.smem = wave_smem_bytes(p, false);
  p.tile_resident = take_if_fits(h, pl, k, WAVE_KERNELS[WK_WAVE], wave_smem_bytes(p, true)) ? 1 : 0;
  if (h->tf.has_soft && (h->cfg.world > 1 || h->n_templates > 1))
    return fail(h, CCSIM_EUNSUPPORTED, "normalised soft scorers (preferred nodeAffinity, ScheduleAnyway spreading, pod-affinity scoring): single template, single GPU only");
  // 2. the lean kernel if eligible
  const bool faithful = h->cfg.sampling == CCSIM_SAMPLING_REFERENCE;
  const bool lean = p.tile_resident && plan_lean(h, pl, faithful, k);
  if (faithful && (!lean || h->cfg.world > 1))
    return fail(h, CCSIM_EUNSUPPORTED, "reference sampling mode needs the lean resident kernel on a single GPU (one template, <=1 taint/static word, no extras)");
  // 3. tie-run batching (ccsim_batched.cuh: node-local predicates and scorers only; + run length, score after the run, run offset
  //    per node) or multi-commit waves on the lean tile
  const bool batched = lean && !faithful && h->n_counters == 0 && h->max_prefer_pop == 0 && h->cfg.world == 1 &&
                       h->cfg.engine != CCSIM_ENGINE_SEQUENTIAL &&
                       take_if_fits(h, pl, k, WAVE_KERNELS[WK_BATCHED], lean_smem_bytes(pl.lp, p.chunk_pad, 12));
  if (h->cfg.engine == CCSIM_ENGINE_BATCHED && !batched)
    return fail(h, CCSIM_EUNSUPPORTED, "batched engine needs one template with node-local predicates only, no PreferNoSchedule taints, a resident tile and a single GPU");
  if (lean && !faithful && !batched) plan_multi(h, pl, k);
  // 4. streaming waves when the lean tile is not taken
  if (!lean && (rc = plan_stream(h, pl, k))) return rc;
  // 5. the parameters, and the persistent grid must be co-resident
  CK(cudaMemcpyAsync(h->d_params, &p, sizeof(DevParams), cudaMemcpyHostToDevice, h->stream));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k->fn, k->block, pl.smem));
  if (occ < 1 || occ * h->sm_count < p.grid) return fail(h, CCSIM_ECUDA, "persistent grid %d does not fit (occupancy %d x %d SMs)", p.grid, occ, h->sm_count);
  pl.kern = k;
  pl.valid = true;
  return CCSIM_OK;
}

extern "C" int ccsim_prepare(ccsim_handle *h, int64_t max_pods) {
  if (!h) return fail(h, CCSIM_EINVAL, "null argument");
  int rc = run_prepare(h, max_pods);
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->stream));     // allocations and restores are done when this returns
  return CCSIM_OK;
}

extern "C" int ccsim_run(ccsim_handle *h, int64_t max_pods, ccsim_result *out) {
  if (!h || !out) return fail(h, CCSIM_EINVAL, "null argument");
  if (!(h->plan.valid && h->plan.max_pods == max_pods)) { int rc = run_prepare(h, max_pods); if (rc) return rc; }
  RunPlan &pl = h->plan;
  pl.valid = false;                          // one launch per preparation: the working columns are consumed by the run
  memset(out, 0, sizeof(*out));
  out->n_nodes = h->n_global;
  if (pl.empty) { out->placed = 0; out->stop_code = CCSIM_STOP_UNSCHEDULABLE; out->pod_node = nullptr; return CCSIM_OK; }
  CK(cudaSetDevice(h->cfg.device));
  const int32_t n = h->n;
  cudaStream_t s = h->stream;
  DevParams &p = pl.p; LeanParams &lp = pl.lp; MultiParams &mp = pl.mp; StreamParams &sp = pl.sp;
  const WaveKernel &k = *pl.kern;
  const int grid = p.grid; const size_t smem = pl.smem;
  const bool stream = k.engine == ENG_STREAM;
  void *args[] = { (void *)&p, stream ? (void *)&sp : (void *)&lp, (void *)&mp };
  CK(cudaEventRecord(h->ev0, s));
  // Cooperative launch = the driver guarantees that the whole persistent grid is co-resident (the kernels never use grid.sync()).
  // Ranks that share a process (ccsim_peer_import_local) may share a device; cooperative launches of different streams are not
  // run concurrently there, so those ranks use a plain launch: the occupancy check above still holds for each grid on its own.
  if (h->peers_local) CK(cudaLaunchKernel(k.fn, dim3(grid), dim3(k.block), args, smem, s));
  else CK(cudaLaunchCooperativeKernel(k.fn, dim3(grid), dim3(k.block), args, smem, s));
  h->launches++;
  CK(cudaEventRecord(h->ev1, s));
  DevOut ho;
  CK(cudaMemcpyAsync(&ho, h->d_out, sizeof(DevOut), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (ho.error) return fail(h, CCSIM_ECUDA, "wave kernel aborted (error %d: %s)", ho.error, ho.error == 1 ? "exchange watchdog / output overflow" : "?");
  float ms = 0.f; CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  if (stream && (p.debug_flags & DBG_CYCLES) && h->cfg.world == 1 && ho.waves > 0) {     // per-CTA cycle split of the streaming kernel (kernel experiments)
    std::vector<unsigned long long> d((size_t)grid * 4);
    CK(cudaMemcpy(d.data(), h->d_xslots + XLINES_OFF, d.size() * 8, cudaMemcpyDeviceToHost));
    const char *nm[4] = {"mbarrier wait", "scan", "exchange", "rest"};
    for (int q = 0; q < 4; q++) {
      double mn = 1e30, mx = 0, sum = 0; int amx = 0, amn = 0;
      for (int c = 0; c < grid; c++) { const double v = (double)d[(size_t)c * 4 + q] / (double)ho.waves; sum += v; if (v > mx) { mx = v; amx = c; } if (v < mn) { mn = v; amn = c; } }
      fprintf(stderr, "[ccsim stream per-CTA cycles/wave] %-14s min %.0f (CTA %d)  mean %.0f  max %.0f (CTA %d)\n", nm[q], mn, amn, sum / grid, mx, amx);
    }
  }
#ifdef CCSIM_PHASE_TIMERS
  fprintf(stderr, "[ccsim %s tile %zu B smem] ", k.name, smem);
  fprintf(stderr, "[ccsim phases, CTA0 cycles/wave] scan=%.0f S1=%.0f publish=%.0f gather=%.0f commit=%.0f S2=%.0f (waves=%lld, %.3f ms)\n",
          (double)ho.phase_cycles[0] / ho.waves, (double)ho.phase_cycles[1] / ho.waves, (double)ho.phase_cycles[2] / ho.waves,
          (double)ho.phase_cycles[3] / ho.waves, (double)ho.phase_cycles[4] / ho.waves, (double)ho.phase_cycles[5] / ho.waves,
          (long long)ho.waves, ms);
  fprintf(stderr, "[ccsim phases 6/7] %.0f %.0f\n", (double)ho.phase_cycles[6] / ho.waves, (double)ho.phase_cycles[7] / ho.waves);
#endif
#ifdef MULTI_GATHER_PROFILE
  if (k.engine == ENG_MULTI && ho.waves > 0) {     // skew of the publishes per wave on the clock all SMs share: latest CTA minus CTA 0
    const long long nw = std::min<long long>(ho.waves, GP_MAX_WAVES);
    std::vector<long long> t((size_t)nw * CCSIM_MAX_GRID), skew((size_t)nw);
    CK(cudaMemcpyFromSymbol(t.data(), gp_pub_ns, t.size() * sizeof(long long)));
    for (long long w = 0; w < nw; w++) {
      long long mx = t[(size_t)w * CCSIM_MAX_GRID];
      for (int c = 1; c < grid; c++) mx = std::max(mx, t[(size_t)w * CCSIM_MAX_GRID + c]);
      skew[(size_t)w] = mx - t[(size_t)w * CCSIM_MAX_GRID];
    }
    std::sort(skew.begin(), skew.end());
    fprintf(stderr, "gather profile: publish skew (latest CTA - CTA 0, %%globaltimer) over %lld waves: median %lld ns, max %lld ns\n",
            nw, skew[(size_t)nw / 2], skew.back());
  }
#endif
  if (h->cfg.world > 1) h->xwave0 += (uint32_t)ho.waves;    // identical on every rank: the engines run the same waves everywhere
  h->last_stat[0] = k.engine; h->last_stat[1] = ho.waves; h->last_stat[2] = ho.placed;
  h->last_stat[3] = ho.stat[0]; h->last_stat[4] = ho.stat[1]; h->last_stat[5] = grid; h->last_stat[6] = k.block; h->last_stat[7] = (int64_t)smem;
  for (int q = 0; q < 8; q++) h->last_stat[8 + q] = ho.phase_cycles[q];
  h->last_key_order_waves = k.engine == ENG_MULTI ? (ho.stat[3] & 0xffffffffll) : 0;
  h->last_sorted_tile_waves = k.engine == ENG_MULTI ? (int64_t)((unsigned long long)ho.stat[3] >> 32) : 0;
  out->placed = ho.placed; out->stop_code = ho.stop_code; out->waves = ho.waves; out->evals = ho.evals; out->run_ms = ms;
  out->examined = ho.examined ? ho.examined : ho.evals;
  h->last_placed = ho.placed;
  if (ho.stop_code == CCSIM_STOP_UNSCHEDULABLE) {
    const int ti = (int)(ho.placed % h->n_templates);
    ccsim_diag_kernel<<<std::min(4 * h->sm_count, (n + 255) / 256), 256, 0, s>>>(p, ti);
    h->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&ho, h->d_out, sizeof(DevOut), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int r = 0; r < CCSIM_R_TOTAL; r++) out->reason_hist[r] = (int64_t)ho.reason_hist[r];
    out->preempt_no_victims = (int64_t)ho.preempt_no_victims;
    out->preempt_not_helpful = (int64_t)h->n - (int64_t)ho.preempt_no_victims;   // per shard, like reason_hist: sums to N - no_victims
  }
  h->h_pod_node.resize((size_t)ho.placed);
  if (ho.placed) CK(cudaMemcpyAsync(h->h_pod_node.data(), h->d_pod_node, (size_t)ho.placed * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  out->pod_node = h->h_pod_node.data();
  return CCSIM_OK;
}

// Entries of tree level l (l >= 1) over all classes of an analysis: sum_c ceil(n_c / 32^l) <= ceil(N / 32^l) + classes
static long long each_level_bound(long long n, int l, int ncls) {
  const long long span = 1ll << (5 * l);
  return (n + span - 1) / span + ncls;
}

extern "C" int ccsim_run_each(ccsim_handle *h, int64_t max_pods, ccsim_result *out) {
  if (!h || !out) return fail(h, CCSIM_EINVAL, "null argument");
  if (!h->have_nodes || !h->have_templates) return fail(h, CCSIM_ESTATE, "load_nodes and set_templates must come first");
  const int T = h->n_templates;
  // the per-analysis kernel covers node-local templates only: placing a clone must change nothing but its node
  if (h->cfg.world > 1) return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: node-sharded runs (world %d) are not supported", h->cfg.world);
  if (h->cfg.sampling == CCSIM_SAMPLING_REFERENCE) return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: reference sampling is not supported");
  // one counter table and one placed mask describe one run; ccsim_set_analyses gives every analysis its own
  if (h->n_counters > 0)
    return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: per-domain counters (topology spread, pod (anti-)affinity) are not supported");
  if (h->w_placed && !h->analyses) return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: hostPorts (placed mask) are not supported");
  for (int t = 0; t < T; t++) {
    const ccsim_template &P = h->h_templates[t];
    if ((P.n_pref_terms > 0 && (P.score_enable & CCSIM_PL_NODE_AFFINITY)) || (P.n_spts > 0 && (P.score_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD)) ||
        (P.n_ipa_score > 0 && (P.score_enable & CCSIM_PL_INTER_POD_AFFINITY)))
      return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: template %d has a normalised soft scorer (preferred nodeAffinity, ScheduleAnyway spreading, pod-affinity scoring)", t);
  }
  CK(cudaSetDevice(h->cfg.device));
  int rc;
  if (h->an.empty() && (rc = build_analyses(h, nullptr))) return rc;   // ccsim_set_templates: node-local analyses, no terms
  // every analysis is bounded like a run of its template alone (check_run_bounds); the sequences hold the largest bound
  int64_t cap = 1;
  int nseg = 1;          // most tree segments of an analysis
  bool terms = false;    // some analysis has counters or a hostPort self-conflict
  for (int t = 0; t < T; t++) {
    const AnalysisState &S = h->an[t];
    const bool fit_off = !(h->h_templates[t].filter_enable & CCSIM_PL_FIT);
    int64_t c = 0;
    if (!run_cap(h, max_pods, fit_off, c))
      return fail(h, CCSIM_EUNSUPPORTED, "template %d: NodeResourcesFit is disabled: the run is unbounded, --max-limit is required", t);
    cap = std::max(cap, c);
    char who[32]; snprintf(who, sizeof(who), "analysis %d: ", t);
    if ((rc = check_counter_bounds(h, max_pods, fit_off, S.terms.n_counters, S.terms.counters, S.range, S.dom_slots, who))) return rc;
    nseg = std::max(nseg, S.terms.n_seg);
    terms |= S.terms.n_counters > 0 || S.terms.port_self;
  }
  const int32_t n = h->n;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const double seq_bytes = (double)T * (double)cap * 4.0;
  if (seq_bytes > (double)free_b)
    return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: the sequence buffers (%d x %lld x 4 B = %.2f GiB) exceed free device memory (%.2f GiB)",
                T, (long long)cap, seq_bytes / (1 << 30), (double)free_b / (1 << 30));
  // tree shape: roots on level L (32^L >= N); levels [1, split) in global memory, [split, L] in shared memory, the lowest split whose
  // shared levels fit in `budget` bytes
  const int L = each_tree_levels(n);
  EachParams ep; memset(&ep, 0, sizeof(ep));
  auto shape = [&](size_t budget) {
    int split = 1;
    for (; split <= L + 1; split++) {
      size_t b = 0;
      for (int l = split; l <= L; l++) b += 8 * (size_t)each_level_bound(n, l, nseg);
      if (b <= budget) break;
    }
    long long g = 0, s = 0;
    for (int l = 1; l <= L; l++) {
      if (l < split) { ep.lev_off[l] = g; g += each_level_bound(n, l, nseg); }
      else { ep.lev_off[l] = s; s += each_level_bound(n, l, nseg); }
    }
    ep.split = split; ep.glev_stride = g; ep.slev_stride = s;
  };
  // one CTA per analysis, the shared levels next to the kernel's static structs, while the device holds every CTA at once (and always
  // for analyses with coupled terms); else node-local analyses share CTAs: A = ceil(T / SMs) of them (<= EACH_MAX_PACK), one warp's
  // placement loop and one share of the opt-in shared memory each
  const WaveKernel *kern = &WAVE_KERNELS[terms ? WK_EACH_TERMS : WK_EACH];
  shape(h->smem_optin - kern->static_smem - 1024);
  size_t smem = 8 * (size_t)ep.slev_stride;
  int per_cta = 1;
  if (!terms) {
    int resident = 0;   // CTAs of the one-per-analysis launch an SM holds
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern->fn, kern->block, smem));
    const uint32_t dbg = getenv("CCSIM_DEBUG_FLAGS") ? (uint32_t)atoi(getenv("CCSIM_DEBUG_FLAGS")) : 0u;
    if (T > std::max(1, resident) * h->sm_count && !(dbg & DBG_EACH_ONE_PER_CTA)) {
      per_cta = std::min<int>(EACH_MAX_PACK, (T + h->sm_count - 1) / h->sm_count);
      kern = &WAVE_KERNELS[WK_EACH_PACKED];
      shape((h->smem_optin - 1024 - (size_t)per_cta * sizeof(EachShared)) / (size_t)per_cta);
      smem = (size_t)per_cta * (sizeof(EachShared) + 8 * (size_t)ep.slev_stride);
    }
  }
  const int grid = (T + per_cta - 1) / per_cta;
  ep.n_levels = L; ep.max_pods = max_pods; ep.seq_cap = cap; ep.pack = per_cta; ep.n_analyses = T;
  {   // everything the run allocates per analysis, and the topology columns ccsim_set_analyses holds, against free device memory
    double topo = 0;
    for (int t = 0; t < T; t++) topo += (double)h->an[t].n_topo * n * 4.0;
    const double need = (double)T * ((double)n * 12.0 + (double)ep.glev_stride * 8.0 + (double)cap * 4.0 + sizeof(EachOut) + sizeof(DevOut)) + topo;
    if (need > (double)free_b)
      return fail(h, CCSIM_EUNSUPPORTED, "per-analysis runs: the per-analysis device state (%d analyses x %d nodes: clone counts and leaves, tree levels, "
                  "sequences, diagnosis outputs, topology columns = %.2f GiB) exceeds free device memory (%.2f GiB)",
                  T, n, need / (1 << 30), (double)free_b / (1 << 30));
  }
  h->plan = RunPlan();
  h->each_ran = false;
  memset(out, 0, sizeof(ccsim_result) * (size_t)T);
  const int split = ep.split;
  free_pool(h, h->each_allocs);
  const size_t tn = (size_t)T * (size_t)n;
  if ((rc = dev_alloc<int32_t>(h, h->each_allocs, &ep.k, tn)) || (rc = dev_alloc<unsigned long long>(h, h->each_allocs, &ep.leaf, tn)) ||
      (rc = dev_alloc<unsigned long long>(h, h->each_allocs, &ep.glev, (size_t)T * ep.glev_stride)) ||
      (rc = dev_alloc<int32_t>(h, h->each_allocs, &ep.seq, (size_t)T * cap)) || (rc = dev_alloc<EachOut>(h, h->each_allocs, &ep.out, (size_t)T)))
    return rc;
  DevOut *d_diag = nullptr;
  if ((rc = dev_alloc<DevOut>(h, h->each_allocs, &d_diag, (size_t)T))) return rc;
  ep.terms = h->d_terms;
  ep.diag = d_diag;
  ep.s_req_cpu = h->s_req_cpu; ep.s_req_mem = h->s_req_mem; ep.s_req_eph = h->s_req_eph; ep.s_nz_cpu = h->s_nz_cpu; ep.s_nz_mem = h->s_nz_mem;
  ep.s_npods = h->s_npods;
  for (int q = 0; q < h->meta.n_scalars; q++) ep.s_req_scalar[q] = h->s_req_scalar[q];
  h->d_each_seq = ep.seq; h->each_seq_cap = cap;
  cudaStream_t s = h->stream;
  std::vector<EachOut> eo((size_t)T);
  std::vector<DevOut> diag((size_t)T);
  float ms = 0.f;
  if (n > 0) {
    DevParams p;
    fill_params(h, p, max_pods);
    CK(cudaMemcpyAsync(h->d_params, &p, sizeof(DevParams), cudaMemcpyHostToDevice, s));   // filter_extras reads p.self
    CK(cudaMemsetAsync(d_diag, 0, sizeof(DevOut) * (size_t)T, s));
    void *args[] = { (void *)&p, (void *)&ep };
    CK(cudaEventRecord(h->ev0, s));
    CK(cudaLaunchKernel(kern->fn, dim3(grid), dim3(kern->block), args, smem, s));
    h->launches++;
    CK(cudaEventRecord(h->ev1, s));
    CK(cudaMemcpyAsync(eo.data(), ep.out, sizeof(EachOut) * (size_t)T, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    for (int t = 0; t < T; t++) if (eo[t].error) return fail(h, CCSIM_ECUDA, "per-analysis kernel: analysis %d overflowed its sequence buffer", t);
    // the terminal diagnosis of every Unschedulable analysis: its final state into the working columns, then the wave kernels' pass
    for (int t = 0; t < T; t++) {
      if (eo[t].stop_code != CCSIM_STOP_UNSCHEDULABLE) continue;
      const int blocks = std::min(4 * h->sm_count, (n + 255) / 256);
      ccsim_each_scatter_kernel<<<blocks, 256, 0, s>>>(p, ep, t);
      DevParams pd = p;   // the analysis's own counters (where the run left them) and columns
      const AnalysisState &S = h->an[t];
      pd.n_counters = S.terms.n_counters; pd.n_topo = S.n_topo;
      for (int j = 0; j < S.terms.n_counters; j++) { pd.counters[j] = S.terms.counters[j]; pd.final_off[j] = S.final_off[j]; }
      pd.final_cnt = S.work;
      for (int k = 0; k < CCSIM_MAX_TOPO_COLS; k++) pd.topo[k] = S.terms.topo[k];
      pd.out = d_diag + t;
      ccsim_diag_kernel<<<blocks, 256, 0, s>>>(pd, t);
      h->launches += 2;
      CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(diag.data(), d_diag, sizeof(DevOut) * (size_t)T, cudaMemcpyDeviceToHost, s));
  } else {
    for (int t = 0; t < T; t++) { eo[t].placed = 0; eo[t].stop_code = CCSIM_STOP_UNSCHEDULABLE; }   // ErrNoNodesAvailable: the host formats it
  }
  h->each_placed.assign((size_t)T, 0);
  h->each_seq.assign((size_t)T, std::vector<int32_t>());
  for (int t = 0; t < T; t++) {
    h->each_placed[t] = eo[t].placed;
    h->each_seq[t].resize((size_t)eo[t].placed);
    if (eo[t].placed) CK(cudaMemcpyAsync(h->each_seq[t].data(), ep.seq + (size_t)t * cap, (size_t)eo[t].placed * 4, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  int64_t waves = 0, placed = 0, rebuilds = 0;
  for (int t = 0; t < T; t++) {
    ccsim_result &r = out[t];
    rebuilds += n > 0 ? eo[t].rebuilds : 0;
    const bool unsched = eo[t].stop_code == CCSIM_STOP_UNSCHEDULABLE;
    r.placed = eo[t].placed; r.stop_code = eo[t].stop_code; r.n_nodes = h->n_global;
    r.waves = eo[t].placed + (unsched ? 1 : 0);
    r.evals = n > 0 ? (int64_t)n + eo[t].placed : 0;        // every node once, then the winner of each placement
    r.examined = r.waves * (int64_t)n;                       // what the reference's scheduling cycles examine
    if (unsched && n > 0) {
      for (int q = 0; q < CCSIM_R_TOTAL; q++) r.reason_hist[q] = (int64_t)diag[t].reason_hist[q];
      r.preempt_no_victims = (int64_t)diag[t].preempt_no_victims;
      r.preempt_not_helpful = (int64_t)n - r.preempt_no_victims;
    }
    r.run_ms = ms;                                           // the whole launch: the analyses run concurrently
    r.pod_node = h->each_seq[t].data();
    waves += r.waves; placed += r.placed;
  }
  h->plan.kern = kern;
  memset(h->last_stat, 0, sizeof(h->last_stat));
  h->last_stat[0] = ENG_EACH; h->last_stat[1] = waves; h->last_stat[2] = placed;
  h->last_stat[3] = std::min(split - 1, L); h->last_stat[4] = L - std::min(split - 1, L);   // upper tree levels in global / shared memory
  h->last_stat[5] = grid; h->last_stat[6] = kern->block; h->last_stat[7] = (int64_t)smem;
  h->last_stat[8] = rebuilds;                                                                 // leaf and level rebuilds, all analyses
  h->last_stat[9] = per_cta;                                                                  // analyses per CTA
  h->last_key_order_waves = 0;
  h->last_sorted_tile_waves = 0;
  h->each_ran = true;
  return CCSIM_OK;
}

extern "C" int ccsim_node_counts(ccsim_handle *h, int32_t t, int32_t *counts, int64_t *first_pod) {
  if (!h || !counts || !first_pod) return fail(h, CCSIM_EINVAL, "null argument");
  if (!h->have_templates || t < 0 || t >= h->n_templates) return fail(h, CCSIM_EINVAL, "template index");
  CK(cudaSetDevice(h->cfg.device));
  if (h->each_ran && t >= (int32_t)h->each_placed.size()) return fail(h, CCSIM_EINVAL, "analysis index");
  const int32_t N = h->n_global;
  int32_t *d_counts = nullptr; unsigned long long *d_first = nullptr;
  CK(cudaMalloc((void **)&d_counts, (size_t)(N ? N : 1) * 4));
  CK(cudaMalloc((void **)&d_first, (size_t)(N ? N : 1) * 8));
  CK(cudaMemsetAsync(d_counts, 0, (size_t)N * 4, h->stream));
  CK(cudaMemsetAsync(d_first, 0xFF, (size_t)N * 8, h->stream));
  // after ccsim_run_each: analysis t's own sequence, every pod of it a clone of template t
  const int32_t *seq = h->each_ran ? h->d_each_seq + (size_t)t * h->each_seq_cap : h->d_pod_node;
  const long long placed = h->each_ran ? h->each_placed[t] : h->last_placed;
  if (placed > 0) {
    ccsim_count_kernel<<<std::min<long long>(4 * h->sm_count, (placed + 255) / 256), 256, 0, h->stream>>>(
        seq, placed, h->each_ran ? 1 : h->n_templates, h->each_ran ? 0 : t, d_counts, d_first);
    h->launches++;
  }
  CK(cudaMemcpyAsync(counts, d_counts, (size_t)N * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(first_pod, d_first, (size_t)N * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  cudaFree(d_counts); cudaFree(d_first);
  return CCSIM_OK;
}

extern "C" int ccsim_device_info(ccsim_handle *h, int32_t *sm_count, int32_t *grid, int32_t *block, int64_t *l2_bytes) {
  if (!h) return CCSIM_EINVAL;
  if (sm_count) *sm_count = h->sm_count;
  if (grid) *grid = h->grid;
  if (block) *block = BLOCK_THREADS;
  if (l2_bytes) *l2_bytes = (int64_t)h->l2_bytes;
  return CCSIM_OK;
}

extern "C" int64_t ccsim_kernel_launches(const ccsim_handle *h) { return h ? h->launches : 0; }

extern "C" const char *ccsim_kernel_name(const ccsim_handle *h) { return h && h->plan.kern ? h->plan.kern->name : ""; }

extern "C" int ccsim_run_stats(const ccsim_handle *h, int64_t out[16]) {
  if (!h || !out) return CCSIM_EINVAL;
  memcpy(out, h->last_stat, sizeof(h->last_stat));
  return CCSIM_OK;
}

extern "C" int64_t ccsim_key_order_waves(const ccsim_handle *h) { return h ? h->last_key_order_waves : 0; }
extern "C" int64_t ccsim_sorted_tile_waves(const ccsim_handle *h) { return h ? h->last_sorted_tile_waves : 0; }

extern "C" int ccsim_flush_l2(ccsim_handle *h) {
  if (!h) return CCSIM_EINVAL;
  CK(cudaSetDevice(h->cfg.device));
  const size_t bytes = std::max<size_t>(2 * h->l2_bytes, (size_t)256 << 20);
  if (h->flush_bytes < bytes) {
    cudaFree(h->d_flush); h->d_flush = nullptr; h->flush_bytes = 0;
    CK(cudaMalloc(&h->d_flush, bytes));
    h->flush_bytes = bytes;
  }
  ccsim_flush_kernel<<<h->sm_count * 4, 512, 0, h->stream>>>((unsigned long long *)h->d_flush, bytes / 8, (unsigned long long)h->launches);
  h->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(h->stream));
  return CCSIM_OK;
}

extern "C" int ccsim_peer_export(ccsim_handle *h, uint8_t handle_out[CCSIM_IPC_HANDLE_BYTES]) {
  if (!h || !handle_out) return fail(h, CCSIM_EINVAL, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  cudaIpcMemHandle_t mh;
  CK(cudaIpcGetMemHandle(&mh, h->d_xslots));
  static_assert(sizeof(mh) == CCSIM_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t size");
  memcpy(handle_out, &mh, sizeof(mh));
  return CCSIM_OK;
}

extern "C" int ccsim_peer_local(ccsim_handle *h, void **ptr_out) {
  if (!h || !ptr_out) return fail(h, CCSIM_EINVAL, "null argument");
  *ptr_out = h->d_xslots;
  return CCSIM_OK;
}

extern "C" int ccsim_peer_import_local(ccsim_handle *h, int32_t world, void *const *ptrs) {
  if (!h || !ptrs) return fail(h, CCSIM_EINVAL, "null argument");
  if (world != h->cfg.world) return fail(h, CCSIM_EINVAL, "world %d != configured %d", world, h->cfg.world);
  for (int r = 0; r < world; r++) {
    if (!ptrs[r]) return fail(h, CCSIM_EINVAL, "null peer pointer %d", r);
    h->x_peer[r] = r == h->cfg.rank ? h->d_xslots : (unsigned long long *)ptrs[r];
  }
  h->peers_local = true;
  h->peers_ready = true;
  return CCSIM_OK;
}

extern "C" int ccsim_peer_import(ccsim_handle *h, int32_t world, const uint8_t *handles) {
  if (!h || !handles) return fail(h, CCSIM_EINVAL, "null argument");
  if (world != h->cfg.world) return fail(h, CCSIM_EINVAL, "world %d != configured %d", world, h->cfg.world);
  CK(cudaSetDevice(h->cfg.device));
  for (int r = 0; r < world; r++) {
    if (r == h->cfg.rank) { h->x_peer[r] = h->d_xslots; continue; }
    cudaIpcMemHandle_t mh;
    memcpy(&mh, handles + (size_t)r * CCSIM_IPC_HANDLE_BYTES, sizeof(mh));
    void *ptr = nullptr;
    CK(cudaIpcOpenMemHandle(&ptr, mh, cudaIpcMemLazyEnablePeerAccess));
    h->x_peer[r] = (unsigned long long *)ptr;
  }
  h->peers_ready = true;
  return CCSIM_OK;
}
