// encoder.hpp — Node/Pod objects -> the flat snapshot of include/ccsim.h (SURVEY.md §8 rows A1-A3, f1).
//
// What the reference builds incrementally through informer events, reproduced here in one pass:
//   node order        nodeTree.addNode / list(): zones in first-seen order, round-robin across zones
//                     (kubernetes/pkg/scheduler/backend/cache/node_tree.go:51-67,119-143); nodes enter in the order of the
//                     source List() minus --exclude-nodes (pkg/framework/simulator.go:203-215)
//   NodeInfo          SetNode: Allocatable (framework/types.go:461-465); AddPodInfo/update: Requested, NonZeroRequested,
//                     len(Pods), UsedPorts, PodsWithRequiredAntiAffinity (types.go:333-343,409-427); pods whose node is
//                     unknown/excluded are dropped (backend/cache/cache.go:439-443,223); terminal pods never enter
//                     (simulator.go:196)
//   PodInfo           CalculateResource (types.go:700-734)
// and the per-template PreFilter/PreScore state is folded into ccsim_template / ccsim_counter (static bits, masks,
// per-domain initial counts).
#pragma once
#include <thread>
#include <mutex>
#include <system_error>
#include <condition_variable>
#include <pthread.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <exception>
#include <unordered_map>
#include <unordered_set>
#include <string_view>
#include <cstring>
#include <functional>
#include "../../../include/ccsim.h"
#include "objects.hpp"

namespace cch {

struct Unsupported : std::runtime_error { using std::runtime_error::runtime_error; };

struct SchedConfig {
  int pct_nodes_to_score = 100;   // canonical contract unless "sampling":"reference" asks for the reference's adaptive sampling
  bool reference_sampling = false;
  uint32_t filter_enable = CCSIM_PL_ALL, score_enable = CCSIM_PL_ALL;
  int w_taint = 3, w_node_affinity = 2, w_fit = 1, w_pts = 2, w_ipa = 2, w_balanced = 1, w_image = 1;
  int hard_pod_affinity_weight = 1;   // InterPodAffinityArgs.HardPodAffinityWeight (apis/config/v1/defaults.go:206-209)
  static uint32_t plugin_bit(const std::string &n) {
    if (n == "NodeUnschedulable") return CCSIM_PL_NODE_UNSCHEDULABLE;
    if (n == "NodeName") return CCSIM_PL_NODE_NAME;
    if (n == "TaintToleration") return CCSIM_PL_TAINT_TOLERATION;
    if (n == "NodeAffinity") return CCSIM_PL_NODE_AFFINITY;
    if (n == "NodePorts") return CCSIM_PL_NODE_PORTS;
    if (n == "NodeResourcesFit") return CCSIM_PL_FIT;
    if (n == "PodTopologySpread") return CCSIM_PL_POD_TOPOLOGY_SPREAD;
    if (n == "InterPodAffinity") return CCSIM_PL_INTER_POD_AFFINITY;
    if (n == "NodeResourcesBalancedAllocation") return CCSIM_PL_BALANCED;
    if (n == "ImageLocality") return CCSIM_PL_IMAGE_LOCALITY;
    return 0;
  }
  static SchedConfig parse(const std::string &text) {
    SchedConfig c;
    if (text.empty()) return c;
    Json j = parse_json(text);
    c.reference_sampling = j.at("sampling").str() == "reference";
    c.pct_nodes_to_score = (int)j.at("percentageOfNodesToScore").i64(c.reference_sampling ? 0 : 100);
    for (auto &x : j.at("disabledFilters").arr) c.filter_enable &= ~plugin_bit(x.str());
    for (auto &x : j.at("disabledScores").arr) c.score_enable &= ~plugin_bit(x.str());
    if (!j.at("hardPodAffinityWeight").is_null()) c.hard_pod_affinity_weight = (int)j.at("hardPodAffinityWeight").i64(1);
    const Json &w = j.at("weights");
    if (w.is_object())
      for (auto &kv : w.obj) {
        // getScoreWeights (framework.go:487-497): an explicit 0 means the default of 1; weights are never negative
        const long long raw = kv.second.i64(1);
        if (raw < 0) throw std::runtime_error("score weight of " + kv.first + " is negative: " + std::to_string(raw));
        if (raw > INT32_MAX) throw std::runtime_error("score weight of " + kv.first + " is too large: " + std::to_string(raw));
        const int v = raw == 0 ? 1 : (int)raw;
        if (kv.first == "TaintToleration") c.w_taint = v; else if (kv.first == "NodeAffinity") c.w_node_affinity = v;
        else if (kv.first == "NodeResourcesFit") c.w_fit = v; else if (kv.first == "PodTopologySpread") c.w_pts = v;
        else if (kv.first == "InterPodAffinity") c.w_ipa = v; else if (kv.first == "NodeResourcesBalancedAllocation") c.w_balanced = v;
        else if (kv.first == "ImageLocality") c.w_image = v;
      }
    return c;
  }
};

struct PodResource { int64_t cpu = 0, mem = 0, eph = 0; std::map<std::string, int64_t> scalar; int64_t non0_cpu = 0, non0_mem = 0; };

// Resource.Add over a ResourceList (framework/types.go:979-1001)
inline void resource_add(PodResource &r, const ResourceList &rl) {
  for (auto &kv : rl) {
    if (kv.first == "cpu") r.cpu += kv.second.milli_value();
    else if (kv.first == "memory") r.mem += kv.second.value();
    else if (kv.first == "ephemeral-storage") r.eph += kv.second.value();
    else if (kv.first == "pods") {}
    else if (is_scalar_resource_name(kv.first)) r.scalar[kv.first] += kv.second.value();
  }
}

inline ResourceList default_non_missing() {
  ResourceList d;
  d["cpu"] = Quantity::parse("100m");          // schedutil.DefaultMilliCPURequest
  d["memory"] = Quantity::parse("209715200");  // schedutil.DefaultMemoryRequest = 200 * 1024 * 1024
  return d;
}

// PodInfo.CalculateResource (framework/types.go:700-734)
inline PodResource calculate_resource_general(const Pod &p);
// The common shape of an EXISTING pod — plain containers, no init containers / overhead / pod-level resources / resize status —
// needs none of resourcehelper.PodRequests' list arithmetic: the pod's request of a resource is the exact sum of its containers'
// quantities (Quantity.Add is exact; Value()/MilliValue() round the SUM up, quantity.go:812-834), and GetNonzeroRequests sees
// every container that names no cpu / memory at 100m / 200Mi (applyNonMissing). Same numbers as the general path
// (CCHOST_CHECK_FAST=1 computes both and compares), without a std::map per container: this runs once per pod of the snapshot.
inline PodResource calculate_resource(const Pod &p) {
  if (!p.init_containers.empty() || !p.overhead.empty() || !p.pod_level_requests.empty() || p.has_pod_level_requests ||
      !p.status_resources.empty() || !p.status_allocated.empty())
    return calculate_resource_general(p);
  static const i128 kDefCpu = Quantity::parse("100m").nanos, kDefMem = Quantity::parse("209715200").nanos;
  PodResource out;
  i128 cpu = 0, mem = 0, eph = 0, z_cpu = 0, z_mem = 0;
  bool any_cpu = false, any_mem = false;
  std::map<std::string, i128> scalar;     // (stays empty — no allocation — unless the pod requests an extended resource)
  for (auto &c : p.containers) {
    bool has_cpu = false, has_mem = false;
    for (auto &kv : c.requests) {
      if (kv.first == "cpu") { cpu += kv.second.nanos; z_cpu += kv.second.nanos; has_cpu = true; }
      else if (kv.first == "memory") { mem += kv.second.nanos; z_mem += kv.second.nanos; has_mem = true; }
      else if (kv.first == "ephemeral-storage") eph += kv.second.nanos;
      else if (kv.first == "pods") {}
      else if (is_scalar_resource_name(kv.first)) scalar[kv.first] += kv.second.nanos;
    }
    if (!has_cpu) z_cpu += kDefCpu;
    if (!has_mem) z_mem += kDefMem;
    any_cpu = true; any_mem = true;
  }
  out.cpu = (int64_t)Quantity::ceil_div(cpu, Quantity::pow10(6));
  out.mem = (int64_t)Quantity::ceil_div(mem, Quantity::pow10(9));
  out.eph = (int64_t)Quantity::ceil_div(eph, Quantity::pow10(9));
  for (auto &kv : scalar) out.scalar[kv.first] = (int64_t)Quantity::ceil_div(kv.second, Quantity::pow10(9));
  out.non0_cpu = any_cpu ? (int64_t)Quantity::ceil_div(z_cpu, Quantity::pow10(6)) : 0;
  out.non0_mem = any_mem ? (int64_t)Quantity::ceil_div(z_mem, Quantity::pow10(9)) : 0;
  static const bool check = getenv("CCHOST_CHECK_FAST") != nullptr;
  if (check) {
    const PodResource g = calculate_resource_general(p);
    if (g.cpu != out.cpu || g.mem != out.mem || g.eph != out.eph || g.scalar != out.scalar || g.non0_cpu != out.non0_cpu || g.non0_mem != out.non0_mem)
      throw std::runtime_error("calculate_resource: fast path differs from the general path for pod " + p.ns + "/" + p.name);
  }
  return out;
}
inline PodResource calculate_resource_general(const Pod &p) {
  PodResource out;
  ResourceList req = p.requests(/*use_status=*/true, /*skip_pod_level=*/false, nullptr);
  ResourceList nm;
  if (!p.has_pod_level_requests) nm = default_non_missing();
  else {
    ResourceList d = default_non_missing();
    for (auto &kv : d) if (!req.count(kv.first)) nm[kv.first] = kv.second;
  }
  ResourceList non0 = req;
  if (!nm.empty()) non0 = p.requests(true, false, &nm);
  resource_add(out, req);
  auto ic = non0.find("cpu"); auto im = non0.find("memory");
  out.non0_cpu = ic == non0.end() ? 0 : ic->second.milli_value();
  out.non0_mem = im == non0.end() ? 0 : im->second.value();
  return out;
}

// Host threads over an index range, in contiguous blocks (the per-node loops of the encoder are independent per node; anything
// order-dependent — dictionary ids in first-seen order — stays in a serial pass over the per-node results).
// host threads for the ingest and the encoder: the hardware's, at most 64 (CCHOST_THREADS overrides; the passes are bound by
// memory allocation and cache misses on the object model, more threads than that only add contention)
inline unsigned host_threads() {
  static const unsigned nt = [] {
    if (const char *e = getenv("CCHOST_THREADS")) { const int v = atoi(e); if (v > 0) return (unsigned)(v > 256 ? 256 : v); }
    const unsigned hw = std::thread::hardware_concurrency();
    return hw == 0 ? 1u : (hw > 64 ? 64u : hw);
  }();
  return nt;
}

// A persistent pool for the host passes. One analysis of the C4 cluster makes ~13 parallel passes (item location x2 and item parsing for
// nodes and pods, node / pod hashing, NodeInfo aggregation, one pass per constraint family ...); creating and joining 64 threads costs
// 1.5-2.5 ms each time, more than most of those passes take. Workers are created on first use and parked on a condition variable; the
// calling thread takes tasks too. One job at a time per process (callers from several host threads queue up); a task that starts a job
// itself runs it inline. The pool is never destroyed (no destructor-order trouble at process exit), and a forked child starts a new one.
class HostPool {
 public:
  static HostPool &instance() {
    HostPool *p = slot().load(std::memory_order_acquire);
    if (!p) {
      static std::mutex mk;
      std::lock_guard<std::mutex> g(mk);
      p = slot().load(std::memory_order_acquire);
      if (!p) {
        static std::once_flag once;
        std::call_once(once, [] { pthread_atfork(nullptr, nullptr, [] { slot().store(nullptr, std::memory_order_release); }); });
        p = new HostPool();
        slot().store(p, std::memory_order_release);
      }
    }
    return *p;
  }
  // fn(c) for every c in [0, n_tasks), on up to n_tasks threads; returns when all are done; the first exception is rethrown
  void run(unsigned n_tasks, const std::function<void(unsigned)> &fn) {
    if (n_tasks == 0) return;
    if (n_tasks == 1 || in_task()) { for (unsigned c = 0; c < n_tasks; c++) fn(c); return; }
    std::lock_guard<std::mutex> serial(run_mu_);
    std::unique_lock<std::mutex> lk(mu_);
    while (n_workers_ + 1 < n_tasks && n_workers_ < kMaxWorkers) {
      try { std::thread(&HostPool::worker, this).detach(); } catch (const std::system_error &) { break; }   // (thread limit reached: fewer workers, same result)
      n_workers_++;
    }
    fn_ = &fn; n_ = n_tasks; next_ = 0; remaining_ = n_tasks; err_ = nullptr; gen_++;
    cv_work_.notify_all();
    drain(lk);                                            // the caller works too
    cv_done_.wait(lk, [&] { return remaining_ == 0; });
    fn_ = nullptr;
    std::exception_ptr e = err_; err_ = nullptr;
    lk.unlock();
    if (e) std::rethrow_exception(e);
  }
 private:
  static constexpr unsigned kMaxWorkers = 255;
  static std::atomic<HostPool *> &slot() { static std::atomic<HostPool *> s{nullptr}; return s; }
  static bool &in_task() { static thread_local bool f = false; return f; }
  // takes tasks of the current job until none is left (mu_ held on entry and on exit)
  void drain(std::unique_lock<std::mutex> &lk) {
    while (next_ < n_) {
      const unsigned c = next_++;
      const std::function<void(unsigned)> *f = fn_;
      lk.unlock();
      in_task() = true;
      std::exception_ptr e;
      try { (*f)(c); } catch (...) { e = std::current_exception(); }
      in_task() = false;
      lk.lock();
      if (e && !err_) err_ = e;
      if (--remaining_ == 0) cv_done_.notify_all();
    }
  }
  void worker() {
    std::unique_lock<std::mutex> lk(mu_);
    uint64_t seen = 0;
    for (;;) {
      cv_work_.wait(lk, [&] { return gen_ != seen; });
      seen = gen_;
      drain(lk);
    }
  }
  std::mutex run_mu_, mu_;
  std::condition_variable cv_work_, cv_done_;
  const std::function<void(unsigned)> *fn_ = nullptr;
  unsigned n_ = 0, next_ = 0, remaining_ = 0, n_workers_ = 0;
  uint64_t gen_ = 0;
  std::exception_ptr err_;
};

template <class F> inline void parallel_for(int n, F fn) {
  unsigned nt = host_threads();
  if (n < 4096 || nt == 1) { for (int i = 0; i < n; i++) fn(i); return; }
  const int per = (n + (int)nt - 1) / (int)nt;
  HostPool::instance().run(nt, [&](unsigned c) { for (int i = (int)c * per, e = std::min(n, i + per); i < e; i++) fn(i); });
}

// String -> small integer index for the encoder's dictionaries (node names, topology values): open addressing over one flat
// array, hashes supplied by the caller — they are computed by the parallel per-node passes, so the serial first-seen-order pass that
// assigns ids (dictionary ids are order-dependent) costs a probe and a short memcmp per node instead of a hash + a heap node.
class FlatIndex {
 public:
  static uint64_t hash(std::string_view k) { return std::hash<std::string_view>()(k); }
  void init(size_t expected) {
    size_t cap = 16;
    while (cap < expected * 2 + 2) cap <<= 1;
    tab_.assign(cap, Slot{nullptr, 0, -1, 0});
    mask_ = cap - 1; size_ = 0;
  }
  // the slot of `k` (inserted with value `v` when new); .second = inserted
  std::pair<int32_t *, bool> emplace(std::string_view k, uint64_t h, int32_t v) {
    if ((size_ + 1) * 2 > tab_.size()) grow();
    for (size_t i = h & mask_;; i = (i + 1) & mask_) {
      Slot &s = tab_[i];
      if (!s.p) { s.p = k.data(); s.len = (uint32_t)k.size(); s.val = v; s.h = h; size_++; return {&s.val, true}; }
      if (s.h == h && s.len == k.size() && memcmp(s.p, k.data(), k.size()) == 0) return {&s.val, false};
    }
  }
  const int32_t *find(std::string_view k, uint64_t h) const {
    if (tab_.empty()) return nullptr;
    for (size_t i = h & mask_;; i = (i + 1) & mask_) {
      const Slot &s = tab_[i];
      if (!s.p) return nullptr;
      if (s.h == h && s.len == k.size() && memcmp(s.p, k.data(), k.size()) == 0) return &s.val;
    }
  }
  const int32_t *find(std::string_view k) const { return find(k, hash(k)); }
  size_t size() const { return size_; }
 private:
  struct Slot { const char *p; uint32_t len; int32_t val; uint64_t h; };
  void grow() {       // (pointers returned by emplace die here: callers that keep them size the table up front with init())
    std::vector<Slot> old; old.swap(tab_);
    tab_.assign(old.size() ? old.size() * 2 : 16, Slot{nullptr, 0, -1, 0});
    mask_ = tab_.size() - 1;
    for (auto &s : old) if (s.p) { size_t i = s.h & mask_; while (tab_[i].p) i = (i + 1) & mask_; tab_[i] = s; }
  }
  std::vector<Slot> tab_;
  size_t mask_ = 0, size_ = 0;
};

struct Encoded {
  int32_t n = 0;
  std::vector<std::string> names;
  std::vector<int64_t> alloc_cpu, alloc_mem, alloc_eph, req_cpu, req_mem, req_eph, nz_cpu, nz_mem;
  std::vector<int32_t> alloc_pods, npods;
  std::vector<std::string> scalar_names;
  std::vector<std::vector<int64_t>> alloc_scalar, req_scalar;
  int taint_words = 1, static_words = 0;
  std::vector<uint64_t> taint_mask, static_mask;   // word-major
  std::vector<Taint> taint_dict;
  uint64_t taint_nosched[CCSIM_MAX_TAINT_WORDS] = {0}, taint_prefer[CCSIM_MAX_TAINT_WORDS] = {0};
  std::vector<int32_t> taint_off;
  std::vector<uint8_t> taint_list;
  std::vector<std::vector<int32_t>> topo;
  std::vector<std::vector<int32_t>> counter_init;
  std::vector<ccsim_counter> counters;
  ccsim_template tmpl;
  std::vector<uint8_t> image_score;   // ImageLocality per node (empty: all zero)
  bool has_placed_mask = false;
  std::string prefilter_msg;   // non-empty: PreFilter rejected the pod for every node (e.g. conflicting metadata.name affinity)

  void fill_nodes(ccsim_nodes &nd) const {
    memset(&nd, 0, sizeof(nd));
    nd.n_nodes = n; nd.n_scalars = (int32_t)scalar_names.size(); nd.taint_words = taint_words; nd.static_words = static_words;
    nd.n_topo_cols = (int32_t)topo.size(); nd.has_placed_mask = has_placed_mask ? 1 : 0;
    nd.alloc_cpu = alloc_cpu.data(); nd.alloc_mem = alloc_mem.data(); nd.alloc_eph = alloc_eph.data(); nd.alloc_pods = alloc_pods.data();
    nd.req_cpu = req_cpu.data(); nd.req_mem = req_mem.data(); nd.req_eph = req_eph.data(); nd.npods = npods.data();
    nd.nz_cpu = nz_cpu.data(); nd.nz_mem = nz_mem.data();
    for (size_t k = 0; k < scalar_names.size(); k++) { nd.alloc_scalar[k] = alloc_scalar[k].data(); nd.req_scalar[k] = req_scalar[k].data(); }
    nd.taint_mask = taint_mask.data(); nd.static_mask = static_mask.data();
    for (size_t k = 0; k < topo.size(); k++) nd.topo[k] = topo[k].data();
    for (int w = 0; w < CCSIM_MAX_TAINT_WORDS; w++) { nd.taint_nosched[w] = taint_nosched[w]; nd.taint_prefer[w] = taint_prefer[w]; }
    nd.taint_list_off = taint_off.data(); nd.taint_list = taint_list.data();
  }
};

class Encoder {
 public:
  Encoder(const SchedConfig &cfg, const Pod &tmpl, const ObjList<Node> &nodes_in, const ObjList<Pod> &pods_in,
          const std::map<std::string, Labels> &ns_labels, const std::set<std::string> &exclude)
      : cfg_(cfg), t_(tmpl), ns_labels_(ns_labels) {
    // ---- node order: nodeTree (zones in first-seen order, round-robin) ----
    std::vector<const Node *> kept;
    for (auto &n : nodes_in) if (exclude.empty() || !exclude.count(n.name)) kept.push_back(&n);
    std::vector<std::string> zkey(kept.size());
    std::vector<uint64_t> nhash(kept.size());
    parallel_for((int)kept.size(), [&](int i) { zkey[i] = kept[i]->zone_key(); nhash[i] = FlatIndex::hash(kept[i]->name); });
    // (one index does both jobs: "already in the tree" and, once the order is known, name -> position; it is sized up front, so
    //  the slots handed out stay where they are)
    std::vector<std::vector<std::pair<const Node *, int32_t *>>> tree;   // one list per zone, zones in first-seen order
    std::unordered_map<std::string_view, int> zone_id;
    node_index_.init(kept.size());
    size_t total = 0;
    int last_zone = -1, cur_zone = 0;
    for (size_t i = 0; i < kept.size(); i++) {
      const Node *n = kept[i];
      auto ins = node_index_.emplace(std::string_view(n->name), nhash[i], -1);
      if (!ins.second) continue;   // "Did not add to the NodeTree because it already exists"
      if (last_zone < 0 || zkey[i] != zkey[(size_t)last_zone]) {     // (runs of nodes of one zone — or a cluster without zone labels — skip the lookup)
        auto it = zone_id.find(std::string_view(zkey[i]));
        if (it == zone_id.end()) { it = zone_id.emplace(std::string_view(zkey[i]), (int)tree.size()).first; tree.emplace_back(); }
        cur_zone = it->second; last_zone = (int)i;
      }
      tree[(size_t)cur_zone].push_back({n, ins.first});
      total++;
    }
    size_t idx = 0;
    nodes_.reserve(total);
    while (nodes_.size() < total) {
      for (auto &v : tree) if (idx < v.size()) { *v[idx].second = (int)nodes_.size(); nodes_.push_back(v[idx].first); }
      idx++;
    }
    // ---- pods: non-terminal, bound to a known node ----
    std::vector<int32_t> where(pods_in.size(), -1);
    std::vector<uint8_t> pflags(pods_in.size(), 0);   // what the rare-case passes of encode() look for, noted while the pod is in cache anyway
    parallel_for((int)pods_in.size(), [&](int j) {
      const Pod &p = pods_in[j];
      if (p.phase == "Succeeded" || p.phase == "Failed") return;
      if (p.node_name.empty()) return;   // pending pods are not replayed (documented deviation, DESIGN.md)
      const int32_t *it = node_index_.find(std::string_view(p.node_name));
      if (!it) return;
      where[j] = *it;
      pflags[j] = (uint8_t)((p.anti_required.empty() ? 0 : 1) | ((p.aff_required.empty() && p.aff_preferred.empty() && p.anti_preferred.empty()) ? 0 : 2) |
                            (p.priority < t_.priority ? 4 : 0));
    });
    pods_on_.build(nodes_.size(), where, pods_in);
    for (size_t j = 0; j < pods_in.size(); j++) {
      if (!pflags[j]) continue;
      if (pflags[j] & 1) anti_required_pods_.push_back({where[j], &pods_in[j]});
      if (pflags[j] & 2) affinity_term_pods_.push_back({where[j], &pods_in[j]});
      if (pflags[j] & 4) lower_priority_pod_ = true;
    }
    // node order, then source-list order within a node: the order in which a pass over pods_on_ would meet them (the topology keys of
    // the InterPodAffinity score get their counter slots in first-seen order)
    std::stable_sort(affinity_term_pods_.begin(), affinity_term_pods_.end(), [](auto &a, auto &b) { return a.first < b.first; });
  }

  // Services / RCs / ReplicaSets / StatefulSets of the snapshot: only helper.DefaultSelector reads them (system-default spreading)
  void set_workloads(const std::vector<WorkloadSelector> *w) { workloads_ = w; }

  Encoded encode() {
    Encoded e;
    memset(&e.tmpl, 0, sizeof(e.tmpl));
    const int n = (int)nodes_.size();
    const bool timing = getenv("CCHOST_TIMING") != nullptr;
    auto tlast = std::chrono::steady_clock::now();
    auto tick = [&](const char *what) {
      if (!timing) return;
      auto now = std::chrono::steady_clock::now();
      fprintf(stderr, "[cchost]   encode/%s %.3f s\n", what, std::chrono::duration<double>(now - tlast).count());
      tlast = now;
    };
    e.n = n;
    guards();
    // ---- template request vectors (A2) ----
    ccsim_template &T = e.tmpl;
    T.filter_enable = cfg_.filter_enable; T.score_enable = cfg_.score_enable;
    T.w_taint = cfg_.w_taint; T.w_node_affinity = cfg_.w_node_affinity; T.w_fit = cfg_.w_fit; T.w_pts = cfg_.w_pts;
    T.w_ipa = cfg_.w_ipa; T.w_balanced = cfg_.w_balanced; T.w_image = cfg_.w_image;
    T.least_w_cpu = 1; T.least_w_mem = 1;
    T.nodename_idx = -1; T.prefilter_bit = -1; T.spts_ignored_bit = -1;
    PodResource fit;     // computePodResourceRequest (fit.go:224-233): PodRequests with pod-level resources, SetMaxResource from zero
    resource_add(fit, t_.requests(false, false, nullptr));
    PodResource cr = calculate_resource(t_);   // what a committed clone adds (types.go:409-427)
    T.req_cpu = cr.cpu; T.req_mem = cr.mem; T.req_eph = cr.eph;
    T.nz_cpu = cr.non0_cpu; T.nz_mem = cr.non0_mem;
    if (fit.cpu != cr.cpu || fit.mem != cr.mem || fit.eph != cr.eph) throw Unsupported("template requests differ between Filter and NodeInfo accounting");
    for (auto &kv : fit.scalar) if (kv.second != 0) e.scalar_names.push_back(kv.first);
    if (e.scalar_names.size() > CCSIM_MAX_SCALARS) throw Unsupported("more than 4 extended resources requested");
    for (size_t k = 0; k < e.scalar_names.size(); k++) T.req_scalar[k] = fit.scalar[e.scalar_names[k]];
    {   // LeastAllocated pod request: pod-level resources skipped, non-zero defaults (resource_allocation.go:118-140; fit.go:186)
      ResourceList d = default_non_missing();
      ResourceList lr = t_.requests(false, true, &d);
      T.least_cpu = lr.count("cpu") ? lr["cpu"].milli_value() : 0;
      T.least_mem = lr.count("memory") ? lr["memory"].value() : 0;
      ResourceList br = t_.requests(true, false, nullptr);   // BalancedAllocation: useRequested, pod-level honoured
      T.bal_cpu = br.count("cpu") ? br["cpu"].milli_value() : 0;
      T.bal_mem = br.count("memory") ? br["memory"].value() : 0;
    }
    if (fit.cpu == 0 && fit.mem == 0 && fit.eph == 0 && fit.scalar.empty()) T.flags |= CCSIM_TF_FIT_ALL_ZERO;
    if (T.bal_cpu == 0 && T.bal_mem == 0) T.flags |= CCSIM_TF_BALANCED_SKIP;

    // ---- node columns (A1) ----
    e.names.resize(n);
    auto z64 = [&](std::vector<int64_t> &v) { v.assign(n, 0); };
    z64(e.alloc_cpu); z64(e.alloc_mem); z64(e.alloc_eph); z64(e.req_cpu); z64(e.req_mem); z64(e.req_eph); z64(e.nz_cpu); z64(e.nz_mem);
    e.alloc_pods.assign(n, 0); e.npods.assign(n, 0);
    e.alloc_scalar.assign(e.scalar_names.size(), std::vector<int64_t>(n, 0));
    e.req_scalar.assign(e.scalar_names.size(), std::vector<int64_t>(n, 0));
    parallel_for(n, [&](int i) {
      const Node &nd = *nodes_[i];
      e.names[i] = nd.name;
      for (auto &kv : nd.allocatable) {   // NewResource(node.Status.Allocatable)
        if (kv.first == "cpu") e.alloc_cpu[i] += kv.second.milli_value();
        else if (kv.first == "memory") e.alloc_mem[i] += kv.second.value();
        else if (kv.first == "ephemeral-storage") e.alloc_eph[i] += kv.second.value();
        else if (kv.first == "pods") e.alloc_pods[i] += (int32_t)kv.second.value();
        else for (size_t k = 0; k < e.scalar_names.size(); k++) if (kv.first == e.scalar_names[k]) e.alloc_scalar[k][i] += kv.second.value();
      }
      for (auto *p : pods_on_[i]) {
        PodResource pr = calculate_resource(*p);
        e.req_cpu[i] += pr.cpu; e.req_mem[i] += pr.mem; e.req_eph[i] += pr.eph;
        e.nz_cpu[i] += pr.non0_cpu; e.nz_mem[i] += pr.non0_mem;
        for (size_t k = 0; k < e.scalar_names.size(); k++) { auto it = pr.scalar.find(e.scalar_names[k]); if (it != pr.scalar.end()) e.req_scalar[k][i] += it->second; }
        e.npods[i] += 1;
      }
    });
    for (int i = 0; i < n; i++) {   // the engine refuses these too, by index; here the node is named
      if (e.alloc_cpu[i] > CCSIM_MAX_SCORED_ALLOCATABLE)
        throw Unsupported("node \"" + e.names[i] + "\": cpu allocatable " + std::to_string(e.alloc_cpu[i]) + "m exceeds " +
                          std::to_string(CCSIM_MAX_SCORED_ALLOCATABLE) + "m (LeastAllocated's int64 score arithmetic)");
      if (e.alloc_mem[i] > CCSIM_MAX_SCORED_ALLOCATABLE)
        throw Unsupported("node \"" + e.names[i] + "\": memory allocatable " + std::to_string(e.alloc_mem[i]) + " exceeds " +
                          std::to_string(CCSIM_MAX_SCORED_ALLOCATABLE) + " (LeastAllocated's int64 score arithmetic)");
    }
    tick("node columns");
    // ---- taints: dictionary in first-seen order ----
    std::map<Taint, int> tid;
    for (int i = 0; i < n; i++)
      for (auto &t : nodes_[i]->taints)
        if (!tid.count(t)) {
          int id = (int)e.taint_dict.size();
          if (id == CCSIM_TAINT_UNSCHEDULABLE_BIT) { e.taint_dict.push_back(Taint{"", "", "__reserved__"}); id++; }   // bit 63 of word 0 is reserved
          tid[t] = id; e.taint_dict.push_back(t);
        }
    if (e.taint_dict.size() > 64 * CCSIM_MAX_TAINT_WORDS || e.taint_dict.size() > 255) throw Unsupported("more than 255 distinct taints in the cluster");
    e.taint_words = std::max<int>(1, (int)(e.taint_dict.size() + 63) / 64);
    e.taint_mask.assign((size_t)e.taint_words * n, 0);
    e.taint_off.assign(n + 1, 0);
    for (int i = 0; i < n; i++) {
      for (auto &t : nodes_[i]->taints) { int id = tid[t]; e.taint_mask[(size_t)(id >> 6) * n + i] |= 1ull << (id & 63); e.taint_list.push_back((uint8_t)id); }
      e.taint_off[i + 1] = (int32_t)e.taint_list.size();
      if (nodes_[i]->unschedulable) e.taint_mask[i] |= 1ull << CCSIM_TAINT_UNSCHEDULABLE_BIT;
    }
    if (e.taint_list.empty()) e.taint_list.push_back(0);
    std::vector<Toleration> prefer_tols;   // getAllTolerationPreferNoSchedule (taint_toleration.go:129-137)
    for (auto &tl : t_.tolerations) if (tl.effect.empty() || tl.effect == "PreferNoSchedule") prefer_tols.push_back(tl);
    for (size_t id = 0; id < e.taint_dict.size(); id++) {
      const Taint &t = e.taint_dict[id];
      const int w = (int)id >> 6; const uint64_t b = 1ull << (id & 63);
      if (t.effect == "NoSchedule" || t.effect == "NoExecute") { e.taint_nosched[w] |= b; if (tolerations_tolerate(t_.tolerations, t)) T.tol_nosched[w] |= b; }
      if (t.effect == "PreferNoSchedule") { e.taint_prefer[w] |= b; if (tolerations_tolerate(prefer_tols, t)) T.tol_prefer[w] |= b; }
    }
    if (tolerations_tolerate(t_.tolerations, Taint{"node.kubernetes.io/unschedulable", "", "NoSchedule"})) T.flags |= CCSIM_TF_TOLERATES_UNSCHEDULABLE;

    tick("taints");
    // ---- static bits ----
    std::vector<std::vector<char>> bits;   // bits[b][i]
    auto new_bit = [&](const std::function<bool(int)> &f) { std::vector<char> v(n); for (int i = 0; i < n; i++) v[i] = f(i) ? 1 : 0; bits.push_back(v); return (int)bits.size() - 1; };
    auto set_mask = [&](uint64_t *m, int b) { m[b >> 6] |= 1ull << (b & 63); };
    // NodeAffinity (nodeaffinity.go:306-332; node_affinity.go:147-227)
    const bool no_affinity = !t_.has_required_node_affinity;
    if (!(no_affinity && !t_.has_node_selector)) {
      T.flags |= CCSIM_TF_HAS_NODE_SELECTOR;   // the Filter is not skipped
      if (!t_.node_selector.empty()) {
        Selector s = Selector::from_set(t_.node_selector);
        set_mask(T.sel_mask, new_bit([&](int i) { return s.matches(nodes_[i]->labels); }));
      }
      if (t_.has_required_node_affinity) {
        T.flags |= CCSIM_TF_HAS_AFFINITY_TERMS;
        if (t_.node_affinity_terms.size() > CCSIM_MAX_AFF_TERMS) throw Unsupported("more than 8 nodeSelectorTerms");
        T.n_aff_terms = (int32_t)t_.node_affinity_terms.size();
        for (size_t k = 0; k < t_.node_affinity_terms.size(); k++) {
          const NodeSelectorTerm &nt = t_.node_affinity_terms[k];
          set_mask(T.aff_term_mask[k], new_bit([&](int i) { return nt.matches(nodes_[i]->labels, nodes_[i]->name); }));
        }
        // PreFilterResult.NodeNames (node_affinity.go:164-194): every term pins metadata.name In [...]
        std::set<std::string> names; bool all_terms_pin = !t_.node_affinity_terms.empty();
        for (auto &nt : t_.node_affinity_terms) {
          bool pinned = false; std::set<std::string> term_names;
          for (auto &r : nt.match_fields)
            if (r.key == "metadata.name" && r.op == "In") {
              std::set<std::string> s(r.values.begin(), r.values.end());
              if (!pinned) { term_names = s; pinned = true; }
              else { std::set<std::string> x; for (auto &v : term_names) if (s.count(v)) x.insert(v); term_names = x; }
            }
          if (!pinned) { all_terms_pin = false; break; }
          names.insert(term_names.begin(), term_names.end());
        }
        if (all_terms_pin) {
          if (names.empty()) e.prefilter_msg = "node(s) didn't match Pod's node affinity/selector";   // errReasonConflict path is host-formatted
          else { T.flags |= CCSIM_TF_PREFILTER_NODES; T.prefilter_bit = new_bit([&](int i) { return names.count(nodes_[i]->name) > 0; }); }
        }
      }
    }
    // NodeAffinity preferred terms -> one static bit each (node_affinity.go:241-290)
    if (t_.node_affinity_preferred.size() > CCSIM_MAX_AFF_TERMS) throw Unsupported("more than 8 preferred nodeAffinity terms");
    T.n_pref_terms = (int32_t)t_.node_affinity_preferred.size();
    for (size_t k = 0; k < t_.node_affinity_preferred.size(); k++) {
      const NodeSelectorTerm &nt = t_.node_affinity_preferred[k].second;
      T.pref_weight[k] = t_.node_affinity_preferred[k].first;
      set_mask(T.pref_mask[k], new_bit([&](int i) { return nt.matches(nodes_[i]->labels, nodes_[i]->name); }));
    }
    // NodePorts (node_ports.go:68-76,157-185)
    std::vector<ContainerPort> want = t_.host_ports();
    if (!want.empty()) {
      T.flags |= CCSIM_TF_HAS_HOST_PORTS;
      e.has_placed_mask = true;
      T.port_tmpl_conflict = 1;   // a clone always conflicts with another clone of the same template
      auto norm = [](const ContainerPort &p, std::string &ip, std::string &proto) { ip = p.host_ip.empty() ? "0.0.0.0" : p.host_ip; proto = p.protocol.empty() ? "TCP" : p.protocol; };
      set_mask(T.port_static_mask, new_bit([&](int i) {
        for (auto *p : pods_on_[i])
          for (auto &u : p->host_ports()) {
            std::string uip, uproto; norm(u, uip, uproto);
            for (auto &w : want) {
              std::string wip, wproto; norm(w, wip, wproto);
              if (w.host_port != u.host_port || wproto != uproto) continue;
              if (wip == "0.0.0.0" || uip == "0.0.0.0" || wip == uip) return true;
            }
          }
        return false;
      }));
    }
    tick("static bits");
    // ---- PodTopologySpread hard constraints (plugin.go:257-278; common.go:86-127; filtering.go:235-308) ----
    const Labels *t_ns_labels = ns_labels_.count(t_.ns) ? &ns_labels_.at(t_.ns) : nullptr;
    std::vector<const TopologySpreadConstraint *> hard;
    for (auto &c : t_.spread) if (c.when_unsatisfiable == "DoNotSchedule" || c.when_unsatisfiable.empty()) hard.push_back(&c);
    if (hard.size() > CCSIM_MAX_PTS) throw Unsupported("more than 8 hard topology spread constraints");
    auto constraint_selector = [&](const TopologySpreadConstraint &c) {   // filterTopologySpreadConstraints (common.go:86-127)
      Selector s = Selector::from_label_selector(c.label_selector);
      if (!c.match_label_keys.empty()) {   // mergeLabelSetWithSelector
        Labels ml;
        for (auto &k : c.match_label_keys) { auto it = t_.labels.find(k); if (it != t_.labels.end()) ml[k] = it->second; }
        if (!ml.empty()) { Selector m = Selector::from_set(ml); if (!s.nothing) for (auto &r : s.reqs) m.reqs.push_back(r); else m = s; s = m; }
      }
      return s;
    };
    std::vector<Selector> hard_sel;
    for (auto *c : hard) hard_sel.push_back(constraint_selector(*c));
    auto required_affinity_match = [&](int i) {   // RequiredNodeAffinity.Match
      if (!t_.node_selector.empty() && !Selector::from_set(t_.node_selector).matches(nodes_[i]->labels)) return false;
      if (t_.has_required_node_affinity) {
        for (auto &nt : t_.node_affinity_terms) if (nt.matches(nodes_[i]->labels, nodes_[i]->name)) return true;
        return false;
      }
      return true;
    };
    auto untolerated = [&](int i) {
      for (auto &t : nodes_[i]->taints) if ((t.effect == "NoSchedule" || t.effect == "NoExecute") && !tolerations_tolerate(t_.tolerations, t)) return true;
      return false;
    };
    // per node, for ALL hard constraints in one pass over the node's labels and pods: the node's value of each constraint's key,
    // eligibility (every constraint key present + the constraint's inclusion policies) and countPodsMatchSelector (common.go:144-158)
    const size_t H = hard.size();
    std::vector<std::vector<char>> eligible_c(H, std::vector<char>(n, 0));
    std::vector<std::vector<int64_t>> node_cnt_c(H, std::vector<int64_t>(n, 0));
    std::vector<std::vector<const std::string *>> value_c(H, std::vector<const std::string *>(n, nullptr));
    std::vector<std::vector<uint64_t>> vhash_c(H, std::vector<uint64_t>(n, 0));
    bool any_aff_policy = false, any_taint_policy = false;
    for (auto *h : hard) { any_aff_policy |= h->node_affinity_policy == "Honor"; any_taint_policy |= h->node_taints_policy == "Honor"; }
    if (H > 0)
      parallel_for(n, [&](int i) {
        const Node &nd = *nodes_[i];
        bool all_keys = true;
        for (size_t c = 0; c < H; c++) {
          auto vit = nd.labels.find(hard[c]->topology_key);
          if (vit != nd.labels.end()) { value_c[c][i] = &vit->second; vhash_c[c][i] = FlatIndex::hash(vit->second); } else all_keys = false;
        }
        if (!all_keys) return;
        const bool aff_ok = !any_aff_policy || required_affinity_match(i);
        const bool taint_ok = !any_taint_policy || !untolerated(i);
        bool any = false;
        for (size_t c = 0; c < H; c++) {
          if (hard[c]->node_affinity_policy == "Honor" && !aff_ok) continue;
          if (hard[c]->node_taints_policy == "Honor" && !taint_ok) continue;
          eligible_c[c][i] = 1;
          any |= !hard_sel[c].empty();
        }
        if (!any) return;
        for (auto *p : pods_on_[i]) {
          if (p->terminating || p->ns != t_.ns) continue;
          for (size_t c = 0; c < H; c++)
            if (eligible_c[c][i] && !hard_sel[c].empty() && hard_sel[c].matches(p->labels)) node_cnt_c[c][i]++;
        }
      });
    for (size_t c = 0; c < hard.size(); c++) {
      const TopologySpreadConstraint &tc = *hard[c];
      // domains: eligible nodes define TpValueToMatchNum; they get ids [0,n_present)
      FlatIndex dom_id; std::vector<int64_t> counts;
      dom_id.init(1024);
      const std::vector<char> &eligible = eligible_c[c];
      const std::vector<int64_t> &node_cnt = node_cnt_c[c];
      const std::vector<const std::string *> &value = value_c[c];
      const std::vector<uint64_t> &vhash = vhash_c[c];
      std::vector<int32_t> col(n, -1);
      for (int i = 0; i < n; i++) {    // domain ids in first-seen order over the eligible nodes
        if (!eligible[i]) continue;
        auto ins = dom_id.emplace(std::string_view(*value[i]), vhash[i], (int32_t)dom_id.size());
        if (ins.second) counts.push_back(0);
        counts[(size_t)*ins.first] += node_cnt[i];
        col[i] = *ins.first;
      }
      const int n_present = (int)dom_id.size();
      for (int i = 0; i < n; i++) {
        if (eligible[i] || !value[i]) continue;
        auto ins = dom_id.emplace(std::string_view(*value[i]), vhash[i], (int32_t)dom_id.size());   // value only on ineligible nodes: matchNum 0, never in the min
        if (ins.second) counts.push_back(0);
        col[i] = *ins.first;
      }
      int colidx = (int)e.topo.size();
      e.topo.push_back(col);
      std::vector<int32_t> init = int32_counts(counts, tc.topology_key);
      const bool self = hard_sel[c].matches(t_.labels);
      // an Everything selector (labelSelector: {}) self-matches (filtering.go:341-344) but is never COUNTED: countPodsMatchSelector
      // returns 0 for selector.Empty() (common.go:144-147), so committed clones do not raise the domain counts either
      add_counter(e, colidx, init, n_present, (self && !hard_sel[c].empty()) ? 1 : 0);
      T.pts[c].counter = (int32_t)e.counters.size() - 1;
      T.pts[c].max_skew = tc.max_skew;
      T.pts[c].self_match = self ? 1 : 0;
      T.pts[c].min_zero = n_present < tc.min_domains ? 1 : 0;
    }
    T.n_pts = (int32_t)hard.size();
    tick("hard spread constraints");
    // ---- InterPodAffinity required terms (interpodaffinity/filtering.go:204-309) ----
    auto term_matches_pod = [&](const AffinityTerm &t, const Pod &p, const Labels *nsl) { return t.matches(p.ns, p.labels, nsl); };
    // incoming pod's terms: namespaceSelector is resolved against the namespace list and merged into Namespaces
    // (mergeAffinityTermNamespacesIfNotEmpty), after which matching uses nil namespace labels
    auto merged = [&](const std::vector<AffinityTerm> &in) {
      std::vector<AffinityTerm> out = in;
      for (auto &t : out) {
        if (!t.ns_selector.nothing && !t.ns_selector.empty())
          for (auto &kv : ns_labels_) if (t.ns_selector.matches(kv.second)) t.namespaces.insert(kv.first);
      }
      return out;
    };
    std::vector<AffinityTerm> aff = merged(t_.aff_required), anti = merged(t_.anti_required);
    auto ipa_counter = [&](const std::string &key, const std::function<int64_t(const Pod &)> &weight, int inc, int32_t &out_idx) {
      // one counter per topology key; node-local when every node has the key with a unique value
      FlatIndex dom_id; std::vector<int32_t> col(n, -1); std::vector<int64_t> counts;
      std::vector<const std::string *> value(n, nullptr);
      std::vector<uint64_t> vhash(n, 0);
      parallel_for(n, [&](int i) { auto it = nodes_[i]->labels.find(key); if (it != nodes_[i]->labels.end()) { value[i] = &it->second; vhash[i] = FlatIndex::hash(it->second); } });
      tick("  ipa/values");
      // kubernetes.io/hostname-style keys: when every node's value is its own (unique) name the domains are the nodes themselves,
      // in node order — no dictionary to build
      std::atomic<bool> own_name{n > 0};
      parallel_for(n, [&](int i) { if (!value[i] || *value[i] != nodes_[i]->name) own_name.store(false, std::memory_order_relaxed); });
      bool unique = true;
      if (own_name.load()) {
        counts.assign(n, 0);
        for (int i = 0; i < n; i++) col[i] = i;
      } else {
        dom_id.init(1024);
        for (int i = 0; i < n; i++) {
          if (!value[i]) { unique = false; continue; }
          auto ins = dom_id.emplace(std::string_view(*value[i]), vhash[i], (int32_t)dom_id.size());
          if (ins.second) counts.push_back(0); else unique = false;
          col[i] = *ins.first;
        }
      }
      tick("  ipa/domain ids");
      std::vector<int64_t> per_node(n, 0);
      parallel_for(n, [&](int i) { if (col[i] < 0) return; for (auto *p : pods_on_[i]) per_node[i] += weight(*p); });
      tick("  ipa/weights");
      for (int i = 0; i < n; i++) if (col[i] >= 0) counts[col[i]] += per_node[i];
      if (unique && n > 0) {
        std::vector<int32_t> init = int32_counts(per_node, key);
        add_counter(e, -1, init, n, inc);
      } else {
        int colidx = (int)e.topo.size();
        e.topo.push_back(col);
        std::vector<int32_t> init = int32_counts(counts, key);
        add_counter(e, colidx, init, (int)init.size(), inc);
      }
      out_idx = (int32_t)e.counters.size() - 1;
    };
    if (!aff.empty()) {
      bool self_all = true;
      for (auto &t : aff) if (!term_matches_pod(t, t_, nullptr)) self_all = false;
      if (self_all) T.flags |= CCSIM_TF_AFF_SELF_MATCH_ALL;
      std::vector<std::string> keys;
      for (auto &t : aff) if (std::find(keys.begin(), keys.end(), t.topology_key) == keys.end()) keys.push_back(t.topology_key);
      if (keys.size() > CCSIM_MAX_IPA) throw Unsupported("more than 8 pod-affinity topology keys");
      int64_t total = 0;
      for (size_t k = 0; k < keys.size(); k++) {
        int nterms = 0; for (auto &t : aff) if (t.topology_key == keys[k]) nterms++;
        auto w = [&](const Pod &p) { for (auto &t : aff) if (!term_matches_pod(t, p, nullptr)) return 0; return nterms; };   // podMatchesAllAffinityTerms
        ipa_counter(keys[k], w, nterms, T.aff_counter[k]);
        const ccsim_counter &cc = e.counters.back();
        for (int d = 0; d < cc.n_domains; d++) total += e.counter_init.back()[d];
      }
      T.n_aff = (int32_t)keys.size();
      T.aff_total_init = total;
    }
    if (!anti.empty()) {
      std::vector<std::string> keys;
      for (auto &t : anti) if (std::find(keys.begin(), keys.end(), t.topology_key) == keys.end()) keys.push_back(t.topology_key);
      if (keys.size() > CCSIM_MAX_IPA) throw Unsupported("more than 8 pod-anti-affinity topology keys");
      for (size_t k = 0; k < keys.size(); k++) {
        auto w = [&](const Pod &p) { int c = 0; for (auto &t : anti) if (t.topology_key == keys[k] && term_matches_pod(t, p, nullptr)) c++; return c; };
        int inc = w(t_);
        ipa_counter(keys[k], w, inc, T.anti_counter[k]);
      }
      T.n_anti = (int32_t)keys.size();
    }
    tick("inter-pod (anti-)affinity counters");
    // existing pods' required anti-affinity against the incoming pod (getExistingAntiAffinityCounts): static bit
    {
      std::set<std::pair<std::string, std::string>> blocked;
      for (auto &ip : anti_required_pods_) {       // (the pods that carry such terms were listed while the pods were assigned to nodes)
        const int i = ip.first;
        for (auto &t : ip.second->anti_required)
          if (t.matches(t_.ns, t_.labels, t_ns_labels)) {
            auto it = nodes_[i]->labels.find(t.topology_key);
            if (it != nodes_[i]->labels.end()) blocked.insert({t.topology_key, it->second});
          }
      }
      if (!blocked.empty())
        set_mask(T.existing_anti_mask, new_bit([&](int i) {
          for (auto &kv : nodes_[i]->labels) if (blocked.count({kv.first, kv.second})) return true;
          return false;
        }));
    }
    tick("existing anti-affinity");
    // ---- PodTopologySpread score: ScheduleAnyway constraints, or the system defaults when a Service / owning controller
    //      selects the pod (scoring.go:60-186; plugin.go:48-59; common.go:64-81) ----
    if (cfg_.score_enable & CCSIM_PL_POD_TOPOLOGY_SPREAD) {
      struct SoftC { int max_skew; std::string key; Selector sel; std::string nap, ntp; };
      std::vector<SoftC> soft;
      const bool require_all = !t_.spread.empty();   // requireAllTopologies (scoring.go:140)
      if (!t_.spread.empty()) {
        for (auto &c : t_.spread)
          if (c.when_unsatisfiable == "ScheduleAnyway") soft.push_back({c.max_skew, c.topology_key, constraint_selector(c), c.node_affinity_policy, c.node_taints_policy});
      } else {
        Selector ds = default_selector();
        if (!ds.empty()) {
          soft.push_back({3, "kubernetes.io/hostname", ds, "Honor", "Ignore"});
          soft.push_back({5, "topology.kubernetes.io/zone", ds, "Honor", "Ignore"});
        }
      }
      if (soft.size() > CCSIM_MAX_PTS) throw Unsupported("more than 8 ScheduleAnyway topology spread constraints");
      if (!soft.empty()) {
        std::vector<char> all_keys(n, 1);
        bool any_missing = false;
        for (int i = 0; i < n; i++)
          for (auto &c : soft) if (!nodes_[i]->labels.count(c.key)) { all_keys[i] = 0; any_missing = true; }
        T.spts_ignored_bit = (require_all && any_missing) ? new_bit([&](int i) { return !all_keys[i]; }) : -1;
        auto matching_pods = [&](int i, const Selector &sel) {   // countPodsMatchSelector (common.go:144-158)
          int64_t cnt = 0;
          if (!sel.empty()) for (auto *p : pods_on_[i]) if (!p->terminating && p->ns == t_.ns && sel.matches(p->labels)) cnt++;
          return cnt;
        };
        for (size_t c = 0; c < soft.size(); c++) {
          const SoftC &sc = soft[c];
          const int inc = (!sc.sel.empty() && sc.sel.matches(t_.labels)) ? 1 : 0;
          ccsim_spts &S = T.spts[c];
          S.max_skew = sc.max_skew; S.has_key_bit = -1;
          if (sc.key == "kubernetes.io/hostname") {   // per-node counts, read at Score (scoring.go:211-212)
            S.hostname = 1;
            std::vector<int32_t> init(n);
            bool everyone = true;
            for (int i = 0; i < n; i++) { init[i] = (int32_t)matching_pods(i, sc.sel); if (!nodes_[i]->labels.count(sc.key)) everyone = false; }
            if (!everyone) S.has_key_bit = new_bit([&](int i) { return nodes_[i]->labels.count(sc.key) > 0; });
            add_counter(e, -1, init, n, inc);
          } else {
            S.hostname = 0;
            std::map<std::string, int> dom_id; std::vector<int64_t> counts; std::vector<int32_t> col(n, -1);
            std::vector<char> counted(n, 0);
            bool everyone = true, explicit_empty = false, missing = false;
            for (int i = 0; i < n; i++) {
              auto it = nodes_[i]->labels.find(sc.key);
              if (it == nodes_[i]->labels.end()) { missing = true; everyone = false; continue; }
              if (it->second.empty()) explicit_empty = true;
              if (!dom_id.count(it->second)) { int id = (int)dom_id.size(); dom_id[it->second] = id; counts.push_back(0); }
              col[i] = dom_id[it->second];
              // processAllNode (scoring.go:157-186)
              if (require_all && !all_keys[i]) { everyone = false; continue; }
              if (sc.nap == "Honor" && !required_affinity_match(i)) { everyone = false; continue; }
              if (sc.ntp == "Honor" && untolerated(i)) { everyone = false; continue; }
              counted[i] = 1;
              counts[col[i]] += matching_pods(i, sc.sel);
            }
            if (!require_all && missing && explicit_empty) throw Unsupported("a topology label with an empty value next to nodes without the label (PodTopologySpread score)");
            int colidx = (int)e.topo.size();
            e.topo.push_back(col);
            std::vector<int32_t> init = int32_counts(counts, sc.key);
            add_counter(e, colidx, init, (int)init.size(), inc);
            if (!everyone && inc) e.counters.back().elig_bit = new_bit([&, counted](int i) { return counted[i] != 0; });
          }
          S.counter = (int32_t)e.counters.size() - 1;
        }
        T.n_spts = (int32_t)soft.size();
      }
    }
    // ---- InterPodAffinity score (scoring.go:51-234): signed weights per (topologyKey, value) ----
    if (cfg_.score_enable & CCSIM_PL_INTER_POD_AFFINITY) {
      std::vector<AffinityTerm> paff = merged(t_.aff_preferred), panti = merged(t_.anti_preferred);
      const int hw = cfg_.hard_pod_affinity_weight;
      // what existing pod `p` contributes to key -> weight (processExistingPod, scoring.go:81-125)
      auto contributions = [&](const Pod &p, std::map<std::string, int64_t> &out) {
        for (auto &t : paff) if (t.matches(p.ns, p.labels, nullptr)) out[t.topology_key] += t.weight;
        for (auto &t : panti) if (t.matches(p.ns, p.labels, nullptr)) out[t.topology_key] -= t.weight;
        if (hw > 0) for (auto &t : p.aff_required) if (t.matches(t_.ns, t_.labels, t_ns_labels)) out[t.topology_key] += hw;
        for (auto &t : p.aff_preferred) if (t.matches(t_.ns, t_.labels, t_ns_labels)) out[t.topology_key] += t.weight;
        for (auto &t : p.anti_preferred) if (t.matches(t_.ns, t_.labels, t_ns_labels)) out[t.topology_key] -= t.weight;
      };
      std::vector<std::string> keys;
      auto note = [&](const std::map<std::string, int64_t> &m) { for (auto &kv : m) if (std::find(keys.begin(), keys.end(), kv.first) == keys.end()) keys.push_back(kv.first); };
      std::map<std::string, int64_t> clone;   // a placed clone is an existing pod of the next cycle
      contributions(t_, clone);
      note(clone);
      std::map<const Pod *, std::map<std::string, int64_t>> per_pod;
      auto visit = [&](const Pod *p) {
        std::map<std::string, int64_t> m; contributions(*p, m);
        if (!m.empty()) { note(m); per_pod[p] = m; }
      };
      if (paff.empty() && panti.empty()) { for (auto &ip : affinity_term_pods_) visit(ip.second); }   // only pods with terms of their own can contribute
      else for (int i = 0; i < n; i++) for (auto *p : pods_on_[i]) visit(p);
      if (keys.size() > CCSIM_MAX_IPA) throw Unsupported("more than 8 topology keys in pod (anti-)affinity scoring terms");
      for (size_t k = 0; k < keys.size(); k++) {
        auto w = [&](const Pod &p) -> int64_t { auto it = per_pod.find(&p); if (it == per_pod.end()) return 0; auto jt = it->second.find(keys[k]); return jt == it->second.end() ? 0 : jt->second; };
        const int64_t inc = clone.count(keys[k]) ? clone[keys[k]] : 0;
        ipa_counter(keys[k], w, int32_counts({inc}, keys[k])[0], T.ipa_score_counter[k]);
      }
      T.n_ipa_score = (int32_t)keys.size();
    }
    // ---- ImageLocality (image_locality.go:54-131; backend/cache/cache.go:680-703): static per node ----
    bool any_images = false;
    for (int i = 0; i < n && !any_images; i++) any_images = !nodes_[i]->images.empty();
    if ((cfg_.score_enable & CCSIM_PL_IMAGE_LOCALITY) && any_images) {      // (no image anywhere: every node scores 0)
      std::map<std::string, std::pair<int64_t, std::set<int>>> states;   // name -> (size as first registered, nodes)
      for (int i = 0; i < n; i++)
        for (auto &im : nodes_[i]->images) {
          auto it = states.find(im.first);
          if (it == states.end()) states[im.first] = {im.second, {i}}; else it->second.second.insert(i);
        }
      auto normalized = [](std::string name) {
        const auto colon = name.rfind(':'), slash = name.rfind('/');
        const long long c = colon == std::string::npos ? -1 : (long long)colon, s = slash == std::string::npos ? -1 : (long long)slash;
        if (c <= s) name += ":latest";
        return name;
      };
      std::vector<std::string> want;
      for (auto &c : t_.init_containers) want.push_back(normalized(c.image));
      for (auto &c : t_.containers) want.push_back(normalized(c.image));
      const int64_t mb = 1024 * 1024, min_thr = 23 * mb, max_thr = 1000 * mb * (int64_t)want.size();
      bool any = false;
      std::vector<uint8_t> col(n, 0);
      for (int i = 0; i < n; i++) {
        int64_t sum = 0;
        std::set<std::string> here; for (auto &im : nodes_[i]->images) here.insert(im.first);
        for (auto &wname : want)
          if (here.count(wname)) {
            const auto &st = states[wname];
            const double spread = (double)st.second.size() / (double)n;
            sum += (int64_t)((double)st.first * spread);
          }
        if (sum < min_thr) sum = min_thr; else if (sum > max_thr) sum = max_thr;
        const int64_t sc = max_thr > min_thr ? 100 * (sum - min_thr) / (max_thr - min_thr) : 0;
        col[i] = (uint8_t)sc;
        if (sc) any = true;
      }
      if (any) e.image_score = col;
    }
    tick("soft scorers");
    if (e.topo.size() > CCSIM_MAX_TOPO_COLS || e.counters.size() > CCSIM_MAX_COUNTERS) throw Unsupported("too many topology columns");
    // ---- pack static bits ----
    if (bits.size() > 64 * CCSIM_MAX_STATIC_WORDS) throw Unsupported("too many static predicate bits");
    e.static_words = (int)(bits.size() + 63) / 64;
    e.static_mask.assign((size_t)std::max(1, e.static_words) * n, 0);
    for (size_t b = 0; b < bits.size(); b++)
      for (int i = 0; i < n; i++) if (bits[b][i]) e.static_mask[(size_t)(b >> 6) * n + i] |= 1ull << (b & 63);
    for (size_t j = 0; j < e.counters.size(); j++) e.counters[j].init = e.counter_init[j].data();
    T.image_score = e.image_score.empty() ? nullptr : e.image_score.data();
    return e;
  }

  const std::vector<const Node *> &nodes() const { return nodes_; }

 private:
  SchedConfig cfg_;
  const Pod &t_;
  const std::map<std::string, Labels> &ns_labels_;
  std::vector<const Node *> nodes_;
  FlatIndex node_index_;   // keys view the Node objects' names (they outlive the encoder)
  // the pods of every node, in the order of the source list: one offsets array + one pointer array (a counting sort; a
  // std::vector per node costs one allocation per node on one core)
  struct PodsOn {
    struct Range { const Pod *const *b, *const *e; const Pod *const *begin() const { return b; } const Pod *const *end() const { return e; } };
    std::vector<uint32_t> off;
    std::vector<const Pod *> ptr;
    void build(size_t n_nodes, const std::vector<int32_t> &where, const ObjList<Pod> &pods) {
      off.assign(n_nodes + 1, 0);
      for (size_t j = 0; j < where.size(); j++) if (where[j] >= 0) off[(size_t)where[j] + 1]++;
      for (size_t i = 0; i < n_nodes; i++) off[i + 1] += off[i];
      ptr.resize(off[n_nodes]);
      std::vector<uint32_t> cur(off.begin(), off.end() - 1);
      for (size_t j = 0; j < where.size(); j++) if (where[j] >= 0) ptr[cur[(size_t)where[j]]++] = &pods[j];
    }
    Range operator[](size_t i) const { return Range{ptr.data() + off[i], ptr.data() + off[i + 1]}; }
  } pods_on_;
  std::vector<std::pair<int, const Pod *>> anti_required_pods_, affinity_term_pods_;   // (node index, pod) of the pods with such terms
  bool lower_priority_pod_ = false;
  const std::vector<WorkloadSelector> *workloads_ = nullptr;

  // helper.DefaultSelector (plugins/helper/spread.go:40-93)
  Selector default_selector() const {
    Labels set;
    Selector sel; sel.nothing = false;
    if (!workloads_) return sel;
    for (auto &w : *workloads_)   // GetPodServices (spread.go:96-113): nil selectors match nothing
      if (w.kind == "Service" && w.ns == t_.ns && w.has_map && Selector::from_set(w.map).matches(t_.labels))
        for (auto &kv : w.map) set[kv.first] = kv.second;
    sel = Selector::from_set(set);
    if (t_.owner_kind.empty()) return sel;
    for (auto &w : *workloads_) {
      if (w.ns != t_.ns || w.name != t_.owner_name || w.kind != t_.owner_kind) continue;
      if (w.kind == "ReplicationController" && t_.owner_api_version == "v1") {
        for (auto &kv : w.map) set[kv.first] = kv.second;
        sel = Selector::from_set(set);
      } else if ((w.kind == "ReplicaSet" || w.kind == "StatefulSet") && t_.owner_api_version == "apps/v1") {
        Selector other = Selector::from_label_selector(w.label_selector);
        if (!other.nothing) for (auto &r : other.reqs) sel.reqs.push_back(r);
      }
      break;
    }
    return sel;
  }

  // Per-domain counts are summed in int64 like the reference's and held as int32 by the engine: a sum outside int32 is refused,
  // naming the topology key, instead of being narrowed.
  static std::vector<int32_t> int32_counts(const std::vector<int64_t> &v, const std::string &key) {
    for (int64_t x : v)
      if (x < INT32_MIN || x > INT32_MAX)
        throw Unsupported("topology key \"" + key + "\": a per-domain count of " + std::to_string(x) + " is outside int32");
    return std::vector<int32_t>(v.begin(), v.end());
  }

  static void add_counter(Encoded &e, int topo_col, const std::vector<int32_t> &init, int n_present, int inc) {
    ccsim_counter c; memset(&c, 0, sizeof(c));
    c.topo_col = topo_col; c.n_domains = (int32_t)init.size(); c.n_present = n_present; c.inc = inc; c.elig_bit = -1;
    e.counter_init.push_back(init);
    e.counters.push_back(c);
  }

  // what the GPU path does not implement is refused, naming the plugin (SURVEY.md §2 rows 30-32, §8f4)
  void guards() const {
    if (t_.has_pvc_volume) throw Unsupported("pod uses PersistentVolumeClaim/ephemeral volumes (VolumeBinding/VolumeZone/NodeVolumeLimits/VolumeRestrictions)");
    if (t_.has_resource_claims) throw Unsupported("pod uses resourceClaims (DynamicResources)");
    if (t_.has_scheduling_gates) throw Unsupported("pod has schedulingGates");
    if (lower_priority_pod_) throw Unsupported("an existing pod has lower priority than the simulated pod (DefaultPreemption would evict it)");
  }
};

}  // namespace cch
