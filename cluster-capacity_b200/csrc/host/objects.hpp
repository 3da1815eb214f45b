// objects.hpp — the slice of the Kubernetes object model the hot path needs (Node, Pod, selectors), parsed from the
// JSON the API server (or `kubectl get -o json`) produces, plus the label/affinity matching helpers.
//
// Reference semantics followed (file:line under /root/reference/vendor):
//   labels.Requirement.Matches            k8s.io/apimachinery/pkg/labels/selector.go:246-293
//   metav1.LabelSelectorAsSelector        k8s.io/apimachinery/pkg/apis/meta/v1/helpers.go (nil -> Nothing, {} -> Everything)
//   Toleration.ToleratesTaint             k8s.io/api/core/v1/toleration.go:38-57
//   AffinityTerm.Matches                  k8s.io/kube-scheduler/framework/types.go:379-384
//   getNamespacesFromPodAffinityTerm      k8s.io/kubernetes/pkg/scheduler/framework/types.go:927-935
//   HostPortInfo.CheckConflict            k8s.io/kube-scheduler/framework/types.go:499-528
//   GetHostPorts                          k8s.io/kubernetes/pkg/scheduler/util/utils.go:175-210
//   PodRequests / AggregateContainerRequests  k8s.io/component-helpers/resource/helpers.go:144-251
#pragma once
#include <mutex>
#include <cstdint>
#include <cstdlib>
#include <stdexcept>
#include <new>
#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <vector>
#include "json.hpp"
#include "quantity.hpp"

namespace cch {

typedef std::map<std::string, std::string> Labels;
typedef std::map<std::string, Quantity> ResourceList;

inline Labels parse_labels(const Json &j) {
  Labels l;
  if (j.is_object()) for (auto &kv : j.obj) l[kv.first] = kv.second.str();
  return l;
}
inline ResourceList parse_resources(const Json &j) {
  ResourceList r;
  if (j.is_object())
    for (auto &kv : j.obj) {
      const Json &v = kv.second;
      r[kv.first] = Quantity::parse(v.type == Json::Number ? v.s : v.str());
    }
  return r;
}
inline void add_resources(ResourceList &dst, const ResourceList &src) { for (auto &kv : src) dst[kv.first].add(kv.second), (void)0; }
inline void add_resources_fmt(ResourceList &dst, const ResourceList &src) {
  for (auto &kv : src) {
    auto it = dst.find(kv.first);
    if (it == dst.end()) dst[kv.first] = kv.second; else it->second.add(kv.second);
  }
}
inline void max_resources(ResourceList &dst, const ResourceList &src) {
  for (auto &kv : src) {
    auto it = dst.find(kv.first);
    if (it == dst.end() || kv.second.nanos > it->second.nanos) dst[kv.first] = kv.second;
  }
}

// ---- label selectors -------------------------------------------------------------------------------------------
struct Requirement {
  std::string key, op;   // In NotIn Exists DoesNotExist Gt Lt (Equals is In with one value)
  std::vector<std::string> values;
  bool matches(const Labels &ls) const {
    auto it = ls.find(key);
    const bool has = it != ls.end();
    if (op == "In") return has && std::find(values.begin(), values.end(), it->second) != values.end();
    if (op == "NotIn") return !has || std::find(values.begin(), values.end(), it->second) == values.end();
    if (op == "Exists") return has;
    if (op == "DoesNotExist") return !has;
    if (op == "Gt" || op == "Lt") {
      if (!has || values.size() != 1) return false;
      char *e1 = nullptr, *e2 = nullptr;
      long long a = strtoll(it->second.c_str(), &e1, 10), b = strtoll(values[0].c_str(), &e2, 10);
      if (it->second.empty() || *e1 || values[0].empty() || *e2) return false;
      return op == "Gt" ? a > b : a < b;
    }
    return false;
  }
};

struct Selector {
  bool nothing = true;                 // labels.Nothing(): matches no object, Empty() is false
  std::vector<Requirement> reqs;       // !nothing && reqs.empty(): Everything, Empty() is true
  bool matches(const Labels &ls) const {
    if (nothing) return false;
    for (auto &r : reqs) if (!r.matches(ls)) return false;
    return true;
  }
  bool empty() const { return !nothing && reqs.empty(); }
  // metav1.LabelSelectorAsSelector
  static Selector from_label_selector(const Json &j) {
    Selector s;
    if (!j.is_object()) return s;      // nil -> Nothing
    s.nothing = false;
    const Json &ml = j.at("matchLabels");
    if (ml.is_object()) for (auto &kv : ml.obj) s.reqs.push_back(Requirement{kv.first, "In", {kv.second.str()}});
    const Json &me = j.at("matchExpressions");
    if (me.is_array())
      for (auto &e : me.arr) {
        Requirement r{e.at("key").str(), e.at("operator").str(), {}};
        for (auto &v : e.at("values").arr) r.values.push_back(v.str());
        s.reqs.push_back(r);
      }
    return s;
  }
  static Selector from_set(const Labels &set) {   // labels.SelectorFromSet
    Selector s;
    s.nothing = false;
    for (auto &kv : set) s.reqs.push_back(Requirement{kv.first, "In", {kv.second}});
    return s;
  }
};

// ---- taints / tolerations --------------------------------------------------------------------------------------
struct Taint { std::string key, value, effect; bool operator<(const Taint &o) const { return std::tie(key, value, effect) < std::tie(o.key, o.value, o.effect); } };
struct Toleration {
  std::string key, op, value, effect;
  bool tolerates(const Taint &t) const {
    if (!effect.empty() && effect != t.effect) return false;
    if (!key.empty() && key != t.key) return false;
    if (op.empty() || op == "Equal") return value == t.value;
    if (op == "Exists") return true;
    return false;
  }
};
inline bool tolerations_tolerate(const std::vector<Toleration> &tols, const Taint &t) {
  for (auto &x : tols) if (x.tolerates(t)) return true;
  return false;
}

// ---- node selector terms (nodeAffinity) ------------------------------------------------------------------------
struct NodeSelectorTerm {
  std::vector<Requirement> match_expressions;
  std::vector<Requirement> match_fields;   // only metadata.name In/NotIn with one value is valid
  bool empty() const { return match_expressions.empty() && match_fields.empty(); }
  bool matches(const Labels &node_labels, const std::string &node_name) const {
    for (auto &r : match_expressions) if (!r.matches(node_labels)) return false;
    if (!match_fields.empty() && !node_name.empty()) {
      Labels f{{"metadata.name", node_name}};
      for (auto &r : match_fields) if (!r.matches(f)) return false;
    }
    return true;
  }
};

// ---- pod (anti-)affinity terms ---------------------------------------------------------------------------------
struct AffinityTerm {
  std::set<std::string> namespaces;
  Selector selector;
  Selector ns_selector;     // nil -> Nothing
  std::string topology_key;
  int weight = 0;           // preferred terms only (WeightedPodAffinityTerm.weight)
  bool matches(const std::string &pod_ns, const Labels &pod_labels, const Labels *ns_labels) const {
    static const Labels none;
    if (namespaces.count(pod_ns) || ns_selector.matches(ns_labels ? *ns_labels : none)) return selector.matches(pod_labels);
    return false;
  }
};

struct ContainerPort { std::string host_ip, protocol; int host_port = 0; };

struct Container {
  std::string name, image;
  ResourceList requests;
  std::vector<ContainerPort> ports;
  bool restart_always = false;   // init containers: restartPolicy: Always (sidecar)
};

struct TopologySpreadConstraint {
  int max_skew = 1;
  std::string topology_key, when_unsatisfiable;
  Json label_selector;           // raw (nil vs {} matters)
  std::vector<std::string> match_label_keys;
  int min_domains = 1;
  std::string node_affinity_policy = "Honor", node_taints_policy = "Ignore";
};

// Retired element arrays of the ingest, kept mapped for the next analysis of the process. First touch of fresh memory is what the
// ingest of a large snapshot mostly waits for: the page faults of the 190 MB Pod array of C4 (200k x 960 B) take ~110 ms here, with 1
// toucher or with 8 (the kernel serialises them), against ~160 ms of actual parsing on one core. A block is handed out
// again when it is large enough and not more than 4x too large; at most 4 blocks / 1 GiB are kept (CCHOST_NO_RECYCLE: none).
class RawBlockCache {
 public:
  static RawBlockCache &get() { static RawBlockCache *c = new RawBlockCache(); return *c; }     // never destroyed (exit order)
  void *take(size_t bytes, size_t &cap) {
    std::lock_guard<std::mutex> g(mu_);
    int best = -1;
    for (int i = 0; i < kSlots; i++)
      if (blk_[i].p && blk_[i].cap >= bytes && blk_[i].cap / 4 <= bytes && (best < 0 || blk_[i].cap < blk_[best].cap)) best = i;
    if (best < 0) return nullptr;
    void *p = blk_[best].p; cap = blk_[best].cap;
    total_ -= cap; blk_[best] = Blk{nullptr, 0};
    return p;
  }
  void give(void *p, size_t cap) {
    if (!p) return;
    static const bool off = getenv("CCHOST_NO_RECYCLE") != nullptr;
    if (!off && cap >= (1u << 20)) {                       // small lists are not worth a slot
      std::lock_guard<std::mutex> g(mu_);
      int slot = -1;
      for (int i = 0; i < kSlots; i++) if (!blk_[i].p) { slot = i; break; }
      if (slot < 0) {                                      // full: the smallest block makes room for a larger one
        int sm = 0;
        for (int i = 1; i < kSlots; i++) if (blk_[i].cap < blk_[sm].cap) sm = i;
        if (blk_[sm].cap < cap) { ::operator delete(blk_[sm].p); total_ -= blk_[sm].cap; blk_[sm] = Blk{nullptr, 0}; slot = sm; }
      }
      if (slot >= 0 && total_ + cap <= kMaxBytes) { blk_[slot] = Blk{p, cap}; total_ += cap; return; }
    }
    ::operator delete(p);
  }
 private:
  static constexpr int kSlots = 4;
  static constexpr size_t kMaxBytes = (size_t)1 << 30;
  struct Blk { void *p; size_t cap; };
  std::mutex mu_;
  Blk blk_[kSlots] = {};
  size_t total_ = 0;
};

// The LISTed objects of a snapshot: a fixed-size array whose elements are constructed IN PLACE by the ingest threads (a
// std::vector would value-initialise 200k x ~1 KB objects on one core before the parse even starts, and first-touch all of
// their pages there).
template <class T> class ObjList {
 public:
  ObjList() = default;
  ObjList(const ObjList &) = delete;
  ObjList &operator=(const ObjList &) = delete;
  ObjList(ObjList &&o) noexcept : p_(o.p_), n_(o.n_), cap_(o.cap_) { o.p_ = nullptr; o.n_ = 0; o.cap_ = 0; }
  ObjList &operator=(ObjList &&o) noexcept { if (this != &o) { clear(); p_ = o.p_; n_ = o.n_; cap_ = o.cap_; o.p_ = nullptr; o.n_ = 0; o.cap_ = 0; } return *this; }
  ~ObjList() { clear(); }
  void clear() { for (size_t i = 0; i < n_; i++) p_[i].~T(); RawBlockCache::get().give(p_, cap_); p_ = nullptr; n_ = 0; cap_ = 0; }
  // raw storage for n elements: the caller constructs every one of them (placement new) before anything else touches the list
  T *allocate_raw(size_t n) {
    clear();
    if (n) {
      const size_t bytes = n * sizeof(T);
      void *q = RawBlockCache::get().take(bytes, cap_);
      if (!q) { q = ::operator new(bytes); cap_ = bytes; }
      p_ = static_cast<T *>(q);
    }
    n_ = n;
    return p_;
  }
  size_t size() const { return n_; }
  bool empty() const { return n_ == 0; }
  const T &operator[](size_t i) const { return p_[i]; }
  T &operator[](size_t i) { return p_[i]; }
  const T *begin() const { return p_; }
  const T *end() const { return p_ + n_; }
  T *begin() { return p_; }
  T *end() { return p_ + n_; }
 private:
  T *p_ = nullptr;
  size_t n_ = 0, cap_ = 0;
};

struct Pod {
  Json raw;
  std::string name, ns, node_name, phase, scheduler_name, preemption_policy;
  Labels labels;
  bool terminating = false;      // metadata.deletionTimestamp set
  std::string owner_api_version, owner_kind, owner_name;   // metav1.GetControllerOf: the ownerReference with controller=true
  int priority = 0;
  std::vector<Container> containers, init_containers;
  ResourceList overhead, pod_level_requests;
  bool has_pod_level_requests = false;
  Labels node_selector;
  bool has_node_selector = false;   // spec.nodeSelector != nil (an empty map still disables the PreFilter Skip)
  bool has_required_node_affinity = false;
  std::vector<NodeSelectorTerm> node_affinity_terms;   // empty terms already dropped
  bool has_preferred_node_affinity = false;
  std::vector<std::pair<int, NodeSelectorTerm>> node_affinity_preferred;   // (weight, preference); weight 0 / empty terms dropped
  std::vector<Toleration> tolerations;
  std::vector<AffinityTerm> aff_required, anti_required, aff_preferred, anti_preferred;
  std::vector<TopologySpreadConstraint> spread;
  bool has_pvc_volume = false, has_resource_claims = false, has_scheduling_gates = false;
  std::map<std::string, ResourceList> status_resources, status_allocated;   // containerStatuses[*].resources.requests / allocatedResources
  bool resize_infeasible = false;

  // WeightedPodAffinityTerm.weight and PreferredSchedulingTerm.weight are int32 in the API: a value outside int32 does not
  // decode there, and is refused here instead of being truncated
  static int term_weight(const Json &w) {
    const int64_t v = w.i64(0);
    if (v < INT32_MIN || v > INT32_MAX) throw std::runtime_error("a preferred term's weight " + std::to_string(v) + " is outside int32");
    return (int)v;
  }

  static std::vector<AffinityTerm> parse_terms(const Json &arr, const std::string &pod_ns, bool weighted) {
    std::vector<AffinityTerm> out;
    if (!arr.is_array()) return out;
    for (auto &e0 : arr.arr) {
      const Json &e = weighted ? e0.at("podAffinityTerm") : e0;
      AffinityTerm t;
      t.topology_key = e.at("topologyKey").str();
      t.selector = Selector::from_label_selector(e.at("labelSelector"));
      const Json &nss = e.at("namespaces");
      const Json &nsel = e.at("namespaceSelector");
      if ((!nss.is_array() || nss.arr.empty()) && !nsel.is_object()) t.namespaces.insert(pod_ns);
      else if (nss.is_array()) for (auto &x : nss.arr) t.namespaces.insert(x.str());
      t.ns_selector = Selector::from_label_selector(nsel);
      if (weighted) t.weight = term_weight(e0.at("weight"));
      out.push_back(t);
    }
    return out;
  }

  static Container parse_container(const Json &c) {
    Container k;
    k.name = c.at("name").str();
    k.image = c.at("image").str();
    k.requests = parse_resources(c.at("resources").at("requests"));
    k.restart_always = c.at("restartPolicy").str() == "Always";
    if (c.at("ports").is_array())
      for (auto &p : c.at("ports").arr) {
        ContainerPort cp;
        cp.host_port = (int)p.at("hostPort").i64(0);
        cp.host_ip = p.at("hostIP").str();
        cp.protocol = p.at("protocol").str();
        k.ports.push_back(cp);
      }
    return k;
  }

  static Pod parse(const Json &j, bool keep_raw = false) {
    Pod p;
    if (keep_raw) p.raw = j;      // only the simulated pod is echoed back (report.go:60-66); existing pods are not
    const Json &md = j.at("metadata"), &sp = j.at("spec"), &st = j.at("status");
    p.name = md.at("name").str();
    p.ns = md.at("namespace").str("default");
    if (p.ns.empty()) p.ns = "default";
    p.labels = parse_labels(md.at("labels"));
    p.terminating = !md.at("deletionTimestamp").is_null();
    if (md.at("ownerReferences").is_array())
      for (auto &o : md.at("ownerReferences").arr)
        if (o.at("controller").truthy()) { p.owner_api_version = o.at("apiVersion").str(); p.owner_kind = o.at("kind").str(); p.owner_name = o.at("name").str(); break; }
    p.node_name = sp.at("nodeName").str();
    p.phase = st.at("phase").str();
    p.scheduler_name = sp.at("schedulerName").str();
    p.preemption_policy = sp.at("preemptionPolicy").str();
    p.priority = (int)sp.at("priority").i64(0);
    if (sp.at("containers").is_array()) for (auto &c : sp.at("containers").arr) p.containers.push_back(parse_container(c));
    if (sp.at("initContainers").is_array()) for (auto &c : sp.at("initContainers").arr) p.init_containers.push_back(parse_container(c));
    p.overhead = parse_resources(sp.at("overhead"));
    p.pod_level_requests = parse_resources(sp.at("resources").at("requests"));
    for (auto &kv : p.pod_level_requests)   // IsSupportedPodLevelResource: cpu, memory, hugepages-*
      if (kv.first == "cpu" || kv.first == "memory" || kv.first.rfind("hugepages-", 0) == 0) p.has_pod_level_requests = true;
    p.has_node_selector = sp.at("nodeSelector").is_object();
    p.node_selector = parse_labels(sp.at("nodeSelector"));
    const Json &na = sp.at("affinity").at("nodeAffinity");
    const Json &req = na.at("requiredDuringSchedulingIgnoredDuringExecution");
    if (req.is_object()) {
      p.has_required_node_affinity = true;
      if (req.at("nodeSelectorTerms").is_array())
        for (auto &t : req.at("nodeSelectorTerms").arr) {
          NodeSelectorTerm nt;
          if (t.at("matchExpressions").is_array())
            for (auto &e : t.at("matchExpressions").arr) {
              Requirement r{e.at("key").str(), e.at("operator").str(), {}};
              for (auto &v : e.at("values").arr) r.values.push_back(v.str());
              nt.match_expressions.push_back(r);
            }
          if (t.at("matchFields").is_array())
            for (auto &e : t.at("matchFields").arr) {
              Requirement r{e.at("key").str(), e.at("operator").str(), {}};
              for (auto &v : e.at("values").arr) r.values.push_back(v.str());
              nt.match_fields.push_back(r);
            }
          if (!nt.empty()) p.node_affinity_terms.push_back(nt);   // nil or empty term selects no objects
        }
    }
    const Json &pref = na.at("preferredDuringSchedulingIgnoredDuringExecution");
    p.has_preferred_node_affinity = pref.is_array() && !pref.arr.empty();
    if (pref.is_array())
      for (auto &pt : pref.arr) {   // NewPreferredSchedulingTerms (nodeaffinity.go:118-139)
        NodeSelectorTerm nt;
        const Json &t = pt.at("preference");
        if (t.at("matchExpressions").is_array())
          for (auto &e : t.at("matchExpressions").arr) {
            Requirement r{e.at("key").str(), e.at("operator").str(), {}};
            for (auto &v : e.at("values").arr) r.values.push_back(v.str());
            nt.match_expressions.push_back(r);
          }
        if (t.at("matchFields").is_array())
          for (auto &e : t.at("matchFields").arr) {
            Requirement r{e.at("key").str(), e.at("operator").str(), {}};
            for (auto &v : e.at("values").arr) r.values.push_back(v.str());
            nt.match_fields.push_back(r);
          }
        const int w = term_weight(pt.at("weight"));
        if (w != 0 && !nt.empty()) p.node_affinity_preferred.push_back({w, nt});
      }
    if (sp.at("tolerations").is_array())
      for (auto &t : sp.at("tolerations").arr)
        p.tolerations.push_back(Toleration{t.at("key").str(), t.at("operator").str(), t.at("value").str(), t.at("effect").str()});
    const Json &pa = sp.at("affinity").at("podAffinity"), &paa = sp.at("affinity").at("podAntiAffinity");
    p.aff_required = parse_terms(pa.at("requiredDuringSchedulingIgnoredDuringExecution"), p.ns, false);
    p.anti_required = parse_terms(paa.at("requiredDuringSchedulingIgnoredDuringExecution"), p.ns, false);
    p.aff_preferred = parse_terms(pa.at("preferredDuringSchedulingIgnoredDuringExecution"), p.ns, true);
    p.anti_preferred = parse_terms(paa.at("preferredDuringSchedulingIgnoredDuringExecution"), p.ns, true);
    if (sp.at("topologySpreadConstraints").is_array())
      for (auto &c : sp.at("topologySpreadConstraints").arr) {
        TopologySpreadConstraint t;
        t.max_skew = (int)c.at("maxSkew").i64(1);
        t.topology_key = c.at("topologyKey").str();
        t.when_unsatisfiable = c.at("whenUnsatisfiable").str();
        t.label_selector = c.at("labelSelector");
        if (c.at("matchLabelKeys").is_array()) for (auto &k : c.at("matchLabelKeys").arr) t.match_label_keys.push_back(k.str());
        if (!c.at("minDomains").is_null()) t.min_domains = (int)c.at("minDomains").i64(1);
        if (c.at("nodeAffinityPolicy").is_string()) t.node_affinity_policy = c.at("nodeAffinityPolicy").str();
        if (c.at("nodeTaintsPolicy").is_string()) t.node_taints_policy = c.at("nodeTaintsPolicy").str();
        p.spread.push_back(t);
      }
    if (sp.at("volumes").is_array())
      for (auto &v : sp.at("volumes").arr) if (v.at("persistentVolumeClaim").is_object() || v.at("ephemeral").is_object()) p.has_pvc_volume = true;
    p.has_resource_claims = sp.at("resourceClaims").is_array() && !sp.at("resourceClaims").arr.empty();
    p.has_scheduling_gates = sp.at("schedulingGates").is_array() && !sp.at("schedulingGates").arr.empty();
    for (const char *field : {"containerStatuses", "initContainerStatuses"})
      if (st.at(field).is_array())
        for (auto &cs : st.at(field).arr) {
          if (cs.at("resources").is_object()) p.status_resources[cs.at("name").str()] = parse_resources(cs.at("resources").at("requests"));
          if (cs.at("allocatedResources").is_object()) p.status_allocated[cs.at("name").str()] = parse_resources(cs.at("allocatedResources"));
        }
    if (st.at("conditions").is_array())
      for (auto &c : st.at("conditions").arr)
        if (c.at("type").str() == "PodResizePending") p.resize_infeasible = c.at("reason").str() == "Infeasible";
    return p;
  }

  // schedutil.GetHostPorts
  std::vector<ContainerPort> host_ports() const {
    std::vector<ContainerPort> out;
    for (auto &c : init_containers) if (c.restart_always) for (auto &p : c.ports) if (p.host_port > 0) out.push_back(p);
    for (auto &c : containers) for (auto &p : c.ports) if (p.host_port > 0) out.push_back(p);
    return out;
  }

  // resourcehelper.PodRequests (UseStatusResources = InPlacePodVerticalScaling, pod-level resources honoured unless skipped)
  ResourceList requests(bool use_status, bool skip_pod_level, const ResourceList *non_missing) const {
    auto container_reqs = [&](const Container &c, bool is_init) {
      ResourceList r = c.requests;
      if (use_status && (!is_init || c.restart_always)) {
        auto it = status_resources.find(c.name);
        if (it != status_resources.end()) {   // determineContainerReqs
          ResourceList m;
          if (!resize_infeasible) max_resources(m, c.requests);
          max_resources(m, it->second);
          auto ia = status_allocated.find(c.name);
          if (ia != status_allocated.end()) max_resources(m, ia->second);
          r = m;
        }
      }
      if (non_missing) for (auto &kv : *non_missing) if (!r.count(kv.first)) r[kv.first] = kv.second;   // applyNonMissing
      return r;
    };
    ResourceList reqs;
    for (auto &c : containers) add_resources_fmt(reqs, container_reqs(c, false));
    ResourceList restartable, init_max;
    for (auto &c : init_containers) {
      ResourceList cr = container_reqs(c, true);
      if (c.restart_always) {
        add_resources_fmt(reqs, cr);
        add_resources_fmt(restartable, cr);
        cr = restartable;
      } else {
        ResourceList tmp;
        add_resources_fmt(tmp, cr);
        add_resources_fmt(tmp, restartable);
        cr = tmp;
      }
      max_resources(init_max, cr);
    }
    max_resources(reqs, init_max);
    if (!skip_pod_level && has_pod_level_requests)
      for (auto &kv : pod_level_requests)
        if (kv.first == "cpu" || kv.first == "memory" || kv.first.rfind("hugepages-", 0) == 0) reqs[kv.first] = kv.second;
    add_resources_fmt(reqs, overhead);
    return reqs;
  }
};

struct Node {
  std::string name;
  Labels labels;
  bool unschedulable = false;
  std::vector<Taint> taints;
  ResourceList allocatable;
  std::vector<std::string> image_names;
  std::vector<std::pair<std::string, int64_t>> images;   // (name, sizeBytes) for every name of every status.images entry

  static Node parse(const Json &j) {
    Node n;
    n.name = j.at("metadata").at("name").str();
    n.labels = parse_labels(j.at("metadata").at("labels"));
    n.unschedulable = j.at("spec").at("unschedulable").truthy();
    if (j.at("spec").at("taints").is_array())
      for (auto &t : j.at("spec").at("taints").arr) n.taints.push_back(Taint{t.at("key").str(), t.at("value").str(), t.at("effect").str()});
    n.allocatable = parse_resources(j.at("status").at("allocatable"));
    if (j.at("status").at("images").is_array())
      for (auto &im : j.at("status").at("images").arr)
        if (im.at("names").is_array()) for (auto &nm : im.at("names").arr) {
          n.image_names.push_back(nm.str());
          n.images.push_back({nm.str(), im.at("sizeBytes").i64(0)});
        }
    return n;
  }
  // utilnode.GetZoneKey (component-helpers/node/topology/helpers.go:31-58)
  std::string zone_key() const {
    auto get = [&](const char *k, std::string &out) { auto it = labels.find(k); if (it == labels.end()) return false; out = it->second; return true; };
    std::string zone, region;
    if (!get("failure-domain.beta.kubernetes.io/zone", zone)) get("topology.kubernetes.io/zone", zone);
    if (!get("failure-domain.beta.kubernetes.io/region", region)) get("topology.kubernetes.io/region", region);
    if (region.empty() && zone.empty()) return "";
    return region + ":" + std::string(1, '\0') + ":" + zone;
  }
};

// The objects helper.DefaultSelector reads (plugins/helper/spread.go:40-113): Services select by a label map, RCs too,
// ReplicaSets / StatefulSets by a LabelSelector.
struct WorkloadSelector {
  std::string kind, ns, name;
  bool has_map = false;      // Service/RC: spec.selector != nil
  Labels map;
  Json label_selector;       // RS/StatefulSet: spec.selector
  static WorkloadSelector parse(const Json &j, const std::string &kind) {
    WorkloadSelector w;
    w.kind = kind;
    w.ns = j.at("metadata").at("namespace").str();
    if (w.ns.empty()) w.ns = "default";
    w.name = j.at("metadata").at("name").str();
    const Json &sel = j.at("spec").at("selector");
    if (kind == "Service" || kind == "ReplicationController") { w.has_map = sel.is_object(); w.map = parse_labels(sel); }
    else w.label_selector = sel;
    return w;
  }
};

// schedutil.IsScalarResourceName (kubernetes/pkg/scheduler/util/utils.go:139-143)
inline bool is_scalar_resource_name(const std::string &n) {
  const bool native = n.find('/') == std::string::npos || n.find("kubernetes.io/") != std::string::npos;
  const bool extended = !native && n.rfind("requests.", 0) != 0;
  return extended || n.rfind("hugepages-", 0) == 0 || n.find("kubernetes.io/") != std::string::npos || n.rfind("attachable-volumes-", 0) == 0;
}

}  // namespace cch
