// cchost.cpp — libcchost.so: the host side of the hot path, mirroring the reference's pkg/framework surface
// (ClusterCapacity New / SyncWithClient / Run / Report / Close and ClusterCapacityReviewPrint) on top of libccsim.
// See include/cchost.h for the mapping to reference file:line.
#include <chrono>
#include <cstdarg>
#include <ctime>
#include <sstream>
#include <thread>
#include <mutex>
#include <exception>
#include <system_error>
#include <cstring>
#include "../../../include/cchost.h"
#include "encoder.hpp"
#include "fastparse.hpp"

using namespace cch;

namespace {

const char *kReasonText[CCSIM_R_FIXED_COUNT] = {
    "node(s) were unschedulable",                                          // nodeunschedulable/node_unschedulable.go:49
    "node(s) didn't match the requested node name",                        // nodename/node_name.go:43
    "node(s) didn't match Pod's node affinity/selector",                   // nodeaffinity/node_affinity.go:64
    "node(s) didn't have free ports for the requested pod ports",          // nodeports/node_ports.go:51
    "Too many pods", "Insufficient cpu", "Insufficient memory", "Insufficient ephemeral-storage",   // noderesources/fit.go:567-616
    "node(s) didn't match pod topology spread constraints (missing required label)",                 // podtopologyspread/filtering.go
    "node(s) didn't match pod topology spread constraints",
    "node(s) didn't match pod affinity rules",                             // interpodaffinity/filtering.go:36-42
    "node(s) didn't match pod anti-affinity rules",
    "node(s) didn't satisfy existing pods anti-affinity rules",
    "node(s) didn't satisfy plugin(s) [NodeAffinity]",                     // schedule_one.go:533
};

// FitError.Error() (framework/types.go:787-838): "0/N nodes are available: <sorted 'count reason'>."
std::string fit_error_body(int n, const std::vector<std::pair<std::string, int64_t>> &hist) {
  std::string msg = "0/" + std::to_string(n) + " nodes are available:";
  std::vector<std::string> strs;
  for (auto &kv : hist) if (kv.second) strs.push_back(std::to_string(kv.second) + " " + kv.first);
  std::sort(strs.begin(), strs.end());
  if (!strs.empty()) {
    msg += " ";
    for (size_t i = 0; i < strs.size(); i++) { if (i) msg += ", "; msg += strs[i]; }
    msg += ".";
  }
  return msg;
}

std::string rfc3339_now() {
  using namespace std::chrono;
  auto now = system_clock::now();
  time_t t = system_clock::to_time_t(now);
  long ns = (long)(duration_cast<nanoseconds>(now.time_since_epoch()).count() % 1000000000LL);
  struct tm g; gmtime_r(&t, &g);
  char buf[64]; strftime(buf, sizeof(buf), "%Y-%m-%dT%H:%M:%S", &g);
  char frac[16]; snprintf(frac, sizeof(frac), "%09ld", ns);
  std::string f(frac);
  while (!f.empty() && f.back() == '0') f.pop_back();
  return std::string(buf) + (f.empty() ? "" : "." + f) + "Z";
}

// ---- YAML emitter for the report (sigs.k8s.io/yaml: JSON -> map -> go-yaml, keys sorted) ----
bool yaml_plain_ok(const std::string &s) {
  if (s.empty()) return false;
  static const char *special[] = {"null", "Null", "NULL", "~", "true", "True", "TRUE", "false", "False", "FALSE", "yes", "Yes", "no", "No", "on", "off", "y", "n"};
  for (auto *w : special) if (s == w) return false;
  char c0 = s[0];
  if (strchr("-?:,[]{}#&*!|>'\"%@` ", c0)) return false;
  if (isdigit((unsigned char)c0) || c0 == '.' || c0 == '+') {   // could parse as a number
    char *e = nullptr; strtod(s.c_str(), &e);
    if (e && *e == 0) return false;
  }
  if (s.back() == ' ' || s.back() == ':') return false;
  for (size_t i = 0; i < s.size(); i++) {
    unsigned char c = (unsigned char)s[i];
    if (c < 0x20 || c == 0x7f) return false;
    if (c == ':' && (i + 1 == s.size() || s[i + 1] == ' ')) return false;
    if (c == '#' && i > 0 && s[i - 1] == ' ') return false;
  }
  return true;
}
std::string yaml_scalar(const Json &j) {
  switch (j.type) {
    case Json::Null: return "null";
    case Json::Bool: return j.b ? "true" : "false";
    case Json::Number: return j.s;
    case Json::String: {
      if (yaml_plain_ok(j.s)) return j.s;
      bool simple = true;
      for (unsigned char c : j.s) if (c < 0x20 || c == '\\' ) simple = false;
      if (simple && j.s.find('\'') == std::string::npos) return "'" + j.s + "'";
      std::string o; json_escape(j.s, o); return o;
    }
    default: return "";
  }
}
void yaml_emit(const Json &j, int indent, std::string &out) {
  std::string pad(indent, ' ');
  if (j.type == Json::Object) {
    std::vector<const std::pair<std::string, Json> *> kv;
    for (auto &p : j.obj) kv.push_back(&p);
    std::sort(kv.begin(), kv.end(), [](auto *a, auto *b) { return a->first < b->first; });
    for (auto *p : kv) {
      const Json &v = p->second;
      std::string key = yaml_plain_ok(p->first) ? p->first : ("\"" + p->first + "\"");
      if (v.type == Json::Object && !v.obj.empty()) { out += pad + key + ":\n"; yaml_emit(v, indent + 2, out); }
      else if (v.type == Json::Array && !v.arr.empty()) { out += pad + key + ":\n"; yaml_emit(v, indent, out); }
      else if (v.type == Json::Object) out += pad + key + ": {}\n";
      else if (v.type == Json::Array) out += pad + key + ": []\n";
      else out += pad + key + ": " + yaml_scalar(v) + "\n";
    }
  } else if (j.type == Json::Array) {
    for (auto &v : j.arr) {
      if ((v.type == Json::Object && !v.obj.empty()) || (v.type == Json::Array && !v.arr.empty())) {
        std::string sub; yaml_emit(v, indent + 2, sub);
        sub[indent] = '-';   // first line: replace the first pad character of the nested block by the dash
        out += sub;
      } else if (v.type == Json::Object) out += pad + "- {}\n";
      else if (v.type == Json::Array) out += pad + "- []\n";
      else out += pad + "- " + yaml_scalar(v) + "\n";
    }
  } else out += pad + yaml_scalar(j) + "\n";
}

}  // namespace

struct cc_handle {
  SchedConfig cfg;
  Pod tmpl;                    // the first (usually only) template
  std::vector<Pod> tmpls;      // all templates: pod k of the run is a clone of tmpls[k % T] (report.go:160)
  std::vector<ccsim_template> enc_tmpls;          // encoded templates over the merged snapshot (T > 1)
  std::vector<std::vector<uint8_t>> enc_images;   // their ImageLocality columns
  int64_t max_pods = 0;
  std::set<std::string> exclude;
  std::vector<int32_t> devices;   // CUDA ordinals: one, or the list of a cc_new_each_on handle
  ObjList<Node> nodes;
  ObjList<Pod> pods;
  std::map<std::string, Labels> ns_labels;
  std::vector<WorkloadSelector> workloads;   // Services / RCs / ReplicaSets / StatefulSets (system-default topology spreading)
  bool synced = false, ran = false, closed = false;
  Encoded enc;
  bool have_enc = false;
  // Status{Pods, StopReason} (pkg/framework/simulator.go:90-93)
  std::vector<int32_t> pod_node;
  std::string stop_reason;
  Json report;   // cached like c.report (simulator.go:161-169)
  bool have_report = false;
  std::string err, out, warn;
  int64_t pending_skipped = 0;   // pods of the snapshot without spec.nodeName (not terminal): not replayed, reported by cc_warnings
  // cc_run_each: one read-only view per podspec (cc_analysis); a view's node names are its base's
  std::vector<std::unique_ptr<cc_handle>> analyses;
  const cc_handle *base = nullptr;
  // cc_new_each: a per-analysis handle; parts[t] holds podspec t's own terms (counters, counter inits, topology columns, PreFilter
  // message, node count; its static bits moved like the merged template's), the node columns of its encoding are dropped after the merge
  bool each = false;
  std::vector<Encoded> parts;
};

// the encoding a handle's node indices refer to (a view's is its base's)
static const Encoded &enc_of(const cc_handle *h) { return h->base ? h->base->enc : h->enc; }

static std::string g_new_err;
static int fail(cc_handle *h, int code, const std::string &m) { if (h) h->err = m; else g_new_err = m; return code; }

// 256-bit static-bit vectors as 4 words; shift left by `off` bits
static void shl256(const uint64_t in[CCSIM_MAX_STATIC_WORDS], int off, uint64_t out[CCSIM_MAX_STATIC_WORDS]) {
  const int ws = off >> 6, bs = off & 63;
  for (int w = CCSIM_MAX_STATIC_WORDS - 1; w >= 0; w--) {
    uint64_t v = 0;
    if (w - ws >= 0) { v = in[w - ws] << bs; if (bs && w - ws - 1 >= 0) v |= in[w - ws - 1] >> (64 - bs); }
    out[w] = v;
  }
}

// Several templates against one snapshot (the roadmap's "list of pods", README.md:305-306; template index = k % T,
// report.go:160): the podspec-independent part of the encoding (node order, NodeInfo columns, taint dictionary: Cluster) is built
// once, every template is encoded against it, and the encodings are merged: the static predicate bits of template t move up by the
// bits of templates 0..t-1; extended resources are the union. A list handle's run is one run: per-domain counters (PodTopologySpread
// / InterPodAffinity terms) stay single-template there. A per-analysis handle (h->each) keeps every part's counters, counter inits,
// topology columns and PreFilter message as that analysis's own (h->parts), and its hostPort self-conflict becomes bit t mod 64.
// Each template's static bits and extended-resource columns fold into the merged ones as soon as it is encoded, so the parts held
// at once are the small ones whatever the number of templates.
static void encode_list(cc_handle *h) {
  const size_t T = h->tmpls.size();
  const auto t0 = std::chrono::steady_clock::now();
  Cluster cluster(h->nodes, h->pods, h->exclude);
  const auto t1 = std::chrono::steady_clock::now();
  const int n = cluster.n();
  std::vector<Encoded> &parts = h->parts;
  parts.clear();
  parts.reserve(T);
  std::vector<std::string> names;                               // extended resources: union of the names the templates request
  std::vector<std::vector<int64_t>> alloc_scalar, req_scalar;   // ... and their columns
  std::vector<int> off(T, 0), nbits(T, 0);                      // static bits: template t's bits start at off[t]
  int total = 0;
  std::vector<uint64_t> smask((size_t)CCSIM_MAX_STATIC_WORDS * n, 0);   // the merged static bits (word-major), while they fit
  for (size_t t = 0; t < T; t++) {
    Encoder enc(h->cfg, h->tmpls[t], cluster, h->ns_labels);
    enc.set_workloads(&h->workloads);
    parts.push_back(enc.encode());
    Encoded &e = parts.back();
    if (!h->each) {
      if (!e.counters.empty()) throw Unsupported("several podspecs of which one has topology spread / pod (anti-)affinity terms or scores (single podspec only)");
      if (!e.prefilter_msg.empty()) throw Unsupported("several podspecs of which one is rejected by PreFilter");
      if (e.has_placed_mask) throw Unsupported("several podspecs with hostPorts");
    }
    for (size_t k = 0; k < e.scalar_names.size(); k++)
      if (std::find(names.begin(), names.end(), e.scalar_names[k]) == names.end()) {
        names.push_back(e.scalar_names[k]); alloc_scalar.push_back(std::move(e.alloc_scalar[k])); req_scalar.push_back(std::move(e.req_scalar[k]));
      }
    e.alloc_scalar.clear(); e.req_scalar.clear();
    // the bits a template really uses: highest set bit over its columns (an encoder allocates them densely from 0)
    int hi = 0;
    for (int w = 0; w < e.static_words; w++) {
      uint64_t acc = 0;
      for (int i = 0; i < n; i++) acc |= e.static_mask[(size_t)w * n + i];
      const ccsim_template &P = e.tmpl;
      acc |= P.sel_mask[w] | P.port_static_mask[w] | P.existing_anti_mask[w];
      for (int k = 0; k < CCSIM_MAX_AFF_TERMS; k++) acc |= P.aff_term_mask[k][w] | P.pref_mask[k][w];
      if (acc) hi = w * 64 + 64 - __builtin_clzll(acc);
    }
    if (e.tmpl.prefilter_bit >= 0) hi = std::max(hi, e.tmpl.prefilter_bit + 1);
    if (e.tmpl.spts_ignored_bit >= 0) hi = std::max(hi, e.tmpl.spts_ignored_bit + 1);
    for (const ccsim_counter &c : e.counters) if (c.elig_bit >= 0) hi = std::max(hi, c.elig_bit + 1);
    for (int c = 0; c < e.tmpl.n_spts; c++) if (e.tmpl.spts[c].has_key_bit >= 0) hi = std::max(hi, e.tmpl.spts[c].has_key_bit + 1);
    off[t] = total; nbits[t] = hi; total += hi;
    if (hi && total <= 64 * CCSIM_MAX_STATIC_WORDS)
      for (int i = 0; i < n; i++) {
        uint64_t in[CCSIM_MAX_STATIC_WORDS] = {0, 0, 0, 0}, out[CCSIM_MAX_STATIC_WORDS];
        for (int w = 0; w < e.static_words; w++) in[w] = e.static_mask[(size_t)w * n + i];
        shl256(in, off[t], out);
        for (int w = 0; w < CCSIM_MAX_STATIC_WORDS; w++) smask[(size_t)w * n + i] |= out[w];
      }
    std::vector<uint64_t>().swap(e.static_mask);
  }
  const auto t2 = std::chrono::steady_clock::now();
  if (names.size() > CCSIM_MAX_SCALARS) throw Unsupported("the podspecs request more than 4 distinct extended resources");
  if (total > 64 * CCSIM_MAX_STATIC_WORDS) throw Unsupported("the podspecs need more than 256 static node-predicate bits together");
  Encoded &m = h->enc;
  m = parts[0];
  cluster.columns_into(m);
  m.scalar_names = names;
  m.alloc_scalar = std::move(alloc_scalar);
  m.req_scalar = std::move(req_scalar);
  m.static_words = (total + 63) / 64;
  smask.resize((size_t)std::max(1, m.static_words) * n);
  m.static_mask = std::move(smask);
  h->enc_tmpls.assign(T, ccsim_template());
  h->enc_images.assign(T, std::vector<uint8_t>());
  for (size_t t = 0; t < T; t++) {
    const Encoded &e = parts[t];
    ccsim_template P = e.tmpl;
    auto mv = [&](uint64_t (&msk)[CCSIM_MAX_STATIC_WORDS]) { uint64_t o[CCSIM_MAX_STATIC_WORDS]; shl256(msk, off[t], o); memcpy(msk, o, sizeof(o)); };
    mv(P.sel_mask); mv(P.port_static_mask); mv(P.existing_anti_mask);
    for (int k = 0; k < CCSIM_MAX_AFF_TERMS; k++) { mv(P.aff_term_mask[k]); mv(P.pref_mask[k]); }
    if (P.prefilter_bit >= 0) P.prefilter_bit += off[t];
    if (P.spts_ignored_bit >= 0) P.spts_ignored_bit += off[t];
    for (int c = 0; c < P.n_spts; c++) if (P.spts[c].has_key_bit >= 0) P.spts[c].has_key_bit += off[t];
    if (h->each) {
      for (ccsim_counter &c : parts[t].counters) if (c.elig_bit >= 0) c.elig_bit += off[t];
      // a clone conflicts with the analysis's own clones: bit t mod 64 (one analysis at a time is diagnosed, so analyses 64 apart never meet)
      if (P.port_tmpl_conflict & 1ull) P.port_tmpl_conflict = 1ull << (t & 63);
      parts[t].tmpl = P;
    }
    // extended resources: re-index into the union
    int64_t rs[CCSIM_MAX_SCALARS] = {0, 0, 0, 0};
    for (size_t k = 0; k < e.scalar_names.size(); k++) rs[std::find(names.begin(), names.end(), e.scalar_names[k]) - names.begin()] = e.tmpl.req_scalar[k];
    memcpy(P.req_scalar, rs, sizeof(rs));
    h->enc_images[t] = e.image_score;
    P.image_score = h->enc_images[t].empty() ? nullptr : h->enc_images[t].data();
    h->enc_tmpls[t] = P;
  }
  m.tmpl = h->enc_tmpls[0];
  if (h->each) {   // the terms are the parts'; each part keeps only them
    for (auto &e : parts) m.has_placed_mask |= e.has_placed_mask;
    m.counters.clear(); m.counter_init.clear(); m.topo.clear(); m.prefilter_msg.clear();
    for (auto &e : parts) {
      Encoded k;
      k.n = e.n; k.counters = std::move(e.counters); k.counter_init = std::move(e.counter_init); k.topo = std::move(e.topo);
      k.prefilter_msg = std::move(e.prefilter_msg); k.tmpl = e.tmpl;
      e = std::move(k);
    }
  } else parts.clear();
  if (getenv("CCHOST_TIMING"))
    fprintf(stderr, "[cchost] encode: cluster (node order, pod assignment, node columns, taints) %.3f s, %zu podspecs %.3f s, merge %.3f s\n",
            std::chrono::duration<double>(t1 - t0).count(), T, std::chrono::duration<double>(t2 - t1).count(),
            std::chrono::duration<double>(std::chrono::steady_clock::now() - t2).count());
}

static void ensure_encoded(cc_handle *h) {
  if (h->have_enc) return;
  if (h->tmpls.size() > 1 || h->each) { encode_list(h); h->have_enc = true; return; }
  auto t0 = std::chrono::steady_clock::now();
  Cluster cluster(h->nodes, h->pods, h->exclude);
  auto t1 = std::chrono::steady_clock::now();
  Encoder enc(h->cfg, h->tmpl, cluster, h->ns_labels);
  enc.set_workloads(&h->workloads);
  h->enc = enc.encode();
  cluster.columns_into(h->enc);
  if (getenv("CCHOST_TIMING"))
    fprintf(stderr, "[cchost] encode: cluster (node order, pod assignment, node columns, taints) %.3f s, podspec (tolerations, static bits, counters) %.3f s\n",
            std::chrono::duration<double>(t1 - t0).count(), std::chrono::duration<double>(std::chrono::steady_clock::now() - t1).count());
  h->enc_tmpls.assign(1, h->enc.tmpl);
  h->have_enc = true;
}

extern "C" const char *cc_last_error(const cc_handle *h) { return h ? h->err.c_str() : g_new_err.c_str(); }

static std::vector<Json> items_of(const char *text);

// each: a per-analysis handle (cc_new_each), up to CCSIM_EACH_MAX_ANALYSES podspecs; else up to CCSIM_MAX_TEMPLATES
static int new_handle(const char *sched_config_json, std::vector<Json> pods, int64_t max_pods, const char *exclude_nodes,
                      std::vector<int32_t> devices, bool each, cc_handle **out) {
  if (pods.empty()) return fail(nullptr, CC_EINVAL, "no podspec");
  if (each && pods.size() > CCSIM_EACH_MAX_ANALYSES)
    return fail(nullptr, CC_EUNSUPPORTED, "more than " + std::to_string(CCSIM_EACH_MAX_ANALYSES) + " podspecs (CCSIM_EACH_MAX_ANALYSES, per-analysis runs)");
  if (!each && pods.size() > CCSIM_MAX_TEMPLATES) return fail(nullptr, CC_EUNSUPPORTED, "more than 64 podspecs");
  cc_handle *h = new cc_handle();
  h->each = each;
  try {
    h->cfg = SchedConfig::parse(sched_config_json ? sched_config_json : "");
    for (auto &j : pods) h->tmpls.push_back(Pod::parse(j, /*keep_raw=*/true));
    h->tmpl = h->tmpls[0];
    h->max_pods = max_pods;
    h->devices = std::move(devices);
    if (exclude_nodes) {
      std::stringstream ss(exclude_nodes); std::string item;
      while (std::getline(ss, item, ',')) if (!item.empty()) h->exclude.insert(item);
    }
    *out = h;
    return CC_OK;
  } catch (const std::exception &e) { delete h; return fail(nullptr, CC_EINVAL, e.what()); }
}

extern "C" int cc_new(const char *sched_config_json, const char *pod_json, int64_t max_pods, const char *exclude_nodes,
                      int32_t device, cc_handle **out) {
  if (!pod_json || !out) return fail(nullptr, CC_EINVAL, "null argument");
  try {
    std::vector<Json> one; one.push_back(parse_json(pod_json));
    return new_handle(sched_config_json, std::move(one), max_pods, exclude_nodes, {device}, false, out);
  } catch (const std::exception &e) { return fail(nullptr, CC_EINVAL, e.what()); }
}

extern "C" int cc_new_list(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                           int32_t device, cc_handle **out) {
  if (!pods_json || !out) return fail(nullptr, CC_EINVAL, "null argument");
  try { return new_handle(sched_config_json, items_of(pods_json), max_pods, exclude_nodes, {device}, false, out); }
  catch (const std::exception &e) { return fail(nullptr, CC_EINVAL, e.what()); }
}

extern "C" int cc_new_each(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                           int32_t device, cc_handle **out) {
  return cc_new_each_on(sched_config_json, pods_json, max_pods, exclude_nodes, &device, 1, out);
}

extern "C" int cc_new_each_on(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                              const int32_t *devices, int32_t n_devices, cc_handle **out) {
  if (!pods_json || !out || (n_devices > 0 && !devices)) return fail(nullptr, CC_EINVAL, "null argument");
  if (n_devices < 1) return fail(nullptr, CC_EINVAL, "empty device list");
  if (n_devices > CC_EACH_MAX_DEVICES)
    return fail(nullptr, CC_EINVAL, "more than " + std::to_string(CC_EACH_MAX_DEVICES) + " devices (" + std::to_string(n_devices) + ", CC_EACH_MAX_DEVICES)");
  for (int32_t g = 0; g < n_devices; g++)
    if (devices[g] < 0) return fail(nullptr, CC_EINVAL, "device list entry " + std::to_string(g) + ": negative CUDA ordinal " + std::to_string(devices[g]));
  try { return new_handle(sched_config_json, items_of(pods_json), max_pods, exclude_nodes, std::vector<int32_t>(devices, devices + n_devices), true, out); }
  catch (const std::exception &e) { return fail(nullptr, CC_EINVAL, e.what()); }
}

static std::vector<Json> items_of(const char *text) {
  std::vector<Json> v;
  if (!text || !*text) return v;
  Json j = parse_json(text);
  if (j.is_array()) v = std::move(j.arr);
  else if (Json *items = const_cast<Json *>(j.find("items")); items && items->is_array()) v = std::move(items->arr);
  else if (j.is_object()) v.push_back(std::move(j));
  return v;
}

// ---- snapshot ingest (SURVEY.md §8 f1): the LISTed objects arrive as one JSON document per kind; the items are independent,
// so their spans are located with one string-aware bracket scan and parsed + converted on all host cores. Order is kept
// (node order feeds nodeTree, node_tree.go:51-67). Documents of another shape take the DOM path. ----
static size_t skip_ws(const char *t, size_t n, size_t p) { while (p < n && (t[p] == ' ' || t[p] == '\n' || t[p] == '\t' || t[p] == '\r')) p++; return p; }
static size_t skip_string(const char *t, size_t n, size_t p) {   // p at the opening quote; returns the position after the closing one
  for (p++; p < n; p++) { if (t[p] == '\\') p++; else if (t[p] == '"') return p + 1; }
  throw std::runtime_error("json: unterminated string");
}
static size_t skip_value(const char *t, size_t n, size_t p) {
  p = skip_ws(t, n, p);
  if (p >= n) throw std::runtime_error("json: unexpected end");
  if (t[p] == '"') return skip_string(t, n, p);
  if (t[p] == '{' || t[p] == '[') {
    int depth = 0;
    for (; p < n; p++) {
      const char c = t[p];
      if (c == '"') { p = skip_string(t, n, p) - 1; continue; }
      if (c == '{' || c == '[') depth++;
      else if (c == '}' || c == ']') { if (--depth == 0) return p + 1; }
    }
    throw std::runtime_error("json: unterminated value");
  }
  while (p < n && t[p] != ',' && t[p] != ']' && t[p] != '}' && t[p] != ' ' && t[p] != '\n' && t[p] != '\t' && t[p] != '\r') p++;
  return p;
}
// The two passes of item_spans_parallel over one chunk [q, end). Scalar reference versions first; the AVX2 versions below do the same
// 32 bytes at a time from compare masks (quotes, brackets: '[' / ']' fold onto '{' / '}' with bit 5 set; a 32-byte block that holds
// a backslash, and in pass 2 everything between two items, goes through the scalar code) and are tested against them.
struct SpanPart { int quotes = 0; long long depth[2] = {0, 0}; };   // depth[s]: change of bracket depth over the bytes seen in relative string state s
static inline void span_pass1_byte(const char *t, size_t &q, int &in, SpanPart &r) {
  const char ch = t[q];
  if (ch == '\\') { q++; return; }
  if (ch == '"') { in ^= 1; r.quotes++; return; }
  if (ch == '{' || ch == '[') r.depth[in]++;
  else if (ch == '}' || ch == ']') r.depth[in]--;
}
static void span_pass1_scalar(const char *t, size_t q, size_t end, SpanPart &r) {
  int in = 0;
  for (; q < end; q++) span_pass1_byte(t, q, in, r);
}
struct SpanEmit { std::vector<size_t> opens, closes; char bad = 0; size_t list_end = (size_t)-1; };
// one byte of pass 2; returns false when the ']' of the item list was met (the rest of the document is not ours)
static inline bool span_pass2_byte(const char *t, size_t &q, int &in, long long &d, SpanEmit &e) {
  const char ch = t[q];
  if (ch == '\\') { q++; return true; }
  if (ch == '"') { if (!in && d == 0) e.bad = 1; in ^= 1; return true; }      // (a string item: not ours either)
  if (in) return true;
  if (ch == '{' || ch == '[') { if (d == 0) { if (ch == '{') e.opens.push_back(q); else e.bad = 1; } d++; }
  else if (ch == '}' || ch == ']') {
    d--;
    if (d == 0) e.closes.push_back(q + 1);
    else if (d < 0) { e.list_end = q; return false; }
  } else if (d == 0 && ch != ',' && ch != ' ' && ch != '\n' && ch != '\t' && ch != '\r') e.bad = 1;   // a scalar item
  return true;
}
static void span_pass2_scalar(const char *t, size_t q, size_t end, int in, long long d, SpanEmit &e) {
  for (; q < end; q++) if (!span_pass2_byte(t, q, in, d, e)) return;
}
#if defined(__x86_64__)
#include <immintrin.h>
static inline uint32_t prefix_xor32(uint32_t x) { x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16; return x; }
__attribute__((target("avx2,popcnt"))) static void span_pass1_avx2(const char *t, size_t q, size_t end, SpanPart &r) {
  const __m256i quote = _mm256_set1_epi8('"'), bslash = _mm256_set1_epi8('\\'), open = _mm256_set1_epi8('{'), close = _mm256_set1_epi8('}');
  const __m256i bit5 = _mm256_set1_epi8(0x20);
  int in = 0;
  while (q < end) {
    if (q + 32 <= end) {
      const __m256i v = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(t + q));
      if (!_mm256_movemask_epi8(_mm256_cmpeq_epi8(v, bslash))) {
        const __m256i w = _mm256_or_si256(v, bit5);
        const uint32_t Q = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(v, quote));
        const uint32_t O = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(w, open)), C = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(w, close));
        uint32_t S = prefix_xor32(Q);            // bit i: an odd number of quotes in bytes 0..i (a bracket is not a quote: inclusive = exclusive there)
        if (in) S = ~S;
        r.depth[0] += __builtin_popcount(O & ~S) - __builtin_popcount(C & ~S);
        r.depth[1] += __builtin_popcount(O & S) - __builtin_popcount(C & S);
        const int nq = __builtin_popcount(Q);
        r.quotes += nq; in ^= nq & 1;
        q += 32;
        continue;
      }
    }
    const size_t stop = std::min(end, q + 32);   // a block with a backslash, or the tail: byte by byte
    for (; q < stop; q++) span_pass1_byte(t, q, in, r);
  }
}
__attribute__((target("avx2,popcnt"))) static void span_pass2_avx2(const char *t, size_t q, size_t end, int in, long long d, SpanEmit &e) {
  const __m256i quote = _mm256_set1_epi8('"'), bslash = _mm256_set1_epi8('\\'), open = _mm256_set1_epi8('{'), close = _mm256_set1_epi8('}');
  const __m256i bit5 = _mm256_set1_epi8(0x20);
  while (q < end) {
    if (d > 0 && q + 32 <= end) {                // inside an item: only quotes and brackets matter
      const __m256i v = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(t + q));
      if (!_mm256_movemask_epi8(_mm256_cmpeq_epi8(v, bslash))) {
        const __m256i w = _mm256_or_si256(v, bit5);
        const uint32_t Q = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(v, quote));
        const uint32_t O = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(w, open)), C = (uint32_t)_mm256_movemask_epi8(_mm256_cmpeq_epi8(w, close));
        uint32_t S = prefix_xor32(Q);
        if (in) S = ~S;
        uint32_t B = (O | C) & ~S;               // brackets outside strings, in order
        bool left = false;
        while (B) {
          const int i = __builtin_ctz(B);
          B &= B - 1;
          if ((O >> i) & 1u) d++;
          else if (--d == 0) {                   // the item ends here: what follows, up to the next '{', is looked at byte by byte
            e.closes.push_back(q + (size_t)i + 1);
            in = 0; q += (size_t)i + 1; left = true;
            break;
          }
        }
        if (!left) { in ^= __builtin_popcount(Q) & 1; q += 32; }
        continue;
      }
      const size_t stop = q + 32;                // a block with a backslash: byte by byte
      for (; q < stop; q++) if (!span_pass2_byte(t, q, in, d, e)) return;
      continue;
    }
    if (!span_pass2_byte(t, q, in, d, e)) return;
    q++;
  }
}
static bool span_simd() { static const bool on = __builtin_cpu_supports("avx2") && __builtin_cpu_supports("popcnt") && !getenv("CCHOST_NO_SIMD"); return on; }
#else
static bool span_simd() { return false; }
static void span_pass1_avx2(const char *, size_t, size_t, SpanPart &) {}
static void span_pass2_avx2(const char *, size_t, size_t, int, long long, SpanEmit &) {}
#endif

// The item list of a big document, located on all host cores. `p` is just behind the '[' of the list. Whether a byte lies inside a
// string is the parity of the unescaped quotes before it, and in valid JSON a backslash only occurs inside strings, so "skip the
// byte after a backslash" finds the same unescaped quotes wherever a chunk starts (chunks start behind a non-backslash byte).
// Pass 1 (parallel): per chunk the quote parity and the bracket-depth change under both start states; a serial prefix gives
// every chunk its true start state and depth; pass 2 (parallel): the '{' that opens depth 1 and the '}' that closes it are the
// item boundaries. Anything unexpected (an item that is not an object, a document that ends early) returns false: the serial
// scan then decides.
static bool item_spans_parallel(const char *t, size_t n, size_t p, std::vector<std::pair<size_t, size_t>> &out) {
  unsigned nt = host_threads();
  if (n - p < (4u << 20) || nt < 2) return false;
  std::vector<size_t> cut(nt + 1);
  cut[0] = p; cut[nt] = n;
  for (unsigned c = 1; c < nt; c++) {
    size_t q = p + (n - p) / nt * c;
    while (q < n && t[q - 1] == '\\') q++;
    cut[c] = std::max(q, cut[c - 1]);
  }
  std::vector<SpanPart> part(nt);
  auto run = [&](auto fn) { HostPool::instance().run(nt, fn); };
  const auto T0 = std::chrono::steady_clock::now();
  const bool simd = span_simd();
  run([&](unsigned c) {
    SpanPart r;
    if (simd) span_pass1_avx2(t, cut[c], cut[c + 1], r); else span_pass1_scalar(t, cut[c], cut[c + 1], r);
    part[c] = r;
  });
  const auto T1 = std::chrono::steady_clock::now();
  std::vector<int> in0(nt); std::vector<long long> d0(nt);
  { int in = 0; long long d = 0;
    for (unsigned c = 0; c < nt; c++) { in0[c] = in; d0[c] = d; d += part[c].depth[in]; in ^= part[c].quotes & 1; } }
  std::vector<SpanEmit> em(nt);
  run([&](unsigned c) {
    if (simd) span_pass2_avx2(t, cut[c], cut[c + 1], in0[c], d0[c], em[c]); else span_pass2_scalar(t, cut[c], cut[c + 1], in0[c], d0[c], em[c]);
  });
  if (getenv("CCHOST_TIMING")) {
    const auto T2 = std::chrono::steady_clock::now();
    fprintf(stderr, "[cchost]     locate: pass 1 %.1f ms, pass 2 %.1f ms on %u threads (%s)\n", std::chrono::duration<double, std::milli>(T1 - T0).count(),
            std::chrono::duration<double, std::milli>(T2 - T1).count(), nt, simd ? "AVX2" : "scalar");
  }
  std::vector<size_t> o, e;
  bool ended = false;
  for (unsigned c = 0; c < nt && !ended; c++) {
    if (em[c].bad) return false;
    o.insert(o.end(), em[c].opens.begin(), em[c].opens.end());
    e.insert(e.end(), em[c].closes.begin(), em[c].closes.end());
    if (em[c].list_end != (size_t)-1) ended = true;
  }
  if (!ended || o.size() != e.size()) return false;
  out.reserve(o.size());
  for (size_t i = 0; i < o.size(); i++) { if (e[i] <= o[i] || (i && o[i] < e[i - 1])) return false; out.push_back({o[i], e[i]}); }
  return true;
}

static bool item_spans(const char *t, size_t n, std::vector<std::pair<size_t, size_t>> &out) {
  size_t p = skip_ws(t, n, 0);
  if (p >= n) return false;
  if (t[p] == '{') {          // a List object: find "items" among its members
    p = skip_ws(t, n, p + 1);
    bool found = false;
    while (p < n && t[p] == '"') {
      const size_t ke = skip_string(t, n, p);
      const bool is_items = (ke - p == 7) && memcmp(t + p, "\"items\"", 7) == 0;
      p = skip_ws(t, n, ke);
      if (p >= n || t[p] != ':') return false;
      p = skip_ws(t, n, p + 1);
      if (is_items) { found = (p < n && t[p] == '['); break; }
      p = skip_ws(t, n, skip_value(t, n, p));
      if (p < n && t[p] == ',') p = skip_ws(t, n, p + 1);
    }
    if (!found) return false;
  } else if (t[p] != '[') return false;
  if (!getenv("CCHOST_SERIAL_SPANS")) {
    if (item_spans_parallel(t, n, p + 1, out)) return true;
    out.clear();
  }
  p = skip_ws(t, n, p + 1);
  if (p < n && t[p] == ']') return true;
  while (p < n) {
    const size_t e = skip_value(t, n, p);
    out.push_back({p, e});
    p = skip_ws(t, n, e);
    if (p < n && t[p] == ',') { p = skip_ws(t, n, p + 1); continue; }
    if (p < n && t[p] == ']') return true;
    throw std::runtime_error("json: expected , or ] in the item list");
  }
  throw std::runtime_error("json: unterminated item list");
}

// one item of a LIST, constructed IN PLACE (an object is ~1 KB of strings, vectors and maps: no temporary, no move): the DOM-free
// fast path first (fastparse.hpp), the general parser when it gives up
static void pod_into(Pod *dst, std::string_view item, bool dom_only) {
  if (!dom_only) {
    new (dst) Pod();
    try { if (fast::pod(item, *dst)) return; } catch (...) { dst->~Pod(); throw; }
    dst->~Pod();
  }
  const Json j = parse_json(item);
  if (!j.is_object()) throw std::runtime_error("json: a list item is not an object");      // (the reference's decoder rejects such a PodList too)
  new (dst) Pod(Pod::parse(j));
}
static void node_into(Node *dst, std::string_view item, bool dom_only) {
  if (!dom_only) {
    new (dst) Node();
    try { if (fast::node(item, *dst)) return; } catch (...) { dst->~Node(); throw; }
    dst->~Node();
  }
  const Json j = parse_json(item);
  if (!j.is_object()) throw std::runtime_error("json: a list item is not an object");
  new (dst) Node(Node::parse(j));
}

template <class T, class F> static ObjList<T> parse_list(const char *text, F one) {
  ObjList<T> out;
  if (!text || !*text) return out;
  const bool timing = getenv("CCHOST_TIMING") != nullptr;
  auto tp0 = std::chrono::steady_clock::now();
  const size_t n = strlen(text);
  std::vector<std::pair<size_t, size_t>> spans;
  const bool located = item_spans(text, n, spans);
  if (timing) fprintf(stderr, "[cchost]   ingest/locate %zu items in %.1f MB: %.3f s\n", spans.size(), n / 1e6, std::chrono::duration<double>(std::chrono::steady_clock::now() - tp0).count());
  if (!located) {   // not a list of items we can locate: DOM of the whole document, items re-serialised for `one`
    std::vector<Json> items = items_of(text);
    T *p = out.allocate_raw(items.size());
    std::exception_ptr err;
    for (size_t i = 0; i < items.size(); i++) {
      try { const std::string t = json_dump(items[i]); one(&p[i], std::string_view(t)); }
      catch (...) { new (&p[i]) T(); if (!err) err = std::current_exception(); }
    }
    if (err) std::rethrow_exception(err);
    return out;
  }
  unsigned nt = host_threads();
  if (spans.size() < 2048) nt = 1;
  T *p = out.allocate_raw(spans.size());       // every element is constructed below, by the thread that parses it
  std::vector<std::exception_ptr> errs(nt);
  auto work = [&](unsigned c) {
    const size_t per = (spans.size() + nt - 1) / nt, b = std::min(spans.size(), (size_t)c * per), e = std::min(spans.size(), b + per);
    for (size_t i = b; i < e; i++) {
      try { one(&p[i], std::string_view(text + spans[i].first, spans[i].second - spans[i].first)); }
      catch (...) { new (&p[i]) T(); if (!errs[c]) errs[c] = std::current_exception(); }
    }
  };
  HostPool::instance().run(nt, work);
  for (auto &e : errs) if (e) std::rethrow_exception(e);
  return out;
}

extern "C" int cc_sync_with_objects(cc_handle *h, const char *nodes_json, const char *pods_json, const char *namespaces_json) {
  if (!h) return CC_EINVAL;
  if (h->closed) return fail(h, CC_ESTATE, "closed");
  if (h->base) return fail(h, CC_ESTATE, "an analysis view is read-only");
  try {
    h->nodes.clear(); h->pods.clear(); h->ns_labels.clear(); h->workloads.clear();
    const bool timing = getenv("CCHOST_TIMING") != nullptr;
    auto t0 = std::chrono::steady_clock::now();
    const bool dom_only = getenv("CCHOST_DOM_ONLY") != nullptr;      // tests: the general parser for every item
    h->nodes = parse_list<Node>(nodes_json, [&](Node *dst, std::string_view it) { node_into(dst, it, dom_only); });
    auto t1 = std::chrono::steady_clock::now();
    h->pods = parse_list<Pod>(pods_json, [&](Pod *dst, std::string_view it) { pod_into(dst, it, dom_only); });
    auto t2 = std::chrono::steady_clock::now();
    if (timing) fprintf(stderr, "[cchost] ingest: %zu nodes %.3f s, %zu pods %.3f s\n", h->nodes.size(), std::chrono::duration<double>(t1 - t0).count(),
                        h->pods.size(), std::chrono::duration<double>(t2 - t1).count());
    h->pending_skipped = 0;
    for (auto &p : h->pods) if (p.node_name.empty() && p.phase != "Succeeded" && p.phase != "Failed") h->pending_skipped++;
    for (auto &j : items_of(namespaces_json)) h->ns_labels[j.at("metadata").at("name").str()] = parse_labels(j.at("metadata").at("labels"));
    h->synced = true; h->have_enc = false; h->ran = false; h->have_report = false;
    return CC_OK;
  } catch (const std::exception &e) { return fail(h, CC_EINVAL, e.what()); }
}

extern "C" int cc_sync_workloads(cc_handle *h, const char *services_json, const char *rcs_json, const char *replicasets_json,
                                 const char *statefulsets_json) {
  if (!h) return CC_EINVAL;
  if (h->closed) return fail(h, CC_ESTATE, "closed");
  if (h->base) return fail(h, CC_ESTATE, "an analysis view is read-only");
  if (!h->synced) return fail(h, CC_ESTATE, "cc_sync_with_objects must come first");
  try {
    h->workloads.clear();
    for (auto &j : items_of(services_json)) h->workloads.push_back(WorkloadSelector::parse(j, "Service"));
    for (auto &j : items_of(rcs_json)) h->workloads.push_back(WorkloadSelector::parse(j, "ReplicationController"));
    for (auto &j : items_of(replicasets_json)) h->workloads.push_back(WorkloadSelector::parse(j, "ReplicaSet"));
    for (auto &j : items_of(statefulsets_json)) h->workloads.push_back(WorkloadSelector::parse(j, "StatefulSet"));
    h->have_enc = false; h->ran = false; h->have_report = false;
    return CC_OK;
  } catch (const std::exception &e) { return fail(h, CC_EINVAL, e.what()); }
}

// Engines (CUDA stream, exchange buffers, kernel attributes: ccsim_create) are kept on an idle list per (device, sampling mode) and
// reused by later analyses of the process instead of being rebuilt for every Run; an engine that failed is destroyed, not reused.
static std::mutex g_eng_mu;
static std::vector<std::pair<ccsim_config, ccsim_handle *>> g_eng_idle;
static bool same_engine_cfg(const ccsim_config &a, const ccsim_config &b) {
  return a.device == b.device && a.sampling == b.sampling && a.pct_nodes_to_score == b.pct_nodes_to_score && a.engine == b.engine;
}
// The code and message of a failed engine step, before they become a handle's error (the shares of cc_run_each fail on threads of
// their own)
struct EngineFailure { int rc = CC_OK; std::string msg; };
static ccsim_handle *engine_acquire(const ccsim_config &cfg, EngineFailure &f) {
  {
    std::lock_guard<std::mutex> g(g_eng_mu);
    for (size_t i = 0; i < g_eng_idle.size(); i++)
      if (same_engine_cfg(g_eng_idle[i].first, cfg)) { ccsim_handle *e = g_eng_idle[i].second; g_eng_idle.erase(g_eng_idle.begin() + (long)i); return e; }
  }
  ccsim_handle *e = nullptr;
  if (ccsim_create(&cfg, &e)) { f.rc = CC_EENGINE; f.msg = std::string("ccsim_create: ") + ccsim_last_error(nullptr); return nullptr; }
  return e;
}
// A libccsim call failed: the engine is destroyed (not reused) and f takes its error
static void engine_failed(ccsim_handle *eng, const char *what, int rc, EngineFailure &f) {
  const std::string m = std::string(what) + ": " + ccsim_last_error(eng);
  ccsim_destroy(eng);
  if (rc == CCSIM_EUNSUPPORTED) { f.rc = CC_EUNSUPPORTED; f.msg = "unsupported on the GPU path: " + m; }
  else { f.rc = CC_EENGINE; f.msg = m; }
}
// at most 4 idle engines per device
static void engine_release(const ccsim_config &cfg, ccsim_handle *e) {
  if (getenv("CCHOST_NO_ENGINE_REUSE")) { ccsim_destroy(e); return; }
  {
    std::lock_guard<std::mutex> g(g_eng_mu);
    if (std::count_if(g_eng_idle.begin(), g_eng_idle.end(), [&](const auto &x) { return x.first.device == cfg.device; }) < 4) {
      g_eng_idle.push_back({cfg, e});
      return;
    }
  }
  ccsim_destroy(e);
}

// The stop reason of a run that ends before the engine: no nodes (ErrNoNodesAvailable, scheduler.go:68; schedule_one.go:165-168), or
// PreFilter rejecting the pod outright (the FitError then carries only the PreFilter message). False when the engine must run.
static bool stop_before_engine(const Encoded &E, std::string &reason) {
  if (E.n == 0) { reason = "Unschedulable: no nodes available to schedule pods"; return true; }
  if (!E.prefilter_msg.empty()) {
    reason = "Unschedulable: 0/" + std::to_string(E.n) + " nodes are available: " + E.prefilter_msg + ". preemption: " +
             fit_error_body(E.n, {{"Preemption is not helpful for scheduling", E.n}});
    return true;
  }
  return false;
}

// Status.StopReason of an engine run whose pod `failed` did not fit (or that reached max_pods): simulator.go:301,332
static std::string stop_reason_of(const Encoded &E, const ccsim_result &res, int64_t max_pods, const Pod &failed) {
  if (res.stop_code == CCSIM_STOP_LIMIT_REACHED) return "LimitReached: Maximum number of pods simulated: " + std::to_string(max_pods);
  std::vector<std::pair<std::string, int64_t>> hist;
  for (int r = 0; r < CCSIM_R_FIXED_COUNT; r++) hist.push_back({kReasonText[r], res.reason_hist[r]});
  for (size_t k = 0; k < E.scalar_names.size(); k++) hist.push_back({"Insufficient " + E.scalar_names[k], res.reason_hist[CCSIM_R_SCALAR0 + k]});
  for (size_t t = 0; t < E.taint_dict.size(); t++)   // taint_toleration.go:120
    hist.push_back({"node(s) had untolerated taint {" + E.taint_dict[t].key + ": " + E.taint_dict[t].value + "}", res.reason_hist[CCSIM_R_TAINT0 + t]});
  std::string msg = fit_error_body(E.n, hist);
  // DefaultPreemption PostFilter (default_preemption.go:132-143; preemption.go:234-279): no victims anywhere
  std::string post;
  if (failed.preemption_policy == "Never") post = "not eligible due to preemptionPolicy=Never.";
  else post = fit_error_body(E.n, {{"No preemption victims found for incoming pod", res.preempt_no_victims},
                                   {"Preemption is not helpful for scheduling", res.preempt_not_helpful}});
  return "Unschedulable: " + msg + " preemption: " + post;   // simulator.go:332
}

// The engine of the handle's configuration, loaded with its encoded snapshot and templates. A per-analysis handle's engine takes the
// analyses `share` lists (global indexes, increasing): analysis share[l] becomes the engine's analysis l. On failure: nullptr, f set.
static ccsim_handle *loaded_engine(const cc_handle *h, const ccsim_config &cfg, const std::vector<int32_t> &share, EngineFailure &f) {
  const Encoded &E = h->enc;
  const bool timing = getenv("CCHOST_TIMING") != nullptr;
  auto tlast = std::chrono::steady_clock::now();
  auto tick = [&](const char *what) {
    if (!timing) return;
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[cchost]   run/%s %.4f s\n", what, std::chrono::duration<double>(now - tlast).count());
    tlast = now;
  };
  ccsim_handle *eng = engine_acquire(cfg, f);
  if (!eng) return nullptr;
  tick("engine (created or taken from the idle list)");
  ccsim_nodes nd; E.fill_nodes(nd);
  const char *what = "ccsim_load_nodes";
  int rc;
  if (!(rc = ccsim_load_nodes(eng, &nd))) {
    tick("ccsim_load_nodes");
    what = "ccsim_set_templates";
    if (h->each) {   // every analysis with its own counters and columns
      what = "ccsim_set_analyses";
      const size_t A = share.size();
      std::vector<ccsim_template> tm(A);
      std::vector<std::vector<ccsim_counter>> ctr(A);
      std::vector<ccsim_analysis_terms> terms(A);
      for (size_t l = 0; l < A; l++) {
        const Encoded &e = h->parts[(size_t)share[l]];
        tm[l] = h->enc_tmpls[(size_t)share[l]];
        // the hostPort self-conflict: bit (index in the launch) mod 64, as the engine reads it (encode_list set the global index's)
        if (tm[l].port_tmpl_conflict) tm[l].port_tmpl_conflict = 1ull << (l & 63);
        ctr[l] = e.counters;
        for (size_t j = 0; j < ctr[l].size(); j++) ctr[l][j].init = e.counter_init[j].data();
        ccsim_analysis_terms &a = terms[l];
        memset(&a, 0, sizeof(a));
        a.n_counters = (int32_t)ctr[l].size(); a.counters = ctr[l].data();
        a.n_topo_cols = (int32_t)e.topo.size();
        for (size_t k = 0; k < e.topo.size() && k < CCSIM_MAX_TOPO_COLS; k++) a.topo[k] = e.topo[k].data();
      }
      if (!(rc = ccsim_set_analyses(eng, (int32_t)A, tm.data(), terms.data()))) { tick(what); return eng; }
    } else if (!(rc = ccsim_set_templates(eng, (int32_t)h->enc_tmpls.size(), h->enc_tmpls.data(), (int32_t)E.counters.size(), E.counters.data()))) {
      tick("ccsim_set_templates");
      return eng;
    }
  }
  engine_failed(eng, what, rc, f);
  return nullptr;
}

static int encode_for_run(cc_handle *h) {
  if (h->closed) return fail(h, CC_ESTATE, "closed");
  if (h->base) return fail(h, CC_ESTATE, "an analysis view is read-only: run its base handle");
  if (!h->synced) return fail(h, CC_ESTATE, "cc_sync_with_objects must come first");
  try {
    ensure_encoded(h);
  } catch (const Unsupported &e) { return fail(h, CC_EUNSUPPORTED, std::string("unsupported on the GPU path: ") + e.what());
  } catch (const std::exception &e) { return fail(h, CC_EINVAL, e.what()); }
  return CC_OK;
}

static ccsim_config engine_config(const cc_handle *h, int32_t device) {
  ccsim_config cfg; memset(&cfg, 0, sizeof(cfg));
  cfg.abi_version = CCSIM_ABI_VERSION; cfg.device = device; cfg.engine = CCSIM_ENGINE_AUTO; cfg.rank = 0; cfg.world = 1;
  if (h->cfg.reference_sampling && h->cfg.pct_nodes_to_score != 100) { cfg.sampling = CCSIM_SAMPLING_REFERENCE; cfg.pct_nodes_to_score = h->cfg.pct_nodes_to_score; }
  return cfg;
}

extern "C" int cc_run(cc_handle *h) {
  if (!h) return CC_EINVAL;
  if (h->each) return fail(h, CC_ESTATE, "a per-analysis handle (cc_new_each) runs with cc_run_each");
  int rc = encode_for_run(h);
  if (rc) return rc;
  const Encoded &E = h->enc;
  h->pod_node.clear();
  h->have_report = false;
  if (stop_before_engine(E, h->stop_reason)) { h->ran = true; return CC_OK; }
  const ccsim_config cfg = engine_config(h, h->devices[0]);
  EngineFailure f;
  ccsim_handle *eng = loaded_engine(h, cfg, {}, f);
  if (!eng) return fail(h, f.rc, f.msg);
  ccsim_result res;
  const auto t0 = std::chrono::steady_clock::now();
  if ((rc = ccsim_run(eng, h->max_pods, &res))) { engine_failed(eng, "ccsim_run", rc, f); return fail(h, f.rc, f.msg); }
  if (getenv("CCHOST_TIMING")) fprintf(stderr, "[cchost]   run/ccsim_run %.4f s\n", std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
  h->pod_node.assign(res.pod_node, res.pod_node + res.placed);
  h->stop_reason = stop_reason_of(E, res, h->max_pods, h->tmpls[(size_t)res.placed % h->tmpls.size()]);   // the pod that did not fit: clone of template placed % T
  engine_release(cfg, eng);
  h->ran = true;
  return CC_OK;
}

// The deal of a per-analysis run over the handle's devices (cc_new_each_on): the coupled analyses (counters, or a hostPort
// self-conflict) in podspec order go to entries 0, 1, ..., G-1, 0, ...; the node-local ones continue the deal where the coupled ones
// stopped, so that every entry gets its part of the expensive analyses and the shares differ by one analysis at most. Entry g's share
// lists its analyses' global indexes in increasing order. A list handle has one device: its share is every analysis.
static std::vector<std::vector<int32_t>> deal_analyses(const cc_handle *h) {
  const size_t G = h->devices.size(), T = h->tmpls.size();
  std::vector<std::vector<int32_t>> share(G);
  size_t next = 0;
  for (const bool coupled : {true, false})
    for (size_t t = 0; t < T; t++)
      if ((h->each && (!h->parts[t].counters.empty() || h->parts[t].tmpl.port_tmpl_conflict)) == coupled) {
        share[next].push_back((int32_t)t);
        next = (next + 1) % G;
      }
  for (auto &s : share) std::sort(s.begin(), s.end());
  return share;
}

// libccsim names an analysis by its index in the launch ("analysis 1: counter 0: ...", "template 1 has ..."): the global index instead
static std::string global_indexes(const std::string &m, const std::vector<int32_t> &share) {
  std::string out;
  size_t p = 0;
  while (p < m.size()) {
    size_t at = std::string::npos, len = 0;
    for (const char *word : {"analysis ", "template "}) {
      const size_t q = m.find(word, p);
      if (q < at) { at = q; len = strlen(word); }
    }
    if (at == std::string::npos) { out.append(m, p, std::string::npos); break; }
    size_t d = at + len, e = d;
    while (e < m.size() && isdigit((unsigned char)m[e])) e++;
    out.append(m, p, d - p);
    const size_t l = e > d && e - d < 10 ? std::stoul(m.substr(d, e - d)) : share.size();
    out += l < share.size() ? std::to_string(share[l]) : m.substr(d, e - d);
    p = e;
  }
  return out;
}

// One device's share of a per-analysis run, in one ccsim_run_each on an engine of its own
struct EachShare {
  ccsim_config cfg;
  std::vector<int32_t> idx;              // its analyses' global indexes, increasing
  ccsim_handle *eng = nullptr;           // after a successful run: the engine, which holds the placement sequences of res
  std::vector<ccsim_result> res;         // res[l]: analysis idx[l]
  EngineFailure f;                       // a failure, named by global indexes
};

static void run_share(const cc_handle *h, EachShare &s) {
  const auto t0 = std::chrono::steady_clock::now();
  ccsim_handle *eng = loaded_engine(h, s.cfg, s.idx, s.f);
  if (eng) {
    s.res.assign(s.idx.size(), ccsim_result());
    if (const int rc = ccsim_run_each(eng, h->max_pods, s.res.data())) engine_failed(eng, "ccsim_run_each", rc, s.f);
    else s.eng = eng;
  }
  if (s.f.rc) { s.f.msg = global_indexes(s.f.msg, s.idx); return; }
  if (getenv("CCHOST_TIMING"))
    fprintf(stderr, "[cchost]   run/ccsim_run_each on device %d: %zu analyses, kernel %s, %.4f s\n", s.cfg.device, s.idx.size(),
            ccsim_kernel_name(eng), std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
}

extern "C" int cc_run_each(cc_handle *h) {
  if (!h) return CC_EINVAL;
  int rc = encode_for_run(h);
  if (rc) return rc;
  const Encoded &E = h->enc;
  const size_t T = h->tmpls.size();
  h->analyses.clear();
  std::vector<std::unique_ptr<cc_handle>> views;
  for (size_t t = 0; t < T; t++) {   // podspec t alone, as a handle of its own would hold it
    std::unique_ptr<cc_handle> v(new cc_handle());
    v->cfg = h->cfg; v->tmpl = h->tmpls[t]; v->tmpls.assign(1, h->tmpls[t]); v->max_pods = h->max_pods; v->exclude = h->exclude;
    v->base = h;
    views.push_back(std::move(v));
  }
  std::string early;
  if (stop_before_engine(E, early)) {
    for (auto &v : views) { v->stop_reason = early; v->ran = true; }
    h->analyses = std::move(views);
    return CC_OK;
  }
  std::vector<EachShare> shares;
  for (std::vector<int32_t> &idx : deal_analyses(h)) {
    shares.emplace_back();
    shares.back().cfg = engine_config(h, h->devices[shares.size() - 1]);
    shares.back().idx = std::move(idx);
  }
  // ccsim_run_each blocks: one host thread per distinct ordinal (the caller's for the first). An ordinal's shares run one after the
  // other on its thread, so that the free-memory check of each engine sees the engines before it; after a failure its later shares
  // do not run (the first failure in list order is the one reported). A share without analyses gets no engine.
  std::vector<int32_t> ords;
  for (int32_t d : h->devices) if (std::find(ords.begin(), ords.end(), d) == ords.end()) ords.push_back(d);
  auto work = [&](int32_t d) {
    for (EachShare &s : shares) {
      if (s.cfg.device != d || s.idx.empty()) continue;
      try { run_share(h, s); } catch (const std::exception &e) { s.f.rc = CC_EENGINE; s.f.msg = e.what(); }
      if (s.f.rc) return;
    }
  };
  std::vector<std::thread> threads;
  for (size_t i = 1; i < ords.size(); i++) {
    try { threads.emplace_back(work, ords[i]); } catch (const std::system_error &) { work(ords[i]); }
  }
  work(ords[0]);
  for (std::thread &th : threads) th.join();
  const EachShare *failed = nullptr;
  for (const EachShare &s : shares) if (s.f.rc) { failed = &s; break; }
  if (!failed)
    for (const EachShare &s : shares)
      for (size_t l = 0; l < s.idx.size(); l++) {
        const size_t t = (size_t)s.idx[l];
        const ccsim_result &r = s.res[l];
        cc_handle &v = *views[t];
        v.ran = true;
        if (h->each && stop_before_engine(h->parts[t], v.stop_reason)) continue;   // PreFilter rejected podspec t: no placements
        v.pod_node.assign(r.pod_node, r.pod_node + r.placed);
        v.stop_reason = stop_reason_of(E, r, h->max_pods, h->tmpls[t]);   // every pod of analysis t is a clone of podspec t
      }
  for (const EachShare &s : shares) if (s.eng) engine_release(s.cfg, s.eng);
  if (failed) return fail(h, failed->f.rc, failed->f.msg);
  h->analyses = std::move(views);
  return CC_OK;
}

extern "C" int cc_analysis(cc_handle *h, int32_t t, cc_handle **view) {
  if (!h || !view) return CC_EINVAL;
  if (h->analyses.empty()) return fail(h, CC_ESTATE, "cc_run_each must come first");
  if (t < 0 || (size_t)t >= h->analyses.size()) return fail(h, CC_EINVAL, "analysis " + std::to_string(t) + " out of range (" + std::to_string(h->analyses.size()) + " podspecs)");
  *view = h->analyses[(size_t)t].get();
  return CC_OK;
}

// getResourceRequest (report.go:111-144): containers only, cpu/memory summed as quantities, scalars as Value()
static Json requirements_json(const Pod &p) {
  Quantity cpu = Quantity::parse("0"); cpu.format = Quantity::DecimalSI;
  Quantity mem = Quantity::parse("0"); mem.format = Quantity::BinarySI;
  std::map<std::string, int64_t> scalars; bool have_scalars = false;
  for (auto &c : p.containers)
    for (auto &kv : c.requests) {
      if (kv.first == "memory") { Quantity q = kv.second; q.add(mem); mem = q; }
      else if (kv.first == "cpu") { Quantity q = kv.second; q.add(cpu); cpu = q; }
      else if (is_scalar_resource_name(kv.first)) { scalars[kv.first] += kv.second.value(); have_scalars = true; }
    }
  Json prim = Json::object();
  prim.set("cpu", Json::string(cpu.str()));
  prim.set("memory", Json::string(mem.str()));
  prim.set("nvdia.com/gpu", Json::string("0"));   // [sic] report.go:35,116
  Json res = Json::object();
  res.set("primaryResources", prim);
  if (have_scalars) { Json s = Json::object(); for (auto &kv : scalars) s.set(kv.first, Json::number(kv.second)); res.set("scalarResources", s); }
  else res.set("scalarResources", Json::null());
  Json req = Json::object();
  req.set("podName", Json::string(p.name));
  req.set("resources", res);
  if (p.has_node_selector) { Json s = Json::object(); for (auto &kv : p.node_selector) s.set(kv.first, Json::string(kv.second)); req.set("nodeSelectors", s); }
  else req.set("nodeSelectors", Json::null());
  return req;
}

static int build_report(cc_handle *h) {
  if (h->have_report) return CC_OK;
  if (!h->ran) return fail(h, CC_ESTATE, "Report() before Run(): no stop reason yet (the reference panics here, report.go:102-106)");
  Json spec = Json::object();
  Json tmpls = Json::array();
  Json reqs = Json::array();
  for (auto &t : h->tmpls) { tmpls.push(t.raw); reqs.push(requirements_json(t)); }
  spec.set("templates", std::move(tmpls));
  spec.set("replicas", Json::number(h->max_pods));
  spec.set("podRequirements", std::move(reqs));
  Json status = Json::object();
  status.set("creationTimestamp", Json::string(rfc3339_now()));
  status.set("replicas", Json::number((long long)h->pod_node.size()));
  // getMainFailReason (report.go:100-109): split at the first ':'
  const std::string &sr = h->stop_reason;
  size_t nl = sr.find('\n');
  std::string first = nl == std::string::npos ? sr : sr.substr(0, nl);
  size_t colon = first.find(':');
  Json fr = Json::object();
  fr.set("failType", Json::string(first.substr(0, colon)));
  std::string m = colon == std::string::npos ? "" : first.substr(colon + 1);
  while (!m.empty() && m.front() == ' ') m.erase(m.begin());
  while (!m.empty() && m.back() == ' ') m.pop_back();
  fr.set("failMessage", Json::string(m));
  status.set("failReason", std::move(fr));
  // parsePodsReview (report.go:146-180): per template (pod k belongs to template k % T), ReplicasOnNodes in order of first placement
  Json pods = Json::array();
  const size_t T = h->tmpls.size();
  for (size_t t = 0; t < T; t++) {
    Json rons = Json::array();
    std::vector<int64_t> count(enc_of(h).n, 0); std::vector<int32_t> order;
    for (size_t k = t; k < h->pod_node.size(); k += T) { const int32_t w = h->pod_node[k]; if (count[w]++ == 0) order.push_back(w); }
    rons.arr.reserve(order.size());
    for (int32_t w : order) { Json r = Json::object(); r.obj.reserve(2); r.set("nodeName", Json::string(enc_of(h).names[w])); r.set("replicas", Json::number(count[w])); rons.push(std::move(r)); }
    Json podres = Json::object();
    podres.set("podName", Json::string(h->tmpls[t].name));
    podres.set("replicasOnNodes", std::move(rons));      // (moved, not copied: one entry per node that received a clone)
    podres.set("failSummary", Json::null());   // never populated by the reference (report.go:174-179)
    pods.push(std::move(podres));
  }
  status.set("pods", std::move(pods));
  h->report = Json::object();
  h->report.set("spec", std::move(spec));
  h->report.set("status", std::move(status));
  h->have_report = true;
  return CC_OK;
}

extern "C" const char *cc_report_json(cc_handle *h) {
  if (!h || build_report(h)) return nullptr;
  h->out = json_dump(h->report);
  return h->out.c_str();
}

extern "C" const char *cc_report_print(cc_handle *h, int32_t verbose, const char *format) {
  if (!h || build_report(h)) return nullptr;
  std::string f = format ? format : "";
  if (f == "json") { h->out = json_dump(h->report) + "\n"; return h->out.c_str(); }
  if (f == "yaml") { h->out.clear(); yaml_emit(h->report, 0, h->out); return h->out.c_str(); }
  if (!f.empty()) { fail(h, CC_EINVAL, "output format \"" + f + "\" not recognized"); return nullptr; }   // report.go:315
  // clusterCapacityReviewPrettyPrint (report.go:235-285)
  std::string o;
  const Json &st = h->report.at("status");
  if (verbose)
    for (auto &req : h->report.at("spec").at("podRequirements").arr) {
      o += req.at("podName").str() + " pod requirements:\n";
      o += "\t- CPU: " + req.at("resources").at("primaryResources").at("cpu").str() + "\n";
      o += "\t- Memory: " + req.at("resources").at("primaryResources").at("memory").str() + "\n";
      const Json &sc = req.at("resources").at("scalarResources");
      if (sc.is_object()) { o += "\t- ScalarResources: map["; bool fst = true; for (auto &kv : sc.obj) { if (!fst) o += " "; o += kv.first + ":" + kv.second.s; fst = false; } o += "]\n"; }
      const Json &ns = req.at("nodeSelectors");
      if (ns.is_object()) {   // labels.SelectorFromSet(...).String(): sorted "k=v" joined by ","
        std::vector<std::string> kv; for (auto &p : ns.obj) kv.push_back(p.first + "=" + p.second.str());
        std::sort(kv.begin(), kv.end());
        o += "\t- NodeSelector: "; for (size_t i = 0; i < kv.size(); i++) { if (i) o += ","; o += kv[i]; } o += "\n";
      }
      o += "\n";
    }
  for (auto &pod : st.at("pods").arr) {
    long long total = 0;
    for (auto &r : pod.at("replicasOnNodes").arr) total += r.at("replicas").i64();
    if (verbose) o += "The cluster can schedule " + std::to_string(total) + " instance(s) of the pod " + pod.at("podName").str() + ".\n";
    else o += std::to_string(total) + "\n";
  }
  if (verbose) {
    o += "\nTermination reason: " + st.at("failReason").at("failType").str() + ": " + st.at("failReason").at("failMessage").str() + "\n";
    if (st.at("replicas").i64() > 0) {
      o += "\nPod distribution among nodes:\n";
      for (auto &pod : st.at("pods").arr) {
        o += pod.at("podName").str() + "\n";
        for (auto &r : pod.at("replicasOnNodes").arr) o += "\t- " + r.at("nodeName").str() + ": " + std::to_string(r.at("replicas").i64()) + " instance(s)\n";
      }
    }
  }
  h->out = o;
  return h->out.c_str();
}

extern "C" const char *cc_warnings(cc_handle *h) {
  if (!h) return "";
  h->warn.clear();
  if (h->pending_skipped > 0)
    h->warn += std::to_string(h->pending_skipped) + " pending pod(s) of the snapshot (no spec.nodeName) were left out: the reference would let its embedded scheduler bind "
               "them and count each as a simulated instance (pkg/framework/simulator.go:193-200,297-312), with no defined order\n";
  return h->warn.c_str();
}
extern "C" const char *cc_stop_reason(cc_handle *h) { return h ? h->stop_reason.c_str() : nullptr; }
extern "C" int64_t cc_scheduled_count(cc_handle *h) { return h ? (int64_t)h->pod_node.size() : 0; }
extern "C" const char *cc_scheduled_node(cc_handle *h, int64_t k) {
  if (!h || k < 0 || k >= (int64_t)h->pod_node.size()) return nullptr;
  return enc_of(h).names[h->pod_node[k]].c_str();
}
extern "C" void cc_close(cc_handle *h) { if (h && !h->base) { h->closed = true; delete h; } }   // a view goes with its base

extern "C" const char *cc_debug_encoded_snapshot(cc_handle *h) {
  if (!h) return nullptr;
  if (h->base) { fail(h, CC_ESTATE, "an analysis view has no snapshot of its own"); return nullptr; }
  try { ensure_encoded(h); }
  catch (const Unsupported &e) { fail(h, CC_EUNSUPPORTED, std::string("unsupported on the GPU path: ") + e.what()); return nullptr; }
  catch (const std::exception &e) { fail(h, CC_EINVAL, e.what()); return nullptr; }
  const Encoded &E = h->enc;
  auto arr64 = [](const std::vector<int64_t> &v) { Json a = Json::array(); for (auto x : v) a.push(Json::number(x)); return a; };
  auto arr32 = [](const std::vector<int32_t> &v) { Json a = Json::array(); for (auto x : v) a.push(Json::number(x)); return a; };
  auto arru64 = [](const uint64_t *v, size_t n) { Json a = Json::array(); for (size_t i = 0; i < n; i++) a.push(Json::number_text(std::to_string((unsigned long long)v[i]))); return a; };
  Json j = Json::object();
  Json names = Json::array(); for (auto &s : E.names) names.push(Json::string(s));
  j.set("names", names);
  Json nd = Json::object();
  nd.set("n", Json::number(E.n));
  nd.set("alloc_cpu", arr64(E.alloc_cpu)); nd.set("alloc_mem", arr64(E.alloc_mem)); nd.set("alloc_eph", arr64(E.alloc_eph));
  nd.set("alloc_pods", arr32(E.alloc_pods));
  nd.set("req_cpu", arr64(E.req_cpu)); nd.set("req_mem", arr64(E.req_mem)); nd.set("req_eph", arr64(E.req_eph));
  nd.set("npods", arr32(E.npods)); nd.set("nz_cpu", arr64(E.nz_cpu)); nd.set("nz_mem", arr64(E.nz_mem));
  Json sn = Json::array(); for (auto &s : E.scalar_names) sn.push(Json::string(s));
  nd.set("scalar_names", sn);
  Json as = Json::array(), rs = Json::array();
  for (auto &v : E.alloc_scalar) as.push(arr64(v));
  for (auto &v : E.req_scalar) rs.push(arr64(v));
  nd.set("alloc_scalar", as); nd.set("req_scalar", rs);
  nd.set("taint_words", Json::number(E.taint_words)); nd.set("static_words", Json::number(E.static_words));
  nd.set("taint_mask", arru64(E.taint_mask.data(), E.taint_mask.size()));
  nd.set("static_mask", arru64(E.static_mask.data(), (size_t)E.static_words * E.n));
  nd.set("taint_nosched", arru64(E.taint_nosched, CCSIM_MAX_TAINT_WORDS)); nd.set("taint_prefer", arru64(E.taint_prefer, CCSIM_MAX_TAINT_WORDS));
  Json td = Json::array();
  for (auto &t : E.taint_dict) { Json x = Json::object(); x.set("key", Json::string(t.key)); x.set("value", Json::string(t.value)); x.set("effect", Json::string(t.effect)); td.push(x); }
  nd.set("taint_dict", td);
  nd.set("taint_off", arr32(E.taint_off));
  { Json tl = Json::array(); for (auto x : E.taint_list) tl.push(Json::number(x)); nd.set("taint_list", tl); }
  Json topo = Json::array(); for (auto &c : E.topo) topo.push(arr32(c));
  nd.set("topo", topo);
  nd.set("has_placed_mask", Json::boolean(E.has_placed_mask));
  j.set("nodes", nd);
  // the template as raw bytes (hex) — the tests memcpy it into the ctypes struct
  std::string hex; const unsigned char *tb = reinterpret_cast<const unsigned char *>(&E.tmpl);
  static const char *d = "0123456789abcdef";
  for (size_t i = 0; i < sizeof(ccsim_template); i++) { hex += d[tb[i] >> 4]; hex += d[tb[i] & 15]; }
  j.set("template_hex", Json::string(hex));
  {   // every template of a list run (image_score pointers are process-local: image_scores carries the columns)
    Json th = Json::array(), is = Json::array();
    for (size_t t = 0; t < h->enc_tmpls.size(); t++) {
      std::string hx; const unsigned char *b = reinterpret_cast<const unsigned char *>(&h->enc_tmpls[t]);
      for (size_t i = 0; i < sizeof(ccsim_template); i++) { hx += d[b[i] >> 4]; hx += d[b[i] & 15]; }
      th.push(Json::string(hx));
      Json col = Json::array();
      if (h->tmpls.size() > 1) for (auto x : h->enc_images[t]) col.push(Json::number(x)); else for (auto x : E.image_score) col.push(Json::number(x));
      is.push(col);
    }
    j.set("templates_hex", th); j.set("image_scores", is);
  }
  Json ctr = Json::array();
  for (size_t k = 0; k < E.counters.size(); k++) {
    Json c = Json::object();
    c.set("topo_col", Json::number(E.counters[k].topo_col)); c.set("n_present", Json::number(E.counters[k].n_present));
    c.set("inc", Json::number(E.counters[k].inc)); c.set("elig_bit", Json::number(E.counters[k].elig_bit)); c.set("init", arr32(E.counter_init[k]));
    ctr.push(c);
  }
  j.set("counters", ctr);
  { Json is = Json::array(); for (auto x : E.image_score) is.push(Json::number(x)); j.set("image_score", is); }   // template_hex holds a process-local pointer
  j.set("prefilter_msg", Json::string(E.prefilter_msg));
  if (h->each) {   // a per-analysis handle: every analysis's own terms
    Json an = Json::array();
    for (const Encoded &e : h->parts) {
      Json a = Json::object(), ac = Json::array(), at = Json::array();
      for (size_t k = 0; k < e.counters.size(); k++) {
        Json c = Json::object();
        c.set("topo_col", Json::number(e.counters[k].topo_col)); c.set("n_present", Json::number(e.counters[k].n_present));
        c.set("inc", Json::number(e.counters[k].inc)); c.set("elig_bit", Json::number(e.counters[k].elig_bit)); c.set("init", arr32(e.counter_init[k]));
        ac.push(c);
      }
      for (auto &c : e.topo) at.push(arr32(c));
      a.set("counters", ac); a.set("topo", at); a.set("prefilter_msg", Json::string(e.prefilter_msg));
      an.push(a);
    }
    j.set("analyses", an);
    Json sh = Json::array();   // the deal of cc_run_each over the handle's devices
    for (const std::vector<int32_t> &s : deal_analyses(h)) sh.push(arr32(s));
    j.set("shares", sh);
  }
  h->out = json_dump(j);
  return h->out.c_str();
}
