/*
 * cchost.h — C-ABI of the host side of the hot path: the H100 counterpart of the reference's pkg/framework API.
 *
 *   cc_new               <- framework.New(kubeSchedulerConfig, kubeConfig, simulatedPod, maxPods, excludeNodes)
 *                           (pkg/framework/simulator.go:107-158)
 *   cc_sync_with_objects <- (*ClusterCapacity).SyncWithClient(client)  (simulator.go:176-295): instead of a clientset the
 *                           caller hands over the LISTed objects as JSON (NodeList / PodList / NamespaceList or bare arrays)
 *   cc_sync_workloads    <- the Services / RCs / ReplicaSets / StatefulSets part of SyncWithClient (simulator.go:217-281): optional;
 *                           only helper.DefaultSelector reads them (system-default topology spreading)
 *   cc_run               <- (*ClusterCapacity).Run()                   (simulator.go:356-381)
 *   cc_report_json       <- (*ClusterCapacity).Report() marshalled     (simulator.go:160-170; report.go:38-98,220-233)
 *   cc_report_print      <- framework.ClusterCapacityReviewPrint(r, verbose, format)  (report.go:235-317)
 *   cc_close             <- (*ClusterCapacity).Close()                 (simulator.go:314-325), idempotent
 *   cc_new_list          <- the roadmap's "accept a list of pods" (README.md:305-306): framework.New with several podspecs, pod k of the
 *                           run is a clone of podspec k % T (the template index parsePodsReview uses, report.go:160)
 *   cc_run_each / cc_analysis <- `cluster-capacity --podspec <file>` once per podspec of a list (the genpod workflow), in one launch
 *                           per device (cc_new_each_on: the podspecs dealt over several GPUs)
 *   cc_stop_reason / cc_scheduled_count / cc_scheduled_node <- Status{StopReason, Pods} as the callers of Report() read them
 *                           (simulator.go:90-93; ScheduledPods in the reference's tests, simulator_test.go:226-240)
 *   cc_warnings          <- nothing in the reference: what this analysis left out that the reference would have done (pending pods)
 *
 * What SyncWithClient+Run do internally here: aggregate NodeInfo exactly as the scheduler cache would
 * (framework/types.go:409-427,700-734), order nodes as nodeTree.list() (backend/cache/node_tree.go:119-143),
 * dictionary-encode taints / label requirements / topology values, compile the pod template, and drive
 * libccsim (include/ccsim.h) on the GPU. There is no CPU scheduling fallback: cc_run fails if no CUDA device exists.
 *
 * All functions return 0 or a negative code; cc_last_error(h) gives the text. Returned strings are owned by the
 * handle and stay valid until the next call on it.
 */
#ifndef CCHOST_H
#define CCHOST_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct cc_handle cc_handle;

#define CC_OK            0
#define CC_EINVAL       -1
#define CC_EUNSUPPORTED -4   /* the podspec/snapshot needs a plugin the GPU path does not implement (named in the error) */
#define CC_ESTATE       -5
#define CC_EENGINE      -7   /* libccsim failed (no GPU, CUDA error) */

/* pod_json: the simulated pod (v1.Pod as JSON, already defaulted/validated by the CLI like ParseAPISpec does).
 * sched_config_json: NULL/"" for the default profile in canonical mode, or a small JSON {"sampling":"reference",
 *   "percentageOfNodesToScore":0,   (reference sampling: adaptive numFeasibleNodesToFind + rotating start index)
 *   "disabledFilters":["NodeResourcesFit",...], "disabledScores":[...], "weights":{"NodeResourcesFit":1,...},
 *   "hardPodAffinityWeight":1}.
 * exclude_nodes: comma-separated node names (--exclude-nodes), may be NULL. device: CUDA ordinal. */
int cc_new(const char *sched_config_json, const char *pod_json, int64_t max_pods, const char *exclude_nodes,
           int32_t device, cc_handle **out);
/* The roadmap's "accept a list of pods" (README.md:305-306): pods_json is a JSON array (or v1 List) of up to 64 v1.Pod; pod k of
 * the simulation is a clone of podspec k % T (the template index the report already uses, report.go:160), the run ends when
 * one of them does not fit or at max_pods. Podspecs with topology-spread / pod-(anti-)affinity terms are single-podspec only. */
int cc_new_list(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                int32_t device, cc_handle **out);
/* A per-analysis handle: the arguments of cc_new_list with up to CCSIM_EACH_MAX_ANALYSES (4096) podspecs, run with cc_run_each only
 * (cc_run fails with CC_ESTATE). Every podspec keeps its own topology-spread and pod-(anti-)affinity counters, topology columns and
 * hostPorts, so podspecs with hard (DoNotSchedule) spread, required pod (anti-)affinity and hostPorts are analysed like
 * cc_new(podspec t) + cc_run; a podspec PreFilter rejects ends its own analysis with cc_run's message and no placements. The
 * podspec-independent part of the encoding (node order, NodeInfo columns, taint dictionary) is built once for all podspecs. */
int cc_new_each(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                int32_t device, cc_handle **out);
/* cc_new_each over a list of CUDA ordinals devices[0..n_devices-1] (cc_new_each(..., d, ...) is the list {d}): cc_run_each deals the
 * analyses over the list and runs every non-empty share on its device, each device holding the whole snapshot; analysis t gives
 * exactly what the one-device handle gives. The deal: the coupled analyses (counters, or a hostPort self-conflict) in podspec order go
 * to entries 0, 1, ..., n_devices-1, 0, ...; the node-local ones continue the deal where the coupled ones stopped. An ordinal may repeat
 * (its shares then run one after the other, each with an engine of its own). CC_EINVAL for an empty list, a negative ordinal or more
 * than CC_EACH_MAX_DEVICES entries; an ordinal without a CUDA device fails at cc_run_each with CC_EENGINE. */
#define CC_EACH_MAX_DEVICES 64
int cc_new_each_on(const char *sched_config_json, const char *pods_json, int64_t max_pods, const char *exclude_nodes,
                   const int32_t *devices, int32_t n_devices, cc_handle **out);
int cc_sync_with_objects(cc_handle *h, const char *nodes_json, const char *pods_json, const char *namespaces_json);
/* Optional, between cc_sync_with_objects and cc_run: the Services / ReplicationControllers / ReplicaSets / StatefulSets
 * SyncWithClient copies (simulator.go:217-281). The scheduler reads them in one place only: helper.DefaultSelector
 * (plugins/helper/spread.go:40-93), which gives a pod WITHOUT topologySpreadConstraints the two system-default soft
 * constraints when a Service (or its owning controller) selects it (podtopologyspread/plugin.go:48-59). Lists or bare
 * arrays as JSON; any may be NULL. */
int cc_sync_workloads(cc_handle *h, const char *services_json, const char *rcs_json, const char *replicasets_json,
                      const char *statefulsets_json);
int cc_run(cc_handle *h);
/* Every podspec of the handle analysed on its own against the synced snapshot, all in one GPU launch per device: analysis t is what
 * cc_new(podspec t) + cc_sync_with_objects + cc_run gives under the same configuration, max_pods and exclude_nodes. On a cc_new_list
 * handle node-local podspecs only: topology spread, pod (anti-)affinity and hostPorts are refused by name; a cc_new_each handle takes
 * them. Always refused by name: normalised soft scorers (preferred node affinity, ScheduleAnyway / system-default spreading,
 * InterPodAffinity scoring, which a required affinity matching the pod's own labels brings under hardPodAffinityWeight > 0),
 * node shards and reference sampling. */
int cc_run_each(cc_handle *h);
/* After cc_run_each: a read-only view of analysis t (podspec t alone and its Status), owned by h and valid until the next
 * cc_run_each or cc_close(h). cc_report_json / cc_report_print / cc_stop_reason / cc_scheduled_* read it like a handle of its own;
 * cc_run, cc_run_each and the syncs fail on it with CC_ESTATE, and cc_close ignores it. */
int cc_analysis(cc_handle *h, int32_t t, cc_handle **view);
const char *cc_report_json(cc_handle *h);
const char *cc_report_print(cc_handle *h, int32_t verbose, const char *format /* "", "json", "yaml" */);
const char *cc_stop_reason(cc_handle *h);
int64_t cc_scheduled_count(cc_handle *h);
/* node name of scheduled pod k (ScheduledPods()[k].Spec.NodeName), NULL if out of range */
const char *cc_scheduled_node(cc_handle *h, int64_t k);
void cc_close(cc_handle *h);
const char *cc_last_error(const cc_handle *h);
/* Deviations of this analysis from what the reference would have done with the same snapshot, one per line ("" when none). Today:
 * pending pods (no spec.nodeName, not Succeeded/Failed) of the source cluster — the reference copies them into its fake cluster
 * (pkg/framework/simulator.go:193-200), its embedded scheduler binds them through ClusterCapacityBinder and postBindHook counts each as
 * a simulated instance and creates one more simulated pod (simulator.go:297-312; the "TODO: remove all pods that are not scheduled
 * yet" of Run, :359): a race with no defined outcome. Here they are left out, and said so. Valid after cc_sync_with_objects. */
const char *cc_warnings(cc_handle *h);

/* Encoder only (no GPU needed): builds the flat snapshot + template exactly as cc_run would and returns it as JSON
 * {"nodes":{...columns...},"templates":[...],"counters":[...],"names":[...]} for tests and for the CPU oracle. */
const char *cc_debug_encoded_snapshot(cc_handle *h);

#ifdef __cplusplus
}
#endif
#endif
