"""Python face of libcchost.so — same names and argument meaning as the reference's pkg/framework:

    cc = framework.New(scheduler_config, None, simulated_pod, max_pods, exclude_nodes)   # simulator.go:107
    cc.SyncWithClient(client)          # simulator.go:176 — `client` is anything with .nodes/.pods/.namespaces lists of dicts
    cc.Run()                           # simulator.go:356 — blocking; raises on error
    review = cc.Report()               # simulator.go:160 — dict with the reference's JSON shape (report.go:38-98)
    framework.ClusterCapacityReviewPrint(review_or_cc, verbose, format)   # report.go:305
    cc.ScheduledPods(); cc.Close()
    for a in cc.RunEach(): a.Report()  # several podspecs, each analysed on its own (`cluster-capacity --podspec` per file);
                                       # NewEach(...) takes podspecs with hard spread, pod (anti-)affinity and hostPorts too,
                                       # NewEach(..., devices=[0, 1, ...]) deals them over several GPUs

All the work happens in C++ (encoder) and CUDA (libccsim); this file only marshals JSON across the C-ABI.
"""
import ctypes as C
import json
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libcchost.so")
_lib = None

EXPORTS = ["cc_new", "cc_new_list", "cc_new_each", "cc_new_each_on", "cc_sync_with_objects", "cc_sync_workloads", "cc_run", "cc_report_json", "cc_report_print", "cc_stop_reason",
           "cc_scheduled_count", "cc_scheduled_node", "cc_close", "cc_last_error", "cc_warnings", "cc_debug_encoded_snapshot", "cc_run_each",
           "cc_analysis"]


class FrameworkError(RuntimeError):
    pass


class UnsupportedError(FrameworkError):
    """The podspec/snapshot needs a scheduler plugin the GPU path does not implement (named in the message)."""


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise FrameworkError("libcchost.so not built: run __graft_entry__.build()")
        L = C.CDLL(SO_PATH)
        L.cc_new.restype = C.c_int
        L.cc_new.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.cc_new_list.restype = C.c_int
        L.cc_new_list.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.cc_sync_with_objects.restype = C.c_int
        L.cc_sync_with_objects.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p]
        L.cc_sync_workloads.restype = C.c_int
        L.cc_sync_workloads.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p]
        L.cc_run.restype = C.c_int
        L.cc_run.argtypes = [C.c_void_p]
        L.cc_new_each.restype = C.c_int
        L.cc_new_each.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.cc_new_each_on.restype = C.c_int
        L.cc_new_each_on.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_char_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]
        L.cc_run_each.restype = C.c_int
        L.cc_run_each.argtypes = [C.c_void_p]
        L.cc_analysis.restype = C.c_int
        L.cc_analysis.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        for f in ("cc_report_json", "cc_stop_reason", "cc_last_error", "cc_warnings", "cc_debug_encoded_snapshot"):
            getattr(L, f).restype = C.c_char_p
            getattr(L, f).argtypes = [C.c_void_p]
        L.cc_report_print.restype = C.c_char_p
        L.cc_report_print.argtypes = [C.c_void_p, C.c_int32, C.c_char_p]
        L.cc_scheduled_count.restype = C.c_int64
        L.cc_scheduled_count.argtypes = [C.c_void_p]
        L.cc_scheduled_node.restype = C.c_char_p
        L.cc_scheduled_node.argtypes = [C.c_void_p, C.c_int64]
        L.cc_close.restype = None
        L.cc_close.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class ListClient:
    """Stand-in for the clientset SyncWithClient LISTs from: plain lists of object dicts."""

    def __init__(self, nodes=(), pods=(), namespaces=(), services=(), replication_controllers=(), replica_sets=(), stateful_sets=()):
        self.nodes, self.pods, self.namespaces = list(nodes), list(pods), list(namespaces)
        # simulator.go:217-281 copies these too; the scheduler reads them only for system-default topology spreading
        self.services, self.replication_controllers = list(services), list(replication_controllers)
        self.replica_sets, self.stateful_sets = list(replica_sets), list(stateful_sets)


class ClusterCapacity:
    def __init__(self, handle, n_podspecs=1):
        self._h = handle
        self._report = None
        self._n = n_podspecs

    def _err(self, rc, what):
        msg = lib().cc_last_error(self._h).decode()
        if rc == -4:
            raise UnsupportedError(msg)
        raise FrameworkError("%s rc=%d: %s" % (what, rc, msg))

    def SyncWithClient(self, client):
        rc = lib().cc_sync_with_objects(self._h, json.dumps(client.nodes).encode(), json.dumps(client.pods).encode(),
                                        json.dumps(getattr(client, "namespaces", [])).encode())
        if rc:
            self._err(rc, "SyncWithClient")
        wl = [getattr(client, a, None) or [] for a in ("services", "replication_controllers", "replica_sets", "stateful_sets")]
        if any(wl):
            rc = lib().cc_sync_workloads(self._h, *[json.dumps(x).encode() for x in wl])
            if rc:
                self._err(rc, "SyncWithClient(workloads)")
        self._report = None

    def Run(self):
        rc = lib().cc_run(self._h)
        if rc:
            self._err(rc, "Run")
        self._report = None

    def RunEach(self):
        """Every podspec analysed on its own against the synced snapshot, in one GPU launch (cc_run_each): a list with one result per
        podspec, in order. Result t has Report(), Print(), StopReason() and ScheduledPods() with the meaning they have on a
        ClusterCapacity built from podspec t alone and Run()."""
        rc = lib().cc_run_each(self._h)
        if rc:
            self._err(rc, "RunEach")
        out = []
        for t in range(self._n):
            v = C.c_void_p()
            rc = lib().cc_analysis(self._h, t, C.byref(v))
            if rc:
                self._err(rc, "RunEach")
            out.append(Analysis(v, self))
        return out

    def Report(self):
        if self._report is None:
            s = lib().cc_report_json(self._h)
            if s is None:
                self._err(-5, "Report")
            self._report = json.loads(s.decode())
        return self._report

    def Print(self, verbose=False, fmt=""):
        s = lib().cc_report_print(self._h, 1 if verbose else 0, fmt.encode())
        if s is None:
            self._err(-1, "ClusterCapacityReviewPrint")
        return s.decode()

    def StopReason(self):
        return lib().cc_stop_reason(self._h).decode()

    def Warnings(self):
        """Deviations from what the reference would have done with this snapshot (cc_warnings): a list of lines, usually empty."""
        return [l for l in lib().cc_warnings(self._h).decode().split("\n") if l]

    def ScheduledPods(self):
        """Node name of every simulated pod, in placement order (ScheduledPods()[k].Spec.NodeName)."""
        n = lib().cc_scheduled_count(self._h)
        return [lib().cc_scheduled_node(self._h, k).decode() for k in range(n)]

    def EncodedSnapshot(self):
        s = lib().cc_debug_encoded_snapshot(self._h)
        if s is None:
            self._err(-4 if "unsupported" in lib().cc_last_error(self._h).decode() else -1, "encode")
        return json.loads(s.decode())

    def Close(self):
        if self._h:
            lib().cc_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.Close()
        except Exception:
            pass


class Analysis(ClusterCapacity):
    """One analysis of RunEach(): a read-only view owned by its ClusterCapacity, which it keeps alive."""

    def __init__(self, handle, owner):
        super().__init__(handle)
        self._owner = owner

    def Close(self):
        self._h = None        # the view goes with its owner's handle
        self._owner = None


def New(kube_scheduler_config, kube_config, simulated_pod, max_pods=0, exclude_nodes=(), device=0):
    """framework.New (simulator.go:107). kube_scheduler_config: None for the default profile or a dict
    {"percentageOfNodesToScore", "disabledFilters", "disabledScores", "weights"}; kube_config is unused (kept for
    signature parity: the analysis never talks to an API server after SyncWithClient).
    simulated_pod: one v1.Pod dict, or a list of up to 64 of them (the roadmap's "list of pods", README.md:305-306: pod k of the
    run is a clone of podspec k % T, the template index report.go:160 already uses)."""
    h = C.c_void_p()
    cfg = json.dumps(kube_scheduler_config).encode() if kube_scheduler_config else None
    if isinstance(simulated_pod, (list, tuple)):
        rc = lib().cc_new_list(cfg, json.dumps(list(simulated_pod)).encode(), int(max_pods), ",".join(exclude_nodes).encode(), device, C.byref(h))
        n = len(simulated_pod)
    else:
        rc = lib().cc_new(cfg, json.dumps(simulated_pod).encode(), int(max_pods), ",".join(exclude_nodes).encode(), device, C.byref(h))
        n = 1
    if rc:
        raise FrameworkError("New rc=%d: %s" % (rc, lib().cc_last_error(None).decode()))
    return ClusterCapacity(h, n)


def NewEach(kube_scheduler_config, kube_config, podspecs, max_pods=0, exclude_nodes=(), device=0, devices=None):
    """A per-analysis ClusterCapacity over up to 4096 podspecs (cc_new_each, CCSIM_EACH_MAX_ANALYSES), for RunEach() only: analysis t
    is what New(podspec t) + Run() gives, hard topology spread, required pod (anti-)affinity and hostPorts included. The cluster is
    encoded once for all of them. Normalised soft scorers (preferred node
    affinity, ScheduleAnyway spreading, InterPodAffinity scoring, which a required affinity matching the pod's own labels brings under
    the default hardPodAffinityWeight), node shards and reference sampling are refused by name.
    devices: a list of CUDA ordinals (cc_new_each_on, up to 64, repeats allowed) instead of `device`: RunEach() deals the analyses over
    them and runs each device's share in a launch of its own, with the same results as on one device."""
    h = C.c_void_p()
    cfg = json.dumps(kube_scheduler_config).encode() if kube_scheduler_config else None
    podspecs = list(podspecs)
    devs = [int(device)] if devices is None else [int(d) for d in devices]
    if any(not -2 ** 31 <= d < 2 ** 31 for d in devs):
        raise FrameworkError("NewEach: a device ordinal outside int32: %r" % devs)
    rc = lib().cc_new_each_on(cfg, json.dumps(podspecs).encode(), int(max_pods), ",".join(exclude_nodes).encode(), (C.c_int32 * len(devs))(*devs),
                              len(devs), C.byref(h))
    if rc:
        raise FrameworkError("NewEach rc=%d: %s" % (rc, lib().cc_last_error(None).decode()))
    return ClusterCapacity(h, len(podspecs))


def ClusterCapacityReviewPrint(cc, verbose=False, fmt=""):
    """framework.ClusterCapacityReviewPrint (report.go:305): prints; an unknown format raises like the reference errors."""
    print(cc.Print(verbose, fmt), end="")
