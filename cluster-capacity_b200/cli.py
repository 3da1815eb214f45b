"""`cluster-capacity` command line — the reference's flag surface (cmd/cluster-capacity/app/options/options.go:65-77) on
top of the GPU path:

    python -m cluster-capacity_b200.cli --podspec examples/pod.yaml --snapshot cluster.json [--max-limit N]
           [--exclude-nodes a,b] [--default-config cfg.yaml] [--verbose] [-o json|yaml] [--kubeconfig KUBECONFIG]
    (--podspec may be repeated or name a directory: several podspecs are simulated round-robin, e.g. the genpod output of 64 namespaces)

The analysis needs the LISTed Node/Pod/Namespace objects. `--snapshot` takes a JSON/YAML file
{"nodes": [...], "pods": [...], "namespaces": [...]} (or a directory with nodes.json / pods.json / namespaces.json);
with `--kubeconfig` (or CC_INCLUSTER) the same lists are fetched through kubectl — the only moment the real API server is
touched, exactly like SyncWithClient (pkg/framework/simulator.go:176-295).
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import yaml

VERSION = "cluster-capacity-b200 0.1 (reference surface: kubernetes-sigs/cluster-capacity @3cb0ea28)"


def parse_api_spec(path, scheduler_name="default-scheduler"):
    """ParseAPISpec (options.go:79-147): YAML or JSON pod, namespace/schedulerName/dnsPolicy/restartPolicy defaults."""
    with open(path) as f:
        pod = yaml.safe_load(f)
    if not isinstance(pod, dict) or "spec" not in pod:
        raise SystemExit("Failed to parse pod spec file: Failed to decode config file: not a Pod")
    md = pod.setdefault("metadata", {})
    if not md.get("namespace"):
        md["namespace"] = "default"
    spec = pod["spec"]
    spec.setdefault("schedulerName", scheduler_name)
    if not spec.get("dnsPolicy"):
        spec["dnsPolicy"] = "ClusterFirst"
    if not spec.get("restartPolicy"):
        spec["restartPolicy"] = "Always"
    for c in spec.get("containers") or []:
        if not c.get("terminationMessagePolicy"):
            c["terminationMessagePolicy"] = "FallbackToLogsOnError"
    errs = []
    if not md.get("name"):
        errs.append("Required value: metadata.name")
    if not spec.get("containers"):
        errs.append("Required value: spec.containers")
    if errs:
        raise SystemExit("Failed to parse pod spec file: Invalid pod: %r" % ", ".join(errs))
    return pod


def load_scheduler_config(path):
    """--default-config: a KubeSchedulerConfiguration (YAML/JSON). Only what changes results on this path is honoured:
    percentageOfNodesToScore and, for profile[0], multiPoint/filter/score enabled-disabled lists and score weights."""
    if not path:
        return None
    with open(path) as f:
        cfg = yaml.safe_load(f) or {}
    out = {"disabledFilters": [], "disabledScores": [], "weights": {}}
    if cfg.get("percentageOfNodesToScore") is not None:
        out["percentageOfNodesToScore"] = int(cfg["percentageOfNodesToScore"])
    prof = (cfg.get("profiles") or [{}])[0]
    plugins = prof.get("plugins") or {}
    for point, key in (("filter", "disabledFilters"), ("score", "disabledScores")):
        for d in (plugins.get(point) or {}).get("disabled") or []:
            out[key].append(d["name"])
    for d in (plugins.get("multiPoint") or {}).get("disabled") or []:
        out["disabledFilters"].append(d["name"])
        out["disabledScores"].append(d["name"])
    # getScoreWeights (framework.go:476-497): a Score-point weight wins over a MultiPoint one, and a weight of 0 (or none: an
    # enabled entry replaces the default one, weight included) means 1. A negative weight is an error.
    for point in ("multiPoint", "score"):
        for e in (plugins.get(point) or {}).get("enabled") or []:
            w = int(e.get("weight") or 0)
            if w < 0:
                raise SystemExit("Invalid scheduler configuration: score weight of %s is negative: %d" % (e["name"], w))
            out["weights"][e["name"]] = w or 1
    return out


# what SyncWithClient LISTs and the scheduler plugins of the hot path read (simulator.go:176-281); PVCs, PDBs and
# StorageClasses are copied by the reference too, but only the out-of-scope volume / preemption plugins look at them
KINDS = ("nodes", "pods", "namespaces", "services", "replicationcontrollers", "replicasets", "statefulsets")


def load_snapshot(path):
    def items(obj):
        if obj is None:
            return []
        if isinstance(obj, dict) and "items" in obj:
            return obj["items"] or []
        return obj
    if os.path.isdir(path):
        out = {}
        for k in KINDS:
            fn = os.path.join(path, k + ".json")
            out[k] = items(json.load(open(fn))) if os.path.exists(fn) else []
        return out
    with open(path) as f:
        d = yaml.safe_load(f)
    return {k: items(d.get(k)) for k in KINDS}


def list_from_cluster(kubeconfig):
    base = ["kubectl"] + (["--kubeconfig", kubeconfig] if kubeconfig else [])
    out = {}
    for k, args in (("nodes", ["get", "nodes"]), ("pods", ["get", "pods", "-A"]), ("namespaces", ["get", "namespaces"]),
                    ("services", ["get", "services", "-A"]), ("replicationcontrollers", ["get", "replicationcontrollers", "-A"]),
                    ("replicasets", ["get", "replicasets.apps", "-A"]), ("statefulsets", ["get", "statefulsets.apps", "-A"])):
        out[k] = json.loads(subprocess.check_output(base + args + ["-o", "json"]))["items"]
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="cluster-capacity", description="Cluster-capacity is used for simulating scheduling of one or multiple pods")
    ap.add_argument("--kubeconfig", default="", help="Path to the kubeconfig file to use for the analysis.")
    ap.add_argument("--podspec", action="append", default=[],
                    help="Path to JSON or YAML file containing pod definition. May be repeated, or name a directory of podspec files: the pods are "
                         "then simulated round-robin (README.md:305-306 'accept a list of pods'; template index = pod number %% #podspecs).")
    ap.add_argument("--max-limit", type=int, default=0, help="Number of instances of pod to be scheduled after which analysis stops. By default unlimited.")
    ap.add_argument("--exclude-nodes", default="", help="Exclude nodes to be scheduled")
    ap.add_argument("--default-config", default="", help="Path to JSON or YAML file containing scheduler configuration.")
    ap.add_argument("--verbose", action="store_true", help="Verbose mode")
    ap.add_argument("-o", "--output", default="", help="Output format. One of: json|yaml")
    ap.add_argument("--snapshot", default="", help="Node/Pod/Namespace lists as a file or directory (instead of a live API server)")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if not a.podspec:
        print("Pod spec file is missing")          # Validate (server.go:83-86)
        ap.print_help()
        return 0
    print("Cluster capacity version %s" % VERSION)
    fw = importlib.import_module("cluster-capacity_b200.framework")
    try:
        files = []
        for path in a.podspec:
            if os.path.isdir(path):
                files += [os.path.join(path, f) for f in sorted(os.listdir(path)) if f.endswith((".yaml", ".yml", ".json"))]
            else:
                files.append(path)
        pods = [parse_api_spec(f) for f in files]
        pod = pods[0] if len(pods) == 1 else pods
        objs = load_snapshot(a.snapshot) if a.snapshot else list_from_cluster(a.kubeconfig)
        cc = fw.New(load_scheduler_config(a.default_config), None, pod, a.max_limit, [x for x in a.exclude_nodes.split(",") if x], device=a.device)
        cc.SyncWithClient(fw.ListClient(objs["nodes"], objs["pods"], objs["namespaces"], objs["services"], objs["replicationcontrollers"],
                                        objs["replicasets"], objs["statefulsets"]))
        for w in cc.Warnings():
            print("warning: " + w, file=sys.stderr)
        cc.Run()
        fw.ClusterCapacityReviewPrint(cc, a.verbose, a.output)
    except (fw.FrameworkError, OSError, subprocess.CalledProcessError) as e:   # the reference prints the error and exits 0 (server.go:68-71)
        print(e)
    return 0


if __name__ == "__main__":
    sys.exit(main())
