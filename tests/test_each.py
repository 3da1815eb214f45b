"""Per-analysis runs (cc_run_each / `cluster-capacity --each`) where no GPU is needed: the encoder's refusals of podspec lists, and
the host side of the analysis views on a cluster without nodes (no engine runs there: every analysis ends before it)."""
import importlib
import io
import json
import re
from contextlib import redirect_stdout

import pytest

import helpers

fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")


def mask(text):
    """a review with its creationTimestamp (the time of the run) replaced"""
    return re.sub(r'(creationTimestamp"?: ?)("[^"]*"|\S+)', r'\1"T"', text)


def podspecs():
    out = []
    for i, v in enumerate(["plain", "selector", "never_preempt"]):
        p = helpers.template(v)
        p["metadata"]["name"] = "%s-%d" % (v.replace("_", "-"), i)
        out.append(p)
    return out


@pytest.mark.parametrize("variant,message", [("spread_zone", "several podspecs of which one has topology spread"),
                                             ("anti_hostname", "several podspecs of which one has topology spread"),
                                             ("hostports", "several podspecs with hostPorts")])
def test_run_each_refuses_coupled_podspecs_in_the_encoder(built, variant, message):
    nodes, pods = helpers.random_cluster(3, n_nodes=10, n_pods=10)
    for p in pods:
        p["spec"].pop("affinity", None)
    cc = fw.New(None, None, [helpers.template("plain"), helpers.template(variant)], 5, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    with pytest.raises(fw.UnsupportedError, match=message):
        cc.RunEach()
    cc.Close()


def test_run_each_needs_a_sync_and_views_need_a_run(built):
    import ctypes as C
    cc = fw.New(None, None, podspecs(), 0, [])
    with pytest.raises(fw.FrameworkError, match="cc_sync_with_objects must come first"):
        cc.RunEach()
    v = C.c_void_p()
    assert fw.lib().cc_analysis(cc._h, 0, C.byref(v)) == -5
    assert "cc_run_each must come first" in fw.lib().cc_last_error(cc._h).decode()
    cc.Close()


def test_analyses_of_an_empty_cluster_read_like_single_runs(built):
    """No nodes: every analysis ends with ErrNoNodesAvailable before the engine. Each view reads like cc_new(podspec t) + cc_run, and is
    read-only."""
    import ctypes as C
    tm = podspecs()
    cc = fw.New(None, None, tm, 7, [])
    cc.SyncWithClient(fw.ListClient([], [], []))
    res = cc.RunEach()
    assert len(res) == len(tm)
    for t, r in enumerate(res):
        one = fw.New(None, None, tm[t], 7, [])
        one.SyncWithClient(fw.ListClient([], [], []))
        one.Run()
        assert r.StopReason() == one.StopReason() == "Unschedulable: no nodes available to schedule pods"
        assert r.ScheduledPods() == one.ScheduledPods() == []
        a, b = r.Report(), one.Report()
        a["status"].pop("creationTimestamp")
        b["status"].pop("creationTimestamp")
        assert a == b and a["spec"]["templates"][0]["metadata"]["name"] == tm[t]["metadata"]["name"]
        for fmt in ("", "json", "yaml"):
            assert mask(r.Print(True, fmt)) == mask(one.Print(True, fmt))
        one.Close()
        # read-only: no run, no sync on a view; closing it leaves the base intact
        assert fw.lib().cc_run(r._h) == -5 and fw.lib().cc_run_each(r._h) == -5
        assert fw.lib().cc_sync_with_objects(r._h, b"[]", b"[]", b"[]") == -5
        fw.lib().cc_close(r._h)
    v = C.c_void_p()
    assert fw.lib().cc_analysis(cc._h, len(tm), C.byref(v)) == -1
    assert res[-1].StopReason().startswith("Unschedulable")      # views stay valid until the base runs again or closes
    cc.Close()


@pytest.mark.parametrize("fmt", ["", "json", "yaml"])
def test_cli_each_prints_one_review_per_podspec(built, tmp_path, fmt):
    import yaml
    specs = tmp_path / "specs"
    specs.mkdir()
    for t, p in enumerate(podspecs()):
        (specs / ("%02d.yaml" % t)).write_text(yaml.safe_dump(p))
    snap = tmp_path / "cluster.json"
    snap.write_text(json.dumps({"nodes": [], "pods": [], "namespaces": []}))

    def run(args):
        buf = io.StringIO()
        with redirect_stdout(buf):
            assert cli.main(args + ["--snapshot", str(snap), "--max-limit", "3", "--verbose"] + (["-o", fmt] if fmt else [])) == 0
        head, body = buf.getvalue().split("\n", 1)
        assert head.startswith("Cluster capacity version")
        return body

    singles = [run(["--podspec", str(specs / f)]) for f in sorted(p.name for p in specs.iterdir())]
    got = run(["--podspec", str(specs), "--each"])
    if fmt == "json":
        assert [json.loads(mask(s)) for s in singles] == json.loads(mask(got))
    elif fmt == "yaml":
        assert mask(got) == mask("---\n".join(singles))
    else:
        assert got == "".join(singles)
