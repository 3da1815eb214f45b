"""GPU: per-analysis runs dealt over a device list (cc_new_each_on / framework.NewEach(devices=...) / `cluster-capacity --each
--devices`). Every analysis of a multi-device handle must read exactly like the one-device handle's: stop reason, placement sequence
and the review in every format (creationTimestamp masked). One H100 is enough: the lists repeat ordinal 0, so that every share runs
on its own engine one after the other; the [0, 1] case runs where two devices are visible."""
import ctypes as C
import importlib
import io
import json
import re
from contextlib import redirect_stdout

import pytest

import helpers
from test_each import mask
from test_each_coupled import NO_HARD_WEIGHT, podspecs, stripped_cluster
from test_each_many import many

fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")

pytestmark = pytest.mark.gpu
NODE_LOCAL = ["plain", "tolerations", "extended", "best_effort", "never_preempt", "selector"]
KERNEL_LINE = re.compile(r"run/ccsim_run_each on device (\d+): (\d+) analyses, kernel (\S+),")


@pytest.fixture(scope="module")
def sms(built):
    return helpers.device_sm_count()


def run_each(tm, nodes, pods, limit, devices, cfg=NO_HARD_WEIGHT):
    """the reviews of one RunEach: (stop reason, sequence, JSON report, verbose prints in the three formats) per analysis"""
    cc = fw.NewEach(cfg, None, tm, limit, [], devices=devices)
    try:
        cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
        return [(r.StopReason(), r.ScheduledPods(), mask(json.dumps(r.Report())), [mask(r.Print(True, f)) for f in ("", "json", "yaml")])
                for r in cc.RunEach()]
    finally:
        cc.Close()


def kernels(capfd):
    """(device, analyses, kernel) of every share that ran since the last call, in the order they finished"""
    return [(int(d), int(a), k) for d, a, k in KERNEL_LINE.findall(capfd.readouterr().err)]


def same_as_one_device(tm, nodes, pods, limit, lists, capfd=None):
    """every device list's reviews against the one-device handle's; with capfd (and CCHOST_TIMING set) the kernels of the shares of
    [0] and of every list, the largest share first"""
    if capfd is not None:
        kernels(capfd)
    one = run_each(tm, nodes, pods, limit, [0])
    assert len(one) == len(tm)
    ran = {(0,): kernels(capfd)} if capfd is not None else {}
    for devices in lists:
        got = run_each(tm, nodes, pods, limit, devices)
        for t in range(len(tm)):
            assert got[t] == one[t], (devices, t)
        if capfd is not None:
            ran[tuple(devices)] = sorted(kernels(capfd), key=lambda x: -x[1])
    return one, ran


# ---- 1. node-local podspecs, across the packing edge -------------------------------------------------------------------------------
def test_node_local_split_across_the_packing_edge(built, sms, capfd, monkeypatch):
    """T = 2 x SMs + 1: on one device every analysis shares CTAs (each<packed>); dealt over two entries one share holds SMs + 1
    analyses (packed) and the other SMs (one CTA each: each), over three every share takes one CTA per analysis"""
    T = 2 * sms + 1
    nodes, pods = stripped_cluster(41, n_nodes=40, n_pods=60)
    tm = [helpers.template(NODE_LOCAL[t % len(NODE_LOCAL)]) for t in range(T)]
    for t, p in enumerate(tm):
        p["metadata"]["name"] = "pod-%03d" % t
    tm[1]["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "100", "memory": "1Gi"}}     # fits nowhere
    monkeypatch.setenv("CCHOST_TIMING", "1")
    one, ran = same_as_one_device(tm, nodes, pods, 0, [[0, 0], [0, 0, 0]], capfd)
    assert ran[(0,)] == [(0, T, "each<packed>")]
    assert ran[(0, 0)] == [(0, sms + 1, "each<packed>"), (0, sms, "each")]
    assert ran[(0, 0, 0)] == [(0, -(-T // 3), "each"), (0, T // 3, "each"), (0, T // 3, "each")]
    assert one[1][1] == [] and "Insufficient cpu" in one[1][0]
    assert all(r[1] and r[0].startswith("Unschedulable") for t, r in enumerate(one) if t != 1)


# ---- 2. coupled podspecs: hard spread, hostname anti-affinity, hostPorts -----------------------------------------------------------
@pytest.mark.parametrize("limit", [0, 25])
def test_coupled_podspecs(built, capfd, monkeypatch, limit):
    nodes, pods = stripped_cluster(42, n_nodes=40, n_pods=60)
    tm = many(23, hostports=(2, 9, 20))
    monkeypatch.setenv("CCHOST_TIMING", "1")
    one, ran = same_as_one_device(tm, nodes, pods, limit, [[0, 0], [0, 0, 0]], capfd)
    # every share holds coupled analyses: one CTA per analysis (each), 12 + 11 and 8 + 8 + 7 of them
    assert ran[(0, 0)] == [(0, 12, "each"), (0, 11, "each")]
    assert ran[(0, 0, 0)] == [(0, 8, "each"), (0, 8, "each"), (0, 7, "each")]
    for t in (2, 9, 20):
        assert len(one[t][1]) == len(set(one[t][1])) > 0
        if not limit:
            assert "node(s) didn't have free ports" in one[t][0]
    assert any("spread" in p["metadata"]["name"] and r[1] for p, r in zip(tm, one))


# ---- 3. a PreFilter-rejected podspec, analyses that reach --max-limit and analyses that do not ---------------------------------------
@pytest.mark.parametrize("devices", [[0, 0], [0, 0, 0]])
def test_prefilter_and_max_limit_mix(built, devices):
    nodes, pods = stripped_cluster(43, n_nodes=30, n_pods=40)
    tm = podspecs(["spread_zone", "plain", "anti_hostname", "selector", "hostports", "tolerations", "extended"])
    tm[1]["spec"]["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
        {"matchFields": [{"key": "metadata.name", "operator": "In", "values": [nodes[0]["metadata"]["name"]]},
                         {"key": "metadata.name", "operator": "In", "values": [nodes[1]["metadata"]["name"]]}]}]}}}
    tm[5]["spec"]["containers"][0]["resources"] = {"requests": {"cpu": "10m", "memory": "1Mi"}}
    limit = 20
    one, _ = same_as_one_device(tm, nodes, pods, limit, [devices])
    assert one[1][1] == [] and "didn't match Pod's node affinity/selector" in one[1][0]
    assert one[5][0] == "LimitReached: Maximum number of pods simulated: %d" % limit


# ---- 4. fewer analyses than entries; one analysis ------------------------------------------------------------------------------------
@pytest.mark.parametrize("variants,devices", [(["spread_zone", "plain"], [0, 0, 0]), (["hostports"], [0, 0]), (["plain"], [0, 0, 0])])
def test_empty_shares(built, capfd, monkeypatch, variants, devices):
    nodes, pods = stripped_cluster(44, n_nodes=30, n_pods=40)
    monkeypatch.setenv("CCHOST_TIMING", "1")
    _, ran = same_as_one_device(podspecs(variants), nodes, pods, 0, [devices], capfd)
    assert len(ran[tuple(devices)]) == len(variants)      # a share without analyses gets no engine and no launch
    assert all(a == 1 for _, a, _ in ran[tuple(devices)])


# ---- 5. refusals name the analysis by its index in the podspec list ----------------------------------------------------------------
def test_refusal_of_a_later_share_names_the_global_index(built):
    """a normalised soft scorer on analysis 3: with two entries it is analysis 1 of the second share's launch"""
    nodes, pods = stripped_cluster(45, n_nodes=20, n_pods=20)
    tm = podspecs(["plain", "selector", "tolerations", "pref_affinity"])
    errs = []
    for devices in ([0], [0, 0]):
        cc = fw.NewEach(None, None, tm, 0, [], devices=devices)
        cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
        with pytest.raises(fw.UnsupportedError) as e:
            cc.RunEach()
        errs.append(str(e.value))
        assert fw.lib().cc_analysis(cc._h, 0, C.byref(C.c_void_p())) == -5      # a failed run leaves no analyses
        cc.Close()
    assert errs[0] == errs[1]
    assert "per-analysis runs: template 3 has a normalised soft scorer" in errs[1]


def test_domain_group_refusal_of_a_later_share_names_the_global_index(built):
    """a hard zone spread over 4 100 two-node zones (more domain groups than an analysis may have) on analysis 1, the first analysis
    of the second share"""
    zones = 4100
    nodes = [helpers.make_node("n%05d" % i, labels={"topology.kubernetes.io/zone": "z%04d" % (i // 2)}) for i in range(2 * zones)]
    tm = podspecs(["anti_hostname", "spread_zone"])
    errs = []
    for devices in ([0], [0, 0]):
        cc = fw.NewEach(None, None, tm, 0, [], devices=devices)
        cc.SyncWithClient(fw.ListClient(nodes, [], []))
        with pytest.raises(fw.UnsupportedError) as e:
            cc.RunEach()
        errs.append(str(e.value))
        cc.Close()
    assert errs[0] == errs[1] == "unsupported on the GPU path: ccsim_set_analyses: per-analysis runs: analysis 1 has %d domain groups (max 4096)" % zones


def test_an_ordinal_without_a_device(built):
    nodes, pods = stripped_cluster(46, n_nodes=20, n_pods=20)
    cc = fw.NewEach(None, None, podspecs(["plain", "selector"]), 0, [], devices=[0, 1000])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    with pytest.raises(fw.FrameworkError, match=r"RunEach rc=-7: ccsim_create: device 1000 out of range"):
        cc.RunEach()
    cc.Close()


# ---- 6. two devices, where there are two ---------------------------------------------------------------------------------------------
def test_two_devices(built):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("fewer than two CUDA devices visible")
    nodes, pods = stripped_cluster(47, n_nodes=40, n_pods=60)
    same_as_one_device(many(31, hostports=(4, 17)), nodes, pods, 0, [[0, 1], [1, 0, 1]])


# ---- 7. the command line -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["", "json", "yaml"])
def test_cli_each_devices(built, tmp_path, fmt):
    nodes, pods = stripped_cluster(48, n_nodes=30, n_pods=40)
    (tmp_path / "snap.json").write_text(json.dumps({"nodes": nodes, "pods": pods, "namespaces": []}))
    d = tmp_path / "specs"
    d.mkdir()
    for i, p in enumerate(podspecs(["spread_zone", "plain", "hostports", "anti_hostname", "selector"])):
        (d / ("%02d.json" % i)).write_text(json.dumps(p))

    def run(extra):
        out = io.StringIO()
        with redirect_stdout(out):
            assert cli.main(["--podspec", str(d), "--each", "--snapshot", str(tmp_path / "snap.json"), "--max-limit", "12", "--verbose"] +
                            (["-o", fmt] if fmt else []) + extra) == 0
        return mask(out.getvalue())
    one = run([])
    assert "instance(s) of the pod" in one or fmt
    assert run(["--devices", "0,0"]) == one == run(["--devices", "0,0,0,0,0,0"])
