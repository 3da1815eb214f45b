"""Per-analysis handles over several devices (cc_new_each_on / framework.NewEach(devices=...) / `cluster-capacity --each --devices`)
where no GPU is needed: the argument checks, the deal of the analyses over the device list, and the views of a cluster without nodes
(no engine runs there: every analysis ends before it)."""
import ctypes as C
import importlib
import io
import json
from contextlib import redirect_stdout

import pytest

import helpers
from test_each import mask
from test_each_coupled import COUPLED, NODE_LOCAL, NO_HARD_WEIGHT, podspecs, stripped_cluster

fw = importlib.import_module("cluster-capacity_b200.framework")
cli = importlib.import_module("cluster-capacity_b200.cli")


def new_each_on(devices, n=None, pods=None):
    """cc_new_each_on straight through the C-ABI: (rc, handle, cc_last_error(NULL))"""
    pods = json.dumps(pods if pods is not None else podspecs(["plain", "selector"])).encode()
    arr = (C.c_int32 * max(1, len(devices)))(*devices)
    h = C.c_void_p()
    rc = fw.lib().cc_new_each_on(None, pods, 5, b"", arr, len(devices) if n is None else n, C.byref(h))
    return rc, h, fw.lib().cc_last_error(None).decode()


def test_cc_new_each_on_argument_checks(built):
    assert "cc_new_each_on" in fw.EXPORTS
    for devices, n, message in (([], None, "empty device list"), ([0], 0, "empty device list"), ([0], -3, "empty device list"),
                                ([0, -1], None, "device list entry 1: negative CUDA ordinal -1"),
                                ([0] * 65, None, "more than 64 devices (65, CC_EACH_MAX_DEVICES)")):
        rc, h, err = new_each_on(devices, n)
        assert rc == -1 and err == message and not h.value, devices
    h = C.c_void_p()
    assert fw.lib().cc_new_each_on(None, b"[]", 5, b"", None, 2, C.byref(h)) == -1
    assert fw.lib().cc_last_error(None).decode() == "null argument"
    # 64 entries, repeated ordinals and ordinals no machine has are accepted: an ordinal without a device fails at cc_run_each
    for devices in ([0] * 64, [3, 3, 1], [1000]):
        rc, h, _ = new_each_on(devices)
        assert rc == 0 and h.value, devices
        fw.lib().cc_close(h)
    # the podspec checks are cc_new_each's
    rc, _, err = new_each_on([0, 1], pods=[])
    assert rc == -1 and err == "no podspec"


def test_new_each_devices_argument(built):
    plain = [helpers.template("plain")]
    for devices, message in (([], "empty device list"), ([1, -2], "device list entry 1: negative CUDA ordinal -2"),
                             (range(65), r"more than 64 devices \(65, CC_EACH_MAX_DEVICES\)"), ([2 ** 32], "outside int32")):
        with pytest.raises(fw.FrameworkError, match=message):
            fw.NewEach(None, None, plain, 3, [], devices=devices)
    with pytest.raises(fw.FrameworkError, match="device list entry 0: negative CUDA ordinal -1"):
        fw.NewEach(None, None, plain, 3, [], device=-1)      # cc_new_each(device) is the list {device}
    fw.NewEach(None, None, plain, 3, [], devices=(0, 0, 1)).Close()


def shares(tm, devices, nodes=(), pods=()):
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, 5, [], devices=devices)
    cc.SyncWithClient(fw.ListClient(list(nodes), list(pods), []))
    out = cc.EncodedSnapshot()["shares"]
    cc.Close()
    return out


def test_the_deal(built):
    """coupled analyses round-robin over the list first, the node-local ones continue the deal; every share in increasing order"""
    nodes, pods = stripped_cluster(5, n_nodes=12, n_pods=20)
    kinds = NODE_LOCAL[:2] + COUPLED + NODE_LOCAL[2:] + ["plain"]         # coupled: 2..7; node-local: 0, 1, 8, 9, 10
    tm = podspecs(kinds)
    assert shares(tm, [0], nodes, pods) == [list(range(len(tm)))]
    assert shares(tm, [0, 1], nodes, pods) == [[0, 2, 4, 6, 8, 10], [1, 3, 5, 7, 9]]
    assert shares(tm, [4, 4, 4], nodes, pods) == [[0, 2, 5, 9], [1, 3, 6, 10], [4, 7, 8]]
    # more devices than analyses: the last entries' shares are empty
    assert shares(tm[:2], [0, 1, 2, 3], nodes, pods) == [[0], [1], [], []]
    assert shares(podspecs(["hostports", "plain", "spread_zone"]), [0, 1], nodes, pods) == [[0, 1], [2]]


@pytest.mark.parametrize("count,devices", [(1, [0, 0]), (3, [0, 0, 0]), (len(NODE_LOCAL[:2] + COUPLED), [0, 1]), (2, [0, 1, 2])])
def test_empty_cluster_views_on_several_devices_read_like_one_device(built, count, devices):
    """no nodes: every analysis ends before the engine, on any device list; each view reads like the one-device handle's"""
    tm = podspecs((NODE_LOCAL[:2] + COUPLED)[:count])
    one = fw.NewEach(None, None, tm, 7, [])
    one.SyncWithClient(fw.ListClient([], [], []))
    several = fw.NewEach(None, None, tm, 7, [], devices=devices)
    several.SyncWithClient(fw.ListClient([], [], []))
    a, b = one.RunEach(), several.RunEach()
    assert len(a) == len(b) == count
    for t in range(count):
        assert b[t].StopReason() == a[t].StopReason() == "Unschedulable: no nodes available to schedule pods"
        assert b[t].ScheduledPods() == a[t].ScheduledPods() == []
        assert b[t].Report()["spec"]["templates"][0]["metadata"]["name"] == tm[t]["metadata"]["name"]
        for fmt in ("", "json", "yaml"):
            assert mask(b[t].Print(True, fmt)) == mask(a[t].Print(True, fmt))
    v = C.c_void_p()
    assert fw.lib().cc_analysis(several._h, count, C.byref(v)) == -1
    one.Close()
    several.Close()


def run_cli(args):
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert cli.main(args) == 0
    return buf.getvalue()


@pytest.fixture
def specs_and_snapshot(tmp_path):
    import yaml
    specs = tmp_path / "specs"
    specs.mkdir()
    for t, p in enumerate(podspecs(["plain", "selector", "spread_zone"])):
        (specs / ("%02d.yaml" % t)).write_text(yaml.safe_dump(p))
    snap = tmp_path / "cluster.json"
    snap.write_text(json.dumps({"nodes": [], "pods": [], "namespaces": []}))
    return ["--podspec", str(specs), "--snapshot", str(snap), "--max-limit", "3", "--verbose"]


def test_cli_devices_needs_each(built, specs_and_snapshot):
    out = run_cli(specs_and_snapshot + ["--devices", "0,1"])
    head, body = out.split("\n", 1)
    assert head.startswith("Cluster capacity version") and body == "--devices is valid with --each only\n"
    for bad in ("0,x", "0,,1", "1.5"):
        body = run_cli(specs_and_snapshot + ["--each", "--devices", bad]).split("\n", 1)[1]
        assert body == "--devices: not a comma-separated list of CUDA ordinals: %r\n" % bad
    body = run_cli(specs_and_snapshot + ["--each", "--devices", "0,-1"]).split("\n", 1)[1]
    assert body == "NewEach rc=-1: device list entry 1: negative CUDA ordinal -1\n"


@pytest.mark.parametrize("fmt", ["", "json", "yaml"])
def test_cli_each_devices_prints_what_one_device_prints(built, specs_and_snapshot, fmt):
    args = specs_and_snapshot + ["--each"] + (["-o", fmt] if fmt else [])
    one = run_cli(args)
    assert "Termination reason: Unschedulable: no nodes available" in one or fmt
    for devices in ("0,0", "0,1,2,3"):
        assert mask(run_cli(args + ["--devices", devices])) == mask(one)
