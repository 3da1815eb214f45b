"""Per-analysis handles (cc_new_each / framework.NewEach) where no GPU is needed: the ccsim_analysis_terms layout, every analysis's own
encoding against the podspec's single encoding, and the host side of the views on a cluster without nodes."""
import ctypes as C
import importlib
import json

import numpy as np
import pytest

import helpers
from test_each import mask

abi = importlib.import_module("cluster-capacity_b200._abi")
engine = importlib.import_module("cluster-capacity_b200.engine")
fw = importlib.import_module("cluster-capacity_b200.framework")

# podspecs with coupled terms, mixed with node-local ones; affinity_zone only without InterPodAffinity scoring (below)
COUPLED = ["hostports", "spread_zone", "spread_two", "spread_everything", "anti_hostname", "anti_zone"]
NODE_LOCAL = ["plain", "selector", "tolerations", "extended"]
NO_HARD_WEIGHT = {"hardPodAffinityWeight": 0}


def podspecs(variants):
    out = []
    for i, v in enumerate(variants):
        p = helpers.template(v)
        p["metadata"]["name"] = "%s-%d" % (v.replace("_", "-"), i)
        out.append(p)
    return out


def stripped_cluster(seed, **kw):
    """a random cluster whose existing pods carry no pod (anti-)affinity: their terms would score the incoming pod"""
    nodes, pods = helpers.random_cluster(seed, **kw)
    for p in pods:
        p["spec"].pop("affinity", None)
    return nodes, pods


def test_analysis_terms_layout():
    assert C.sizeof(abi.AnalysisTerms) == 8 + 8 + 8 * abi.MAX_TOPO_COLS
    assert abi.AnalysisTerms.counters.offset == 8 and abi.AnalysisTerms.topo.offset == 16
    assert "ccsim_set_analyses" in engine.EXPORTS and "cc_new_each" in fw.EXPORTS


def static_bit_column(enc, bit):
    nd = enc["nodes"]
    n, w = nd["n"], bit >> 6
    return [(int(nd["static_mask"][w * n + i]) >> (bit & 63)) & 1 for i in range(n)]


@pytest.mark.parametrize("seed", [3, 4])
def test_each_encoding_is_every_podspecs_single_encoding(built, seed):
    nodes, pods = stripped_cluster(seed, n_nodes=30, n_pods=50)
    tm = podspecs(["plain"] + COUPLED + ["selector", "affinity_zone", "extended"])
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, 9, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    enc = cc.EncodedSnapshot()
    _, merged, ctr, _, _, _ = helpers.from_encoded(enc)
    assert not ctr and not enc["nodes"]["topo"] and len(enc["analyses"]) == len(tm)
    assert enc["nodes"]["has_placed_mask"]
    for t, p in enumerate(tm):
        one = fw.New(NO_HARD_WEIGHT, None, p, 9, [])
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        single = one.EncodedSnapshot()
        _, (st,), sctr, _, _, _ = helpers.from_encoded(single)
        a = enc["analyses"][t]
        assert a["topo"] == single["nodes"]["topo"] and a["prefilter_msg"] == single["prefilter_msg"]
        assert len(a["counters"]) == len(single["counters"])
        for c, s in zip(a["counters"], single["counters"]):
            assert (c["topo_col"], c["n_present"], c["inc"], c["init"]) == (s["topo_col"], s["n_present"], s["inc"], s["init"])
            assert (c["elig_bit"] < 0) == (s["elig_bit"] < 0)
            if s["elig_bit"] >= 0:     # moved with the podspec's other static bits: the same nodes carry it
                assert static_bit_column(enc, c["elig_bit"]) == static_bit_column(single, s["elig_bit"])
        mt = merged[t]
        for f in ("n_pts", "n_aff", "n_anti", "aff_total_init", "flags", "filter_enable", "score_enable", "req_cpu", "req_mem"):
            assert getattr(mt, f) == getattr(st, f), (t, f)
        assert [(x.counter, x.max_skew, x.self_match, x.min_zero) for x in mt.pts] == [(x.counter, x.max_skew, x.self_match, x.min_zero) for x in st.pts]
        assert list(mt.aff_counter) == list(st.aff_counter) and list(mt.anti_counter) == list(st.anti_counter)
        assert mt.port_tmpl_conflict == (1 << t if st.port_tmpl_conflict else 0)
        one.Close()
    cc.Close()


def test_each_handle_keeps_list_refusals_apart(built):
    """the same podspecs on a list handle are still refused; cc_run on a per-analysis handle fails with CC_ESTATE"""
    nodes, pods = stripped_cluster(3, n_nodes=10, n_pods=10)
    tm = podspecs(["plain", "spread_zone"])
    lst = fw.New(None, None, tm, 5, [])
    lst.SyncWithClient(helpers.list_client(fw, nodes, pods))
    with pytest.raises(fw.UnsupportedError, match="several podspecs of which one has topology spread"):
        lst.RunEach()
    lst.Close()
    cc = fw.NewEach(None, None, tm, 5, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    assert fw.lib().cc_run(cc._h) == -5
    assert "cc_run_each" in fw.lib().cc_last_error(cc._h).decode()
    cc.Close()


def test_each_handle_on_an_empty_cluster_reads_like_single_runs(built):
    tm = podspecs(NODE_LOCAL[:2] + COUPLED)
    cc = fw.NewEach(None, None, tm, 7, [])
    cc.SyncWithClient(fw.ListClient([], [], []))
    assert fw.lib().cc_run(cc._h) == -5
    res = cc.RunEach()
    assert len(res) == len(tm)
    for t, r in enumerate(res):
        one = fw.New(None, None, tm[t], 7, [])
        one.SyncWithClient(fw.ListClient([], [], []))
        one.Run()
        assert r.StopReason() == one.StopReason() == "Unschedulable: no nodes available to schedule pods"
        assert r.ScheduledPods() == one.ScheduledPods() == []
        for fmt in ("", "json", "yaml"):
            assert mask(r.Print(True, fmt)) == mask(one.Print(True, fmt))
        one.Close()
    cc.Close()
