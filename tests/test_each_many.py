"""Per-analysis handles past 64 podspecs (cc_new_each / framework.NewEach, up to CCSIM_EACH_MAX_ANALYSES) where no GPU is needed:
every analysis's encoding against the podspec's single encoding, the hostPort self-conflict bit of analyses 64 and up, and the
podspec bounds of per-analysis and list handles."""
import importlib

import pytest

import helpers
from test_each_coupled import NO_HARD_WEIGHT, static_bit_column, stripped_cluster

abi = importlib.import_module("cluster-capacity_b200._abi")
fw = importlib.import_module("cluster-capacity_b200.framework")

# podspecs without static node-predicate bits, so that a thousand of them stay inside the 256 bits a handle has; a nodeSelector
# (one bit) every 16th podspec, and hostPorts (one bit) where a test asks for them
CYCLE = ["plain", "tolerations", "extended", "spread_zone", "anti_hostname", "anti_zone", "best_effort", "never_preempt", "spread_everything",
         "affinity_zone"]
NODE_FIELDS = ("alloc_cpu", "alloc_mem", "alloc_eph", "alloc_pods", "req_cpu", "req_mem", "req_eph", "npods", "nz_cpu", "nz_mem",
               "taint_words", "taint_mask", "taint_nosched", "taint_prefer", "taint_dict", "taint_off", "taint_list")


def many(count, hostports=()):
    out = []
    for t in range(count):
        v = "hostports" if t in hostports else ("selector" if t % 16 == 5 else CYCLE[t % len(CYCLE)])
        p = helpers.template(v)
        p["metadata"]["name"] = "%s-%04d" % (v.replace("_", "-"), t)
        p["metadata"]["namespace"] = "ns-%04d" % t
        out.append(p)
    return out


def single_encoding(p, nodes, pods):
    one = fw.New(NO_HARD_WEIGHT, None, p, 9, [])
    try:
        one.SyncWithClient(helpers.list_client(fw, nodes, pods))
        return one.EncodedSnapshot()
    finally:
        one.Close()


def same_analysis(enc, merged_t, a, single):
    """analysis a of a per-analysis encoding against its podspec's single encoding, field by field"""
    _, (st,), _, _, _, _ = helpers.from_encoded(single)
    assert a["topo"] == single["nodes"]["topo"] and a["prefilter_msg"] == single["prefilter_msg"]
    assert len(a["counters"]) == len(single["counters"])
    for c, s in zip(a["counters"], single["counters"]):
        assert (c["topo_col"], c["n_present"], c["inc"], c["init"]) == (s["topo_col"], s["n_present"], s["inc"], s["init"])
        assert (c["elig_bit"] < 0) == (s["elig_bit"] < 0)
        if s["elig_bit"] >= 0:
            assert static_bit_column(enc, c["elig_bit"]) == static_bit_column(single, s["elig_bit"])
    mt = merged_t
    for f in ("n_pts", "n_aff", "n_anti", "aff_total_init", "flags", "filter_enable", "score_enable", "req_cpu", "req_mem", "req_eph",
              "nz_cpu", "nz_mem", "n_aff_terms"):
        assert getattr(mt, f) == getattr(st, f), f
    assert [(x.counter, x.max_skew, x.self_match, x.min_zero) for x in mt.pts] == [(x.counter, x.max_skew, x.self_match, x.min_zero) for x in st.pts]
    assert list(mt.aff_counter) == list(st.aff_counter) and list(mt.anti_counter) == list(st.anti_counter)
    assert list(mt.tol_nosched) == list(st.tol_nosched) and list(mt.tol_prefer) == list(st.tol_prefer)
    # a selector's static bit moved with the podspec: the same nodes carry it
    for w in range(abi.MAX_STATIC_WORDS):
        for b in range(64):
            if (int(st.sel_mask[w]) >> b) & 1:
                moved = [k for k in range(256) if (int(mt.sel_mask[k >> 6]) >> (k & 63)) & 1]
                assert len(moved) == 1 and static_bit_column(enc, moved[0]) == static_bit_column(single, 64 * w + b)
    return mt, st


@pytest.mark.parametrize("count", [65, 200, 1000])
def test_every_analysis_is_its_podspecs_single_encoding(built, count):
    nodes, pods = stripped_cluster(7, n_nodes=24, n_pods=40)
    tm = many(count, hostports=(64,))
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, 9, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    enc = cc.EncodedSnapshot()
    _, merged, ctr, _, _, _ = helpers.from_encoded(enc)
    assert not ctr and len(enc["analyses"]) == count == len(merged)
    first = single_encoding(tm[0], nodes, pods)
    for f in NODE_FIELDS:     # the cluster's columns, built once for the handle, are every single encoding's
        assert enc["nodes"][f] == first["nodes"][f], f
    assert enc["names"] == first["names"]
    ext = single_encoding(tm[CYCLE.index("extended")], nodes, pods)     # the union of the extended resources: this podspec's
    for f in ("scalar_names", "alloc_scalar", "req_scalar"):
        assert enc["nodes"][f] == ext["nodes"][f] and ext["nodes"]["scalar_names"] == ["example.com/foo"], f
    # every podspec of the shorter lists; a sample of every variant of the longest
    check = range(count) if count <= 200 else sorted(set(range(0, count, 37)) | set(range(60, 70)) | {count - 1})
    for t in check:
        mt, st = same_analysis(enc, merged[t], enc["analyses"][t], single_encoding(tm[t], nodes, pods))
        assert mt.port_tmpl_conflict == ((1 << (t % 64)) if st.port_tmpl_conflict else 0), t
    cc.Close()


def test_hostports_past_64_take_bit_t_mod_64(built):
    nodes, pods = stripped_cluster(8, n_nodes=20, n_pods=30)
    tm = many(140, hostports=(0, 64, 130))
    cc = fw.NewEach(NO_HARD_WEIGHT, None, tm, 9, [])
    cc.SyncWithClient(helpers.list_client(fw, nodes, pods))
    enc = cc.EncodedSnapshot()
    _, merged, _, _, _, _ = helpers.from_encoded(enc)
    assert enc["nodes"]["has_placed_mask"]
    assert [t for t in range(140) if merged[t].port_tmpl_conflict] == [0, 64, 130]
    assert merged[0].port_tmpl_conflict == merged[64].port_tmpl_conflict == 1
    assert merged[130].port_tmpl_conflict == 1 << 2
    for t in (64, 130):      # the existing-pod conflicts stay the podspec's own static bit
        same_analysis(enc, merged[t], enc["analyses"][t], single_encoding(tm[t], nodes, pods))
    cc.Close()


def test_podspec_bounds(built):
    assert abi.EACH_MAX_ANALYSES == 4096
    with open(__file__.rsplit("/tests/", 1)[0] + "/include/ccsim.h") as f:
        assert "#define CCSIM_EACH_MAX_ANALYSES 4096" in f.read()
    plain = helpers.template("plain")
    # the bound itself is accepted and encodes; one more is refused by name
    cc = fw.NewEach(None, None, [plain] * abi.EACH_MAX_ANALYSES, 3, [])
    cc.SyncWithClient(fw.ListClient([helpers.make_node("n0")], [], []))
    assert len(cc.EncodedSnapshot()["analyses"]) == abi.EACH_MAX_ANALYSES
    cc.Close()
    with pytest.raises(fw.FrameworkError, match=r"more than 4096 podspecs \(CCSIM_EACH_MAX_ANALYSES, per-analysis runs\)"):
        fw.NewEach(None, None, [plain] * (abi.EACH_MAX_ANALYSES + 1), 3, [])
    # list handles keep 64, with their message
    with pytest.raises(fw.FrameworkError, match="rc=-4: more than 64 podspecs$"):
        fw.New(None, None, [plain] * 65, 3, [])
    fw.New(None, None, [plain] * 64, 3, []).Close()
