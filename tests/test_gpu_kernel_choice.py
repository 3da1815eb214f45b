"""GPU: which wave-kernel instantiation a workload gets, or which refusal it meets, asserted from ccsim_prepare alone over small
workloads, one row per rule of the engine choice (DESIGN.md §4): generic, lean if eligible, tie-run batching or multi-commit on top
of lean, streaming when lean is not taken, and the refusals in the order they fire. A refused prepare leaves no kernel name and
launches nothing. Then one tiny run per instantiation pins the engine code and block size ccsim_run_stats reports for it.

The expectations are written from the rules, not recorded from a run."""
import importlib
import re

import numpy as np
import pytest

import helpers
from test_gpu_kernel_edges import _extended, _nodes

abi = importlib.import_module("cluster-capacity_b200._abi")
synth = importlib.import_module("cluster-capacity_b200.synth")
engine = importlib.import_module("cluster-capacity_b200.engine")

pytestmark = pytest.mark.gpu
MiB = 1 << 20
AUTO, SEQ, BATCHED = abi.ENGINE_AUTO, abi.ENGINE_SEQUENTIAL, abi.ENGINE_BATCHED
SAMPLING = dict(sampling=abi.SAMPLING_REFERENCE)
N = 3000

UNBOUNDED = "the run is unbounded, --max-limit is required"
SAMPLING_NEEDS_LEAN = "reference sampling mode needs the lean resident kernel"
BATCHED_NEEDS = "batched engine needs"
SOFT_ONLY = r"normalised soft scorers \(.*\): single template, single GPU only"
OVERFLOW = r"counter \d+, domain \d+: .* can leave int32"


@pytest.fixture(scope="module")
def sm_count(built):
    return helpers.device_sm_count()


# ---- workloads -----------------------------------------------------------------------------------------------------------------
def node_local(sm=None):
    return synth.c2(n=N, seed=11)


def prefer_classes(sm=None):
    return synth.c3(n=N, prefer_taints=True)


def extended(sm=None):
    return _extended(N)


def node_name(sm=None):
    snap, tmpl, ctr = synth.c2(n=N, seed=12, fit_only=False)
    tmpl[0].nodename_idx = 17
    return snap, tmpl, ctr


def two_taint_words(sm=None):
    snap, _ = _nodes(N, 13, taint_mask=np.zeros((2, N), np.uint64))
    return snap, [abi.default_template(150, 100 * MiB)], []


def c4_small(sm=None):
    return synth.c4(n=N, n_existing=2 * N, zones=8, racks=32, regions=4)


def c4_pod_affinity(sm=None):
    snap, tmpl, ctr = c4_small()
    tmpl[0].n_aff, tmpl[0].aff_counter[0] = 1, len(ctr)
    ctr.append(abi.make_counter(0, np.ones(8, np.int32), inc=1))
    return snap, tmpl, ctr


def c4_negative_inc(sm=None):
    snap, tmpl, ctr = c4_small()
    ctr[3] = abi.make_counter(-1, ctr[3]._keep, inc=-1)
    return snap, tmpl, ctr


def c4_wide_tile(sm):
    """Every CTA of the full grid holds 769 nodes: one more than a multi-commit tile (one node per thread)."""
    n = sm * 769
    return synth.c4(n=n, n_existing=2 * n, zones=8, racks=32, regions=4)


def soft(sm=None):
    return helpers.soft_cluster(31, n=N)


def soft_overflow(sm=None):
    """soft() with a zone count a few placements short of INT32_MAX."""
    snap, tmpl, ctr = soft()
    init = ctr[0]._keep.copy()
    init[0] = np.iinfo(np.int32).max - 5
    ctr[0] = abi.make_counter(0, init, inc=1, elig_bit=2)
    return snap, tmpl, ctr


def preferred_affinity(k, fit_off=False):
    """k templates with one preferred nodeAffinity term each: soft scorers without counters (the last one with NodeResourcesFit
    disabled if fit_off)."""
    snap, _, _ = synth.c2(n=N, seed=14, fit_only=False)
    tmpl = []
    for q in range(k):
        t = abi.default_template(150 + 50 * q, 100 * MiB)
        t.n_pref_terms, t.pref_weight[0] = 1, 10
        tmpl.append(t)
    if fit_off:
        tmpl[-1].filter_enable &= ~abi.PL_FIT
    return snap, tmpl, []


def several_templates(sm=None):
    return synth.c5(n=N, n_templates=4, seed=15)


def several_templates_masked(sm=None):
    """Several templates, none tolerating a NoSchedule taint that one node in ten carries: the mask columns matter."""
    snap, _ = _nodes(N, 16, taint_mask=(np.arange(N) % 10 == 0).astype(np.uint64).reshape(1, N), taint_nosched=[1])
    return snap, [abi.default_template(100 + 150 * k, (64 + 100 * k) * MiB) for k in range(3)], []


def fit_disabled(sm=None):
    snap, tmpl, ctr = node_local()
    tmpl[0].filter_enable &= ~abi.PL_FIT
    return snap, tmpl, ctr


# ---- the decision table ----------------------------------------------------------------------------------------------------------
class Refused(str):
    """An expected refusal: a regular expression the error message must match."""


def prepared(snap, tmpl, ctr, max_pods=0, **engine_kw):
    """prepare() on a fresh handle: the kernel it chose, or the refusal's message. A refused prepare must leave no kernel name and
    must not have launched anything."""
    with engine.Engine(device=0, **engine_kw) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        launches = eng.kernel_launches()
        try:
            eng.prepare(max_pods)
        except engine.EngineError as e:
            assert helpers.kernel_name(eng) == "", str(e)
            assert eng.kernel_launches() == launches, str(e)
            return Refused(str(e))
        return helpers.kernel_name(eng)


def sharded(snap, tmpl, ctr, max_pods=0, kind=AUTO, **engine_kw):
    """The kernel every rank of a two-rank node-sharded run chose, or the refusal's message (every rank refused alike, with the same
    state left behind as prepared() asserts)."""
    engs = helpers.sharded_engines(snap, tmpl, ctr, 2, kind, **engine_kw)
    try:
        got = []
        for e in engs:
            launches = e.kernel_launches()
            try:
                e.prepare(max_pods)
                got.append(helpers.kernel_name(e))
            except engine.EngineError as ex:
                assert helpers.kernel_name(e) == "" and e.kernel_launches() == launches, str(ex)
                got.append(Refused(str(ex)))
    finally:
        for e in engs:
            e.close()
    assert len(set(got)) == 1, got
    return got[0]


ROWS = [
    # id, workload, world, max_pods, engine options, expected kernel or Refused(message)
    ("node_local-auto", node_local, 1, 0, {}, "batched"),
    ("node_local-sequential", node_local, 1, 0, dict(engine=SEQ), "lean<false>"),
    ("node_local-batched", node_local, 1, 0, dict(engine=BATCHED), "batched"),
    ("prefer_classes-auto", prefer_classes, 1, 0, {}, "lean<false>"),
    ("prefer_classes-batched", prefer_classes, 1, 0, dict(engine=BATCHED), Refused(BATCHED_NEEDS)),
    ("sampling-auto", node_local, 1, 0, SAMPLING, "lean<true>"),
    ("sampling-sequential", node_local, 1, 0, dict(engine=SEQ, **SAMPLING), "lean<true>"),
    ("sampling-extended", extended, 1, 0, SAMPLING, Refused(SAMPLING_NEEDS_LEAN)),
    ("sampling-world2", node_local, 2, 0, SAMPLING, Refused(SAMPLING_NEEDS_LEAN)),
    ("generic-extended", extended, 1, 0, {}, "wave<true>"),
    ("generic-node_name", node_name, 1, 0, {}, "wave<true>"),
    ("generic-two_taint_words", two_taint_words, 1, 0, {}, "wave<true>"),
    ("counters-auto", c4_small, 1, 0, {}, "multi<false>"),
    ("counters-sequential", c4_small, 1, 0, dict(engine=SEQ), "lean<false>"),
    ("counters-world2-auto", c4_small, 2, 0, {}, "multi<true>"),
    ("counters-world2-sequential", c4_small, 2, 0, dict(kind=SEQ), "lean<false>"),
    ("counters-pod_affinity", c4_pod_affinity, 1, 0, {}, "lean<false>"),
    ("counters-negative_inc", c4_negative_inc, 1, 0, {}, "lean<false>"),
    ("counters-wide_tile", c4_wide_tile, 1, 0, {}, "lean<false>"),
    ("counters-batched", c4_small, 1, 0, dict(engine=BATCHED), Refused(BATCHED_NEEDS)),
    ("soft", soft, 1, 0, {}, "wave<true>"),
    ("soft-two_templates", lambda sm: preferred_affinity(2), 1, 0, {}, Refused(SOFT_ONLY)),
    ("soft-world2", soft, 2, 0, {}, Refused(SOFT_ONLY)),
    ("templates", several_templates, 1, 0, {}, "stream<2>"),
    ("templates-masks", several_templates_masked, 1, 0, {}, "stream<1>"),
    ("fit_disabled-unlimited", fit_disabled, 1, 0, {}, Refused(UNBOUNDED)),
    ("fit_disabled-limit", fit_disabled, 1, 5, {}, "batched"),
    # precedence: two refusals met at once, the first in the cascade wins
    ("first-unbounded-then-soft", lambda sm: preferred_affinity(2, fit_off=True), 1, 0, {}, Refused(UNBOUNDED)),
    ("first-overflow-then-soft", soft_overflow, 2, 0, {}, Refused(OVERFLOW)),
    ("first-soft-then-sampling", lambda sm: preferred_affinity(2), 1, 0, SAMPLING, Refused(SOFT_ONLY)),
    ("soft-one_template-sampling", lambda sm: preferred_affinity(1), 1, 0, SAMPLING, Refused(SAMPLING_NEEDS_LEAN)),
]


@pytest.mark.parametrize("make,world,max_pods,kw,want", [r[1:] for r in ROWS], ids=[r[0] for r in ROWS])
def test_kernel_choice(built, sm_count, make, world, max_pods, kw, want):
    got = (prepared if world == 1 else sharded)(*make(sm_count), max_pods=max_pods, **kw)
    print("\n  %s" % got, end="")
    if isinstance(want, Refused):
        assert isinstance(got, Refused) and re.search(want, got), got
    else:
        assert not isinstance(got, Refused) and got == want, got


def test_stream_all_forced(built, monkeypatch):
    monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    assert prepared(*several_templates()) == "stream<0>"


def test_state_refusals(built):
    """An empty cluster prepares without a kernel; prepare() before set_templates(), and a sharded handle before its peers are
    imported, are refused."""
    assert prepared(abi.Snapshot(0, np.zeros(0), np.zeros(0), np.zeros(0)), [abi.default_template(150, 100 * MiB)], []) == ""
    snap, tmpl, ctr = node_local()
    with engine.Engine(device=0) as eng:
        eng.load_nodes(snap)
        with pytest.raises(engine.EngineError, match="load_nodes and set_templates must come first"):
            eng.prepare(0)
        assert helpers.kernel_name(eng) == "" and eng.kernel_launches() == 0
    with engine.Engine(device=0, rank=0, world=2) as eng:
        eng.load_nodes(snap)
        eng.set_templates(tmpl, ctr)
        with pytest.raises(engine.EngineError, match="ccsim_peer_import must come first"):
            eng.prepare(0)
        assert helpers.kernel_name(eng) == "" and eng.kernel_launches() == 0


# ---- one tiny run per instantiation: engine code and block size ---------------------------------------------------------------------
GENERIC, LEAN, TIE_RUN, MULTI, STREAMING = engine.Engine.ENGINE_NAMES
RUNS = [
    # kernel, workload, world, engine options, CCSIM_STREAM_ALL, engine, block
    ("wave<true>", extended, 1, {}, False, GENERIC, 512),
    ("lean<false>", node_local, 1, dict(engine=SEQ), False, LEAN, 768),
    ("lean<true>", node_local, 1, SAMPLING, False, LEAN, 768),
    ("batched", node_local, 1, {}, False, TIE_RUN, 768),
    ("multi<false>", c4_small, 1, {}, False, MULTI, 768),
    ("multi<true>", c4_small, 2, {}, False, MULTI, 768),
    ("stream<0>", several_templates, 1, {}, True, STREAMING, 576),
    ("stream<1>", several_templates_masked, 1, {}, False, STREAMING, 576),
    ("stream<2>", several_templates, 1, {}, False, STREAMING, 576),
]


@pytest.mark.parametrize("kernel,make,world,kw,stream_all,want_engine,want_block", RUNS, ids=[r[0] for r in RUNS])
def test_run_stats_per_kernel(built, sm_count, monkeypatch, kernel, make, world, kw, stream_all, want_engine, want_block):
    if stream_all:
        monkeypatch.setenv("CCSIM_STREAM_ALL", "1")
    snap, tmpl, ctr = make(sm_count)
    if world == 1:
        with engine.Engine(device=0, **kw) as eng:
            eng.load_nodes(snap)
            eng.set_templates(tmpl, ctr)
            res = eng.run(50)
            stats = [eng.run_stats()]
        assert res.placed > 0
    else:
        (res, stats), = helpers.run_sharded(snap, tmpl, ctr, 50, world, AUTO, [50])
        assert all(r.placed > 0 for r in res)
    for st in stats:
        assert (st["kernel"], st["engine"], st["block"]) == (kernel, want_engine, want_block), st
