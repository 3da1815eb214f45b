"""ctypes binding of libccsim.so — the CUDA hot path behind include/ccsim.h.

There is NO CPU fallback: if the shared object is missing, or no CUDA device is visible, every entry point raises.
(The CPU oracle under oracle/ is test infrastructure and is never imported from here.)
"""
import ctypes as C
import os

import numpy as np

from . import _abi as abi

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("CCSIM_SO") or os.path.join(_HERE, "libccsim.so")   # CCSIM_SO: kernel-variant experiments only
_lib = None

EXPORTS = ["ccsim_create", "ccsim_destroy", "ccsim_last_error", "ccsim_abi_version", "ccsim_load_nodes",
           "ccsim_set_templates", "ccsim_run", "ccsim_prepare", "ccsim_node_counts", "ccsim_peer_export", "ccsim_peer_import",
           "ccsim_device_info", "ccsim_kernel_launches", "ccsim_kernel_name", "ccsim_flush_l2", "ccsim_run_stats", "ccsim_peer_local",
           "ccsim_peer_import_local", "ccsim_key_order_waves", "ccsim_sorted_tile_waves", "ccsim_run_each", "ccsim_set_analyses"]


class EngineError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise EngineError("libccsim.so not built (%s): run __graft_entry__.build(); there is no CPU fallback" % SO_PATH)
        L = C.CDLL(SO_PATH)
        L.ccsim_create.restype = C.c_int
        L.ccsim_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        L.ccsim_destroy.restype = None
        L.ccsim_destroy.argtypes = [C.c_void_p]
        L.ccsim_last_error.restype = C.c_char_p
        L.ccsim_last_error.argtypes = [C.c_void_p]
        L.ccsim_abi_version.restype = C.c_int
        L.ccsim_load_nodes.restype = C.c_int
        L.ccsim_load_nodes.argtypes = [C.c_void_p, C.POINTER(abi.Nodes)]
        L.ccsim_set_templates.restype = C.c_int
        L.ccsim_set_templates.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.Template), C.c_int32, C.POINTER(abi.Counter)]
        L.ccsim_set_analyses.restype = C.c_int
        L.ccsim_set_analyses.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.Template), C.POINTER(abi.AnalysisTerms)]
        L.ccsim_prepare.restype = C.c_int
        L.ccsim_prepare.argtypes = [C.c_void_p, C.c_int64]
        L.ccsim_run.restype = C.c_int
        L.ccsim_run.argtypes = [C.c_void_p, C.c_int64, C.POINTER(abi.Result)]
        L.ccsim_run_each.restype = C.c_int
        L.ccsim_run_each.argtypes = [C.c_void_p, C.c_int64, C.POINTER(abi.Result)]
        L.ccsim_node_counts.restype = C.c_int
        L.ccsim_node_counts.argtypes = [C.c_void_p, C.c_int32, abi.P32, abi.P64]
        L.ccsim_device_info.restype = C.c_int
        L.ccsim_device_info.argtypes = [C.c_void_p, abi.P32, abi.P32, abi.P32, abi.P64]
        L.ccsim_kernel_launches.restype = C.c_int64
        L.ccsim_kernel_launches.argtypes = [C.c_void_p]
        L.ccsim_kernel_name.restype = C.c_char_p
        L.ccsim_kernel_name.argtypes = [C.c_void_p]
        L.ccsim_flush_l2.restype = C.c_int
        L.ccsim_flush_l2.argtypes = [C.c_void_p]
        L.ccsim_peer_local.restype = C.c_int
        L.ccsim_peer_local.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.ccsim_peer_import_local.restype = C.c_int
        L.ccsim_peer_import_local.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.ccsim_run_stats.restype = C.c_int
        L.ccsim_run_stats.argtypes = [C.c_void_p, abi.P64]
        L.ccsim_key_order_waves.restype = C.c_int64
        L.ccsim_key_order_waves.argtypes = [C.c_void_p]
        L.ccsim_sorted_tile_waves.restype = C.c_int64
        L.ccsim_sorted_tile_waves.argtypes = [C.c_void_p]
        L.ccsim_peer_export.restype = C.c_int
        L.ccsim_peer_export.argtypes = [C.c_void_p, abi.PU8]
        L.ccsim_peer_import.restype = C.c_int
        L.ccsim_peer_import.argtypes = [C.c_void_p, C.c_int32, abi.PU8]
        _lib = L
    return _lib


class RunResult:
    def __init__(self, res):
        self.placed = int(res.placed)
        self.stop_code = int(res.stop_code)
        self.n_nodes = int(res.n_nodes)
        self.waves = int(res.waves)
        self.evals = int(res.evals)
        self.examined = int(res.examined)
        self.run_ms = float(res.run_ms)
        self.reason_hist = np.array(res.reason_hist[:], dtype=np.int64)
        self.preempt_no_victims = int(res.preempt_no_victims)
        self.preempt_not_helpful = int(res.preempt_not_helpful)
        if self.placed:
            self.pod_node = np.ctypeslib.as_array(res.pod_node, shape=(self.placed,)).copy()
        else:
            self.pod_node = np.zeros(0, np.int32)


class Engine:
    """One ccsim handle (one GPU / one node-axis shard)."""

    def __init__(self, device=0, engine=abi.ENGINE_AUTO, rank=0, world=1, sampling=abi.SAMPLING_CANONICAL, pct_nodes_to_score=0):
        cfg = abi.Config()
        cfg.abi_version = abi.ABI_VERSION
        cfg.device, cfg.engine, cfg.rank, cfg.world = device, engine, rank, world
        cfg.sampling, cfg.pct_nodes_to_score = sampling, pct_nodes_to_score
        self._h = C.c_void_p()
        rc = lib().ccsim_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise EngineError("ccsim_create rc=%d: %s" % (rc, lib().ccsim_last_error(None).decode()))
        self._keep = None

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s rc=%d: %s" % (what, rc, lib().ccsim_last_error(self._h).decode()))

    def load_nodes(self, snapshot):
        nd = snapshot.c_struct()
        self._check(lib().ccsim_load_nodes(self._h, C.byref(nd)), "ccsim_load_nodes")
        self._n = snapshot.n

    def set_templates(self, templates, counters=()):
        T = (abi.Template * len(templates))(*templates)
        Cn = (abi.Counter * max(1, len(counters)))(*counters)
        self._check(lib().ccsim_set_templates(self._h, len(templates), T, len(counters), Cn), "ccsim_set_templates")
        self._n_templates = len(templates)

    def set_analyses(self, templates, terms):
        """Templates for run_each() with every analysis's own terms (ccsim_set_analyses). terms[t] = (counters, topo columns):
        abi.Counter structs whose topo_col index the analysis's int32 numpy columns of n_nodes domain ids."""
        T = (abi.Template * len(templates))(*templates)
        A = (abi.AnalysisTerms * len(templates))()
        keep = []
        for t, (counters, cols) in enumerate(terms):
            Cn = (abi.Counter * max(1, len(counters)))(*counters)
            cols = [np.ascontiguousarray(c, dtype=np.int32) for c in cols]
            keep += [Cn, cols]
            A[t].n_counters, A[t].n_topo_cols, A[t].counters = len(counters), len(cols), Cn
            for k, c in enumerate(cols):
                A[t].topo[k] = c.ctypes.data_as(abi.P32)
        self._check(lib().ccsim_set_analyses(self._h, len(templates), T, A), "ccsim_set_analyses")
        self._n_templates = len(templates)

    def prepare(self, max_pods=0):
        """The allocation / restore half of run(max_pods); see ccsim_prepare."""
        self._check(lib().ccsim_prepare(self._h, max_pods), "ccsim_prepare")

    def run(self, max_pods=0):
        res = abi.Result()
        self._check(lib().ccsim_run(self._h, max_pods, C.byref(res)), "ccsim_run")
        return RunResult(res)

    def run_each(self, max_pods=0):
        """Every loaded template analysed on its own (ccsim_run_each): one RunResult per template, each what run() gives for a
        handle holding that template alone."""
        res = (abi.Result * self._n_templates)()
        self._check(lib().ccsim_run_each(self._h, max_pods, res), "ccsim_run_each")
        return [RunResult(r) for r in res]

    def connect_peers(self, dist):
        """Node-sharded multi-GPU run: all-gather the CUDA IPC handles of the exchange buffers over torch.distributed
        and map every peer's buffer (the per-wave exchange itself then happens inside the persistent kernel)."""
        import torch
        mine = np.zeros(64, np.uint8)
        self._check(lib().ccsim_peer_export(self._h, mine.ctypes.data_as(abi.PU8)), "ccsim_peer_export")
        world = dist.get_world_size()
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        t = torch.from_numpy(mine).to(dev)
        out = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        allh = np.concatenate([o.cpu().numpy() for o in out]).astype(np.uint8)
        self._check(lib().ccsim_peer_import(self._h, world, allh.ctypes.data_as(abi.PU8)), "ccsim_peer_import")

    @staticmethod
    def connect_local(engines):
        """All ranks live in this process (rank r = engines[r]): hand every engine the others' exchange-buffer pointers. The
        runs must then be started concurrently (one host thread per rank): the persistent kernels talk to each other."""
        ptrs = (C.c_void_p * len(engines))()
        for r, e in enumerate(engines):
            p = C.c_void_p()
            e._check(lib().ccsim_peer_local(e._h, C.byref(p)), "ccsim_peer_local")
            ptrs[r] = p
        for e in engines:
            e._check(lib().ccsim_peer_import_local(e._h, len(engines), ptrs), "ccsim_peer_import_local")

    def node_counts(self, t=0):
        counts = np.zeros(max(1, self._n), np.int32)
        first = np.zeros(max(1, self._n), np.int64)
        self._check(lib().ccsim_node_counts(self._h, t, counts.ctypes.data_as(abi.P32), first.ctypes.data_as(abi.P64)),
                    "ccsim_node_counts")
        return counts[: self._n], first[: self._n]

    def device_info(self):
        sm, grid, block, l2 = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
        lib().ccsim_device_info(self._h, C.byref(sm), C.byref(grid), C.byref(block), C.byref(l2))
        return dict(sm_count=sm.value, grid=grid.value, block=block.value, l2_bytes=l2.value)

    ENGINE_NAMES = ("generic", "lean sequential", "tie-run batching", "multi-commit", "streaming (TMA)")   # what ccsim_run may choose
    EACH_ENGINE = "per-analysis max-tree"                                                                # engine code 5: ccsim_run_each

    def run_stats(self):
        """Latency anatomy of the last run (see ccsim_run_stats in include/ccsim.h)."""
        v = np.zeros(16, np.int64)
        self._check(lib().ccsim_run_stats(self._h, v.ctypes.data_as(abi.P64)), "ccsim_run_stats")
        st = {"engine": self.ENGINE_NAMES[int(v[0])] if int(v[0]) < len(self.ENGINE_NAMES) else self.EACH_ENGINE, "kernel": self.kernel_name(), "waves": int(v[1]), "placed": int(v[2]),
              "candidates": int(v[3]), "bar_raised_waves": int(v[4]), "grid": int(v[5]), "block": int(v[6]), "smem_bytes": int(v[7]),
              "phase_cycles": [int(x) for x in v[8:16]]}
        if int(v[0]) == 5:      # per-analysis runs: where the upper levels of the max-trees live, rebuilds of all analyses, analyses per CTA
            st["global_levels"], st["shared_levels"], st["rebuilds"], st["per_cta"] = int(v[3]), int(v[4]), int(v[8]), int(v[9])
        return st

    def key_order_waves(self):
        """Waves of the last run the multi-commit kernel replayed in key order (see ccsim_key_order_waves in include/ccsim.h)."""
        return int(lib().ccsim_key_order_waves(self._h))

    def sorted_tile_waves(self):
        """Waves of the last run the multi-commit kernel selected each tile's candidates from the tile sorted by key (see
        ccsim_sorted_tile_waves in include/ccsim.h)."""
        return int(lib().ccsim_sorted_tile_waves(self._h))

    def kernel_launches(self):
        return int(lib().ccsim_kernel_launches(self._h))

    def kernel_name(self):
        """The wave-kernel instantiation the last prepare() / run() chose, e.g. "lean<true>" or "stream<0>" (see ccsim_kernel_name);
        "" before any, and for an empty cluster."""
        return lib().ccsim_kernel_name(self._h).decode()

    def flush_l2(self):
        self._check(lib().ccsim_flush_l2(self._h), "ccsim_flush_l2")

    def close(self):
        if self._h:
            lib().ccsim_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
