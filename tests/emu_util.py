"""Helpers for the CPU kernel-logic tests: load the EMULATED kernel library
(tests/emu, test infrastructure) and drive the C ABI with numpy buffers."""
import ctypes as C
import importlib.util
import os

import numpy as np

from gcc_b200 import _capi

HERE = os.path.dirname(os.path.abspath(__file__))
_libs = {}


def lib(production_hub_deg=False):
    """The emulated library.  production_hub_deg: the build with the product's hub threshold (GCCB_HUB_DEG = 256)
    instead of the tests' 3, for the warp gathers of rows with up to 256 neighbours."""
    if production_hub_deg not in _libs:
        spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        path = mod.build(hub_deg=None) if production_hub_deg else mod.build()
        _libs[production_hub_deg] = _capi.bind(C.CDLL(path), require_all=False)
    return _libs[production_hub_deg]


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class NpBatch:
    """Host-memory mirror of gccb_batch_t for the emulator."""

    def __init__(self, B, node_cap, edge_cap):
        self.B, self.node_cap, self.edge_cap = B, node_cap, edge_cap
        self.node_off = np.zeros((2, B + 1), np.int32)
        self.edge_off = np.zeros((2, B + 1), np.int32)
        self.indptr = np.zeros((2, node_cap + 1), np.int32)
        self.indices = np.zeros((2, edge_cap), np.int32)
        self.sub_deg = np.zeros((2, node_cap), np.int32)
        self.graph_id = np.zeros((2, node_cap), np.int32)
        self.orig_id = np.zeros((2, node_cap), np.int32)
        self.counters = np.zeros((2 * B, 4), np.int64)
        self.flags = np.zeros(1, np.int32)
        self.c = _capi.Batch(B, node_cap, edge_cap, 0, ptr(self.node_off), ptr(self.edge_off),
                             ptr(self.indptr), ptr(self.indices), ptr(self.sub_deg),
                             ptr(self.graph_id), ptr(self.orig_id), ptr(self.counters),
                             ptr(self.flags))

    @classmethod
    def from_subgraphs(cls, views, node_cap=None, edge_cap=None):
        """views: [list of B dicts(subv, indptr, indices, n, m)] x 2 (oracle output)."""
        B = len(views[0])
        N = max(sum(s["n"] for s in v) for v in views)
        E = max(sum(s["m"] for s in v) for v in views)
        b = cls(B, node_cap or N + 3, edge_cap or E + 5)
        for v, subs in enumerate(views):
            noff = eoff = 0
            for g, s in enumerate(subs):
                n, m = s["n"], s["m"]
                b.node_off[v, g], b.edge_off[v, g] = noff, eoff
                b.indptr[v, noff:noff + n] = eoff + s["indptr"][:n]
                b.indices[v, eoff:eoff + m] = noff + s["indices"]
                b.sub_deg[v, noff:noff + n] = np.diff(s["indptr"])
                b.graph_id[v, noff:noff + n] = g
                b.orig_id[v, noff:noff + n] = s["subv"]
                b.counters[v * B + g, :2] = (n, m)
                noff += n
                eoff += m
            b.node_off[v, B], b.edge_off[v, B] = noff, eoff
            b.indptr[v, noff] = eoff
        return b

    def view_graphs(self, v):
        """Split view v back into per-graph dicts (local ids)."""
        out = []
        for g in range(self.B):
            a, z = self.node_off[v, g], self.node_off[v, g + 1]
            ip = self.indptr[v, a:z + 1].copy()
            idx = self.indices[v, ip[0]:ip[-1]] - a
            out.append(dict(subv=self.orig_id[v, a:z].copy(), indptr=ip - ip[0], indices=idx,
                            n=z - a, m=len(idx)))
        return out


class NpGraph:
    def __init__(self, g, rw_hops, restart_prob, key):
        from oracle import rwr as orwr   # tests only
        self.indptr = np.ascontiguousarray(g.indptr, np.int64)
        self.indices = np.ascontiguousarray(g.indices, np.int32)
        self.btable = orwr.budget_table(int(np.diff(g.indptr).max()), rw_hops, restart_prob)
        self.rt = orwr.restart_threshold(restart_prob)
        self.key = key
        self.cdf = orwr.seed_cdf(g.indptr)
        self.c = _capi.Graph(ptr(self.indptr), ptr(self.indices), g.num_nodes, ptr(self.btable),
                             len(self.btable), int(self.btable.max()), self.rt, 0, key)
