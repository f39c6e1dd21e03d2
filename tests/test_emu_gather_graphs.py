"""gccb_gather_graphs under the CPU emulator: both views of a whole-graph batch, bit-exact against
labeled.fill_whole_graphs (the host assembly of a whole-graph batch), on TU-style multigraphs with parallel edges,
self loops, an isolated vertex and seeds that are not vertex 0; and the capacity contract of the sampler (flag
raised, batch published empty) for node and edge overflow."""
import ctypes as C
import types

import numpy as np
import torch

from emu_util import NpBatch, lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets.graph_dataset import seed_first_union
from gcc_b200.datasets.labeled import _listed_csr, fill_whole_graphs

ARRAYS = ("node_off", "edge_off", "indptr", "indices", "sub_deg", "graph_id", "orig_id", "counters")


def _sym(pairs, n, name):
    """Every listed pair in both directions (a self loop once per listing), as a TU _A.txt lists them."""
    src, dst = [], []
    for u, v in pairs:
        src.append(u)
        dst.append(v)
        if u != v:
            src.append(v)
            dst.append(u)
    return _listed_csr(np.array(src, np.int64), np.array(dst, np.int64), n, name)


def _graphs():
    rng = np.random.RandomState(5)
    gs = [
        # hub on 3, a doubled pair (0, 1), a self loop on 2, vertex 5 isolated
        _sym([(3, 0), (3, 1), (3, 2), (3, 4), (0, 1), (0, 1), (2, 2)], 6, "g0"),
        _sym([(0, 1)], 2, "g1"),                                         # seed 0
        _sym([(1, 1), (1, 1), (0, 2)], 4, "g2"),                          # two self loops on 1, vertex 3 isolated
    ]
    for i in range(5):
        n = int(rng.randint(4, 12))
        pairs = [(j, (j + 1) % n) for j in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(n)]
        pairs += [pairs[1], pairs[1]]                                    # parallel edges
        gs.append(_sym(pairs, n, "r%d" % i))
    return gs


class _Set:
    def __init__(self, graphs):
        self.seeds, self.items, ip, ix, no, eo = seed_first_union(graphs)
        self.indptr, self.indices = ip.astype(np.int64), ix.astype(np.int32)
        self.node_off, self.edge_off = no, eo
        self.c = _capi.GraphSet(ptr(self.indptr), ptr(self.indices), ptr(self.node_off), ptr(self.edge_off),
                                len(graphs))


def _torch_view(b):
    """fill_whole_graphs writes through torch: CPU tensors sharing the NpBatch's memory."""
    t = types.SimpleNamespace(B=b.B, node_cap=b.node_cap, edge_cap=b.edge_cap, pos=torch.zeros(1))
    for k in ARRAYS:
        setattr(t, k, torch.from_numpy(getattr(b, k)))
    return t


def _gather(s, ids, node_cap, edge_cap):
    b = NpBatch(len(ids), node_cap, edge_cap)
    for k in ("indptr", "indices", "sub_deg", "graph_id", "orig_id"):
        getattr(b, k)[:] = -7                                            # untouched entries stay visible
    gids = np.asarray(ids, np.int64)
    assert lib().gccb_gather_graphs(C.byref(s.c), ptr(gids), C.byref(b.c), None) == 0
    return b


def _view_arrays(b, v):
    B = b.B
    N, E = int(b.node_off[v, B]), int(b.edge_off[v, B])
    return dict(node_off=b.node_off[v], edge_off=b.edge_off[v], indptr=b.indptr[v, :N + 1],
                indices=b.indices[v, :E], sub_deg=b.sub_deg[v, :N], graph_id=b.graph_id[v, :N],
                orig_id=b.orig_id[v, :N], counters=b.counters[v * B:(v + 1) * B])


def test_gather_graphs_matches_host_assembly():
    graphs = _graphs()
    s = _Set(graphs)
    assert s.seeds[0] == 3 and s.seeds[2] == 1                          # seeds that are not vertex 0
    ids = [0, 4, 2, 2, 7, 1, 5]                                          # out of order, one graph twice
    N = int(sum(np.diff(s.node_off)[ids]))
    E = int(sum(np.diff(s.edge_off)[ids]))
    got = _gather(s, ids, N, E)                                          # exactly full: no overflow
    assert got.flags[0] == 0
    for v in (0, 1):
        want = NpBatch(len(ids), N, E)
        fill_whole_graphs(_torch_view(want), [s.items[i] for i in ids], view=v)
        a, w = _view_arrays(got, v), _view_arrays(want, v)
        for k in ARRAYS:
            assert a[k].shape == w[k].shape and np.array_equal(a[k], w[k]), (v, k, a[k], w[k])
    # the doubled pair, the self loops and the isolated vertex survive
    g0 = got.indices[0, got.indptr[0, 0]:got.indptr[0, 6]]
    assert len(g0) == len(graphs[0].indices) == 13       # (4 hub edges + 2 parallel) x 2 + 1 self loop
    assert got.sub_deg[0, 5] == 0                                        # isolated vertex of graph 0


def test_gather_graphs_overflow_publishes_empty():
    s = _Set(_graphs())
    ids = [0, 3, 6]
    N = int(sum(np.diff(s.node_off)[ids]))
    E = int(sum(np.diff(s.edge_off)[ids]))
    for node_cap, edge_cap, flag in ((N - 1, E, _capi.FLAG_NODE_OVERFLOW), (N, E - 1, _capi.FLAG_EDGE_OVERFLOW)):
        b = _gather(s, ids, node_cap, edge_cap)
        assert b.flags[0] == flag
        for v in (0, 1):
            assert b.node_off[v, len(ids)] == -1 and b.edge_off[v, len(ids)] == -1
        for k in ("indptr", "indices", "sub_deg", "graph_id", "orig_id"):
            assert (getattr(b, k) == -7).all(), k                        # nothing filled
