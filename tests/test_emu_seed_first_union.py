"""gccb_seed_first_union under the CPU emulator: the whole-graph set relabelled seed first on the device equals
seed_first_union (the host relabel, one graph at a time) array for array -- indptr, indices and seeds -- on random
corpora with degree ties, seeds at the first and last vertex, parallel edges and self loops on the seed, isolated
vertices, one-vertex graphs and a corpus of one graph; a row that is not non-decreasing raises GCCB_FLAG_BAD_ROW and
is named by its graph."""
import ctypes as C

import numpy as np
import pytest

from emu_util import lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import first_bad_graph, seed_first_union
from gcc_b200.datasets.labeled import _listed_csr


def _graph(rng, n, m, name, extra=()):
    """m random directed entries (both directions listed, as TU files list them) plus `extra` pairs."""
    pairs = [tuple(rng.randint(0, n, 2)) for _ in range(m)] + list(extra)
    src = [u for u, v in pairs] + [v for u, v in pairs if u != v]
    dst = [v for u, v in pairs] + [u for u, v in pairs if u != v]
    return _listed_csr(np.array(src, np.int64), np.array(dst, np.int64), n, name)


def _union(graphs):
    """The raw union (no relabel) in the gccb_graph_set_t layout."""
    sizes = [g.num_nodes for g in graphs]
    u = synthetic.disjoint_union(graphs)
    node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    indptr = np.ascontiguousarray(u.indptr, np.int64)
    return indptr, np.ascontiguousarray(u.indices, np.int32), node_off, indptr[node_off].copy()


def _device(graphs):
    indptr, indices, node_off, edge_off = _union(graphs)
    G, V, E = len(graphs), len(indptr) - 1, len(indices)
    s = _capi.GraphSet(ptr(indptr), ptr(indices), ptr(node_off), ptr(edge_off), G)
    seeds = np.full(G, -5, np.int64)
    out_ip = np.full(V + 1, -5, np.int64)
    out_ix = np.full(max(E, 1), -5, np.int32)
    flags = np.zeros(1, np.int32)
    assert lib().gccb_seed_first_union(C.byref(s), V, E, ptr(seeds), ptr(out_ip), ptr(out_ix), ptr(flags),
                                       None) == 0
    return seeds, out_ip, out_ix[:E], int(flags[0])


def _check(graphs):
    seeds, ip, ix, flags = _device(graphs)
    w_seeds, _, w_ip, w_ix, _, _ = seed_first_union(graphs)
    assert flags == 0
    assert np.array_equal(seeds, w_seeds)
    assert np.array_equal(ip, w_ip)
    assert ip.dtype == np.int64 and np.array_equal(ix.astype(np.int64), w_ix)
    return seeds


def test_random_corpora_match_host_relabel():
    rng = np.random.RandomState(3)
    for trial in range(4):
        graphs = []
        for i in range(int(rng.randint(20, 60))):
            n = int(rng.randint(1, 40))
            graphs.append(_graph(rng, n, int(rng.randint(0, 3 * n)), "r%d_%d" % (trial, i)))
        _check(graphs)


def test_edge_cases():
    rng = np.random.RandomState(7)
    star = lambda n, hub: [(hub, v) for v in range(n) if v != hub]
    graphs = [
        _graph(rng, 1, 0, "single"),                                              # one vertex, no row
        _graph(rng, 1, 0, "loop", [(0, 0)]),                                      # one vertex with a self loop
        _graph(rng, 9, 0, "seed_first", star(9, 0)),                             # seed at vertex 0
        _graph(rng, 9, 0, "seed_last", star(9, 8)),                              # seed at the last vertex
        _graph(rng, 8, 0, "tie", [(2, 3), (2, 4), (5, 6), (5, 7)]),              # 2 and 5 tie: the first wins
        _graph(rng, 7, 0, "parallel", star(6, 4) + [(4, 1), (4, 1), (4, 4), (2, 4), (6, 4), (6, 4)]),
        _graph(rng, 12, 0, "isolated", [(3, 5), (5, 9)]),                        # isolated vertices, seed not 0
        _graph(rng, 6, 0, "empty_rows", []),                                     # every vertex isolated: seed 0
    ]
    seeds = _check(graphs)
    assert seeds.tolist()[:8] == [0, 0, 0, 8, 2, 4, 5, 0]
    # one graph holding the whole corpus, with parallel edges and a self loop on its seed
    _check([_graph(rng, 300, 900, "one", star(300, 137) + [(137, 137), (137, 12), (137, 12)])])


def test_unsorted_row_raises_flag_and_names_its_graph():
    rng = np.random.RandomState(11)
    graphs = [_graph(rng, 10, 20, "g%d" % i) for i in range(6)]
    indptr, indices, node_off, _ = _union(graphs)
    assert first_bad_graph(indptr, indices, node_off) is None
    # swap two entries of one row of graph 4 that differ
    r = next(r for r in range(node_off[4], node_off[5])
             if indptr[r + 1] - indptr[r] >= 2 and indices[indptr[r]] != indices[indptr[r + 1] - 1])
    bad = [g for g in graphs]
    ix = bad[4].indices.copy()
    a, b = indptr[r] - indptr[node_off[4]], indptr[r + 1] - 1 - indptr[node_off[4]]
    ix[a], ix[b] = ix[b], ix[a]
    bad[4] = synthetic.CSRGraph(bad[4].indptr, ix, bad[4].num_nodes, "bad")
    _, _, _, flags = _device(bad)
    assert flags == _capi.FLAG_BAD_ROW
    indptr, indices, node_off, _ = _union(bad)
    assert first_bad_graph(indptr, indices, node_off) == 4


def test_id_outside_its_graph_raises_flag():
    rng = np.random.RandomState(12)
    graphs = [_graph(rng, 8, 16, "g%d" % i) for i in range(3)]
    indptr, indices, node_off, edge_off = _union(graphs)
    indices = indices.copy()
    indices[edge_off[1]] = node_off[2]                         # a row of graph 1 names graph 2's first vertex
    s = _capi.GraphSet(ptr(indptr), ptr(indices), ptr(node_off), ptr(edge_off), 3)
    V, E = len(indptr) - 1, len(indices)
    seeds, ip, ix, flags = np.zeros(3, np.int64), np.zeros(V + 1, np.int64), np.zeros(E, np.int32), np.zeros(1, np.int32)
    assert lib().gccb_seed_first_union(C.byref(s), V, E, ptr(seeds), ptr(ip), ptr(ix), ptr(flags), None) == 0
    assert flags[0] == _capi.FLAG_BAD_ROW
    assert first_bad_graph(indptr, indices, node_off) == 1


@pytest.mark.parametrize("n_nodes", [-1, 2 ** 31 + 1])
def test_refused_arguments(n_nodes):
    s = _capi.GraphSet(None, None, None, None, 1)
    one = np.zeros(4, np.int64)
    assert lib().gccb_seed_first_union(C.byref(s), 1, 0, ptr(one), ptr(one), None, ptr(one), None) == \
        _capi.GCCB_ERR_BADARG
    indptr, node_off = np.zeros(2, np.int64), np.array([0, 1], np.int64)
    s = _capi.GraphSet(ptr(indptr), None, ptr(node_off), ptr(node_off), 1)
    assert lib().gccb_seed_first_union(C.byref(s), n_nodes, 0, ptr(one), ptr(one), None, ptr(one), None) == \
        _capi.GCCB_ERR_BADARG
