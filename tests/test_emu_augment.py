"""CPU: the step_dist key seeds and the neighbour-sampled ego-nets (gcc_b200/csrc/sampler.cu: gccb_pair_seeds,
gccb_sample_batch_pairs, gccb_ns_batch) under the fiber emulator, against tests/augment_oracle.py integer for
integer; the step and endpoint distributions against closed forms; the dataset refusals."""
import ctypes as C

import numpy as np
import pytest
from scipy.stats import chi2

import augment_oracle as ao
import emu_util
from emu_util import NpBatch, NpGraph, ptr
from gcc_b200.datasets import downstream, synthetic
from oracle import rwr as orwr

CHI2_P = 1e-6          # the draws are fixed by the key: a bound this loose only guards against a wrong distribution


def _csr(n, edges, name="g"):
    """Directed CSR of (src, dst) pairs, rows sorted (the gccb_graph_t contract)."""
    e = np.array(sorted(edges), dtype=np.int64).reshape(-1, 2)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(e[:, 0], minlength=n))]).astype(np.int64)
    return synthetic.CSRGraph(indptr, e[:, 1].astype(np.int32), n, name)


def _undirected(n, pairs, name="g"):
    return _csr(n, [(a, b) for a, b in pairs] + [(b, a) for a, b in pairs], name)


def _multigraph(seed=3, n=60, hubs=2):
    """Hubs joined to every other vertex by 1..3 parallel edges, random edges of multiplicity 1..2, self loops."""
    rng = np.random.RandomState(seed)
    src, dst = [], []

    def add(a, b, t):
        src.extend([a] * t)
        dst.extend([b] * t)
    for h in range(hubs):
        for v in range(hubs, n):
            add(h, v, int(rng.randint(1, 4)))
    for a, b in rng.randint(hubs, n, size=(80, 2)):
        if a != b:
            add(int(a), int(b), int(rng.randint(1, 3)))
    add(0, 0, 1)
    add(hubs + 1, hubs + 1, 2)
    return downstream.multigraph_from_edge_index(np.array([src, dst]), "multigraph")


def _pair_seeds(L, g, key, seeds_q, sids, step_dist):
    G = NpGraph(g, 16, 0.8, key)
    cdf = ao.step_cdf(step_dist)
    seeds_q = np.ascontiguousarray(seeds_q, np.int64)
    sids = np.ascontiguousarray(sids, np.int64)
    out = np.full(len(seeds_q), -7, np.int64)
    rc = L.gccb_pair_seeds(C.byref(G.c), cdf.ctypes.data, len(cdf), ptr(seeds_q), ptr(sids), len(seeds_q), ptr(out),
                           None)
    assert rc == 0, L.gccb_last_error()
    return out


# ---- key seeds ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("step_dist", [[0.2, 0.3, 0.5], [0.4, 0.6], [1.0]])
def test_pair_seeds_match_oracle(step_dist):
    # vertex 5 has no neighbours: 4 -> 5 is a dead end for the second hop
    g = _csr(7, [(0, 1), (0, 2), (1, 0), (1, 2), (1, 4), (2, 0), (2, 3), (3, 2), (3, 4), (4, 5), (4, 3), (6, 4)])
    L = emu_util.lib()
    key = 0xA11CE
    B = 600
    seeds_q = np.arange(B) % 7
    seeds_q[seeds_q == 5] = 4
    sids = np.arange(1000, 1000 + B)
    got = _pair_seeds(L, g, key, seeds_q, sids, step_dist)
    cdf = ao.step_cdf(step_dist)
    want = [ao.pair_seed(g.indptr, g.indices, key, int(s), int(q), cdf) for s, q in zip(sids, seeds_q)]
    assert got.tolist() == [w[1] for w in want]
    steps = {w[0] for w in want}
    assert steps == set(range(len(step_dist)))                  # every step is taken
    dead = [i for i, (w, q) in enumerate(zip(want, seeds_q)) if w[0] == 2 and w[1] == 5]
    assert dead or len(step_dist) < 3                           # the walk stopped at the dead end
    if len(step_dist) == 1:
        assert np.array_equal(got, seeds_q)


def test_pair_seeds_reuse_of_a_hop_draw_fails():
    """The 2-hop oracle with hop 2 drawing hop 1's word disagrees with the kernel."""
    g = _undirected(20, [(i, i + 1) for i in range(19)], "path")
    L = emu_util.lib()
    key, B = 77, 300
    seeds_q, sids = np.full(B, 10), np.arange(B)
    got = _pair_seeds(L, g, key, seeds_q, sids, [0.0, 0.0, 1.0])

    def reused(s):
        cur = 10
        for _ in (1, 2):
            w = orwr._philox_at(key, s, 0, 1, 0, ao.TAG_KHOP)
            beg, deg = int(g.indptr[cur]), int(g.indptr[cur + 1] - g.indptr[cur])
            cur = int(g.indices[beg + ((w[1] * deg) >> 32)])
        return cur
    assert got.tolist() != [reused(int(s)) for s in sids]


def test_step_frequencies_match_step_dist():
    """On a directed 3-cycle the k seed is q + step (mod 3): the step counts of 10^5 samples against step_dist."""
    g = _csr(3, [(0, 1), (1, 2), (2, 0)], "cycle")
    L = emu_util.lib()
    N = 100000
    p = np.array([0.5, 0.3, 0.2])
    got = _pair_seeds(L, g, 0xC0FFEE, np.zeros(N, np.int64), np.arange(N), p)
    counts = np.bincount(got, minlength=3)
    stat = float(((counts - N * p) ** 2 / (N * p)).sum())
    assert stat < chi2.isf(CHI2_P, 2), (counts, stat)


def _chi2_ok(got, probs):
    N = len(got)
    keys = sorted(probs)
    counts = np.array([(got == k).sum() for k in keys])
    assert counts.sum() == N, "an endpoint outside the closed form's support"
    exp = N * np.array([probs[k] for k in keys])
    stat = float(((counts - exp) ** 2 / exp).sum())
    return stat < chi2.isf(CHI2_P, max(len(keys) - 1, 1))


def test_endpoint_distributions_path_and_star():
    L = emu_util.lib()
    N = 20000
    path = _undirected(21, [(i, i + 1) for i in range(20)], "path")
    one = _pair_seeds(L, path, 5, np.full(N, 10), np.arange(N), [0.0, 1.0])
    two = _pair_seeds(L, path, 5, np.full(N, 10), np.arange(N), [0.0, 0.0, 1.0])
    assert _chi2_ok(one, {9: 0.5, 11: 0.5})
    assert _chi2_ok(two, {8: 0.25, 10: 0.5, 12: 0.25})
    leaves = 12
    star = _undirected(leaves + 1, [(0, i) for i in range(1, leaves + 1)], "star")
    from_leaf = _pair_seeds(L, star, 9, np.full(N, 3), np.arange(N), [0.0, 0.0, 1.0])
    from_center = _pair_seeds(L, star, 9, np.zeros(N, np.int64), np.arange(N), [0.0, 1.0])
    assert _chi2_ok(from_leaf, {i: 1.0 / leaves for i in range(1, leaves + 1)})
    assert _chi2_ok(from_center, {i: 1.0 / leaves for i in range(1, leaves + 1)})
    assert np.all(_pair_seeds(L, star, 9, np.zeros(100, np.int64), np.arange(100), [0.0, 0.0, 1.0]) == 0)


# ---- RWR with separate view seeds ------------------------------------------------------------------------------
def _check_views(b, views, B):
    for v in (0, 1):
        assert b.node_off[v, B] == sum(s["n"] for s in views[v])
        assert b.edge_off[v, B] == sum(s["m"] for s in views[v])
        for gi, (a, w) in enumerate(zip(b.view_graphs(v), views[v])):
            assert np.array_equal(a["subv"], w["subv"]), (v, gi)
            assert np.array_equal(a["indptr"], w["indptr"]), (v, gi)
            assert np.array_equal(a["indices"], w["indices"]), (v, gi)
            c = b.counters[v * B + gi]
            assert (c[0], c[1], c[3]) == (w["n"], w["m"], w["sumdeg"]), (v, gi)
        n = b.node_off[v, B]
        assert np.array_equal(b.sub_deg[v, :n], np.diff(b.indptr[v, :n + 1]))


def test_paired_rwr_matches_oracle_on_a_multigraph():
    g = _multigraph()
    L = emu_util.lib()
    key, B, hops = 0x5EED, 6, 12
    G = NpGraph(g, hops, 0.8, key)
    seeds_q, sids = np.zeros(B, np.int64), np.zeros(B, np.int64)
    assert L.gccb_draw_seeds(ptr(G.cdf), g.num_nodes, key, 0, B, ptr(seeds_q), ptr(sids), None) == 0
    seeds_q[:2] = [0, 1]                                        # hubs: budgets far above their neighbours'
    seeds_k = _pair_seeds(L, g, key, seeds_q, sids, [0.0, 1.0])
    want = ao.pairs_batch(G.indptr, G.indices, key, sids, seeds_q, seeds_k, G.btable, G.rt)
    for s in want[0]:
        assert s["traces"] > 0
    N = max(sum(s["n"] for s in v) for v in want)
    E = max(sum(s["m"] for s in v) for v in want)
    b = NpBatch(B, N + 7, E + 11)
    ws = np.zeros(L.gccb_sample_batch_workspace(B, int(G.btable.max()), b.edge_cap), np.uint8)
    rc = L.gccb_sample_batch_pairs(C.byref(G.c), ptr(seeds_q), ptr(seeds_k), ptr(sids), C.byref(b.c), ptr(ws),
                                   ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    assert b.flags[0] == 0
    _check_views(b, want, B)
    for gi in range(B):                                         # the k view's row 0 is its own seed
        assert b.orig_id[1, b.node_off[1, gi]] == seeds_k[gi]
        assert b.counters[B + gi, 2] == want[1][gi]["steps"]
    # the k view's budget is the q seed's: the k seed's own budget gives other walks
    deg = np.diff(G.indptr)
    own = [orwr.rwr_subgraph(G.indptr, G.indices, key, int(s), 1, int(k), int(G.btable[deg[k]]), G.rt)
           for s, k in zip(sids, seeds_k)]
    assert any(o["steps"] != w["steps"] or not np.array_equal(o["subv"], w["subv"]) for o, w in zip(own, want[1]))


# ---- neighbour sampling ----------------------------------------------------------------------------------------
def _ns(L, g, key, seeds_q, seeds_k, hops, k, node_cap=None, edge_cap=None, want=None):
    B = len(seeds_q)
    sids = np.arange(100, 100 + B, dtype=np.int64)
    seeds_q = np.ascontiguousarray(seeds_q, np.int64)
    seeds_k = np.ascontiguousarray(seeds_k, np.int64)
    G = NpGraph(g, 8, 0.8, key)
    if want is None:
        want = ao.ns_batch(G.indptr, G.indices, key, sids, seeds_q, seeds_k, hops, k)
    N = max(sum(s["n"] for s in v) for v in want)
    E = max(sum(s["m"] for s in v) for v in want)
    b = NpBatch(B, node_cap or N + 5, edge_cap or E + 9)
    ws = np.zeros(L.gccb_ns_batch_workspace(B, k, b.edge_cap), np.uint8)
    rc = L.gccb_ns_batch(C.byref(G.c), ptr(seeds_q), ptr(seeds_k), ptr(sids), hops, k, C.byref(b.c), ptr(ws),
                         ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return b, want, sids


def test_ns_whole_neighbourhood_when_degree_is_small():
    g = _undirected(30, [(i, (i + 1) % 30) for i in range(30)] + [(i, (i + 7) % 30) for i in range(0, 30, 3)], "ring")
    L = emu_util.lib()
    b, want, _ = _ns(L, g, 1, [0, 4, 9], [2, 4, 20], 3, 5)
    assert b.flags[0] == 0
    _check_views(b, want, 3)
    # deg <= k everywhere: layer h is the h-ball
    ball = {0}
    for _ in range(3):
        ball |= {int(u) for v in ball for u in g.indices[g.indptr[v]:g.indptr[v + 1]]}
    assert set(want[0][0]["subv"].tolist()) == ball


def test_ns_hubs_and_parallel_edges_match_oracle():
    g = _multigraph(n=80)
    L = emu_util.lib()
    k = 3
    seeds_q, seeds_k = [0, 5, 17, 40], [1, 5, 30, 2]
    b, want, sids = _ns(L, g, 0xBEEF, seeds_q, seeds_k, 2, k)
    assert b.flags[0] == 0
    _check_views(b, want, 4)
    # a hub seed's first layer: exactly k distinct entries, so at most k vertices (parallel edges collapse)
    deg = np.diff(g.indptr)
    assert deg[0] > k and len(ao.ns_nodes(g.indptr, g.indices, 0xBEEF, int(sids[0]), 0, 0, 1, k)) <= k + 1
    # sampling WITH replacement, or one Philox stream for every hop, gives other node sets
    floyd, philox = ao._floyd, ao.philox_np
    try:
        ao._floyd = lambda words, d, kk: [(int(w) * d) >> 32 for w in words[:kk]]
        repl = ao.ns_batch(g.indptr, g.indices, 0xBEEF, sids, seeds_q, seeds_k, 2, k)
        ao._floyd = floyd
        ao.philox_np = lambda c0, c1, c2, c3, key: philox(c0, c1, c2, (np.asarray(c3, dtype=np.uint64) & ~np.uint64(0xFF)) | np.uint64(1), key)
        same_tag = ao.ns_batch(g.indptr, g.indices, 0xBEEF, sids, seeds_q, seeds_k, 2, k)
    finally:
        ao._floyd, ao.philox_np = floyd, philox
    for bad in (repl, same_tag):
        assert any(not np.array_equal(x["subv"], y["subv"]) for v in (0, 1) for x, y in zip(bad[v], want[v]))


def test_ns_early_stop_gives_the_full_loop():
    """rw_hops = 50 on a 9-vertex component with a hub: the kernel stops once the union is closed; the oracle runs
    all 50 layers."""
    small = [(0, i) for i in range(1, 9)] + [(i, i + 1) for i in range(1, 8)]
    big = [(i, i + 1) for i in range(9, 59)]
    g = _undirected(60, small + big, "two_components")
    L = emu_util.lib()
    b, want, _ = _ns(L, g, 42, [0, 3], [5, 8], 50, 2)
    assert b.flags[0] == 0
    _check_views(b, want, 2)
    assert all(s["n"] == 9 for v in want for s in v)
    assert all(b.counters[s, 2] < 50 for s in range(4))           # stopped early


def test_ns_a_layer_adding_nothing_new_does_not_stop_the_loop():
    """From the centre of a 40-leaf star with k = 2: layer 1 draws two leaves, layer 2 is the centre alone (nothing
    new), layer 3 draws two leaves afresh.  Stopping at layer 2 would keep 3 vertices."""
    star = _undirected(41, [(0, i) for i in range(1, 41)], "star")
    L = emu_util.lib()
    b, want, _ = _ns(L, star, 8, [0, 0, 0], [0, 0, 0], 5, 2)
    assert b.flags[0] == 0
    _check_views(b, want, 3)
    assert all(s["n"] > 3 for v in want for s in v)
    # layer 2 of every view adds nothing: its union after 2 layers equals the one after 1 layer
    for v in (0, 1):
        for i, sid in enumerate(range(100, 103)):
            assert ao.ns_nodes(star.indptr, star.indices, 8, sid, v, 0, 2, 2) == \
                ao.ns_nodes(star.indptr, star.indices, 8, sid, v, 0, 1, 2)


def test_ns_overflow_publishes_the_view_empty():
    star = _undirected(201, [(0, i) for i in range(1, 201)], "star")
    L = emu_util.lib()
    # views over node_cap: every ego-net here has at least 2 vertices
    b, want, _ = _ns(L, star, 3, [1, 2, 0], [1, 2, 3], 2, 5, node_cap=5)
    assert min(s["n"] for v in want for s in v) >= 2
    assert b.flags[0] & 1 and (b.node_off[:, 3] == -1).all() and (b.edge_off[:, 3] == -1).all()
    # one ego-net over the kernel's per-ego-net limit (64 vertices at num_neighbors = 300)
    assert L.gccb_ns_ego_cap(300) == 64
    want = [[dict(n=1, m=0)] * 2, [dict(n=1, m=0)] * 2]
    b, _, _ = _ns(L, star, 3, [0, 5], [5, 5], 1, 300, node_cap=500, edge_cap=500, want=want)
    assert b.flags[0] & 1 and b.node_off[0, 2] == -1
    assert b.node_off[1, 2] == 4                                # view 1: two leaves and the centre each


def test_ns_overflow_at_the_largest_node_cap():
    """256 ego-nets over the per-ego-net cap in one view, each counted node_cap + 1 vertices: at the largest node_cap
    gccb_ns_batch takes, batch_offsets_kernel's int scan over 256 samples must not wrap, and the view is published
    empty.  One more is refused."""
    from gcc_b200.datasets.graph_dataset import NS_NODE_CAP_MAX
    star = _undirected(201, [(0, i) for i in range(1, 201)], "star")
    L = emu_util.lib()
    B, k = 256, 300                                             # cap 64: the centre's first layer (200) overflows
    G = NpGraph(star, 8, 0.8, 5)
    seeds, sids = np.zeros(B, np.int64), np.arange(B, dtype=np.int64)
    b = NpBatch(B, NS_NODE_CAP_MAX, 64)
    assert 256 * (b.node_cap + 1) < 2 ** 31 <= 256 * (b.node_cap + 2)
    ws = np.zeros(L.gccb_ns_batch_workspace(B, k, b.edge_cap), np.uint8)
    args = (C.byref(G.c), ptr(seeds), ptr(seeds), ptr(sids), 1, k)
    rc = L.gccb_ns_batch(*args, C.byref(b.c), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    assert b.flags[0] & 1
    assert (b.node_off[:, B] == -1).all() and (b.edge_off[:, B] == -1).all()
    assert (b.counters[:, 0] == NS_NODE_CAP_MAX + 1).all()
    b.c.node_cap = NS_NODE_CAP_MAX + 1
    assert L.gccb_ns_batch(*args, C.byref(b.c), ptr(ws), ws.nbytes, None) == -2      # GCCB_ERR_CAPACITY


# ---- dataset refusals (before any device is touched) -----------------------------------------------------------
def test_refusals():
    from gcc_b200.datasets.graph_dataset import GraphClassificationDataset, LoadBalanceGraphDataset
    g = _undirected(4, [(0, 1), (1, 2), (2, 3)])
    with pytest.raises(NotImplementedError, match="graph_transform"):
        LoadBalanceGraphDataset(dgl_graphs_file=g, graph_transform=lambda x: x)
    with pytest.raises(NotImplementedError, match="other"):
        LoadBalanceGraphDataset(dgl_graphs_file=g, aug="other")
    with pytest.raises(ValueError):
        LoadBalanceGraphDataset(dgl_graphs_file=g, aug="ns", num_neighbors=0)
    with pytest.raises(ValueError):
        LoadBalanceGraphDataset(dgl_graphs_file=g, step_dist=[0.25, 0.25, 0.25, 0.25])
    with pytest.raises(NotImplementedError, match="step_dist"):
        GraphClassificationDataset([g, g], step_dist=[0.5, 0.5, 0.0])
