"""CPU: the sampler's wide path (gcc_b200/csrc/sampler.cu: rwr_walk_wide_kernel, induce_fill_wide_kernel) under the
fiber emulator, compared bit-for-bit with the oracle.  The emulator library is built with a walk CTA trace of
GCCB_WALK_KEYS = 1024 ints instead of the product's 32,768, so that a seed of degree >= 486 under the plain-degree
budget table (budget > 960) is a wide ego-net and these graphs stay small."""
import ctypes as C
import glob
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from emu_util import NpBatch, lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import budget_for_degree
from oracle import rwr as orwr

HERE = os.path.dirname(os.path.abspath(__file__))
WALK_KEYS = 1024
BUDGET_MAX = WALK_KEYS - 64
HOPS, RESTART = 16, 0.8
_lib = []


def wide_lib():
    """The emulated library of tests/emu/build_emu.py (its sources, flags and test hub threshold) compiled with
    -DGCCB_WALK_KEYS=WALK_KEYS, in a directory of its own under that script's build directory."""
    if not _lib:
        spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
        emu = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(emu)
        out = os.path.join(emu.OUT, "walk_keys_%d" % WALK_KEYS)
        path = os.path.join(out, "libgccb200_emu.so")
        defs = ["-DGCCB_EMU", "-DGCCB_HUB_DEG=%d" % emu.HUB_DEG_TESTS, "-DGCCB_WALK_KEYS=%d" % WALK_KEYS]
        os.makedirs(out, exist_ok=True)
        hdrs = glob.glob(os.path.join(emu.CSRC, "*.cuh")) + \
            [os.path.join(emu.HERE, "cuda_emu.h"), os.path.join(emu.ROOT, "include", "gccb200.h")]
        objs, relink = [], not os.path.exists(path)
        for src in emu.sources():
            obj = os.path.join(out, os.path.basename(src) + ".o")
            if not os.path.exists(obj) or any(os.path.getmtime(obj) < os.path.getmtime(d) for d in [src] + hdrs):
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC"] + defs +
                                      ["-I", emu.HERE, "-x", "c++", "-c", src, "-o", obj])
                relink = True
            objs.append(obj)
        if relink:
            subprocess.check_call(["g++", "-shared", "-o", path] + objs)
        _lib.append(_capi.bind(C.CDLL(path), require_all=False))
    return _lib[0]


class PlainGraph:
    """gccb_graph_t with the plain-degree budget table of generate.py / --finetune (graph_dataset.py:243-254)."""

    def __init__(self, g, key):
        self.indptr = np.ascontiguousarray(g.indptr, np.int64)
        self.indices = np.ascontiguousarray(g.indices, np.int32)
        self.deg = np.diff(self.indptr)
        self.btable = np.array([budget_for_degree(d, HOPS, RESTART, 1.0) for d in range(int(self.deg.max()) + 1)],
                               np.int32)
        self.rt = orwr.restart_threshold(RESTART)
        self.key = key
        self.c = _capi.Graph(ptr(self.indptr), ptr(self.indices), g.num_nodes, ptr(self.btable), len(self.btable),
                             int(self.btable.max()), self.rt, 0, key)

    def budget(self, v):
        return int(self.btable[self.deg[v]])


def _run(g, seeds_q, seeds_k=None, key=0x5EED, first=0, node_cap=None, edge_cap=None):
    """Both views of B samples with the given seeds through gccb_sample_batch (seeds_k None) or
    gccb_sample_batch_pairs; returns (batch, oracle views [2][B], graph)."""
    L = wide_lib()
    G = PlainGraph(g, key)
    seeds_q = np.asarray(seeds_q, np.int64)
    seeds_k = seeds_q if seeds_k is None else np.asarray(seeds_k, np.int64)
    B = len(seeds_q)
    sids = np.arange(first, first + B, dtype=np.int64)
    views = [[orwr.rwr_subgraph(G.indptr, G.indices, key, int(sids[i]), v, int((seeds_q, seeds_k)[v][i]),
                                G.budget(seeds_q[i]), G.rt) for i in range(B)] for v in (0, 1)]
    N = max(sum(s["n"] for s in v) for v in views)
    E = max(sum(s["m"] for s in v) for v in views)
    b = NpBatch(B, node_cap or N + 7, edge_cap or E + 11)
    ws = np.zeros(L.gccb_sample_batch_workspace(B, int(G.btable.max()), b.edge_cap), np.uint8)
    if seeds_k is seeds_q:
        rc = L.gccb_sample_batch(C.byref(G.c), ptr(seeds_q), ptr(sids), C.byref(b.c), ptr(ws), ws.nbytes, None)
    else:
        rc = L.gccb_sample_batch_pairs(C.byref(G.c), ptr(seeds_q), ptr(seeds_k), ptr(sids), C.byref(b.c), ptr(ws),
                                       ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return b, views, G


def _check(b, views, vlist=(0, 1)):
    B = b.B
    for v in vlist:
        got = b.view_graphs(v)
        assert b.node_off[v, B] == sum(s["n"] for s in views[v])
        assert b.edge_off[v, B] == sum(s["m"] for s in views[v])
        for gi, (a, w) in enumerate(zip(got, views[v])):
            assert np.array_equal(a["subv"], w["subv"]), (v, gi)
            assert np.array_equal(a["indptr"], w["indptr"]), (v, gi)
            assert np.array_equal(a["indices"], w["indices"]), (v, gi)
            c = b.counters[v * B + gi]
            assert (c[0], c[1], c[2], c[3]) == (w["n"], w["m"], w["steps"], w["sumdeg"]), (v, gi)
        n = b.node_off[v, B]
        assert np.array_equal(b.sub_deg[v, :n], np.diff(b.indptr[v, :n + 1]))
        assert np.array_equal(b.graph_id[v, :n], np.repeat(np.arange(B), np.diff(b.node_off[v])))


def _three_centres(leaves):
    src = np.repeat(np.arange(3), leaves)
    dst = 3 + np.tile(np.arange(leaves), 3)
    return synthetic.from_pairs(src, dst, leaves + 3, "k3_%d" % leaves)


def _hub_beside_centre(leaves=500, hub_leaves=20000):
    """Centre 0 with `leaves` leaves and a neighbour 1 (the hub) of hub_leaves further leaves: the centre's ego-net
    is wide and holds the hub, whose row (degree > 16 n) is induced by the reverse probe."""
    src = np.concatenate([np.zeros(leaves + 1, np.int64), np.ones(hub_leaves, np.int64)])
    dst = np.concatenate([np.arange(1, leaves + 2), leaves + 2 + np.arange(hub_leaves)])
    return synthetic.from_pairs(src, dst, leaves + 2 + hub_leaves, "hub_beside_centre")


def test_library_walks_wide_above_the_lowered_limit():
    """The workspace of wide_lib() takes the wide formula above BUDGET_MAX: its batches below do run the wide path."""
    L = wide_lib()
    cap = lambda mb: (mb + 64 + 1 + 3) & ~3
    assert L.gccb_sample_batch_workspace(2, BUDGET_MAX, 100) == (3 * 4 * cap(BUDGET_MAX) + 16 + 200) * 4
    assert L.gccb_sample_batch_workspace(2, BUDGET_MAX + 1, 100) == \
        (3 * 4 * cap(BUDGET_MAX) + 16 + 200 + 6 * 102 + 4 * WALK_KEYS * 2) * 4


def test_star_centre_is_wide_and_matches_oracle():
    g = synthetic.star_graph(1000)
    b, views, G = _run(g, [0, 0])
    assert G.budget(0) > BUDGET_MAX
    assert b.flags[0] == 0
    _check(b, views)


def test_three_centres_wide_matches_oracle():
    g = _three_centres(600)
    b, views, G = _run(g, [0, 1, 2])
    assert min(G.budget(c) for c in range(3)) > BUDGET_MAX
    assert b.flags[0] == 0
    _check(b, views)


def test_batch_mixing_wide_and_ordinary_samples():
    g = _three_centres(600)
    seeds = [5, 0, 7, 2, 3, 1, 600]
    b, views, G = _run(g, seeds, key=0xABCDEF12345, first=40)
    wide = [G.budget(s) > BUDGET_MAX for s in seeds]
    assert any(wide) and not all(wide)
    assert b.flags[0] == 0
    _check(b, views)


def test_wide_egonet_hub_row_takes_the_reverse_probe():
    g = _hub_beside_centre()
    b, views, G = _run(g, [0, 3, 0])
    assert G.budget(0) > BUDGET_MAX
    w = views[0][0]
    assert 1 in set(w["subv"].tolist()) and G.deg[1] > 16 * w["n"]
    assert b.flags[0] == 0
    _check(b, views)


def test_pairs_wide_q_seed_gives_both_views_its_budget():
    g = _three_centres(600)
    # sample 0: q wide, k a leaf (both views walk the centre's budget); sample 1: q a leaf, k a centre (both ordinary)
    b, views, G = _run(g, [0, 5, 1], seeds_k=[4, 2, 1], key=77)
    assert G.budget(0) > BUDGET_MAX and G.budget(5) <= BUDGET_MAX
    assert b.flags[0] == 0
    _check(b, views)


def test_node_overflow_of_a_view_with_a_wide_egonet_is_flagged_not_fatal():
    g = synthetic.star_graph(1000)
    _, views, _ = _run(g, [0, 9])
    n = min(sum(s["n"] for s in v) for v in views)
    b, _, _ = _run(g, [0, 9], node_cap=n - 5, edge_cap=1 << 16)
    assert b.flags[0] & 1
    assert b.node_off[0, 2] == -1 and b.node_off[1, 2] == -1


def test_view_without_room_in_the_wide_region_overflows_its_edges():
    """The wide node sets live in a region of edge_cap + B entries per view: an ego-net that finds no room there is
    counted with m = n - 1 edges, which pushes its view over edge_cap."""
    g = synthetic.star_graph(1000)
    b, views, _ = _run(g, [0, 9], node_cap=1 << 14, edge_cap=100)
    assert min(s["n"] for s in (views[0][0], views[1][0])) > 100 + 2
    assert b.flags[0] & 2
    assert b.node_off[0, 2] == -1 and b.node_off[1, 2] == -1


def test_pool_exhaustion_second_look_on_a_wide_egonet():
    """As test_emu_sampler's: view 0 overflows its edges and eats the pool (2 * edge_cap), so the wide ego-net of the
    still valid view 1 is induced by the fill kernel's own look at its rows, from the node set in the region."""
    g = synthetic.star_graph(1000)
    for key in range(1, 40):
        _, views, _ = _run(g, [0], key=key)
        m0, m1 = (sum(s["m"] for s in v) for v in views)
        if m0 > m1 + 8:
            break
    else:
        pytest.skip("no key with m0 > m1")
    cap = (m0 + m1) // 2 - 2
    assert m1 <= cap < m0 and 2 * cap < m0 + m1
    b, views, _ = _run(g, [0], key=key, edge_cap=cap)
    assert b.flags[0] & 2 and b.node_off[0, 1] == -1 and b.node_off[1, 1] >= 0
    _check(b, views, vlist=(1,))


@pytest.mark.parametrize("B,edge_cap", [(1, 100), (32, 123457), (256, 4_000_000)])
def test_workspace_unchanged_for_budgets_that_fit(B, edge_cap):
    L = lib()                                   # the product's walk CTA trace: 32,768 ints
    for mb in (1, 64, 1000, 16384, 32704):
        cap_n = (mb + 64 + 1 + 3) & ~3
        assert L.gccb_sample_batch_workspace(B, mb, edge_cap) == (3 * 2 * B * cap_n + 16 + 2 * edge_cap) * 4
    # above: ordinary slots at the limit's cap_n, the wide regions by edge_cap, key arrays per wide walk CTA
    cap_n = (32704 + 64 + 1 + 3) & ~3
    for mb in (32705, 79064, 989000):
        keys = 1 << (mb + 64 - 1).bit_length()
        want = 3 * 2 * B * cap_n + 16 + 2 * edge_cap + 6 * (edge_cap + B) + min(2 * B, 32) * keys
        assert L.gccb_sample_batch_workspace(B, mb, edge_cap) == want * 4


def test_budget_beyond_int32_positions_is_an_explicit_error():
    L = lib()
    g = synthetic.star_graph(3)
    G = PlainGraph(g, 1)
    G.c.max_budget = (1 << 30) - 63                  # pow2 >= budget + HOPCAP would be 2^31
    b = NpBatch(1, 64, 64)
    seeds = np.zeros(1, np.int64)
    ws = np.zeros(64, np.uint8)
    rc = L.gccb_sample_batch(C.byref(G.c), ptr(seeds), ptr(seeds), C.byref(b.c), ptr(ws), ws.nbytes, None)
    assert rc != 0
    err = L.gccb_last_error()
    assert "walk budget %d" % ((1 << 30) - 63) in (err.decode() if isinstance(err, bytes) else err)
