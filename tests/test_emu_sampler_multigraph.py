"""CPU: the sampler kernels (gcc_b200/csrc/sampler.cu) on multigraphs, run under the fiber emulator and compared
bit-for-bit with the oracle, which induces entry by entry.  A neighbour repeated c times in a row is c parallel
edges (the gccb_graph_t contract): the walk picks it with probability c / deg and the ego-net keeps c copies.

Every path that induces a row is reached with parallel edges into the row's vertex:
  - the CTA-wide hub list of the walk kernel (rows of degree > 16 n);
  - the per-warp reverse probe, taken by hub rows beyond that list (a build with GCCB_HUB_LIST = 1);
  - the fill kernel's second look after the scratch pool ran out, for hub and streamed rows;
  - the streamed scan of ordinary rows, in all three."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import emu_util
from emu_util import NpBatch, NpGraph, ptr
from gcc_b200 import _capi
from gcc_b200.datasets import downstream
from oracle import rwr as orwr

HUBS, LEAVES = 3, 3000


def _hub_multigraph(seed=7):
    """Three hubs joined to every leaf by t = 1..5 parallel edges, leaf-leaf edges of multiplicity 1..3, the hubs
    joined to each other twice, a self loop on hub 0 and on one leaf.  Built like the Panther graphs: the pairs
    listed t times, each added in both directions."""
    rng = np.random.RandomState(seed)
    n = HUBS + LEAVES
    src, dst = [], []

    def add(a, b, t):
        src.extend([a] * t)
        dst.extend([b] * t)
    for h in range(HUBS):
        for leaf in range(HUBS, n):
            add(h, leaf, int(rng.randint(1, 6)))
        for h2 in range(h + 1, HUBS):
            add(h, h2, 2)
    for a, b in rng.randint(HUBS, n, size=(4000, 2)):
        if a != b:
            add(int(a), int(b), int(rng.randint(1, 4)))
    add(0, 0, 1)
    add(HUBS + 5, HUBS + 5, 1)
    return downstream.multigraph_from_edge_index(np.array([src, dst]), "hub_multigraph")


_G = None


def _graph():
    global _G
    if _G is None:
        _G = _hub_multigraph()
    return _G


_hub1 = None


def _lib_hub_list_1():
    """The emulated library with GCCB_HUB_LIST = 1: all hub rows of an ego-net but one take the warp path."""
    global _hub1
    if _hub1 is None:
        emu_util.lib()                                              # builds the default objects
        spec = importlib.util.spec_from_file_location("build_emu", os.path.join(emu_util.HERE, "emu", "build_emu.py"))
        be = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(be)
        out = os.path.join(be.OUT, "hub_list_1")
        os.makedirs(out, exist_ok=True)
        src = os.path.join(be.CSRC, "sampler.cu")
        obj, lib = os.path.join(out, "sampler.cu.o"), os.path.join(out, "libgccb200_emu_hub1.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-DGCCB_EMU", "-DGCCB_HUB_DEG=3",
                               "-DGCCB_HUB_LIST=1", "-I", be.HERE, "-x", "c++", "-c", src, "-o", obj])
        others = [os.path.join(be.OUT, os.path.basename(s) + ".o") for s in be.sources()
                  if os.path.basename(s) != "sampler.cu"]
        subprocess.check_call(["g++", "-shared", "-o", lib, obj] + others)
        _hub1 = _capi.bind(C.CDLL(lib), require_all=False)
    return _hub1


def _run(L, g, B, rw_hops, key, edge_cap=None):
    G = NpGraph(g, rw_hops, 0.8, key)
    seeds = np.zeros(B, np.int64)
    sids = np.zeros(B, np.int64)
    assert L.gccb_draw_seeds(ptr(G.cdf), g.num_nodes, key, 0, B, ptr(seeds), ptr(sids), None) == 0
    want = orwr.rwr_batch(G.indptr, G.indices, key, sids, seeds, G.btable, G.rt, int(G.btable.max()) + 65, 1 << 20)
    views = [[want[2 * i + v] for i in range(B)] for v in (0, 1)]
    N = max(sum(s["n"] for s in v) for v in views)
    E = max(sum(s["m"] for s in v) for v in views)
    b = NpBatch(B, N + 7, edge_cap or E + 11)
    ws = np.zeros(L.gccb_sample_batch_workspace(B, int(G.btable.max()), b.edge_cap), np.uint8)
    rc = L.gccb_sample_batch(C.byref(G.c), ptr(seeds), ptr(sids), C.byref(b.c), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    # rowstart scratch of the walk kernel (sampler.cu workspace layout): -1 = row left to the fill kernel
    cap_n = (int(G.btable.max()) + 64 + 1 + 3) & ~3
    rowstart = ws.view(np.int32)[2 * 2 * B * cap_n:3 * 2 * B * cap_n].reshape(2 * B, cap_n)
    return b, views, rowstart.copy()


def _hub_rows(g, s):
    """Local ids of the ego-net's rows the kernels treat as hubs (parent degree > 16 n)."""
    deg = np.diff(g.indptr)[s["subv"]]
    return np.flatnonzero(deg > 16 * s["n"])


def _check_view(b, views, v, B):
    got = b.view_graphs(v)
    assert b.node_off[v, B] == sum(s["n"] for s in views[v])
    assert b.edge_off[v, B] == sum(s["m"] for s in views[v])
    for gi, (a, w) in enumerate(zip(got, views[v])):
        assert np.array_equal(a["subv"], w["subv"]), (v, gi)
        assert np.array_equal(a["indptr"], w["indptr"]), (v, gi)
        assert np.array_equal(a["indices"], w["indices"]), (v, gi)
    n = b.node_off[v, B]
    assert np.array_equal(b.sub_deg[v, :n], np.diff(b.indptr[v, :n + 1]))


def _multi_hub_hits(g, views):
    """Parallel edges out of hub rows into the ego-net, summed over all ego-nets (the count the probes must keep)."""
    total = 0
    for v in views:
        for s in v:
            for i in _hub_rows(g, s):
                row = s["indices"][s["indptr"][i]:s["indptr"][i + 1]]
                _, c = np.unique(row, return_counts=True)
                total += int((c - 1).sum())
    return total


@pytest.mark.parametrize("hub_list", ["cta", "warp"])
def test_multigraph_sampler_matches_oracle(hub_list):
    g = _graph()
    L = emu_util.lib() if hub_list == "cta" else _lib_hub_list_1()
    B = 6
    b, views, _ = _run(L, g, B, 48, key=0x5EED1234)
    assert b.flags[0] == 0
    # the reached ground: ego-nets with several hub rows, whose induced rows repeat local ids
    assert max(len(_hub_rows(g, s)) for v in views for s in v) >= 2
    assert _multi_hub_hits(g, views) > 0
    for v in (0, 1):
        _check_view(b, views, v, B)
        for gi, w in enumerate(views[v]):
            c = b.counters[v * B + gi]
            assert (c[0], c[1], c[2], c[3]) == (w["n"], w["m"], w["steps"], w["sumdeg"])


def test_multigraph_fill_kernel_second_look():
    """Pool exhaustion (as in test_sampler_pool_exhaustion_falls_back_to_a_second_look): view 0 overflows its
    edge_cap and eats the scratch pool, so hub rows of the still valid view 1 are induced by the fill kernel."""
    g = _graph()
    L = emu_util.lib()
    B = 4
    for key in range(1, 60):
        _, views, _ = _run(L, g, B, 48, key=key)
        m0, m1 = (sum(s["m"] for s in v) for v in views)
        if m0 <= m1 or not any(len(_hub_rows(g, s)) for s in views[1]):
            continue
        b, views, rowstart = _run(L, g, B, 48, key=key, edge_cap=m1)
        assert b.flags[0] & 2 and b.node_off[0, B] == -1 and b.node_off[1, B] >= 0
        looked_again = [(gi, i) for gi, s in enumerate(views[1]) for i in _hub_rows(g, s)
                        if rowstart[B + gi, i] == -1]
        repeats = sum(len(r) - len(np.unique(r)) for r in
                      (views[1][gi]["indices"][views[1][gi]["indptr"][i]:views[1][gi]["indptr"][i + 1]]
                       for gi, i in looked_again))
        if not repeats:
            continue
        _check_view(b, views, 1, B)
        return
    pytest.fail("no key whose view 1 leaves a hub row to the fill kernel")
