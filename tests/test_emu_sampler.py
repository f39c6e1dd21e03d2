"""CPU: sampler kernels (gcc_b200/csrc/sampler.cu) run under the fiber emulator and
compared bit-for-bit with the oracle.  Kernel LOGIC only -- the real parity gate is
tests/test_gpu_*.py on an H100."""
import ctypes as C

import numpy as np
import pytest

from emu_util import NpBatch, NpGraph, lib, ptr
from gcc_b200.datasets import synthetic
from oracle import rwr as orwr


def _run(g, B, rw_hops, key, first=0, node_cap=None, edge_cap=None):
    L = lib()
    G = NpGraph(g, rw_hops, 0.8, key)
    seeds = np.zeros(B, np.int64)
    sids = np.zeros(B, np.int64)
    assert L.gccb_draw_seeds(ptr(G.cdf), g.num_nodes, key, first, B, ptr(seeds), ptr(sids), None) == 0
    want_seeds = orwr.draw_seeds(G.cdf, key, range(first, first + B))
    assert np.array_equal(seeds, want_seeds) and np.array_equal(sids, np.arange(first, first + B))
    want = orwr.rwr_batch(G.indptr, G.indices, key, sids, seeds, G.btable, G.rt,
                          int(G.btable.max()) + 65, 1 << 16)
    views = [[want[2 * i + v] for i in range(B)] for v in (0, 1)]
    N = max(sum(s["n"] for s in v) for v in views)
    E = max(sum(s["m"] for s in v) for v in views)
    b = NpBatch(B, node_cap or N + 7, edge_cap or E + 11)
    ws = np.zeros(L.gccb_sample_batch_workspace(B, int(G.btable.max()), b.edge_cap), np.uint8)
    rc = L.gccb_sample_batch(C.byref(G.c), ptr(seeds), ptr(sids), C.byref(b.c), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return b, views, want


def _three_centres(leaves):
    src = np.repeat(np.arange(3), leaves)
    dst = 3 + np.tile(np.arange(leaves), 3)
    return synthetic.from_pairs(src, dst, leaves + 3, "k3_%d" % leaves)


@pytest.mark.parametrize("name,B,hops", [("er", 5, 24), ("star", 3, 16), ("cl", 4, 40), ("hub", 4, 16), ("bigstar", 2, 400),
                                         ("k3", 2, 8000)])
def test_sampler_matches_oracle(name, B, hops):
    g = {"er": lambda: synthetic.erdos_renyi(300, 1200, seed=2),
         "star": lambda: synthetic.star_graph(40),
         # the hub row of the ego-net has several hundred induced neighbours: more than one parking buffer
         # (GCCB_HIT_STAGE = 128), i.e. the count-then-record path of the walk kernel
         "bigstar": lambda: synthetic.star_graph(700),
         "cl": lambda: synthetic.chung_lu(2000, 12000, seed=3),
         # hub degree >> ego-net size: exercises the reverse-probe induction path
         "hub": lambda: synthetic.chung_lu(6000, 60000, exponent=0.9, seed=5),
         # ego-nets of more than 1024 vertices whose three centre rows (degree 30000 > 16 n) take the CTA-wide
         # reverse probe in several chunks of keys
         "k3": lambda: _three_centres(30000)}[name]()
    b, views, want = _run(g, B, hops, key=0xABCDEF12345)
    assert b.flags[0] == 0
    if name == "k3":
        assert max(s_["n"] for v_ in views for s_ in v_) > 1024
    for v in (0, 1):
        got = b.view_graphs(v)
        assert b.node_off[v, B] == sum(s["n"] for s in views[v])
        assert b.edge_off[v, B] == sum(s["m"] for s in views[v])
        for gi, (a, w) in enumerate(zip(got, views[v])):
            assert np.array_equal(a["subv"], w["subv"]), (v, gi)
            assert np.array_equal(a["indptr"], w["indptr"]), (v, gi)
            assert np.array_equal(a["indices"], w["indices"]), (v, gi)
            c = b.counters[v * B + gi]
            assert (c[0], c[1], c[2], c[3]) == (w["n"], w["m"], w["steps"], w["sumdeg"])
        n = b.node_off[v, B]
        assert np.array_equal(b.sub_deg[v, :n], np.diff(b.indptr[v, :n + 1]))
        assert np.array_equal(b.graph_id[v, :n], np.repeat(np.arange(B), np.diff(b.node_off[v])))


def test_sampler_capacity_overflow_is_flagged_not_fatal():
    g = synthetic.erdos_renyi(300, 1200, seed=2)
    b, views, _ = _run(g, 4, 24, key=5, node_cap=20, edge_cap=10000)
    assert b.flags[0] & 1
    assert b.node_off[0, 4] == -1 or b.node_off[1, 4] == -1


def test_sampler_pool_exhaustion_falls_back_to_a_second_look():
    """The scratch pool holds 2 * edge_cap hits.  When view 0 needs more than edge_cap (it is published empty)
    it also eats the pool, and the rows of the still valid view 1 must be induced by the fill kernel's own
    scan -- bit-exact all the same."""
    g = synthetic.chung_lu(2000, 12000, seed=3)
    for key in range(1, 40):
        b0, views, _ = _run(g, 4, 40, key=key)
        m0, m1 = (sum(s["m"] for s in v) for v in views)
        if m0 > m1 + 8:
            break
    else:
        pytest.skip("no key with m0 > m1")
    cap = (m0 + m1) // 2 - 2
    assert m1 <= cap < m0 and 2 * cap < m0 + m1
    b, views, _ = _run(g, 4, 40, key=key, edge_cap=cap)
    assert b.flags[0] & 2 and b.node_off[0, 4] == -1 and b.node_off[1, 4] >= 0
    for gi, (a, w) in enumerate(zip(b.view_graphs(1), views[1])):
        assert np.array_equal(a["subv"], w["subv"]) and np.array_equal(a["indptr"], w["indptr"])
        assert np.array_equal(a["indices"], w["indices"]), gi
