"""CPU: the embedding baselines (gcc_b200/tasks/baselines.py, csrc/baselines.cu) against
tests/golden/baselines_golden.npz, which the reference's own ProNE and GraphWave produced
(tests/golden/make_golden_baselines.py).  The kernels run under the CPU emulator (tests/emu)."""
import os

import networkx as nx
import numpy as np
import pytest
import scipy.sparse as sp

import emu_util
from gcc_b200.tasks import baselines

ptr = emu_util.ptr


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "baselines_golden.npz"))


def _graph(z, name):
    build = baselines.multigraph_from_pairs if z[name + "_multi"] else baselines.graph_from_pairs
    return build(z[name + "_edge_index"])


def _dense(g):
    n = len(g.indptr) - 1
    return sp.csr_matrix((g.vals, g.indices, g.indptr), shape=(n, n)).toarray()


NAMES = ["usa", "hindex", "kdd", "icdm", "hub", "split"]


@pytest.mark.parametrize("name", NAMES)
def test_graph_builders_match_networkx(z, name):
    ei = z[name + "_edge_index"]
    G = nx.MultiGraph() if z[name + "_multi"] else nx.Graph()
    G.add_edges_from(ei.T.tolist())
    nodes = sorted(G.nodes())
    want = nx.adjacency_matrix(G, nodelist=nodes).toarray()
    g = _graph(z, name)
    assert g.nodes.tolist() == nodes
    assert np.array_equal(_dense(g), want)
    for v in range(len(nodes)):
        assert np.all(np.diff(g.indices[g.indptr[v]:g.indptr[v + 1]]) > 0)


def test_builders_self_loops_and_multiplicities():
    ei = np.array([[5, 7, 7, 5, 9, 9, 9], [7, 5, 5, 5, 9, 9, 5]])
    simple = _dense(baselines.graph_from_pairs(ei))
    multi = _dense(baselines.multigraph_from_pairs(ei))
    # ids 5, 7, 9 -> 0, 1, 2
    assert simple.tolist() == [[1, 1, 1], [1, 0, 0], [1, 0, 1]]
    assert multi.tolist() == [[1, 3, 1], [3, 0, 0], [1, 0, 2]]


@pytest.mark.parametrize("name", NAMES)
def test_scales_and_chebyshev_coefficients(z, name):
    n = int(z[name + "_n"])
    taus = baselines.graphwave_scales(n)
    np.testing.assert_allclose(taus, z[name + "_taus"], rtol=1e-14)
    # The coefficients fall below the rounding error of their own sums (1e-17 against terms of order 1) well
    # before k = 30, so the bound is relative to the largest coefficient, not to each one.
    for s, tau in enumerate(taus):
        want = z[name + "_cheb"][s]
        assert np.abs(baselines.cheb_coeffs(tau) - want).max() <= 1e-13 * np.abs(want).max()


def test_bessel_coefficients(z):
    np.testing.assert_allclose([baselines.bessel_i(i, 0.5) for i in range(5)], z["bessel"], rtol=1e-14)


def _emu_graphwave(g, bc, dim=64, scale=100):
    lib = emu_util.lib()
    n = len(g.indptr) - 1
    T = dim // 4
    cheb = np.ascontiguousarray(np.concatenate([baselines.cheb_coeffs(t) for t in baselines.graphwave_scales(n)]))
    times = np.ascontiguousarray(np.linspace(0, scale, T))
    ws = np.zeros(lib.gccb_graphwave_workspace(n, bc), np.uint8)
    chi = np.full((n, 4 * T), np.nan)
    rc = lib.gccb_graphwave(ptr(g.indptr), ptr(g.indices), ptr(g.vals), n, ptr(cheb), baselines.ORDER, ptr(times),
                            T, bc, ptr(ws), ws.nbytes, ptr(chi), None)
    assert rc == 0
    return chi


@pytest.mark.parametrize("name", ["usa", "kdd", "hub"])
def test_emu_graphwave_matches_reference(z, name):
    g = _graph(z, name)
    chi = _emu_graphwave(g, bc=len(g.indptr) - 1)
    assert np.abs(chi - z[name + "_chi"]).max() <= 1e-6


def test_emu_graphwave_independent_of_block_size(z):
    g = _graph(z, "icdm")
    ref = _emu_graphwave(g, bc=len(g.indptr) - 1)
    assert np.abs(ref - z["icdm_chi"]).max() <= 1e-6
    for bc in (1, 7):
        assert np.array_equal(_emu_graphwave(g, bc), ref)


@pytest.mark.parametrize("name", ["usa", "split"])
def test_emu_prone_factor_matches_reference(z, name):
    lib = emu_util.lib()
    g = _graph(z, name)
    n = len(g.indptr) - 1
    ws = np.zeros(lib.gccb_prone_factor_workspace(n), np.uint8)
    F, FT = np.zeros_like(g.vals), np.zeros_like(g.vals)
    assert lib.gccb_prone_factor(ptr(g.indptr), ptr(g.indices), ptr(g.vals), n, ptr(ws), ws.nbytes, ptr(F), ptr(FT),
                                 None) == 0
    want = sp.coo_matrix((z[name + "_F_val"], (z[name + "_F_row"], z[name + "_F_col"])), shape=(n, n)).toarray()
    got = sp.csr_matrix((F, g.indices, g.indptr), shape=(n, n)).toarray()
    got_t = sp.csr_matrix((FT, g.indices, g.indptr), shape=(n, n)).toarray()
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 1e-12 * scale
    assert np.abs(got_t - want.T).max() <= 1e-12 * scale


@pytest.mark.parametrize("name", ["hindex", "kdd", "hub"])
def test_emu_prone_propagation_matches_reference(z, name):
    lib = emu_util.lib()
    g = _graph(z, name)
    n = len(g.indptr) - 1
    a = np.ascontiguousarray(z[name + "_a"], np.float64)
    k = a.shape[1]
    bessel = np.ascontiguousarray([baselines.bessel_i(i, 0.5) for i in range(5)])
    ws = np.zeros(lib.gccb_prone_propagate_workspace(n, k), np.uint8)
    mm = np.full_like(a, np.nan)
    assert lib.gccb_prone_propagate(ptr(g.indptr), ptr(g.indices), ptr(g.vals), n, ptr(a), k, 0.2, ptr(bessel), 5,
                                    ptr(ws), ws.nbytes, ptr(mm), None) == 0
    want = z[name + "_mm"]
    assert np.abs(mm - want).max() <= 1e-9 * np.abs(want).max()


def test_emu_spmm_epilogue():
    """Y = alpha dr ((A + sigma I)(dc X)) + beta X + gamma Z against dense numpy, repeated columns as weights."""
    lib = emu_util.lib()
    rng = np.random.RandomState(1)
    indptr = np.array([0, 3, 4, 6, 8], np.int64)
    indices = np.array([1, 1, 3, 0, 0, 3, 0, 2], np.int32)        # row 0 lists column 1 twice
    n, k, ld = 4, 5, 6
    A = np.zeros((n, n))
    for i in range(n):
        for e in range(indptr[i], indptr[i + 1]):
            A[i, indices[e]] += 1
    X, Z = rng.randn(n, ld), rng.randn(n, ld)
    dr, dc = rng.rand(n) + 0.5, rng.rand(n) + 0.5
    Y = np.zeros((n, ld))
    assert lib.gccb_spmm_f64(ptr(indptr), ptr(indices), None, n, k, ld, -0.7, 1.0, ptr(dr), ptr(dc), 0.3, ptr(X),
                             -1.5, ptr(Z), ptr(Y), None) == 0
    want = -0.7 * dr[:, None] * ((A + np.eye(n)) @ (dc[:, None] * X)) + 0.3 * X - 1.5 * Z
    np.testing.assert_allclose(Y[:, :k], want[:, :k], rtol=1e-13, atol=1e-13)
    assert np.all(Y[:, k:] == 0)


def test_emu_spmm_offset_blocks():
    """Blocks that start 8 bytes past a 16-byte boundary with an even row stride give the same result as aligned
    ones: the product takes its single-column path for them."""
    lib = emu_util.lib()
    rng = np.random.RandomState(2)
    indptr = np.array([0, 2, 3, 5], np.int64)
    indices = np.array([0, 2, 1, 0, 2], np.int32)
    vals = rng.rand(5)
    n, k = 3, 4
    buf_x, buf_y = np.zeros(n * k + 1), np.zeros(n * k + 1)
    x = buf_x[1:].reshape(n, k)
    x[:] = rng.randn(n, k)
    y = buf_y[1:].reshape(n, k)
    assert x.ctypes.data % 16 == 8 and y.ctypes.data % 16 == 8
    assert lib.gccb_spmm_f64(ptr(indptr), ptr(indices), ptr(vals), n, k, k, 2.0, 0.0, None, None, 0.5, ptr(x), 0.0,
                             None, ptr(y), None) == 0
    A = sp.csr_matrix((vals, indices, indptr), shape=(n, n)).toarray()
    np.testing.assert_allclose(y, 2.0 * A @ x + 0.5 * x, rtol=1e-13, atol=1e-13)


def test_gaussian_block_is_seeded(z):
    lib = emu_util.lib()
    out = [np.zeros((300, 26)) for _ in range(3)]
    for o, key in zip(out, (5, 5, 6)):
        assert lib.gccb_gaussian_f64(ptr(o), 300, 26, key, None) == 0
    assert np.array_equal(out[0], out[1]) and not np.array_equal(out[0], out[2])
    x = out[0].ravel()
    assert abs(x.mean()) < 0.05 and abs(x.std() - 1) < 0.05
