"""CPU: eigensolver kernels (gcc_b200/csrc/posenc.cu) under the fiber emulator --
spectral parity with the oracle (dense float64 eigh) and with the reference's own
outputs (tests/golden/posenc_golden.npz).  Kernel LOGIC only; see test_gpu_*.

The `solver` fixture runs a test through the shipped dispatch ("default": GCCB200_DENSE_MAX unset, the dense
tridiagonal solver up to 96 vertices and the Chebyshev-filtered subspace iteration above) and through the dense
solver up to 228 vertices ("dense": GCCB200_DENSE_MAX=228); gccb_posenc reads the variable on every call."""
import ctypes as C
import os

import numpy as np
import pytest

from emu_util import NpBatch, lib, ptr
from gcc_b200.datasets import synthetic
from oracle import posenc as opos

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(params=["default", "dense"])
def solver(request, monkeypatch):
    if request.param == "dense":
        monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    else:
        monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
    return request.param


def _sub(g):
    return dict(subv=np.arange(g.num_nodes, dtype=np.int32), indptr=g.indptr.astype(np.int32),
                indices=g.indices.astype(np.int32), n=g.num_nodes, m=len(g.indices))


def _posenc(views, normalize):
    L = lib()
    b = NpBatch.from_subgraphs(views)
    pos = np.full((2, b.node_cap, 32), np.nan, np.float32)
    eig = np.full((2 * b.B, 32), np.nan, np.float32)
    ws = np.zeros(L.gccb_posenc_workspace(b.B, b.node_cap), np.uint8)
    rc = L.gccb_posenc(C.byref(b.c), 32, normalize, ptr(pos), ptr(eig), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return b, pos, eig


def _views(graphs):
    half = len(graphs) // 2
    return [[_sub(g) for g in graphs[:half]], [_sub(g) for g in graphs[half:]]]


def _check_spectral(sub, u, lam):
    n = sub["n"]
    k = min(n - 2, 32)
    lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n).toarray()
    if k <= 0:
        assert np.all(u == 0) and np.all(lam == 0)
        return
    w_exact, _ = opos.eig_topk_exact(lap, k)
    assert np.all(u[:, k:] == 0) and np.all(lam[k:] == 0)
    assert np.allclose(lam[:k], w_exact, atol=1e-5), np.abs(lam[:k] - w_exact).max()
    theta, resid, ortho = opos.spectral_report(lap, u[:, :k].astype(np.float64))
    assert resid.max() < 1e-4, resid.max()
    assert ortho < 1e-4, ortho
    assert np.allclose(theta, w_exact, atol=1e-5)


def test_spectral_parity_small_and_degenerate(solver):
    graphs = [synthetic.path_graph(2), synthetic.path_graph(3), synthetic.path_graph(9),
              synthetic.star_graph(20), synthetic.triangle_tail(4),
              synthetic.erdos_renyi(40, 90, seed=1), synthetic.star_graph(50),
              synthetic.erdos_renyi(60, 100, seed=4)]
    half = len(graphs) // 2
    views = [[_sub(g) for g in graphs[:half]], [_sub(g) for g in graphs[half:]]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    for v in (0, 1):
        for gi, sub in enumerate(views[v]):
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            _check_spectral(sub, pos[v, a:z], eig[v * b.B + gi])


def test_size_classes_and_normalisation(solver):
    g1 = synthetic.erdos_renyi(90, 240, seed=7)           # n <= 96: dense solver
    g2 = synthetic.star_graph(90)                         # extreme degeneracy (eigenvalue 0 x 89)
    g3 = synthetic.erdos_renyi(150, 420, seed=9)          # 96 < n <= 160: shared-memory ChFSI (dense: n <= 228)
    views = [[_sub(g1), _sub(g3)], [_sub(g2), _sub(synthetic.path_graph(30))]]
    assert 64 < g1.num_nodes <= 96 < g3.num_nodes <= 160 and 64 < g2.num_nodes
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    for v in (0, 1):
        for gi, sub in enumerate(views[v]):
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            _check_spectral(sub, pos[v, a:z], eig[v * b.B + gi])
    b, posn, _ = _posenc(views, normalize=1)
    for v in (0, 1):
        n = b.node_off[v, b.B]
        assert np.allclose(np.linalg.norm(posn[v, :n], axis=1), 1.0, atol=1e-5)
        raw = pos[v, :n]
        want = raw / np.linalg.norm(raw, axis=1, keepdims=True)
        assert np.allclose(posn[v, :n], want, atol=1e-6)


def test_posenc_matches_reference_golden(solver):
    z = np.load(os.path.join(G, "posenc_golden.npz"))
    subs = []
    for ci in range(int(z["num_cases"])):
        ip, ix = z["indptr%d" % ci].astype(np.int32), z["indices%d" % ci].astype(np.int32)
        subs.append(dict(subv=np.arange(len(ip) - 1, dtype=np.int32), indptr=ip, indices=ix,
                         n=len(ip) - 1, m=len(ix)))
    if len(subs) % 2:
        subs.append(subs[0])
    half = len(subs) // 2
    views = [subs[:half], subs[half:]]
    b, pos, _ = _posenc(views, normalize=1)
    checked = 0
    for ci in range(int(z["num_cases"])):
        v, gi = (0, ci) if ci < half else (1, ci - half)
        a, zz = b.node_off[v, gi], b.node_off[v, gi + 1]
        got, want = pos[v, a:zz], z["pos%d" % ci]
        n = zz - a
        k = min(n - 2, 32)
        if k <= 0:
            assert np.all(got == 0) and np.all(want == 0)
        elif bool(z["simple%d" % ci]):
            s = np.sign((got[:, :k] * want[:, :k]).sum(axis=0))
            assert np.allclose(got[:, :k] * s, want[:, :k], atol=5e-5), (ci, np.abs(got[:, :k] * s - want[:, :k]).max())
            assert np.all(got[:, k:] == 0)
            checked += 1
    assert checked >= 8


def test_dense_max_below_96_is_the_default(monkeypatch):
    """GCCB200_DENSE_MAX below the first dense class acts as 96: the output is bit-identical to the default dispatch's,
    on ego-nets on both sides of the boundary."""
    graphs = [synthetic.path_graph(9), synthetic.star_graph(50), synthetic.erdos_renyi(60, 100, seed=4),
              synthetic.chung_lu(95, 250, seed=2), synthetic.erdos_renyi(150, 420, seed=9),
              synthetic.chung_lu(156, 420, seed=3)]
    assert sorted(g.num_nodes > 96 for g in graphs) == [False] * 4 + [True] * 2
    views = _views(graphs)
    monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
    _, pos, eig = _posenc(views, normalize=1)
    monkeypatch.setenv("GCCB200_DENSE_MAX", "0")
    _, pos0, eig0 = _posenc(views, normalize=1)
    assert np.array_equal(pos, pos0, equal_nan=True) and np.array_equal(eig, eig0, equal_nan=True)


def test_posenc_refuses_a_misaligned_workspace():
    """The debug area at the start of the workspace holds int64 counters."""
    L = lib()
    b = NpBatch.from_subgraphs(_views([synthetic.path_graph(9), synthetic.path_graph(5)]))
    pos = np.zeros((2, b.node_cap, 32), np.float32)
    ws = np.zeros(L.gccb_posenc_workspace(b.B, b.node_cap) + 8, np.uint8)
    assert L.gccb_posenc(C.byref(b.c), 32, 1, ptr(pos), None, C.c_void_p(ws.ctypes.data + 4), ws.nbytes - 4,
                         None) != 0
    assert b"aligned" in L.gccb_last_error()


def test_huge_egonet_one_block_in_shared_memory():
    g = synthetic.chung_lu(560, 1500, exponent=0.8, seed=3)    # 480 < n <= 1000: X in smem, Y in workspace
    assert 480 < g.num_nodes <= 1000
    views = [[_sub(g)], [_sub(synthetic.path_graph(5))]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    _check_spectral(views[0][0], pos[0, :g.num_nodes], eig[0])


def test_large_egonet_goes_through_chfsi(solver):
    g = synthetic.chung_lu(260, 700, seed=3)              # hub-and-leaves: large degenerate cluster
    assert g.num_nodes > 200
    views = [[_sub(g)], [_sub(synthetic.path_graph(5))]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    _check_spectral(views[0][0], pos[0, :g.num_nodes], eig[0])
    _check_spectral(views[1][0], pos[1, :5], eig[1])


def test_dense_solver_class_boundaries_and_degenerate_spectra(monkeypatch):
    """The dense tridiagonal solver at the edges of its three classes (96 / 144 / 228), on the smallest ego-nets
    (k = 1, 2, 3), on exactly degenerate spectra (stars: eigenvalue 0 x 199; a disconnected union) and on paths
    (the matrix is already tridiagonal: every reflector is the identity); tighter bars than the shared ones --
    the fp32 model of the kernel measures eigenvalues to 5e-7 and residuals / orthonormality to 4e-6."""
    monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    graphs = [synthetic.path_graph(3), synthetic.path_graph(4), synthetic.path_graph(5), synthetic.star_graph(33),
              synthetic.path_graph(96), synthetic.chung_lu(100, 250, seed=1), synthetic.chung_lu(150, 400, seed=2),
              synthetic.chung_lu(156, 420, seed=3), synthetic.path_graph(228), synthetic.star_graph(200),
              synthetic.disjoint_union([synthetic.star_graph(30), synthetic.star_graph(30), synthetic.path_graph(20)]),
              synthetic.erdos_renyi(228, 2000, seed=3), synthetic.chung_lu(240, 640, exponent=0.8, seed=5),
              synthetic.erdos_renyi(34, 60, seed=2)]
    sizes = [g.num_nodes for g in graphs]
    assert max(sizes) <= 228 and any(96 < n <= 144 for n in sizes) and any(144 < n for n in sizes), sizes
    half = len(graphs) // 2
    views = [[_sub(g) for g in graphs[:half]], [_sub(g) for g in graphs[half:]]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    for v in (0, 1):
        for gi, sub in enumerate(views[v]):
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            u, lam = pos[v, a:z], eig[v * b.B + gi]
            _check_spectral(sub, u, lam)
            n = sub["n"]
            k = min(n - 2, 32)
            lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n).toarray()
            w_exact, _ = opos.eig_topk_exact(lap, k)
            theta, resid, ortho = opos.spectral_report(lap, u[:, :k].astype(np.float64))
            assert np.abs(lam[:k] - w_exact).max() < 2e-6 and resid.max() < 2e-5 and ortho < 2e-5, (
                n, np.abs(lam[:k] - w_exact).max(), resid.max(), ortho)


def test_dense_solver_fifteen_fold_cluster_regression(monkeypatch):
    """A sampled C2 ego-net (n = 173) whose 15-fold eigenvalue 1/sqrt 2 made the first cluster member come out of
    Gram-Schmidt with a residual of 2.8e-4 when all inverse iterations ran before the orthogonalisation (the
    iterates of a cluster get more collinear with every iteration); with the two-stage order it is 4e-7."""
    monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    z = np.load(os.path.join(G, "egonet_cluster15.npz"))
    ip, ix = z["indptr"].astype(np.int32), z["indices"].astype(np.int32)
    n = len(ip) - 1
    sub = dict(subv=np.arange(n, dtype=np.int32), indptr=ip, indices=ix, n=n, m=len(ix))
    views = [[sub], [_sub(synthetic.path_graph(5))]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0
    lap = opos.normalized_adjacency(ip, ix, n).toarray()
    w = np.linalg.eigvalsh(lap)
    assert np.sum(np.abs(w - 2 ** -0.5) < 1e-9) == 15
    theta, resid, ortho = opos.spectral_report(lap, pos[0, :n, :32].astype(np.float64))
    assert resid.max() < 2e-5 and ortho < 2e-5, (resid.max(), ortho)


def test_dense_solver_random_structures(monkeypatch):
    """Fuzz of the dense solver over the structures ego-nets are made of: random trees, trees with a few extra edges,
    hubs with pendant paths (the multiple eigenvalues 1/sqrt 2, sqrt(2/3), 0), dense random graphs, disconnected
    unions, rings (every eigenvalue double) -- 24 graphs of 3..228 vertices, all classes.  240 such graphs measured
    eigenvalues to 7e-7, residuals to 1e-6 and orthonormality to 3e-6."""
    monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    rng = np.random.default_rng(1)

    def rand_graph(n):
        kind = int(rng.integers(0, 6))
        if kind in (0, 1):
            src = np.arange(1, n)
            dst = np.array([rng.integers(0, i) for i in range(1, n)])
            if kind == 1:
                ex = rng.integers(0, n, (max(1, n // 20), 2))
                src, dst = np.concatenate([src, ex[:, 0]]), np.concatenate([dst, ex[:, 1]])
        elif kind == 2:
            src = np.arange(1, n)
            dst = np.where(rng.random(n - 1) < 0.6, 0, np.maximum(np.arange(1, n) - 1, 0))
        elif kind == 3:
            e = rng.integers(0, n, (3 * n, 2))
            src, dst = e[:, 0], e[:, 1]
        elif kind == 4:
            h = n // 2
            src = np.concatenate([np.arange(1, h), np.arange(h + 1, n)])
            dst = np.concatenate([np.zeros(h - 1, int), np.full(n - h - 1, h)])
        else:
            src, dst = np.arange(n), (np.arange(n) + 1) % n
        return synthetic.from_pairs(np.asarray(src, np.int64), np.asarray(dst, np.int64), n)

    graphs = []
    while len(graphs) < 24:
        g = rand_graph(int(rng.integers(5, 229)))
        if g.num_nodes >= 3:
            graphs.append(g)
    views = [[_sub(g) for g in graphs[0::2]], [_sub(g) for g in graphs[1::2]]]
    b, pos, eig = _posenc(views, normalize=0)
    assert b.flags[0] == 0 and np.all(np.isfinite(pos[0, :b.node_off[0, b.B]])) and np.all(np.isfinite(pos[1, :b.node_off[1, b.B]]))
    for v in (0, 1):
        for gi, sub in enumerate(views[v]):
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            n = sub["n"]
            k = min(n - 2, 32)
            lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n).toarray()
            w_exact, _ = opos.eig_topk_exact(lap, k)
            theta, resid, ortho = opos.spectral_report(lap, pos[v, a:z, :k].astype(np.float64))
            assert np.abs(eig[v * b.B + gi, :k] - w_exact).max() < 2e-6 and resid.max() < 2e-5 and ortho < 2e-5, (
                n, np.abs(eig[v * b.B + gi, :k] - w_exact).max(), resid.max(), ortho)


@pytest.mark.parametrize("pos_dim", [5, 16])
def test_dense_solver_other_feature_widths(monkeypatch, pos_dim):
    """positional_embedding_size below 32 (train.py:94 is a free parameter): k = min(n - 2, pos_dim) columns, the rest
    zero; the top-k cut may fall inside a multiple eigenvalue (the star's 0 x 39)."""
    monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    views = [[_sub(synthetic.chung_lu(90, 240, seed=2)), _sub(synthetic.path_graph(7))],
             [_sub(synthetic.star_graph(40)), _sub(synthetic.chung_lu(150, 400, seed=3))]]
    L = lib()
    b = NpBatch.from_subgraphs(views)
    pos = np.full((2, b.node_cap, pos_dim), np.nan, np.float32)
    eig = np.full((2 * b.B, pos_dim), np.nan, np.float32)
    ws = np.zeros(L.gccb_posenc_workspace(b.B, b.node_cap), np.uint8)
    assert L.gccb_posenc(C.byref(b.c), pos_dim, 0, ptr(pos), ptr(eig), ptr(ws), ws.nbytes, None) == 0
    assert b.flags[0] == 0
    for v in (0, 1):
        for gi, sub in enumerate(views[v]):
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            n = sub["n"]
            k = min(n - 2, pos_dim)
            lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n).toarray()
            w, _ = opos.eig_topk_exact(lap, k)
            theta, resid, ortho = opos.spectral_report(lap, pos[v, a:z, :k].astype(np.float64))
            assert np.all(pos[v, a:z, k:] == 0) and np.all(eig[v * b.B + gi, k:] == 0)
            assert np.abs(eig[v * b.B + gi, :k] - w).max() < 2e-6 and resid.max() < 2e-5 and ortho < 2e-5
