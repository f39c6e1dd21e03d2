"""GPU: GraphWave and ProNE (gcc_b200/tasks/baselines.py, csrc/baselines.cu) against the reference's own outputs in
tests/golden/baselines_golden.npz, a float64 scipy restatement on a 20k-vertex graph, and the exporter command line
feeding the existing evaluators."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse as sp

from gcc_b200.tasks import baselines

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NAMES = ["usa", "hindex", "kdd", "icdm", "hub", "split"]


@pytest.fixture(scope="module")
def z():
    return np.load(os.path.join(GOLDEN, "baselines_golden.npz"))


def _graph(z, name):
    build = baselines.multigraph_from_pairs if z[name + "_multi"] else baselines.graph_from_pairs
    return build(z[name + "_edge_index"])


def _gram(r):
    return r @ r.T


@pytest.mark.parametrize("name", NAMES)
def test_graphwave_matches_reference_for_any_block_size(z, name):
    g = _graph(z, name)
    n = len(g.indptr) - 1
    whole = baselines.GraphWave(64).train(g)
    assert np.abs(whole - z[name + "_chi"]).max() <= 1e-6
    assert np.array_equal(baselines.GraphWave(64).train(g), whole)
    for bc in (1, 7, n):
        assert np.array_equal(baselines.GraphWave(64, block_cols=bc).train(g), whole)


def _chung_lu(n, avg_deg, seed):
    rng = np.random.RandomState(seed)
    w = (np.arange(1, n + 1) / n) ** -0.6
    p = w / w.sum()
    m = n * avg_deg // 2
    ei = np.stack([rng.choice(n, m, p=p), rng.choice(n, m, p=p)])
    ei = np.concatenate([ei, np.stack([np.arange(n), (np.arange(n) + 1) % n])], axis=1)   # every vertex has an edge
    return ei


def _chi_columns(g, cols, dim=64, scale=100):
    """GraphWave's chi rows `cols` restated in float64 scipy: heat columns by the Chebyshev recursion on the
    identity columns, threshold, characteristic function."""
    n = len(g.indptr) - 1
    A = sp.csr_matrix((g.vals, g.indices, g.indptr), shape=(n, n))
    d = np.asarray(A.sum(axis=0)).ravel()
    dinv = np.where(d > 1e-10, 1.0 / np.sqrt(np.maximum(d, 1e-300)), 0.0)
    N = sp.diags(dinv) @ A @ sp.diags(dinv)
    times = np.linspace(0, scale, dim // 4)
    out = []
    for tau in baselines.graphwave_scales(n):
        c = baselines.cheb_coeffs(tau)
        t0 = np.zeros((n, len(cols)))
        t0[cols, np.arange(len(cols))] = 1.0
        t1 = -(N @ t0)
        heat = c[0] * t0 + c[1] * t1
        for k in range(2, baselines.ORDER + 1):
            t0, t1 = t1, -2.0 * (N @ t1) - t0
            heat += c[k] * t1
        heat[heat <= 1e-4 / n] = 0.0
        arg = times[None, :, None] * heat.T[:, None, :]            # [col, time, row]
        part = np.stack([np.cos(arg).sum(2), np.sin(arg).sum(2)], axis=2) / n
        out.append(part.reshape(len(cols), -1))
    return np.concatenate(out, axis=1)


def test_graphwave_20k_vertices_in_several_blocks():
    g = baselines.graph_from_pairs(_chung_lu(20000, 8, seed=3))
    n = len(g.indptr) - 1
    assert n == 20000
    gw = baselines.GraphWave(64, workspace_bytes=1 << 30)             # about 1,500 columns per block: 14 blocks
    chi = gw.train(g)
    cols = np.sort(np.random.RandomState(0).choice(n, 64, replace=False))
    want = _chi_columns(g, cols)
    assert np.abs(chi[cols] - want).max() <= 1e-6
    assert np.isfinite(chi).all()


@pytest.mark.parametrize("name", NAMES)
def test_prone_factor_matches_reference(z, name):
    g = _graph(z, name)
    n = len(g.indptr) - 1
    _, F, FT = baselines.ProNE(int(z[name + "_dim"])).factorize(g)
    want = sp.coo_matrix((z[name + "_F_val"], (z[name + "_F_row"], z[name + "_F_col"])), shape=(n, n)).toarray()
    got = sp.csr_matrix((F.cpu().numpy(), g.indices, g.indptr), shape=(n, n)).toarray()
    got_t = sp.csr_matrix((FT.cpu().numpy(), g.indices, g.indptr), shape=(n, n)).toarray()
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 1e-12 * scale
    assert np.abs(got_t - want.T).max() <= 1e-12 * scale


@pytest.mark.parametrize("name", NAMES)
def test_prone_propagation_teacher_forced(z, name):
    g = _graph(z, name)
    a = z[name + "_a"].astype(np.float64)
    mm, emb = baselines.ProNE(int(z[name + "_dim"])).propagate(g, a)
    want = z[name + "_mm"]
    assert np.abs(mm.cpu().numpy() - want).max() <= 1e-10 * np.abs(want).max()
    assert np.abs(_gram(emb.cpu().numpy()) - _gram(z[name + "_emb"])).max() <= 1e-8


def _sklearn_range_svd(F, omega, d, n_iter=5):
    """sklearn's randomized_svd with the LU power-iteration normaliser, on a given start block."""
    Q = omega
    for _ in range(n_iter):
        Q, _ = scipy.linalg.lu(F @ Q, permute_l=True)
        Q, _ = scipy.linalg.lu(F.T @ Q, permute_l=True)
    Q, _ = scipy.linalg.qr(F @ Q, mode="economic")
    Uh, s, _ = scipy.linalg.svd(Q.T @ F, full_matrices=False)
    U = (Q @ Uh)[:, :d] * np.sqrt(s[:d])
    return s[:d], U / np.linalg.norm(U, axis=1, keepdims=True)


@pytest.mark.parametrize("name", NAMES)
def test_prone_tsvd_with_supplied_start(z, name):
    g = _graph(z, name)
    n, d = int(z[name + "_n"]), int(z[name + "_dim"])
    omega = np.random.RandomState(7).randn(n, min(d + 10, n))
    F = sp.coo_matrix((z[name + "_F_val"], (z[name + "_F_row"], z[name + "_F_col"])), shape=(n, n)).toarray()
    s_want, r_want = _sklearn_range_svd(F, omega, d)
    s, r = baselines.ProNE(d).tsvd(g, omega)
    np.testing.assert_allclose(s.cpu().numpy(), s_want, rtol=1e-9)
    assert np.abs(_gram(r.cpu().numpy()) - _gram(r_want)).max() <= 1e-6


def test_prone_default_start_is_reproducible(z):
    g = _graph(z, "hub")
    runs = [baselines.ProNE(64, seed=3).train(g) for _ in range(2)]
    assert np.array_equal(runs[0], runs[1])
    assert runs[0].shape == (181, 64)
    np.testing.assert_allclose(np.linalg.norm(runs[0], axis=1), 1.0, rtol=1e-12)
    other = baselines.ProNE(64, seed=4).train(g)
    assert not np.array_equal(other, runs[0])


def test_prone_needs_as_many_vertices_as_dimensions(z):
    with pytest.raises(ValueError, match="ProNE"):
        baselines.ProNE(64).train(_graph(z, "usa"))


def test_prone_refuses_blocks_of_another_graph_size(z):
    g = _graph(z, "hub")
    n = len(g.indptr) - 1
    model = baselines.ProNE(16)
    for rows in (n - 1, n + 1):
        with pytest.raises(ValueError, match="omega"):
            model.tsvd(g, np.ones((rows, 26)))
        with pytest.raises(ValueError, match="expected %d rows" % n):
            model.propagate(g, np.ones((rows, 16)))


@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    t = np.load(os.path.join(GOLDEN, "tasks_golden.npz"))
    root = tmp_path_factory.mktemp("baselines") / "data"
    for k in t.files:
        if k.startswith("files/"):
            p = root / k[len("files/"):]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_text(str(t[k]))
    return root


def _export(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-s", "-m", "gcc_b200.tasks.baselines"] + args, cwd=cwd, env=env,
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return out.stdout


def test_exporter_graphwave_through_evaluators(z, data_root, tmp_path):
    from gcc_b200.tasks.node_classification import NodeClassification
    from gcc_b200.tasks.similarity_search import SimilaritySearch
    cwd = data_root.parent
    _export(["--task", "node_classification", "--dataset", "usa_airport", "--model", "graphwave", "--hidden-size", "64",
             "--output-dir", str(tmp_path / "gpu")], cwd)
    _export(["--task", "similarity_search", "--dataset", "kdd_icdm", "--model", "graphwave", "--hidden-size", "64",
             "--output-dir", str(tmp_path / "gpu")], cwd)
    usa = np.load(tmp_path / "gpu" / "usa_airport.npy")
    ref = np.zeros_like(usa)
    ref[_graph(z, "usa").nodes] = z["usa_chi"]
    assert usa.shape[1] == 64 and np.abs(usa - ref).max() <= 1e-6
    (tmp_path / "ref").mkdir()
    np.save(tmp_path / "ref" / "usa_airport.npy", ref)
    for name in ("kdd", "icdm"):
        np.save(tmp_path / "ref" / (name + ".npy"), z[name + "_chi"].astype(np.float64))
    res = {}
    for src in ("gpu", "ref"):
        nc = NodeClassification("usa_airport", "from_numpy", 64, 10, 0, root=str(data_root),
                                emb_path=str(tmp_path / src / "usa_airport.npy"))
        ss = SimilaritySearch("kdd", "icdm", "from_numpy_align", 64, root=str(data_root),
                              emb_path_1=str(tmp_path / src / "kdd.npy"), emb_path_2=str(tmp_path / src / "icdm.npy"))
        res[src] = dict(nc.train(), **ss.train())
    for k, v in res["ref"].items():
        assert abs(res["gpu"][k] - v) <= 0.01, (k, res)


def test_exporter_prone_layout(z, data_root, tmp_path):
    from gcc_b200.datasets import downstream
    from gcc_b200.tasks.node_classification import NodeClassification
    from gcc_b200.tasks.similarity_search import SimilaritySearch
    cwd = data_root.parent
    _export(["--task", "node_classification", "--dataset", "usa_airport", "--model", "prone", "--hidden-size", "16",
             "--output-dir", str(tmp_path)], cwd)
    _export(["--task", "similarity_search", "--dataset", "kdd_icdm", "--model", "prone", "--hidden-size", "16",
             "--output-dir", str(tmp_path)], cwd)
    usa = np.load(tmp_path / "usa_airport.npy")
    assert usa.shape == (downstream.node_dataset_graph("usa_airport", str(data_root)).num_nodes, 16)
    nodes = _graph(z, "usa").nodes
    np.testing.assert_allclose(np.linalg.norm(usa[nodes], axis=1), 1.0, rtol=1e-12)
    assert not np.delete(usa, nodes, axis=0).any()
    for name in ("kdd", "icdm"):
        e = np.load(tmp_path / (name + ".npy"))
        assert e.shape == (int(z[name + "_n"]), 16)
        np.testing.assert_allclose(np.linalg.norm(e, axis=1), 1.0, rtol=1e-12)
    nc = NodeClassification("usa_airport", "from_numpy", 16, 10, 0, root=str(data_root),
                            emb_path=str(tmp_path / "usa_airport.npy"))
    assert 0.0 <= nc.train()["Micro-F1"] <= 1.0
    ss = SimilaritySearch("kdd", "icdm", "from_numpy_align", 16, root=str(data_root),
                          emb_path_1=str(tmp_path / "kdd.npy"), emb_path_2=str(tmp_path / "icdm.npy"))
    assert set(ss.train()) == {"Recall @ 20", "Recall @ 40"}
