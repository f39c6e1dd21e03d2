"""CPU: the downstream datasets (gcc_b200/datasets/downstream.py) and the frozen-embedding evaluators
(gcc_b200/tasks) against tests/golden/tasks_golden.npz, which the reference's own readers, graph builder and
evaluators produced (tests/golden/make_golden_tasks.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from gcc_b200 import tasks
from gcc_b200.datasets import downstream, labeled
from gcc_b200.tasks.graph_classification import GraphClassification
from gcc_b200.tasks.node_classification import NodeClassification
from gcc_b200.tasks.similarity_search import SimilaritySearch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "tasks_golden.npz"))


@pytest.fixture
def data_root(z, tmp_path):
    """The fixture's input files under <tmp>/data, the layout the reference reads."""
    for k in z.files:
        if k.startswith("files/"):
            p = tmp_path / "data" / k[len("files/"):]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_text(str(z[k]))
    return tmp_path / "data"


def _multiset(src, dst):
    return sorted(zip(np.asarray(src).tolist(), np.asarray(dst).tolist()))


def _csr_edges(g):
    row = np.repeat(np.arange(g.num_nodes), np.diff(g.indptr))
    return _multiset(row, g.indices)


def _check_graph(z, tag, g):
    assert g.num_nodes == int(z[tag + "_graph_n"])
    assert _csr_edges(g) == _multiset(z[tag + "_graph_src"], z[tag + "_graph_dst"])
    for v in range(g.num_nodes):                                  # the gccb_graph_t contract: rows non-decreasing
        assert np.all(np.diff(g.indices[g.indptr[v]:g.indptr[v + 1]]) >= 0)


@pytest.mark.parametrize("name,tag", [("usa_airport", "usa"), ("h-index-rand-1", "hindex")])
def test_edgelist_multigraph_matches_reference(z, data_root, name, tag):
    e = downstream.create_node_classification_dataset(name, str(data_root))
    assert np.array_equal(e.data.edge_index.numpy(), z[tag + "_edge_index"])
    assert np.array_equal(e.data.y.numpy(), z[tag + "_y"])
    g = downstream.node_dataset_graph(name, str(data_root))
    _check_graph(z, tag, g)
    # parallel edges and the self loop survive: more entries than the de-duplicating finetune graph
    simple = labeled.graph_from_edge_index(e.data.edge_index.numpy())
    assert len(g.indices) == 2 * z[tag + "_edge_index"].shape[1] > len(simple.indices)


def test_panther_readers_match_reference(z, data_root):
    s = downstream.create_node_classification_dataset("kdd", str(data_root))
    assert np.array_equal(s.data.edge_index.numpy(), z["kdd_edge_index"])
    g = downstream.node_dataset_graph("kdd", str(data_root))
    _check_graph(z, "kdd", g)
    row = np.repeat(np.arange(g.num_nodes), np.diff(g.indptr))
    _, mult = np.unique(row * g.num_nodes + g.indices, return_counts=True)
    assert mult.max() >= 10                                       # t = 5, listed both ways, doubled by the builder
    ss = downstream.SSDataset(str(data_root / "panther"), "kdd", "icdm")
    for i, d in enumerate(ss.data):
        assert np.array_equal(d.edge_index.numpy(), z["ss%d_edge_index" % i])
        want = dict(zip(z["ss%d_dict_keys" % i].tolist(), z["ss%d_dict_ids" % i].tolist()))
        assert d.y == want
        assert max(want.values()) >= int(d.edge_index.max()) + 1        # ids without edges are appended


def test_tu_reader_keeps_listed_entries(tmp_path):
    d = tmp_path / "TOY"
    d.mkdir()
    # graph 1: a repeated pair (1,2) and a self loop on 3; graph 2: a single edge
    (d / "TOY_A.txt").write_text("1, 2\n2, 1\n1, 2\n2, 1\n3, 3\n2, 3\n3, 2\n4, 5\n5, 4\n")
    (d / "TOY_graph_indicator.txt").write_text("1\n1\n1\n2\n2\n")
    (d / "TOY_graph_labels.txt").write_text("1\n-1\n")
    graphs, labels = labeled.read_tu_dataset(str(tmp_path), "TOY", multigraph=True)
    assert labels.tolist() == [1, 0]
    assert graphs[0].indptr.tolist() == [0, 2, 5, 7] and graphs[0].indices.tolist() == [1, 1, 0, 0, 2, 1, 2]
    assert graphs[1].indices.tolist() == [1, 0]
    simple, _ = labeled.read_tu_dataset(str(tmp_path), "TOY")
    assert simple[0].indices.tolist() == [1, 0, 2, 1]


def test_node_classification_evaluator_matches_reference(z):
    t = NodeClassification.__new__(NodeClassification)
    t.seed = int(z["nc_seed"])
    assert t._evaluate(z["nc_x"], z["nc_y"], 10) == {"Micro-F1": float(z["nc_result"])}


def test_graph_classification_evaluator_matches_reference(z):
    t = GraphClassification.__new__(GraphClassification)
    t.seed = int(z["gc_seed"])
    assert t.svc_classify(z["gc_x"], z["gc_y"]) == {"Micro-F1": float(z["gc_result"])}


def test_similarity_search_evaluator_matches_reference(z):
    d1 = dict(zip(z["ss_d1_keys"].tolist(), z["ss_d1_ids"].tolist()))
    d2 = dict(zip(z["ss_d2_keys"].tolist(), z["ss_d2_ids"].tolist()))
    res = SimilaritySearch._evaluate(None, z["ss_e1"], z["ss_e2"], d1, d2)
    assert res == {"Recall @ 20": float(z["ss_recall20"]), "Recall @ 40": float(z["ss_recall40"])}


def test_build_model_baselines_are_named():
    for name, what in (("prone", "ProNE"), ("graphwave", "GraphWave")):
        with pytest.raises(NotImplementedError, match=what):
            tasks.build_model(name, 8)
    assert tasks.build_model("zero", 8).train(np.arange(5)).shape == (5, 8)


def _run(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-s", "-m"] + args, cwd=cwd, env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return out.stdout


def test_task_clis_on_reference_files(z, data_root, tmp_path):
    """Each evaluator's command line on the fixture's files with a saved `.npy`; node rows map to node ids."""
    rng = np.random.RandomState(0)
    n_usa = downstream.node_dataset_graph("usa_airport", str(data_root)).num_nodes
    np.save(tmp_path / "usa_airport.npy", rng.randn(n_usa, 8).astype(np.float32))
    out = _run(["gcc_b200.tasks.node_classification", "--dataset", "usa_airport", "--model", "from_numpy",
                "--hidden-size", "8", "--emb-path", str(tmp_path / "usa_airport.npy")], tmp_path)
    assert out.startswith("{'Micro-F1': ")
    for name in ("kdd", "icdm"):
        n = downstream.node_dataset_graph(name, str(data_root)).num_nodes
        np.save(tmp_path / (name + ".npy"), rng.randn(n, 8).astype(np.float32))
    out = _run(["gcc_b200.tasks.similarity_search", "--dataset", "kdd_icdm", "--model", "from_numpy_align",
                "--hidden-size", "8", "--emb-path-1", str(tmp_path / "kdd.npy"), "--emb-path-2",
                str(tmp_path / "icdm.npy")], tmp_path)
    assert out.startswith("{'Recall @ 20': ") and "'Recall @ 40': " in out
