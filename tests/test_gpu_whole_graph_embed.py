"""GPU (H100): whole-graph rows from generate.py through EmbedEngine -- the TU sets' rows byte for byte what the
labeled dataset's batches give through the encoder (GIN hidden 64 and 128, GAT), a TU directory by path, the run-ahead
ring against the serial loop, shards against one run, `--nodes` subsets, a skewed corpus on ring buffers sized from
its largest batch, a .bin corpus from x2dgl embedded with --whole-graphs and searched and classified through the task
command lines, and the device relabel against seed_first_union on 10^5 graphs."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from test_gpu_downstream import _write_tu
from test_gpu_generate import _ckpt, _model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _main(ckpt, dataset, gpu=0, B=16, **kw):
    import generate
    return generate.main(types.SimpleNamespace(load_path=ckpt, dataset=dataset, graph_nodes=0, graph_edges=0,
                                               batch_size=B, gpu=gpu, **kw))


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("kind", ["gin64", "gin128", "gat64"])
def test_tu_rows_equal_the_labeled_dataset_path(tmp_path, monkeypatch, kind):
    """The five names keep their rows: the engine's file equals, byte for byte, the rows of
    GraphClassificationDatasetLabeled.batches() through the encoder at the same batch size (generate.py's former
    path); a TU directory given by path writes the same bytes under its own name."""
    from gcc_b200.datasets import downstream
    from gcc_b200.datasets.labeled import GraphClassificationDatasetLabeled
    _write_tu(tmp_path / "data", "IMDB-BINARY", n_graphs=45)
    monkeypatch.chdir(tmp_path)
    ckpt = _ckpt(tmp_path, kind)
    _main(ckpt, "imdb-binary", B=8)
    model = _model(kind).cuda().eval()
    ds = GraphClassificationDatasetLabeled(downstream.graph_dataset_graphs("imdb-binary"),
                                           positional_embedding_size=32, batch_size=8)
    with torch.no_grad():
        want = torch.cat([model(g).cpu() for g, _ in ds.batches()]).numpy()
    got = np.load(str(tmp_path / "imdb-binary.npy"))
    assert got.shape == want.shape == (45, model.cfg.hidden)
    assert got.tobytes() == want.tobytes(), np.abs(got - want).max()
    _main(ckpt, str(tmp_path / "data" / "IMDB-BINARY"), B=8)
    assert _bytes(str(tmp_path / "IMDB-BINARY.npy")) == _bytes(str(tmp_path / "imdb-binary.npy"))


@pytest.fixture(scope="module")
def tu300(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("tu300")
    _write_tu(tmp, "SET300", n_graphs=300, seed=4)
    return tmp, str(tmp / "SET300"), _ckpt(tmp, "gin64")


def test_prefetch_and_serial_write_identical_files(tu300):
    tmp, path, ckpt = tu300
    out = str(tmp / "SET300.npy")
    _main(ckpt, path, prefetch=0)
    serial = _bytes(out)
    _main(ckpt, path, prefetch=4)
    assert _bytes(out) == serial


def test_shards_write_the_file_one_run_writes(tu300):
    tmp, path, ckpt = tu300
    out = str(tmp / "SET300.npy")
    _main(ckpt, path, gpu=[0])
    one = _bytes(out)
    gpus = [0, 1] if torch.cuda.device_count() > 1 else [0, 0]
    _main(ckpt, path, gpu=gpus)
    assert _bytes(out) == one


def test_nodes_subset_matches_the_full_run(tu300):
    tmp, path, ckpt = tu300
    out = str(tmp / "SET300.npy")
    _main(ckpt, path)
    full = np.load(out).copy()
    ids = np.array([5, 0, 299, 17, 17, 100, 250, 3], np.int64)
    np.save(str(tmp / "ids.npy"), ids)
    _main(ckpt, path, nodes=str(tmp / "ids.npy"))
    sub = np.load(out)
    print("--nodes: max |subset - full| = %.3e" % np.abs(sub - full[ids]).max())
    assert np.allclose(sub, full[ids], rtol=1e-4, atol=1e-5)
    with pytest.raises(SystemExit, match="graph ids must lie in 0..299"):
        np.save(str(tmp / "bad.npy"), np.array([300]))
        _main(ckpt, path, nodes=str(tmp / "bad.npy"))


def test_skewed_corpus_runs_on_buffers_of_its_largest_batch():
    """Thousands of small graphs and one of 50,000 vertices: the ring holds the largest actual batch (the big
    graph's), far less than the B largest graphs would need, and the big graph's row is finite."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import WholeGraphDataset, whole_graph_plan
    from gcc_b200.datasets.labeled import _listed_csr
    from gcc_b200.embed import EmbedEngine
    rng = np.random.RandomState(8)
    graphs = []
    for i in range(3000):
        n = int(rng.randint(4, 30))
        e = np.concatenate([np.stack([np.arange(n), (np.arange(n) + 1) % n], 1), rng.randint(0, n, (n, 2))])
        graphs.append(_listed_csr(np.concatenate([e[:, 0], e[:, 1]]), np.concatenate([e[:, 1], e[:, 0]]), n, "s%d" % i))
    big = synthetic.chung_lu(50000, 150000, exponent=0.5, seed=2)
    graphs.insert(1234, big)
    B = 64
    ds = WholeGraphDataset(graphs, positional_embedding_size=32, batch_size=B)
    model = _model("gin64").cuda().eval()
    eng = EmbedEngine(ds, model, prefetch=4)
    rows = eng.run(range(len(graphs)))
    sizes = np.array([g.num_nodes for g in graphs])
    nnz = np.array([len(g.indices) for g in graphs])
    assert (eng.node_cap, eng.edge_cap) == whole_graph_plan(sizes, nnz, np.arange(len(graphs)), B)
    t = 1234 // B
    assert eng.node_cap == sizes[t * B:(t + 1) * B].sum() + 8 and eng.edge_cap == nnz[t * B:(t + 1) * B].sum() + 8
    top = int(np.sort(sizes)[::-1][:B].sum()) + 8                # the former sizing: the B largest graphs
    print("skewed corpus: ring of %d vertices / %d edge entries (B largest graphs: %d vertices)"
          % (eng.node_cap, eng.edge_cap, top))
    assert eng.node_cap < top
    assert all(b.node_cap == eng.node_cap and b.edge_cap == eng.edge_cap for b in eng.bufs)
    assert np.isfinite(rows).all() and np.abs(rows[1234]).sum() > 0


def test_own_corpus_end_to_end(tmp_path, monkeypatch):
    """Edge-list files -> x2dgl .bin -> generate.py --whole-graphs -> tasks.knn and tasks.graph_classification."""
    from gcc_b200.datasets import x2dgl
    rng = np.random.RandomState(3)
    d = tmp_path / "edges"
    d.mkdir()
    files = []
    for i in range(24):
        n = int(rng.randint(20, 60))
        e = [(j, (j + 1) % n) for j in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(n * (1 + i % 2))]
        e = [(u, v) for u, v in e if u != v]
        p = d / ("g%02d.txt" % i)
        p.write_text("".join("%d %d\n" % uv for uv in e))
        files.append(str(p))
    corpus = str(tmp_path / "mine.bin")
    x2dgl.main(["--graph-dir", str(d), "--save-file", corpus, "--graph-files"] + files)
    ckpt = _ckpt(tmp_path, "gin64")
    rows = _main(ckpt, corpus, B=8, whole_graphs=True).numpy()
    assert rows.shape == (24, 64) and np.isfinite(rows).all()
    assert os.path.exists(str(tmp_path / "mine.graphs.npy")) and not os.path.exists(str(tmp_path / "mine.npy"))
    np.savez(str(tmp_path / "labels.npz"), graph_labels=np.arange(24) % 2)
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda args: subprocess.run([sys.executable, "-s", "-m"] + args, cwd=str(tmp_path), env=env,
                                      capture_output=True, text=True)
    out = run(["gcc_b200.tasks.knn", "--emb-path", str(tmp_path / "mine.graphs.npy"), "--k", "5", "--output",
               str(tmp_path / "nn")])
    assert out.returncode == 0, out.stderr
    ids = np.load(str(tmp_path / "nn.ids.npy"))
    assert ids.shape == (24, 5) and (ids != np.arange(24)[:, None]).all()
    out = run(["gcc_b200.tasks.graph_classification", "--dataset", str(tmp_path / "labels.npz"), "--model",
               "from_numpy_graph", "--hidden-size", "64", "--emb-path", str(tmp_path / "mine.graphs.npy")])
    assert out.returncode == 0, out.stderr
    print(out.stdout.strip())
    assert out.stdout.startswith("{'Micro-F1': ")


def test_device_build_equals_seed_first_union():
    from gcc_b200 import _lib
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import DeviceGraphSet, seed_first_union
    rng = np.random.RandomState(9)
    G = 100_000
    n = rng.randint(1, 12, G)
    m = rng.randint(0, 3, G) * n
    graphs, a = [], 0
    # one vectorised corpus: random entries per graph, sorted rows (parallel edges and self loops kept)
    node_off = np.concatenate([[0], np.cumsum(n)])
    gid = np.repeat(np.arange(G), m)
    src = node_off[gid] + (rng.random_sample(len(gid)) * n[gid]).astype(np.int64)
    dst = node_off[gid] + (rng.random_sample(len(gid)) * n[gid]).astype(np.int64)
    order = np.lexsort((dst, src))
    V = int(node_off[-1])
    indptr = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=V), out=indptr[1:])
    union = synthetic.CSRGraph(indptr, dst[order].astype(np.int32), V, "corpus")
    for g in range(G):
        a, b = node_off[g], node_off[g + 1]
        ip = indptr[a:b + 1] - indptr[a]
        graphs.append(synthetic.CSRGraph(ip, (union.indices[indptr[a]:indptr[b]] - a).astype(np.int32), int(b - a),
                                         "g%d" % g))
    w_seeds, _, w_ip, w_ix, w_no, w_eo = seed_first_union(graphs)
    for s in (DeviceGraphSet(graphs, "cuda"), DeviceGraphSet.from_union(union, n, "cuda")):
        assert np.array_equal(s.seeds, w_seeds)
        assert np.array_equal(s.indptr.cpu().numpy(), w_ip)
        assert np.array_equal(s.indices.cpu().numpy().astype(np.int64), w_ix)
        assert np.array_equal(s.node_off_host, w_no) and np.array_equal(s.edge_off.cpu().numpy(), w_eo)
    bad = union.indices.copy()
    r = int(next(r for r in np.flatnonzero(np.diff(indptr) >= 2)[::-1] if bad[indptr[r]] != bad[indptr[r] + 1]))
    bad[indptr[r]], bad[indptr[r] + 1] = bad[indptr[r] + 1], bad[indptr[r]]
    g_bad = int(np.searchsorted(node_off, r, side="right") - 1)
    with pytest.raises(_lib.GccbError, match="graph %d has a row" % g_bad):
        DeviceGraphSet.from_union(synthetic.CSRGraph(indptr, bad, V, "bad"), n, "cuda")
