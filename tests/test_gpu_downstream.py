"""GPU: the freeze-evaluation recipe end to end on small files in each reference format -- a short train.py
pretraining run, generate.py on airports / h-index (Edgelist), Panther (kdd, icdm) and a TU set, then the three
task command lines on the saved rows.  The node datasets are multigraphs (parallel edges, Panther weights, self
loops): the device sampler must induce them bit-exactly like the oracle, and the encoder must match the oracle
encoder in eval mode on the device's positional features."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _write_tu(root, name, n_graphs=40, seed=0):
    """A TU set: class 1 graphs have a hub; a repeated pair and a self loop in every third graph."""
    rng = np.random.RandomState(seed)
    d = root / name
    d.mkdir(parents=True)
    a_rows, ind, labels, base = [], [], [], 0
    for g in range(n_graphs):
        n = int(rng.randint(8, 20))
        pairs = [(i, (i + 1) % n) for i in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(n // 2)]
        if g % 2:
            pairs += [(0, i) for i in range(2, n)]
        if g % 3 == 0:
            pairs += [pairs[0], (1, 1)]
        for u, v in pairs:
            a_rows.append("%d, %d" % (base + u + 1, base + v + 1))
            if u != v:
                a_rows.append("%d, %d" % (base + v + 1, base + u + 1))
        ind += [g + 1] * n
        labels.append(1 if g % 2 else -1)
        base += n
    (d / (name + "_A.txt")).write_text("\n".join(a_rows) + "\n")
    (d / (name + "_graph_indicator.txt")).write_text("\n".join(map(str, ind)) + "\n")
    (d / (name + "_graph_labels.txt")).write_text("\n".join(map(str, labels)) + "\n")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    """<tmp>/data with every format, and a checkpoint from a short pretraining run."""
    import train
    tmp = tmp_path_factory.mktemp("downstream")
    z = np.load(os.path.join(GOLDEN, "tasks_golden.npz"))
    for k in z.files:
        if k.startswith("files/"):
            p = tmp / "data" / k[len("files/"):]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_text(str(z[k]))
    _write_tu(tmp / "data", "IMDB-BINARY")
    args = train.parse_option(["--moco", "--max-steps", "4", "--dataset", "synthetic-er", "--graph-nodes", "2000",
                               "--graph-edges", "10000", "--batch-size", "16", "--num-workers", "1",
                               "--num-copies", "1", "--num-samples", "64", "--epochs", "1", "--nce-k", "64",
                               "--hidden-size", "64", "--num-layer", "3", "--rw-hops", "32", "--print-freq", "1000",
                               "--model-path", str(tmp / "m"), "--tb-path", str(tmp / "tb")])
    train.main(args)
    return tmp, os.path.join(args.model_folder, "current.pth"), args.model_folder


def _generate(work, monkeypatch, name, batch_size=16):
    import generate
    tmp, ckpt, folder = work
    monkeypatch.chdir(tmp)
    generate.main(types.SimpleNamespace(load_path=ckpt, dataset=name, graph_nodes=0, graph_edges=0,
                                        batch_size=batch_size, gpu=0))
    return np.load(os.path.join(folder, name + ".npy"))


def _encoder(ckpt):
    import generate
    from gcc_b200.models import GraphEncoder
    c = torch.load(ckpt, map_location="cpu", weights_only=False)
    opt = c["opt"]
    model = GraphEncoder(degree_input=True, **{kw: getattr(opt, a) for kw, a in generate.ENCODER_KWARGS.items()})
    model.load_state_dict(c["model"])
    return model.cuda().eval(), opt


def _view(buf, v):
    """View v of a BatchBuffers on the host: per-graph dicts (local ids) and the batched arrays."""
    B = buf.B
    noff = buf.node_off[v].cpu().numpy().astype(np.int64)
    N, E = int(noff[B]), int(buf.edge_off[v, B])
    ip = buf.indptr[v, :N + 1].cpu().numpy().astype(np.int64)
    ix = buf.indices[v, :E].cpu().numpy().astype(np.int64)
    orig = buf.orig_id[v, :N].cpu().numpy()
    graphs = []
    for g in range(B):
        a, b = noff[g], noff[g + 1]
        graphs.append(dict(subv=orig[a:b], indptr=ip[a:b + 1] - ip[a], indices=ix[ip[a]:ip[b]] - a))
    return graphs, ip, ix, noff


def _hub_multigraph():
    """Two hubs joined to 2000 leaves by t = 1..5 parallel edges, a sparse leaf layer, a self loop on a hub."""
    from gcc_b200.datasets import downstream
    rng = np.random.RandomState(11)
    src, dst = [], []
    for h in (0, 1):
        for leaf in range(2, 2002):
            t = int(rng.randint(1, 6))
            src += [h] * t
            dst += [leaf] * t
    e = rng.randint(2, 2002, size=(3000, 2))
    src += e[:, 0].tolist() + [0]
    dst += e[:, 1].tolist() + [0]
    return downstream.multigraph_from_edge_index(np.array([src, dst]), "hubs")


@pytest.mark.parametrize("name", ["usa_airport", "kdd", "hubs"])
def test_multigraph_ego_nets_match_oracle(work, monkeypatch, name):
    """generate.py's node dataset on a multigraph: sampler outputs bit-exact against the oracle, the encoder
    within 1e-3 of the oracle encoder (eval mode) on the device's positional features, and the saved rows equal
    (f(q) + f(k)) / 2 of those batches."""
    from gcc_b200.datasets import downstream
    from gcc_b200.datasets.data_util import BatchedSubgraphs
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    from oracle import model as om
    from oracle import rwr as orwr
    tmp, ckpt, folder = work
    monkeypatch.chdir(tmp)
    g = _hub_multigraph() if name == "hubs" else downstream.node_dataset_graph(name)
    model, opt = _encoder(ckpt)
    params = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    B = 16
    ds = NodeClassificationDataset(g, rw_hops=opt.rw_hops, subgraph_size=opt.subgraph_size,
                                   restart_prob=opt.restart_prob, positional_embedding_size=opt.positional_embedding_size,
                                   device="cuda", seed=getattr(opt, "seed", 0), batch_size=B)
    dg = ds.graph
    seeds = np.arange(B, dtype=np.int64)
    want = orwr.rwr_batch(g.indptr, g.indices, dg.key, seeds, seeds, dg.budget_table.cpu().numpy(),
                          dg.restart_thresh, dg.max_budget + 65, 1 << 17)
    hub_multi = 0
    q_k = []
    for view_q, view_k, count in ds:
        buf = view_q.buffers
        for v in (0, 1):
            graphs, ip, ix, noff = _view(buf, v)
            for i, (a, w) in enumerate(zip(graphs, [want[2 * j + v] for j in range(B)])):
                assert np.array_equal(a["subv"], w["subv"]), (v, i)
                assert np.array_equal(a["indptr"], w["indptr"]), (v, i)
                assert np.array_equal(a["indices"], w["indices"]), (v, i)
                deg = np.diff(g.indptr)[w["subv"]]
                for r in np.flatnonzero(deg > 16 * w["n"]):
                    row = w["indices"][w["indptr"][r]:w["indptr"][r + 1]]
                    hub_multi += len(row) - len(np.unique(row))
            with torch.no_grad():
                feat = model(BatchedSubgraphs(buf, v)).cpu().numpy()
            N = int(noff[B])
            seed_flag = np.zeros(N, np.int64)
            seed_flag[noff[:-1]] = 1
            feat_o, _, _ = om.gin_encoder_forward(params, ip, ix, buf.pos[v, :N].cpu(), seed_flag,
                                                  buf.sub_deg[v, :N].cpu().numpy(), noff, num_layers=opt.num_layer,
                                                  max_degree=opt.max_degree, norm=True, bn_train=False,
                                                  dropout_keep=None)
            err = np.abs(feat - feat_o.numpy()).max()
            print(name, "view", v, "encoder max |device - oracle| = %.2e" % err)
            assert err <= 1e-3, err
            q_k.append(feat)
        break
    if name == "hubs":
        assert hub_multi > 0                              # parallel edges out of hub rows were induced
    emb = _generate(work, monkeypatch, name) if name != "hubs" else None
    if emb is not None:
        assert emb.shape == (g.num_nodes, opt.hidden_size)
        assert np.allclose(emb[:B], (q_k[0] + q_k[1]) / 2, rtol=1e-5, atol=1e-6)


def test_graph_dataset_rows_are_whole_graph_encodings(work, monkeypatch):
    from gcc_b200.datasets import downstream
    from gcc_b200.datasets.labeled import GraphClassificationDatasetLabeled
    tmp, ckpt, folder = work
    emb = _generate(work, monkeypatch, "imdb-binary", batch_size=8)
    graphs, labels = downstream.graph_dataset_graphs("imdb-binary")
    assert emb.shape[0] == len(graphs) == 40
    assert any(len(g.indices) != len(np.unique(np.repeat(np.arange(g.num_nodes), np.diff(g.indptr)) * g.num_nodes
                                               + g.indices)) for g in graphs)          # some graphs are multigraphs
    model, opt = _encoder(ckpt)
    for i in (0, 3, 17):
        one = GraphClassificationDatasetLabeled(([graphs[i]], labels[i:i + 1]), positional_embedding_size=opt.positional_embedding_size,
                                                batch_size=1)
        (gq, _), = list(one.batches())
        with torch.no_grad():
            row = model(gq).cpu().numpy()[0]
        assert np.allclose(emb[i], row, rtol=1e-4, atol=1e-5), (i, np.abs(emb[i] - row).max())


def _task(tmp, args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-s", "-m"] + args, cwd=tmp, env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    print(out.stdout.strip())
    return out.stdout


def test_task_clis_on_generated_rows(work, monkeypatch):
    tmp, ckpt, folder = work
    for name in ("usa_airport", "h-index-rand-1", "kdd", "icdm", "imdb-binary"):
        _generate(work, monkeypatch, name)
    H = "64"
    npy = lambda n: os.path.join(folder, n + ".npy")
    for name in ("usa_airport", "h-index-rand-1"):
        out = _task(tmp, ["gcc_b200.tasks.node_classification", "--dataset", name, "--model", "from_numpy",
                          "--hidden-size", H, "--emb-path", npy(name)])
        assert out.startswith("{'Micro-F1': ")
    out = _task(tmp, ["gcc_b200.tasks.graph_classification", "--dataset", "imdb-binary", "--model",
                      "from_numpy_graph", "--hidden-size", H, "--emb-path", npy("imdb-binary")])
    assert out.startswith("{'Micro-F1': ")
    out = _task(tmp, ["gcc_b200.tasks.similarity_search", "--dataset", "kdd_icdm", "--model", "from_numpy_align",
                      "--hidden-size", H, "--emb-path-1", npy("kdd"), "--emb-path-2", npy("icdm")])
    assert out.startswith("{'Recall @ 20': ") and "'Recall @ 40': " in out
