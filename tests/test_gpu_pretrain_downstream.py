"""GPU: pretraining on the reference's named datasets (train.py:547-586) -- a downstream node dataset in epoch
order with its short last batch, the short-batch MoCo / E2E step against the float64 oracle step, whole-graph
batches of a TU set from gccb_gather_graphs, and train.py end to end on `--dataset usa_airport | imdb-binary | dgl`.
The data are the small reference-format files of tasks_golden.npz written into a temporary ./data."""
import os
import types

import numpy as np
import pytest
import torch

from test_gpu_downstream import _write_tu

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
H, L = 64, 3


@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("pretrain_downstream")
    z = np.load(os.path.join(GOLDEN, "tasks_golden.npz"))
    for k in z.files:
        if k.startswith("files/"):
            p = tmp / "data" / k[len("files/"):]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_text(str(z[k]))
    _write_tu(tmp / "data", "IMDB-BINARY")
    return tmp


def _node_ds(B, rw_hops=32):
    from gcc_b200.datasets import downstream
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    return NodeClassificationDataset(downstream.node_dataset_graph("usa_airport"), rw_hops=rw_hops,
                                     restart_prob=0.8, positional_embedding_size=32, device="cuda", seed=7,
                                     batch_size=B)


def _engine(ds, moco, prefetch, K=64, index=0):
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    torch.manual_seed(5)

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                            node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True)

    model, ema = mk(), mk()
    ema.load_state_dict(model.state_dict())
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).cuda()
    contrast.index = index
    return PretrainEngine(ds, model.cuda(), ema.cuda(), contrast, moco=moco, prefetch=prefetch)


def _view(buf, v):
    """View v of a batch as the oracle step takes it."""
    b = buf.B
    n, m = int(buf.node_off[v, b]), int(buf.edge_off[v, b])
    noff = buf.node_off[v].cpu().numpy().astype(np.int64)
    seed = np.zeros(n, np.int64)
    seed[noff[:b]] = 1
    return dict(indptr=buf.indptr[v, :n + 1].cpu().numpy().astype(np.int64),
                indices=buf.indices[v, :m].cpu().numpy().astype(np.int64),
                pos=buf.pos[v, :n].cpu().double().numpy(), seed=seed,
                sub_deg=buf.sub_deg[v, :n].cpu().numpy(), node_off=noff)


@pytest.mark.parametrize("prefetch", [0, 2])
def test_node_dataset_epoch_order_and_ego_nets(data_root, monkeypatch, prefetch):
    from oracle import rwr as orwr
    monkeypatch.chdir(data_root)
    B, epochs = 16, 3
    ds = _node_ds(B)
    N = ds.total
    assert N % B != 0
    steps = ds.steps_per_epoch()
    eng = _engine(ds, moco=True, prefetch=prefetch)
    dg = ds.graph
    indptr, indices = dg.indptr.cpu().numpy(), dg.indices.cpu().numpy()
    used_ids, per_epoch = [], [[] for _ in range(epochs)]
    for j in range(epochs * steps):
        eng.step(lr=0.005)
        s = eng.read_stats()                                     # syncs; the slot is intact until the next step
        buf = eng.cur_buf
        b = buf.B
        assert s["batch_size"] == b == (N % B if j % steps == steps - 1 else B)
        assert np.isfinite(s["loss"])
        seeds = buf.seeds.cpu().numpy()
        ids = buf.sample_ids.cpu().numpy()
        used_ids += ids.tolist()
        want = orwr.rwr_batch(indptr, indices, dg.key, ids, seeds, dg.budget_table.cpu().numpy(),
                              dg.restart_thresh, dg.max_budget + 65, 1 << 17)
        for v in (0, 1):
            noff = buf.node_off[v].cpu().numpy().astype(np.int64)
            N_v = int(noff[b])
            ip = buf.indptr[v, :N_v + 1].cpu().numpy().astype(np.int64)
            ix = buf.indices[v, :int(buf.edge_off[v, b])].cpu().numpy().astype(np.int64)
            orig = buf.orig_id[v, :N_v].cpu().numpy()
            assert s["nodes_q" if v == 0 else "nodes_k"] == N_v
            for i in range(b):
                a, z = noff[i], noff[i + 1]
                w = want[2 * i + v]
                assert np.array_equal(orig[a:z], w["subv"]), (j, v, i)
                assert np.array_equal(ip[a:z + 1] - ip[a], w["indptr"]), (j, v, i)
                assert np.array_equal(ix[ip[a]:ip[z]] - a, w["indices"]), (j, v, i)
            if v == 0:
                per_epoch[j // steps] += orig[noff[:b]].tolist()     # row 0 of each graph: the seed
    for e in range(epochs):
        assert per_epoch[e] == list(range(N)), e
    assert len(set(used_ids)) == len(used_ids) == epochs * N     # fresh walk randomness every epoch


def _snapshot(eng):
    m = eng.model
    st = dict(params={k: v.detach().cpu().double().clone() for k, v in m.state_dict().items()},
              ema={k: v.detach().cpu().double().clone() for k, v in eng.model_ema.state_dict().items()},
              memory=eng.contrast.memory.detach().cpu().double().clone(), index=eng.contrast.index,
              adam_m={}, adam_v={}, adam_t=eng.adam_t)
    for k, (o, shape) in m._slices.items():
        n = int(np.prod(shape))
        st["adam_m"][k] = eng.adam_m[o:o + n].view(shape).cpu().double().clone()
        st["adam_v"][k] = eng.adam_v[o:o + n].view(shape).cpu().double().clone()
    return st


def _skip(k):
    return ("mlp.linears" in k and k.endswith("bias")) or (k.endswith("running_mean") and "apply_func" in k) \
        or k.endswith("num_batches_tracked") or k.endswith(".eps")


@pytest.mark.parametrize("moco", [True, False])
def test_short_batch_step_matches_oracle(data_root, monkeypatch, moco):
    """usa_airport (40 nodes) in batches of 14: 14, 14, then a short batch of 12.  MoCo starts its queue at 28, so
    the short batch enqueues at 56 with K = 64 and wraps to rows 0..3.  The third step is checked against the
    float64 oracle step from the engine's own state.  The run-ahead ring must train on the same batches, bit for
    bit, and reach the same state as the serial run.  That state is compared to rounding, not bit for bit: the
    loss and the degree-embedding gradient are float atomic sums, so two serial runs differ in the last bits too."""
    from oracle import step as ostep
    monkeypatch.chdir(data_root)
    B, K = 14, 64
    runs = {}
    for prefetch in (0, 2):
        eng = _engine(_node_ds(B), moco=moco, prefetch=prefetch, K=K, index=28)
        losses, batches = [], []
        for j in range(3):
            if j == 2 and prefetch == 0:
                torch.cuda.synchronize()
                state = _snapshot(eng)
            eng.step(lr=0.005)
            losses.append(eng.read_stats()["loss"])
            batches.append([_view(eng.cur_buf, v) for v in (0, 1)])
        buf = eng.cur_buf
        assert buf.B == 12
        if prefetch == 0:
            if moco:
                assert state["index"] == 56
            r = ostep.train_step(state, _view(buf, 0), _view(buf, 1), num_layers=L, moco=moco, T=0.07, lr=0.005,
                                 dropout_key=eng.model.dropout_key, step_index=2)
            assert np.isclose(losses[2], r["loss"], rtol=1e-3), (losses[2], r["loss"])
            sd = {k: v.detach().cpu().numpy() for k, v in eng.model.state_dict().items()}
            for k, v in state["params"].items():
                if _skip(k):
                    continue
                diff = np.abs(sd[k] - v.numpy())
                assert diff.max() <= 2 * 0.005 + 1e-6, (k, diff.max())
                assert (diff > 5e-5).mean() < 0.02, (k, (diff > 5e-5).mean())
            if moco:
                sde = {k: v.detach().cpu().numpy() for k, v in eng.model_ema.state_dict().items()}
                for k, v in state["ema"].items():
                    if not _skip(k):
                        assert np.allclose(sde[k], v.numpy(), atol=2e-5), (k, np.abs(sde[k] - v.numpy()).max())
                mem = eng.contrast.memory.cpu().numpy()
                assert np.allclose(mem, state["memory"].numpy(), atol=1e-4)
                rows = [(56 + i) % K for i in range(12)]
                assert np.allclose(mem[rows], r["feat_k"].numpy(), atol=1e-4)
                assert eng.contrast.index == state["index"] == 4 == int(eng.index_dev.item())
            else:
                assert r["out"].shape == (12, 12)
        runs[prefetch] = dict(losses=losses, batches=batches, index=eng.contrast.index,
                              params=eng.model.flat_params[:eng.model.n_live].cpu().numpy(),
                              ema=eng.model_ema.flat_params[:eng.model.n_live].cpu().numpy(),
                              memory=eng.contrast.memory.cpu().numpy())
    a, b = runs[0], runs[2]
    for j in range(3):
        for v in (0, 1):
            for k, x in a["batches"][j][v].items():
                assert np.array_equal(x, b["batches"][j][v][k]), (j, v, k)
    assert np.allclose(a["losses"], b["losses"], rtol=1e-5, atol=0), (a["losses"], b["losses"])
    assert a["index"] == b["index"]
    for k in ("params", "ema"):
        diff = np.abs(a[k] - b[k])
        assert diff.max() <= 2 * 0.005 + 1e-6 and (diff > 5e-5).mean() < 0.02, (k, diff.max(), (diff > 5e-5).mean())
    assert np.allclose(a["memory"], b["memory"], atol=1e-5)


def test_graph_dataset_batches_are_whole_graphs(data_root, monkeypatch):
    from gcc_b200.datasets.data_util import BatchedSubgraphs
    from gcc_b200.datasets.graph_dataset import BatchBuffers, GraphClassificationDataset
    from gcc_b200.datasets.labeled import fill_whole_graphs
    from gcc_b200.models import GraphEncoder
    monkeypatch.chdir(data_root)
    B = 6
    ds = GraphClassificationDataset("imdb-binary", positional_embedding_size=32, device="cuda", batch_size=B)
    assert ds.total == 40 and ds.steps_per_epoch() == 7
    torch.manual_seed(1)
    model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                         node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True).cuda().eval()
    names = ("node_off", "edge_off", "indptr", "indices", "sub_deg", "graph_id", "orig_id")
    for j in range(ds.steps_per_epoch()):
        buf = ds.sample_batch(first_sample=j * B)
        b = buf.B
        assert b == (4 if j == 6 else B)
        buf.check_flags()
        items = [ds.items[i] for i in range(j * B, j * B + b)]
        for v in (0, 1):
            ref = BatchBuffers(b, ds.node_cap, ds.edge_cap, 32, None, "cuda")
            fill_whole_graphs(ref, items, view=v)
            N, E = int(ref.node_off[v, b]), int(ref.edge_off[v, b])
            got = dict(node_off=buf.node_off[v], edge_off=buf.edge_off[v], indptr=buf.indptr[v, :N + 1],
                       indices=buf.indices[v, :E], sub_deg=buf.sub_deg[v, :N], graph_id=buf.graph_id[v, :N],
                       orig_id=buf.orig_id[v, :N])
            want = dict(node_off=ref.node_off[v], edge_off=ref.edge_off[v], indptr=ref.indptr[v, :N + 1],
                        indices=ref.indices[v, :E], sub_deg=ref.sub_deg[v, :N], graph_id=ref.graph_id[v, :N],
                        orig_id=ref.orig_id[v, :N])
            for k in names:
                assert torch.equal(got[k], want[k]), (j, v, k)
            assert torch.equal(buf.counters[v * b:(v + 1) * b], ref.counters[v * b:(v + 1) * b])
        N = int(buf.node_off[0, b])
        assert torch.equal(buf.pos[0, :N], buf.pos[1, :N]), (j, (buf.pos[0, :N] - buf.pos[1, :N]).abs().max())
        with torch.no_grad():
            fq, fk = model(BatchedSubgraphs(buf, 0)), model(BatchedSubgraphs(buf, 1))
        assert fq.shape == (b, H) and torch.equal(fq, fk)


def _train(tmp, extra):
    import train
    args = train.parse_option(["--batch-size", "16", "--epochs", "2", "--nce-k", "64",
                               "--hidden-size", str(H), "--num-layer", str(L), "--rw-hops", "32", "--print-freq", "2",
                               "--model-path", str(tmp / "m"), "--tb-path", str(tmp / "tb")] + extra)
    train.main(args)
    ckpt = os.path.join(args.model_folder, "current.pth")
    c = torch.load(ckpt, map_location="cpu", weights_only=False)
    assert c["epoch"] == 2
    assert set(c) == {"opt", "model", "contrast", "optimizer", "epoch"} | ({"model_ema"} if args.moco else set())
    assert all(torch.isfinite(v).all() for v in c["model"].values() if v.is_floating_point())
    return ckpt, args.model_folder


def test_train_py_on_named_datasets(data_root, monkeypatch):
    import generate
    from gcc_b200.datasets import dgl_bin, synthetic
    monkeypatch.chdir(data_root)
    dgl_bin.write_dgl_bin(str(data_root / "data" / "small.bin"),
                          [synthetic.erdos_renyi(600, 3000, seed=1), synthetic.erdos_renyi(400, 2000, seed=2)])
    first, folder = _train(data_root, ["--dataset", "usa_airport", "--moco"])
    _train(data_root, ["--dataset", "imdb-binary"])
    _train(data_root, ["--dataset", "dgl", "--moco", "--num-workers", "1", "--num-copies", "1", "--num-samples", "64"])
    emb = generate.main(types.SimpleNamespace(load_path=first, dataset="usa_airport", graph_nodes=0, graph_edges=0,
                                              batch_size=16, gpu=0))
    assert emb.shape == (40, H) and torch.isfinite(emb).all()
    assert os.path.exists(os.path.join(folder, "usa_airport.npy"))
