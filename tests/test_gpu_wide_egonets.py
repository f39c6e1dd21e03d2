"""GPU (H100): ego-nets whose walk budget does not fit the walk CTA's shared memory (the sampler's wide path) in the
datasets that meet them: a node dataset around a hub of 40,000 neighbours (plain-degree budget about 79,000) against
the oracle bit for bit, its positional features against scipy, generate.py's embedding pass over every node, and
pretraining steps on a graph with a hub of 500,000 neighbours (deg^0.75 budget about 37,000)."""
import argparse
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WALK_BUDGET_MAX = 32768 - 64
FLAG_EIG_NOCONV = 8


def _with_hub(n_rest, pairs, hub_deg, seed):
    """Vertex 0 joined to vertices 1..hub_deg, beside a Chung-Lu graph on vertices 1..n_rest."""
    from gcc_b200.datasets import synthetic
    g = synthetic.chung_lu(n_rest, pairs, exponent=0.5, seed=seed)
    src = np.repeat(np.arange(g.num_nodes, dtype=np.int64), np.diff(g.indptr)) + 1
    dst = g.indices.astype(np.int64) + 1
    src = np.concatenate([src, np.zeros(hub_deg, np.int64)])
    dst = np.concatenate([dst, np.arange(1, hub_deg + 1, dtype=np.int64)])
    out = synthetic.from_pairs(src, dst, max(g.num_nodes, hub_deg) + 1, "hub%d" % hub_deg)
    assert np.diff(out.indptr)[0] == hub_deg
    return out


_G40 = {}


def _g40():
    if not _G40:
        _G40["g"] = _with_hub(60000, 300000, 40000, seed=11)
    return _G40["g"]


def _nodes(g, B):
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    return NodeClassificationDataset(dataset=g, rw_hops=256, restart_prob=0.8, positional_embedding_size=32,
                                     device="cuda", seed=5, batch_size=B)


def _split(buf, v):
    noff = buf.node_off[v].cpu().numpy()
    indptr, indices, orig = (t[v].cpu().numpy() for t in (buf.indptr, buf.indices, buf.orig_id))
    out = []
    for g in range(buf.B):
        a, z = noff[g], noff[g + 1]
        ip = indptr[a:z + 1]
        out.append(dict(subv=orig[a:z], indptr=ip - ip[0], indices=indices[ip[0]:ip[-1]] - a, n=z - a))
    return out


def _spectral_sparse(sub, u, lam):
    """test_gpu_parity._spectral_check's tolerances, with scipy's Lanczos for the exact top-k (a dense eigh of a
    40,000-vertex ego-net does not fit)."""
    from scipy.sparse import linalg

    from oracle import posenc as opos
    n = sub["n"]
    k = min(n - 2, 32)
    lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n)
    w = np.sort(linalg.eigsh(lap, k=k, which="LA", return_eigenvectors=False, tol=1e-10, maxiter=100000))
    assert np.allclose(lam[:k], w, atol=2e-5), np.abs(lam[:k] - w).max()
    _, resid, ortho = opos.spectral_report(lap, u[:, :k].astype(np.float64))
    assert resid.max() < 3e-4 and ortho < 1e-4, (resid.max(), ortho)
    assert np.all(u[:, k:] == 0)


def test_node_dataset_around_a_40k_hub_matches_oracle_and_its_features_are_spectral():
    from oracle import rwr as orwr
    g = _g40()
    ds = _nodes(g, 64)
    deg = np.diff(g.indptr)
    bt = ds.graph.budget_table.cpu().numpy()
    assert ds.graph.max_budget > WALK_BUDGET_MAX and bt[deg[0]] > 75000
    buf = ds.sample_batch(first_sample=0, posenc=True)           # items 0..63: the hub and 63 of its neighbours
    torch.cuda.synchronize()
    assert int(buf.flags.item()) & ~FLAG_EIG_NOCONV == 0
    counters = buf.counters.cpu().numpy()
    for v in (0, 1):
        for i, s in enumerate(_split(buf, v)):
            w = orwr.rwr_subgraph(g.indptr, g.indices, ds.graph.key, i, v, i, int(bt[deg[i]]), ds.graph.restart_thresh)
            assert np.array_equal(s["subv"], w["subv"]), (v, i)
            assert np.array_equal(s["indptr"], w["indptr"]), (v, i)
            assert np.array_equal(s["indices"], w["indices"]), (v, i)
            assert tuple(counters[v * 64 + i]) == (w["n"], w["m"], w["steps"], w["sumdeg"]), (v, i)
    assert np.isfinite(buf.pos.cpu().numpy()).all() and np.isfinite(buf.eigvals.cpu().numpy()).all()
    # the raw eigenvectors (not row-normalised), as test_gpu_parity checks them
    from gcc_b200 import _lib
    _lib.check(_lib.get().gccb_posenc(C.byref(buf.c), 32, 0, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                                      _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    pos, eig = buf.pos.cpu().numpy(), buf.eigvals.cpu().numpy()
    s = _split(buf, 0)[0]
    assert s["n"] > 30000
    noff = buf.node_off[0].cpu().numpy()
    _spectral_sparse(s, pos[0, noff[0]:noff[1]], eig[0])


def test_generate_embeds_every_node_of_a_graph_with_a_40k_hub():
    import generate
    from gcc_b200.models import GraphEncoder
    g = _g40()
    torch.manual_seed(0)
    model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=64,
                         node_hidden_dim=64, num_layers=5, norm=True, gnn_model="gin", degree_input=True).cuda().eval()
    ds = _nodes(g, 256)
    with torch.no_grad():                                        # the hub's batch: each view's rows are unit-norm
        q, k, _ = next(iter(ds))
        for f in (model(q), model(k)):
            assert torch.isfinite(f).all() and torch.allclose(f.norm(dim=1), torch.ones(256, device="cuda"), atol=1e-4)
    emb = generate.test_moco(ds, model, argparse.Namespace(hidden_size=64, device="cuda"))
    assert emb.shape == (g.num_nodes, 64) and torch.isfinite(emb).all()
    nrm = emb.norm(dim=1)                                        # the mean of two unit vectors
    assert (nrm > 0).all() and (nrm <= 1 + 1e-5).all()


def test_pretraining_steps_on_a_graph_with_a_500k_hub():
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    g = _with_hub(520000, 1_000_000, 500000, seed=12)
    B = 32
    ds = LoadBalanceGraphDataset(rw_hops=256, restart_prob=0.8, positional_embedding_size=32, dgl_graphs_file=g,
                                 num_samples=B * 8, batch_size=B, seed=3)
    assert ds.graph.max_budget > WALK_BUDGET_MAX
    seeds = torch.arange(B, dtype=torch.int64, device="cuda") * 7919 + 1
    seeds[3] = 0
    buf = ds.sample_batch(first_sample=0, seeds=seeds)
    torch.cuda.synchronize()
    assert int(buf.flags.item()) & ~FLAG_EIG_NOCONV == 0
    counters = buf.counters.cpu().numpy()
    assert counters[3, 2] > WALK_BUDGET_MAX and counters[B + 3, 2] > WALK_BUDGET_MAX   # the hub's walks: wide
    assert np.isfinite(buf.pos[0, :int(buf.node_off[0, B])].cpu().numpy()).all()

    def encoder():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=64,
                            node_hidden_dim=64, num_layers=5, norm=True, gnn_model="gin", degree_input=True)
    torch.manual_seed(3)
    model, ema = encoder().cuda(), encoder().cuda()
    ema.load_state_dict(model.state_dict())
    contrast = MemoryMoCo(64, None, 64, 0.07, use_softmax=True).cuda()
    eng = PretrainEngine(ds, model, ema, contrast, moco=True, prefetch=0)
    for _ in range(4):
        eng.step(lr=0.001)
        torch.cuda.synchronize()
        assert int(eng.cur_buf.flags.item()) & 3 == 0            # no node / edge overflow
        assert np.isfinite(eng.read_stats()["loss"])
