"""GPU (H100): the step_dist key seeds and the neighbour-sampled ego-nets against tests/augment_oracle.py bit for
bit on C2-sized batches, their positional features, PretrainEngine steps on such datasets against the oracle step,
run-ahead against serial, the sync-free epoch, the unchanged default launch sequence and generate.py's path."""
import ctypes as C

import numpy as np
import pytest
import torch

import augment_oracle as ao

pytestmark = pytest.mark.gpu

STEP = [0.5, 0.3, 0.2]
_C2 = {}


def _c2():
    if not _C2:
        from gcc_b200.datasets import synthetic
        g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
        host = lambda x: x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
        _C2.update(g=g, indptr=host(g.indptr).astype(np.int64), indices=host(g.indices).astype(np.int32))
    return _C2


def _dataset(graph, B, rw_hops, seed=7, **kw):
    from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
    return LoadBalanceGraphDataset(rw_hops=rw_hops, restart_prob=0.8, positional_embedding_size=32,
                                   dgl_graphs_file=graph, num_samples=B * 4, batch_size=B, seed=seed, **kw)


def _split(buf, v):
    noff = buf.node_off[v].cpu().numpy()
    indptr, indices, orig = (t[v].cpu().numpy() for t in (buf.indptr, buf.indices, buf.orig_id))
    out = []
    for g in range(buf.B):
        a, z = noff[g], noff[g + 1]
        ip = indptr[a:z + 1]
        out.append(dict(subv=orig[a:z], indptr=ip - ip[0], indices=indices[ip[0]:ip[-1]] - a, n=z - a))
    return out


def _spectral(buf, n_check):
    from gcc_b200 import _lib
    from test_gpu_parity import _spectral_check
    lib = _lib.get()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 0, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                               _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    raw, eig = buf.pos.cpu().numpy(), buf.eigvals.cpu().numpy()
    for v in (0, 1):
        noff = buf.node_off[v].cpu().numpy()
        for gi, s in enumerate(_split(buf, v)[:n_check]):
            _spectral_check(s, raw[v, noff[gi]:noff[gi + 1]], eig[v * buf.B + gi])


@pytest.mark.parametrize("mode", ["rwr_step", "ns2_step", "ns3", "ns5"])
def test_c2_batches_match_oracle(mode):
    c2 = _c2()
    ip, ix = c2["indptr"], c2["indices"]
    B = 64 if mode == "ns5" else 256
    if mode == "rwr_step":
        ds = _dataset(c2["g"], B, 256, seed=11, step_dist=STEP)
    elif mode == "ns5":
        # five layers at k = 5: unions of up to 3,906 vertices (cap 4,096), up to 3,125 candidates per layer, so
        # ns_expand's loops over several chunks of GCCB_ST and its sorts above 1,024 entries
        ds = _dataset(c2["g"], B, 5, seed=11, aug="ns", num_neighbors=5, step_dist=STEP, node_cap=B * 4096)
    else:
        ds = _dataset(c2["g"], B, 2 if mode == "ns2_step" else 3, seed=11, aug="ns", num_neighbors=5,
                      step_dist=STEP if mode == "ns2_step" else [1.0, 0.0, 0.0])
    buf = ds.sample_batch(first_sample=512, posenc=False)
    torch.cuda.synchronize()
    buf.check_flags()
    seeds, sids = buf.seeds.cpu().numpy(), buf.sample_ids.cpu().numpy()
    if ds.step_cdf is not None:
        cdf = ao.step_cdf(STEP)
        want_k = [ao.pair_seed(ip, ix, ds.graph.key, int(s), int(q), cdf) for s, q in zip(sids, seeds)]
        assert buf.seeds_k.cpu().numpy().tolist() == [w[1] for w in want_k]
        assert {w[0] for w in want_k} == {0, 1, 2}
        seeds_k = np.array([w[1] for w in want_k])
    else:
        seeds_k = seeds
    if mode == "rwr_step":
        want = ao.pairs_batch(ip, ix, ds.graph.key, sids, seeds, seeds_k, ds.graph.budget_table.cpu().numpy(),
                              ds.graph.restart_thresh)
    else:
        want = ao.ns_batch(ip, ix, ds.graph.key, sids, seeds, seeds_k, ds.rw_hops, 5)
    cnt = buf.counters.cpu().numpy()
    for v in (0, 1):
        for gi, (a, w) in enumerate(zip(_split(buf, v), want[v])):
            assert np.array_equal(a["subv"], w["subv"]), (v, gi)
            assert np.array_equal(a["indptr"], w["indptr"]), (v, gi)
            assert np.array_equal(a["indices"], w["indices"]), (v, gi)
            assert (cnt[v * B + gi][0], cnt[v * B + gi][1], cnt[v * B + gi][3]) == (w["n"], w["m"], w["sumdeg"])
            if mode == "rwr_step":
                assert cnt[v * B + gi][2] == w["steps"]
    if mode == "ns5":
        assert max(s["n"] for v in want for s in v) > 2 * 1024          # unions over two chunks of GCCB_ST
    else:                                                               # (dense float64 checks: small ego-nets)
        _spectral(buf, 24)


def _encoder():
    from gcc_b200.models import GraphEncoder
    return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=64,
                        node_hidden_dim=64, num_layers=5, norm=True, gnn_model="gin", degree_input=True)


def _engine(ds, prefetch=True):
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.engine import PretrainEngine
    torch.manual_seed(3)
    model, ema = _encoder(), _encoder()
    ema.load_state_dict(model.state_dict())
    model, ema = model.cuda(), ema.cuda()
    contrast = MemoryMoCo(64, None, 64, 0.07, use_softmax=True).cuda()
    return PretrainEngine(ds, model, ema, contrast, moco=True, prefetch=prefetch), model, contrast


@pytest.mark.parametrize("kw", [dict(step_dist=STEP), dict(aug="ns", rw_hops=3, num_neighbors=5),
                                dict(aug="ns", rw_hops=2, num_neighbors=5, step_dist=STEP)])
def test_engine_step_matches_oracle(kw):
    from gcc_b200.datasets import synthetic
    from oracle import step as ostep
    kw = dict(kw)
    hops = kw.pop("rw_hops", 48)
    B = 16
    ds = _dataset(synthetic.chung_lu(5000, 40000, seed=4), B, hops, seed=9, **kw)
    eng, model, contrast = _engine(ds)
    sd0 = {k: v.detach().cpu().double().clone() for k, v in model.state_dict().items()}
    state = dict(params={k: v.clone() for k, v in sd0.items()}, ema={k: v.clone() for k, v in sd0.items()},
                 memory=contrast.memory.detach().cpu().double().clone(), index=0, adam_m={}, adam_v={}, adam_t=0)
    eng.step(lr=0.005)
    torch.cuda.synchronize()
    s = eng.read_stats()
    buf = eng.cur_buf
    if "step_dist" in kw:
        assert not torch.equal(buf.seeds_k, buf.seeds)

    def view(v):
        n, m = int(buf.node_off[v, B]), int(buf.edge_off[v, B])
        noff = buf.node_off[v].cpu().numpy().astype(np.int64)
        seed = np.zeros(n, np.int64)
        seed[noff[:B]] = 1
        return dict(indptr=buf.indptr[v, :n + 1].cpu().numpy().astype(np.int64),
                    indices=buf.indices[v, :m].cpu().numpy().astype(np.int64),
                    pos=buf.pos[v, :n].cpu().double().numpy(), seed=seed,
                    sub_deg=buf.sub_deg[v, :n].cpu().numpy(), node_off=noff)

    r = ostep.train_step(state, view(0), view(1), num_layers=5, moco=True, T=0.07, lr=0.005,
                         dropout_key=model.dropout_key, step_index=0)
    assert np.isclose(s["loss"], r["loss"], rtol=1e-3), (s["loss"], r["loss"])
    assert np.isclose(s["grad_norm"], r["grad_norm"], rtol=2e-3)
    assert np.allclose(eng.feat_q.cpu().numpy(), r["feat_q"].numpy(), rtol=1e-3, atol=1e-4)
    sd1 = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    # the weight check of test_gpu_parity.test_engine_step_matches_oracle_and_learns: the first Adam update is
    # sign-like, and biases feeding a BatchNorm have an exactly-zero true gradient
    for k, v in state["params"].items():
        if ("mlp.linears" in k and k.endswith("bias")) or (k.endswith("running_mean") and "apply_func" in k) \
                or k.endswith("num_batches_tracked") or k.endswith(".eps"):
            continue
        diff = np.abs(sd1[k] - v.numpy())
        assert diff.max() <= 2 * 0.005 + 1e-6, (k, diff.max())
        assert (diff > 5e-5).mean() < 0.02, (k, (diff > 5e-5).mean())
    assert np.allclose(contrast.memory.cpu().numpy(), state["memory"].numpy(), atol=1e-4)


@pytest.mark.parametrize("kw", [dict(step_dist=STEP), dict(aug="ns", num_neighbors=5, step_dist=STEP)])
def test_run_ahead_equals_serial_and_epoch_is_sync_free(kw):
    from gcc_b200.datasets import synthetic
    B = 32
    g = synthetic.chung_lu(5000, 40000, seed=5)
    hops = 3 if kw.get("aug") == "ns" else 32
    ahead, _, _ = _engine(_dataset(g, B, hops, seed=21, **kw), prefetch=4)
    serial, _, _ = _engine(_dataset(g, B, hops, seed=21, **kw), prefetch=0)
    for _ in range(6):
        got = []
        for eng in (ahead, serial):
            eng.step(lr=0.001)
            torch.cuda.synchronize()
            b = eng.cur_buf
            cut = [b.seeds.cpu(), b.seeds_k.cpu(), b.node_off.cpu()]
            for v in (0, 1):                                    # the filled part: the ring's buffers differ beyond it
                n, m = int(b.node_off[v, B]), int(b.edge_off[v, B])
                cut += [b.orig_id[v, :n].cpu(), b.indptr[v, :n + 1].cpu(), b.indices[v, :m].cpu()]
            got.append(cut)
        for a, z in zip(*got):
            assert torch.equal(a, z)
    # one epoch (total // B steps) with no host sync
    ds = ahead.ds
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(ds.total // B):
            ahead.step(lr=0.001)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert np.isfinite(ahead.read_stats()["loss"])


def _sampler_kernels(ds):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ds.sample_batch(first_sample=0, posenc=False)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return [n.split("(")[0].replace("void ", "") for n in names if "gccb" in n or "kernel" in n]


def test_default_launch_sequence_unchanged():
    from gcc_b200 import _lib
    from gcc_b200.datasets import synthetic
    g = synthetic.chung_lu(5000, 40000, seed=6)
    ds = _dataset(g, 32, 32)
    lib = _lib.get()
    c0 = lib.gccb_launch_count()
    ds.sample_batch(first_sample=0, posenc=False)
    assert lib.gccb_launch_count() - c0 == 4                     # draw seeds, walk, offsets, fill
    names = _sampler_kernels(ds)
    assert names == ["gccb::draw_seeds_kernel", "gccb::rwr_walk_unique_kernel<0>", "gccb::batch_offsets_kernel",
                     "gccb::induce_fill_kernel"], names
    assert "pair_seeds_kernel" in _sampler_kernels(_dataset(g, 32, 32, step_dist=STEP))[1]
    assert "rwr_walk_unique_kernel<2>" in _sampler_kernels(_dataset(g, 32, 3, aug="ns"))[1]


def test_node_dataset_step_dist_through_generate():
    import argparse

    import generate
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    g = synthetic.chung_lu(700, 4000, seed=8)
    nodes = NodeClassificationDataset(dataset=g, rw_hops=16, restart_prob=0.8, positional_embedding_size=32,
                                      step_dist=STEP, device="cuda", seed=3, batch_size=256)
    model = _encoder().cuda().eval()
    emb = generate.test_moco(nodes, model, argparse.Namespace(hidden_size=64, device="cuda"))
    assert emb.shape == (g.num_nodes, 64) and torch.isfinite(emb).all()
