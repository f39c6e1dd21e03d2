"""GPU parity, round 2: the cases VERDICT r01 found uncovered -- every eigensolver size class, one full
BASELINE-config-2 batch (1M / 20M Chung-Lu, B = 256, rw_hops 256) bit-exact against the C oracle with a
spectral check of all 512 ego-nets, the fused InfoNCE / E2E heads at their real sizes, hidden = 256, the
skip-step protocol under run-ahead, and replica identity on 2 GPUs."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_parity import _dataset, _fill_batch, _split

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Residual bars (||L x - theta x||, unit x, evaluated in float64 on the float32 output):
#   n <= 160 (93% of a config-2 batch): 1e-4 -- round 2 reaches 4e-5 there (round-1 bar: 3e-4);
#   n > 160 (hub-like ego-nets): the documented stagnation bar of posenc.cu (GCCB_CF_STAG = 2e-3, +25% for the
#   float64 re-evaluation): their spectrum has a near-degenerate cluster (around 1/sqrt 2: pendant paths of a hub)
#   wider than the 48-column block, which converges only to the cluster's own spread.  The eigenVALUES are still
#   exact to 5e-5 (error quadratic in the residual) and the basis is orthonormal to 1e-4.
#   Inside that cluster (spread up to ~1e-3) WHICH members make the top-32 cut is not resolved either, so the
#   eigenvalue bar for n > 160 is the cluster spread, 1e-3 (2e-5 everywhere else).
RES_SMALL, RES_HUB, HUB_N, LAM_SMALL, LAM_HUB = 1e-4, 2.5e-3, 160, 2e-5, 1e-3
# The dense tridiagonal solver (posenc.cu solver (0); n <= 96 by default, GCCB200_DENSE_MAX=228 up to 228) is a direct
# method: eigenvalues to 2e-6, residuals and orthonormality to 2e-5 (measured on the fp32 model: 5e-7 / 4e-6 / 3e-6),
# hub-like ego-nets included.
DENSE_N, RES_DENSE, LAM_DENSE = {"default": 96, "dense": 228}, 2e-5, 2e-6


@pytest.fixture(params=["default", "dense"])
def solver(request, monkeypatch):
    """gccb_posenc reads GCCB200_DENSE_MAX on every call: unset is the shipped dispatch, 228 sends every ego-net up
    to 228 vertices to the dense solver."""
    if request.param == "dense":
        monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    else:
        monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
    return request.param


def _bars(n, solver):
    if n <= DENSE_N[solver]:
        return RES_DENSE, LAM_DENSE
    return (RES_HUB, LAM_HUB) if n > HUB_N else (RES_SMALL, LAM_SMALL)


def _eig_class(n, solver):
    """The size class posenc.cu sends an n-vertex ego-net to (eig_class)."""
    if n <= DENSE_N[solver]:
        return "dense<=%d" % next(c for c in (96, 144, 228) if n <= c)
    return "chfsi<=%s" % next((c for c in (160, 384, 1536, 3584) if n <= c), "L2")


def _spectral(sub, u, lam, res_bar, tol_l):
    from oracle import posenc as opos
    n = sub["n"]
    k = min(n - 2, 32)
    if k <= 0:
        assert np.all(u == 0)
        return 0.0, 0.0
    lap = opos.normalized_adjacency(sub["indptr"], sub["indices"], n).toarray()
    w = np.linalg.eigvalsh(lap)[-k:]
    assert np.allclose(lam[:k], w, atol=tol_l), (n, np.abs(lam[:k] - w).max())
    theta, resid, ortho = opos.spectral_report(lap, u[:, :k].astype(np.float64))
    assert resid.max() < res_bar and ortho < 1e-4, (n, resid.max(), ortho)
    assert np.all(u[:, k:] == 0)
    return float(resid.max()), float(ortho)


def _posenc_raw(buf):
    from gcc_b200 import _lib
    lib = _lib.get()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 0, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                               _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return buf.pos.cpu().numpy().copy(), buf.eigvals.cpu().numpy().copy()


def test_eigensolver_every_size_class(solver):
    """One explicit ego-net per solver class: the dense solver (n 40, 93), shared-memory ChFSI (152, 309), cluster
    ChFSI with 192-row slabs (505, 1445, and a 701-vertex star: eigenvalue 0 x 699) and 448-row slabs (2859); with
    the dense solver up to 228, the 152-vertex ego-net goes through its n <= 228 class instead."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import BatchBuffers
    graphs = [synthetic.erdos_renyi(40, 90, seed=1), synthetic.chung_lu(95, 250, seed=2),
              synthetic.chung_lu(156, 420, seed=3), synthetic.chung_lu(320, 900, exponent=0.7, seed=4),
              synthetic.chung_lu(560, 1500, exponent=0.8, seed=3), synthetic.chung_lu(1700, 5000, exponent=0.9, seed=4),
              synthetic.chung_lu(3500, 9000, exponent=0.9, seed=5), synthetic.star_graph(700)]
    subs = [dict(indptr=g.indptr.astype(np.int32), indices=g.indices.astype(np.int32), n=g.num_nodes) for g in graphs]
    sizes = [s["n"] for s in subs]
    cls = [_eig_class(n, solver) for n in sizes]
    want = {"default": ["chfsi<=1536", "chfsi<=160", "chfsi<=3584", "chfsi<=384", "dense<=96"],
            "dense": ["chfsi<=1536", "chfsi<=3584", "chfsi<=384", "dense<=228", "dense<=96"]}
    assert sorted(set(cls)) == want[solver], (sizes, cls)
    B = 4
    views = [subs[:4], subs[4:]]
    N = max(sum(s["n"] for s in v) for v in views)
    E = max(sum(len(s["indices"]) for s in v) for v in views)
    buf = BatchBuffers(B, N + 8, E + 8, 32, 64, "cuda")
    _fill_batch(buf, views)
    raw, eig = _posenc_raw(buf)
    buf.check_flags()
    noff = buf.node_off.cpu().numpy()
    it, res = buf.eig_debug()
    report = []
    for i, s in enumerate(subs):
        v, gi = divmod(i, B)
        bar, lbar = _bars(s["n"], solver)
        r, o = _spectral(s, raw[v, noff[v, gi]:noff[v, gi + 1]], eig[v * B + gi], bar, lbar)
        report.append((s["n"], int(it[v * B + gi]), r))
    print("eigensolver classes [%s] (n, iterations, max residual):" % solver, report)


def test_dense_eigensolver_class_boundaries(monkeypatch):
    """The dense tridiagonal solver at the edges of its classes (96 / 144 / 228), on exactly degenerate spectra
    (a 200-leaf star, a disconnected union), on paths (already tridiagonal), on k = 1..3, and on the sampled
    ego-net with a 15-fold eigenvalue (tests/golden/egonet_cluster15.npz)."""
    monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import BatchBuffers
    graphs = [synthetic.path_graph(3), synthetic.path_graph(4), synthetic.path_graph(5), synthetic.star_graph(33),
              synthetic.path_graph(96), synthetic.chung_lu(100, 250, seed=1), synthetic.chung_lu(150, 400, seed=2),
              synthetic.chung_lu(156, 420, seed=3), synthetic.path_graph(228), synthetic.star_graph(200),
              synthetic.disjoint_union([synthetic.star_graph(30), synthetic.star_graph(30), synthetic.path_graph(20)]),
              synthetic.erdos_renyi(228, 2000, seed=3), synthetic.chung_lu(240, 640, exponent=0.8, seed=5)]
    subs = [dict(indptr=g.indptr.astype(np.int32), indices=g.indices.astype(np.int32), n=g.num_nodes) for g in graphs]
    z = np.load(os.path.join(ROOT, "tests", "golden", "egonet_cluster15.npz"))
    subs.append(dict(indptr=z["indptr"].astype(np.int32), indices=z["indices"].astype(np.int32), n=len(z["indptr"]) - 1))
    assert max(s["n"] for s in subs) <= DENSE_N["dense"]
    B = len(subs) // 2
    views = [subs[:B], subs[B:]]
    N = max(sum(s["n"] for s in v) for v in views)
    E = max(sum(len(s["indices"]) for s in v) for v in views)
    buf = BatchBuffers(B, N + 8, E + 8, 32, 64, "cuda")
    _fill_batch(buf, views)
    raw, eig = _posenc_raw(buf)
    assert int(buf.flags.item()) == 0
    noff = buf.node_off.cpu().numpy()
    it, res = buf.eig_debug()
    worst = 0.0
    for i, s in enumerate(subs):
        v, gi = divmod(i, B)
        r, o = _spectral(s, raw[v, noff[v, gi]:noff[v, gi + 1]], eig[v * B + gi], RES_DENSE, LAM_DENSE)
        assert o < 2e-5, (s["n"], o)
        worst = max(worst, r)
    print("dense eigensolver: worst residual %.2e (fp64 re-evaluation), kernel-side %.2e" % (worst, float(res.max())))
    raw2, eig2 = _posenc_raw(buf)                          # deterministic run to run
    assert np.array_equal(raw, raw2) and np.array_equal(eig, eig2)


@pytest.fixture(scope="module")
def c2_batch():
    """One batch of BASELINE config 2 on the device + the C oracle's answer for the same samples."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
    from oracle import rwr as orwr
    g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
    B = 256
    ds = LoadBalanceGraphDataset(rw_hops=256, restart_prob=0.8, positional_embedding_size=32, dgl_graphs_file=g,
                                 num_samples=2000, num_workers=12, num_copies=6, batch_size=B, seed=0)
    buf = ds.sample_batch(first_sample=0, posenc=False)
    torch.cuda.synchronize()
    buf.check_flags()
    indptr, indices = g.indptr.cpu().numpy(), g.indices.cpu().numpy()
    seeds = orwr.draw_seeds(orwr.seed_cdf(indptr), 0, range(B))
    bt = orwr.budget_table(int(np.diff(indptr).max()), 256, 0.8)
    want = orwr.rwr_batch(indptr, indices, 0, np.arange(B), seeds, bt, orwr.restart_threshold(0.8),
                          int(bt.max()) + 65, 1 << 21)
    return dict(ds=ds, buf=buf, want=want, seeds=seeds, B=B, max_budget=int(bt.max()))


def test_c2_batch_sampler_bit_exact(c2_batch):
    """All 512 ego-nets of a config-2 batch (walk budgets up to ~3.3k, hub rows reverse-probed): seeds,
    vertex order, induced CSR and counters equal the C oracle's integer for integer."""
    buf, want, B = c2_batch["buf"], c2_batch["want"], c2_batch["B"]
    assert np.array_equal(buf.seeds.cpu().numpy(), c2_batch["seeds"])
    cnt = buf.counters.cpu().numpy()
    sizes = []
    for v in (0, 1):
        got = _split(buf, v)
        for gi in range(B):
            w = want[2 * gi + v]
            assert np.array_equal(got[gi]["subv"], w["subv"]), (v, gi)
            assert np.array_equal(got[gi]["indptr"], w["indptr"]), (v, gi)
            assert np.array_equal(got[gi]["indices"], w["indices"]), (v, gi)
            assert tuple(cnt[v * B + gi]) == (w["n"], w["m"], w["steps"], w["sumdeg"])
            sizes.append(w["n"])
    print("C2 batch: ego-net sizes mean %.1f max %d; walk budget max %d" % (np.mean(sizes), max(sizes), c2_batch["max_budget"]))
    assert max(sizes) > 384                                # a hub ego-net (cluster eigensolver class) is present


def test_c2_batch_posenc_spectral_every_egonet(c2_batch, solver):
    """Spectral parity of ALL 512 ego-nets of the batch, with the residual bar of each solver class."""
    buf, B = c2_batch["buf"], c2_batch["B"]
    raw, eig = _posenc_raw(buf)
    flags = int(buf.flags.item())
    buf.flags.zero_()
    it, res = buf.eig_debug()
    it, res = it.cpu().numpy(), res.cpu().numpy()
    noff = buf.node_off.cpu().numpy()
    worst_small = worst_hub = 0.0
    nhub = 0
    for v in (0, 1):
        for gi, s in enumerate(_split(buf, v)):
            hub = s["n"] > HUB_N
            bar, lbar = _bars(s["n"], solver)
            r, _ = _spectral(s, raw[v, noff[v, gi]:noff[v, gi + 1]], eig[v * B + gi], bar, lbar)
            if hub:
                worst_hub, nhub = max(worst_hub, r), nhub + 1
            else:
                worst_small = max(worst_small, r)
    ch = it > 0
    print("C2 batch eigensolver [%s]: NOCONV flag %d; ChFSI ego-nets %d, iterations mean %.2f max %d; worst residual "
          "n<=160: %.2e, n>160 (%d): %.2e; kernel-side residual max %.2e" % (
              solver, (flags >> 3) & 1, int(ch.sum()), it[ch].mean() if ch.any() else 0.0, it.max(), worst_small, nhub,
              worst_hub, res.max()))


def test_c2_batch_engine_step_matches_oracle(c2_batch):
    """One full MoCo step (K = 16384, 5-layer GIN hid 64, B = 256) on the config-2 batch against the CPU
    oracle step fed the same batch and positional features: loss, feat_q, pre-clip gradient norm <= 1e-3."""
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    from oracle import step as ostep
    ds, B = c2_batch["ds"], c2_batch["B"]
    torch.manual_seed(1)
    H, L, K = 64, 5, 16384

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                            node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True)

    model, ema = mk(), mk()
    ema.load_state_dict(model.state_dict())
    model, ema = model.cuda(), ema.cuda()
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).cuda()
    eng = PretrainEngine(ds, model, ema, contrast, moco=True, prefetch=0)
    sd0 = {k: v.detach().cpu().double().clone() for k, v in model.state_dict().items()}
    state = dict(params={k: v.clone() for k, v in sd0.items()}, ema={k: v.clone() for k, v in sd0.items()},
                 memory=contrast.memory.detach().cpu().double().clone(), index=0, adam_m={}, adam_v={}, adam_t=0)
    eng.step(lr=0.005)
    s = eng.read_stats()
    buf = eng.cur_buf

    def view(v):
        n, m = int(buf.node_off[v, B]), int(buf.edge_off[v, B])
        noff = buf.node_off[v].cpu().numpy().astype(np.int64)
        seed = np.zeros(n, np.int64)
        seed[noff[:B]] = 1
        return dict(indptr=buf.indptr[v, :n + 1].cpu().numpy().astype(np.int64),
                    indices=buf.indices[v, :m].cpu().numpy().astype(np.int64),
                    pos=buf.pos[v, :n].cpu().double().numpy(), seed=seed,
                    sub_deg=buf.sub_deg[v, :n].cpu().numpy(), node_off=noff)

    r = ostep.train_step(state, view(0), view(1), num_layers=L, moco=True, T=0.07, lr=0.005,
                         dropout_key=model.dropout_key, step_index=0)
    assert np.isclose(s["loss"], r["loss"], rtol=1e-3), (s["loss"], r["loss"])
    assert np.isclose(s["grad_norm"], r["grad_norm"], rtol=2e-3), (s["grad_norm"], r["grad_norm"])
    fq, fk = eng.feat_q.cpu().numpy(), eng.feat_k.cpu().numpy()
    assert np.allclose(fq, r["feat_q"].numpy(), rtol=1e-3, atol=1e-4), np.abs(fq - r["feat_q"].numpy()).max()
    assert np.allclose(fk, r["feat_k"].numpy(), rtol=1e-3, atol=1e-4)
    print("C2 step: loss %.6f (oracle %.6f), grad norm %.5f (oracle %.5f), nodes %d/%d" % (
        s["loss"], r["loss"], s["grad_norm"], r["grad_norm"], s["nodes_q"], s["nodes_k"]))


@pytest.mark.parametrize("B,K,d", [(256, 16384, 64), (1024, 65536, 256), (100, 1000, 128)])
def test_fused_infonce_real_sizes(B, K, d):
    """gccb_infonce_fused at the config-2 and config-4 head sizes against float64 torch: loss, mean positive
    logit and dq (memory_moco.py:33-44 + criterions.py:12-17 + backward)."""
    from gcc_b200 import _lib
    lib = _lib.get()
    g = torch.Generator(device="cuda").manual_seed(B + K)
    q = torch.nn.functional.normalize(torch.randn(B, d, device="cuda", generator=g), dim=1)
    k = torch.nn.functional.normalize(q + 0.3 * torch.randn(B, d, device="cuda", generator=g), dim=1)
    stdv = 1.0 / (d / 3) ** 0.5
    mem = (torch.rand(K, d, device="cuda", generator=g) * 2 * stdv - stdv)
    mem[:K // 2] = torch.nn.functional.normalize(mem[:K // 2], dim=1)          # a half-filled queue: both regimes
    stats = torch.zeros(4, device="cuda")
    dq = torch.zeros(B, d, device="cuda")
    ws = torch.empty(lib.gccb_infonce_workspace(B, d, K), dtype=torch.uint8, device="cuda")
    _lib.check(lib.gccb_infonce_fused(_lib.dptr(q), _lib.dptr(k), _lib.dptr(mem), B, d, K, 0.07, _lib.dptr(stats),
                                      _lib.dptr(dq), _lib.dptr(ws), ws.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tc = d >= 128 and B >= 128 and K % 64 == 0      # tensor-core path (moco.cu: nce_use_tc)
    q64 = q.double().requires_grad_(True)
    # tensor-core path: the two big products take bf16 operands -> the oracle rounds q / queue the same way for the
    # negatives (the positive logit stays fp32 in the kernel)
    rnd = (lambda t: t.to(torch.bfloat16).double()) if tc else (lambda t: t.double())
    qn = q64 + (rnd(q) - q.double()).detach()
    out = torch.cat([(q64 * k.double()).sum(1, keepdim=True), qn @ rnd(mem).t()], 1) / 0.07
    loss = torch.nn.functional.cross_entropy(out, torch.zeros(B, dtype=torch.long, device="cuda"))
    loss.backward()
    tol = 1e-4 if tc else 1e-5
    assert np.isclose(float(stats[0]), float(loss), rtol=tol), (float(stats[0]), float(loss))
    assert np.isclose(float(stats[1]), float(out[:, 0].mean()), rtol=1e-5)
    want = q64.grad
    scale = float(want.abs().max())
    err = float((dq.double() - want).abs().max() / scale)
    # dq = P . queue with P rounded to bf16 on the tensor-core path: 2^-9 relative per probability
    assert err < (1e-2 if tc else 1e-3), err
    if tc:
        q0 = q.double().requires_grad_(True)
        out0 = torch.cat([(q0 * k.double()).sum(1, keepdim=True), q0 @ mem.double().t()], 1) / 0.07
        l0 = torch.nn.functional.cross_entropy(out0, torch.zeros(B, dtype=torch.long, device="cuda"))
        print("tensor-core InfoNCE B=%d K=%d d=%d: loss %.6f; bf16-operand oracle %.6f; unrounded fp64 %.6f (rel %.1e); "
              "dq max err / scale vs rounded oracle %.1e" % (B, K, d, float(stats[0]), float(loss), float(l0),
                                                             abs(float(stats[0]) - float(l0)) / float(l0), err))


@pytest.mark.parametrize("B,d", [(32, 32), (256, 64), (100, 256)])
def test_e2e_head_matches_float64(B, d):
    """gccb_e2e_nce (train.py:397-401 + criterions.py:27-33): loss, mean diagonal logit, dq and dk."""
    from gcc_b200 import _lib
    lib = _lib.get()
    g = torch.Generator(device="cuda").manual_seed(B * d)
    q = torch.nn.functional.normalize(torch.randn(B, d, device="cuda", generator=g), dim=1)
    k = torch.nn.functional.normalize(q + 0.5 * torch.randn(B, d, device="cuda", generator=g), dim=1)
    stats = torch.zeros(4, device="cuda")
    dq, dk = torch.zeros(B, d, device="cuda"), torch.zeros(B, d, device="cuda")
    ws = torch.empty(B * B * 4, dtype=torch.uint8, device="cuda")
    _lib.check(lib.gccb_e2e_nce(_lib.dptr(q), _lib.dptr(k), B, d, 0.07, _lib.dptr(stats), _lib.dptr(dq), _lib.dptr(dk),
                                _lib.dptr(ws), ws.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    q64, k64 = q.double().requires_grad_(True), k.double().requires_grad_(True)
    out = k64 @ q64.t() / 0.07
    loss = torch.nn.functional.cross_entropy(out, torch.arange(B, device="cuda"))
    loss.backward()
    assert np.isclose(float(stats[0]), float(loss), rtol=1e-5)
    assert np.isclose(float(stats[1]), float(out.diagonal().mean()), rtol=1e-5)
    for got, want in ((dq, q64.grad), (dk, k64.grad)):
        scale = float(want.abs().max())
        assert torch.allclose(got.double(), want, rtol=1e-3, atol=1e-5 * scale)


@pytest.mark.parametrize("H,tc", [(256, 1), (256, 0), (128, 1)])
def test_gin_wide_forward_backward_vs_oracle(H, tc):
    """BASELINE config 4 width: GraphEncoder(hidden 256 / 128, 5 layers) forward + backward through the module
    API against the torch-CPU float64 oracle with autograd.
      tc = 0: fp32 SIMT kernels vs the plain oracle: embeddings <= 1e-3, gradients <= 5e-3 of their scale.
      tc = 1: wgmma path (bf16 operands, fp32 accumulation in registers) vs the oracle with ITS GEMM operands rounded
              to bf16 the same way: embeddings <= 2e-3 (rms 3e-4) of the (unit) row norm -- what is left is the tensor core's
              forward rounding-boundary flips (an fp32 vs fp64 operand landing on the other side of a bf16
              boundary) through 8 chained GEMMs + BatchNorms.  Gradients: this BatchNorm/ReLU stack is very
              sensitive to operand rounding -- the ORACLE's own gradients move by 10-35% of their scale when its
              operands are rounded to bf16 (profiles/wide_grad_check.py measures it) -- so the bar for the tensor-core
              backward (which also rounds dz) is statistical: per weight tensor relative L2 error <= 8e-2 and
              cosine >= 0.995 against the bf16-operand oracle.
    fp32 (tc = 0) gradients are compared elementwise, allowing isolated ReLU-kink flips (one pre-activation within
    fp32 noise of zero moves one row or column of a gradient): >= 99% of the entries within 5e-3, none beyond 5e-2.
    Against the UNROUNDED fp64 oracle the tensor-core embeddings are printed, not asserted (bf16 operands)."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.data_util import BatchedSubgraphs
    from gcc_b200.models import GraphEncoder
    from gcc_b200.models import layout as glayout
    from oracle import model as om
    torch.manual_seed(5)
    g = synthetic.chung_lu(4000, 30000, seed=6)
    B, L = 24, 5
    ds = _dataset(g, B, 64, seed=3)
    buf = ds.sample_batch(first_sample=0)
    torch.cuda.synchronize()
    buf.check_flags()
    model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                         node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True)
    model.cfg.tensor_cores = tc
    model = model.cuda()
    model.train()
    model.gnn.drop.eval()                                   # dropout off: its mask parity is covered elsewhere
    gq = BatchedSubgraphs(buf, 0)
    sd0 = {k: v.detach().cpu().double().clone() for k, v in model.state_dict().items()}
    feat = model(gq)
    R = torch.randn(B, H, device="cuda")
    (feat * R).sum().backward()
    torch.cuda.synchronize()
    n, m = int(buf.node_off[0, B]), int(buf.edge_off[0, B])
    noff = buf.node_off[0].cpu().numpy().astype(np.int64)
    seed = np.zeros(n, np.int64)
    seed[noff[:B]] = 1
    P = {k: (v.clone().requires_grad_(True) if not k.endswith(("running_mean", "running_var", ".eps", "num_batches_tracked")) else v)
         for k, v in sd0.items()}
    args = (buf.indptr[0, :n + 1].cpu().numpy().astype(np.int64), buf.indices[0, :m].cpu().numpy().astype(np.int64),
            buf.pos[0, :n].cpu().double(), seed, buf.sub_deg[0, :n].cpu().numpy(), noff)
    f, _, _ = om.gin_encoder_forward(P, *args, num_layers=L, bn_train=True,
                                     gemm_operand_dtype=torch.bfloat16 if tc else None)
    got_f, want_f = feat.detach().cpu().numpy(), f.detach().numpy()
    if tc:
        # rows have unit norm.  The flips are a noise quantity that moves with the inputs: 3.5e-4 .. 1.04e-3 (max) were
        # measured on the same ego-nets with positional features from the two eigensolvers, hence a 2e-3 bar on the
        # largest entry and 3e-4 on the root mean square
        dmax, drms = np.abs(got_f - want_f).max(), float(np.sqrt(np.mean((got_f - want_f) ** 2)))
        assert dmax < 2e-3 and drms < 3e-4, (dmax, drms)
        print("hidden %d tensor-core embeddings vs the bf16-operand oracle: max |diff| %.2e, rms %.2e" % (H, dmax, drms))
    else:
        assert np.allclose(got_f, want_f, rtol=1e-3, atol=1e-4), np.abs(got_f - want_f).max()
    if tc:
        with torch.no_grad():
            f64, _, _ = om.gin_encoder_forward({k: v.detach() for k, v in P.items()}, *args, num_layers=L, bn_train=True)
        print("hidden %d tensor-core embeddings vs the unrounded fp64 oracle: max |diff| %.2e (unit-norm rows)" % (
            H, np.abs(got_f - f64.numpy()).max()))
    (f * R.cpu().double()).sum().backward()
    checked = 0
    worst_l2, worst_cos = 0.0, 1.0
    for name, p in model.named_parameters():
        if p.grad is None or name.startswith(("set2set", "lin_readout")):
            continue
        if "mlp.linears" in name and name.endswith("bias"):
            continue                                    # exactly-zero true gradient (feeds a BatchNorm)
        want = P[name].grad
        want = np.zeros(tuple(p.shape)) if want is None else want.numpy()
        got = p.grad.cpu().numpy().astype(np.float64)
        scale = max(np.abs(want).max(), 1e-6)
        if tc:
            if scale < 1e-2:
                continue                                # near-zero gradients (apply_func.bn.weight at init): no signal
            l2 = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-12)
            cos = float((got * want).sum() / max(np.linalg.norm(got) * np.linalg.norm(want), 1e-12))
            worst_l2, worst_cos = max(worst_l2, l2), min(worst_cos, cos)
            assert l2 <= 8e-2 and cos >= 0.995, (name, l2, cos)
        else:
            bad = np.abs(got - want) > 5e-3 * np.abs(want) + 5e-3 * scale
            assert bad.mean() <= 1e-2 and np.abs(got - want).max() <= 5e-2 * scale, \
                (name, float(bad.mean()), np.abs(got - want).max(), scale)
        checked += 1
    if tc:
        print("hidden %d tensor-core gradients vs the bf16-operand oracle: worst relative L2 %.3f, worst cosine %.5f" % (
            H, worst_l2, worst_cos))
    assert checked >= 30


def test_overflowed_batch_is_skipped_under_prefetch():
    """ADVICE r01: with run-ahead on, a batch whose view overflows node_cap is published empty; the step must
    leave weights, Adam state, queue and BatchNorm running statistics untouched, and read_stats() must raise
    whichever ring buffer carried the flag."""
    from gcc_b200 import _lib
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.datasets import synthetic
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    torch.manual_seed(0)
    g = synthetic.erdos_renyi(1000, 5000, seed=0)
    ds = _dataset(g, 16, 64, node_cap=100, edge_cap=100000)     # far too small: every batch overflows

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=64,
                            node_hidden_dim=64, num_layers=3, norm=True, gnn_model="gin", degree_input=True)

    model, ema = mk(), mk()
    ema.load_state_dict(model.state_dict())
    model, ema = model.cuda(), ema.cuda()
    contrast = MemoryMoCo(64, None, 64, 0.07, use_softmax=True).cuda()
    eng = PretrainEngine(ds, model, ema, contrast, moco=True, prefetch=4)
    snap = [t.detach().clone() for t in (model.flat_params, ema.flat_params, contrast.memory, model._running,
                                          ema._running, eng.adam_m, eng.adam_v)]
    for _ in range(7):                                           # steps land on several ring slots
        eng.step(lr=0.005)
    torch.cuda.synchronize()
    now = (model.flat_params, ema.flat_params, contrast.memory, model._running, ema._running, eng.adam_m, eng.adam_v)
    for a, b in zip(snap, now):
        assert torch.equal(a, b)
    assert int(eng.index_dev.item()) == 0
    assert torch.isfinite(eng.stats).all()
    with pytest.raises(_lib.GccbError):
        eng.read_stats()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_replicas_stay_identical():
    """5 data-parallel steps on 2 GPUs over NCCL: parameters, EMA parameters and queues hash identically on
    both ranks, and the summed gradient equals the sum of the two single-GPU shards (tests/dist_replica_check.py)."""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29517",
                        os.path.join(ROOT, "tests", "dist_replica_check.py")], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and "REPLICAS IDENTICAL" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
