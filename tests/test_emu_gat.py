"""CPU: the GAT encoder kernels (csrc/gat.cu) under the fiber emulator against the float64 restatement
(tests/gat_oracle.py): the forward's stashed intermediates and output, and every parameter gradient of the backward,
on a sampled batch, a batch of multigraphs (parallel edges, self loops, an isolated vertex, a one-node graph) and a
short batch.  The default emulator build sends every row with more than 3 entries through the CTA-wide hub path; the
build with the product's threshold runs the one-warp-per-row path.  Also: launch counts, the flat layout against
layout.py, and the refusal of unsupported configurations."""
import ctypes as C

import numpy as np
import pytest
import torch

import gat_oracle
from emu_util import NpBatch, lib, ptr
from gcc_b200 import _capi
from gcc_b200.models import layout as glayout
from test_emu_gin import _batch, _oracle_view


def _params(cfg, rng):
    sl, total = glayout.gat_param_slices(cfg)
    flat = np.zeros(total, np.float32)
    sd = {}
    for key, (off, shape) in sl.items():
        n = int(np.prod(shape))
        if key == "degree_embedding.weight":
            val = rng.normal(0, 1.0, n)
        elif key.endswith(("attn_l", "attn_r")):
            val = rng.normal(0, 0.5, n)
        elif len(shape) == 1:
            val = rng.normal(0, 0.1, n)
        else:
            val = rng.normal(0, 1.0 / np.sqrt(shape[1]), n)
        flat[off:off + n] = val
        sd[key] = torch.from_numpy(flat[off:off + n].reshape(shape).copy()).double()
    return flat, sd, sl


def _multigraph_batch(short=False):
    """Symmetric multigraphs: parallel edges (0-1 twice), self loops (2-2, 3-3 twice), an isolated vertex (4), a
    one-node graph without edges and a one-node graph with a self loop; a hub row (vertex 0 of the star, 11 entries).
    short: three graphs in buffers sized for more (an epoch's last batch)."""
    def graph(n, pairs):
        rows = [[] for _ in range(n)]
        for u, v in pairs:
            rows[u].append(v)
            if u != v:
                rows[v].append(u)
        indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
        indices = np.array(sum([sorted(r) for r in rows], []), np.int64)
        return dict(subv=np.arange(n), indptr=indptr, indices=indices, n=n, m=len(indices))
    g1 = graph(5, [(0, 1), (0, 1), (1, 2), (2, 2), (3, 3), (3, 3), (0, 3)])
    g2 = graph(1, [])
    g3 = graph(10, [(0, i) for i in range(1, 10)] + [(1, 2), (0, 0)])
    g4 = graph(1, [(0, 0)])
    views = [[g1, g2, g3, g4], [g3, g4, g1, g2]]
    if short:
        views = [v[:3] for v in views]
    b = NpBatch.from_subgraphs(views, node_cap=40 if short else None, edge_cap=80 if short else None)
    rng = np.random.default_rng(5)
    pos = rng.normal(0, 0.3, (2, b.node_cap, 32)).astype(np.float32)
    return b, views, pos


def _run(Lb, cfg, b, view, pos, flat, w):
    acts = np.zeros(Lb.gccb_gat_acts_bytes(C.byref(cfg), b.B, b.node_cap), np.uint8)
    feat = np.zeros((b.B, cfg.hidden), np.float32)
    rc = Lb.gccb_gat_forward(C.byref(cfg), C.byref(b.c), view, ptr(pos), ptr(flat), ptr(acts), acts.nbytes, ptr(feat),
                             None)
    assert rc == 0, Lb.gccb_last_error()
    grads = np.zeros_like(flat)
    ws = np.zeros(Lb.gccb_gat_backward_workspace(C.byref(cfg), b.B, b.node_cap), np.uint8)
    rc = Lb.gccb_gat_backward(C.byref(cfg), C.byref(b.c), view, ptr(flat), ptr(acts), ptr(w), ptr(grads), ptr(ws),
                              ws.nbytes, None)
    assert rc == 0, Lb.gccb_last_error()
    return feat, grads, acts


def _check(Lb, cfg, b, views, pos, seed=0):
    rng = np.random.default_rng(seed)
    flat, sd, sl = _params(cfg, rng)
    st = _capi.GatStash()
    assert Lb.gccb_gat_stash_layout(C.byref(cfg), b.B, b.node_cap, C.byref(st)) == 0
    H, L, nh = cfg.hidden, cfg.num_layers, cfg.num_heads
    for view in (0, 1):
        w = rng.normal(0, 1, (b.B, H)).astype(np.float32)
        feat, grads, acts = _run(Lb, cfg, b, view, pos, flat, w)
        ov = _oracle_view(b, views, pos, view)
        N = int(b.node_off[view, b.B])
        P = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        rec = {}
        f_o = gat_oracle.gat_encoder_forward(P, ov["indptr"], ov["indices"], torch.from_numpy(ov["pos"]).double(),
                                             ov["seed"], ov["sub_deg"], ov["node_off"], L, nh, cfg.set2set_iter,
                                             cfg.set2set_layers, max_degree=cfg.max_degree, record=rec)
        cap = b.node_cap
        for l in range(L):
            h = acts[st.h[l]:st.h[l] + N * H * 4].view(np.float32).reshape(N, H)
            want = rec["h"][l].detach().numpy()
            assert np.allclose(h, want, rtol=1e-4, atol=1e-4 * max(1.0, np.abs(want).max())), (view, l)
            att = acts[st.att[l]:st.att[l] + 4 * cap * nh * 4].view(np.float32).reshape(4, cap, nh)
            assert np.allclose(att[0, :N], rec["el"][l].detach().numpy(), rtol=1e-4, atol=1e-5)
            assert np.allclose(att[1, :N], rec["er"][l].detach().numpy(), rtol=1e-4, atol=1e-5)
            assert np.allclose(att[3, :N], rec["den"][l].detach().numpy(), rtol=1e-4, atol=1e-5)
        want = f_o.detach().numpy()
        assert np.allclose(feat, want, rtol=1e-4, atol=1e-5), np.abs(feat - want).max()
        loss = (f_o * torch.from_numpy(w).double()).sum()
        names = list(sl)
        g_o = torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)
        # a tensor whose true gradient vanishes (attn_r when every logit of a row sits on the same side of the
        # leaky_relu kink, so er_v shifts the row's softmax uniformly) is held to fp32 noise of the largest gradient
        floor = 1e-3 * max(float(go.abs().max()) for go in g_o if go is not None)
        for k_, go in zip(names, g_o):
            off, shape = sl[k_]
            got = grads[off:off + int(np.prod(shape))].reshape(shape)
            want = go.numpy() if go is not None else np.zeros(shape)
            scale = max(np.abs(want).max(), floor)
            assert np.allclose(got, want, rtol=1e-3, atol=1e-4 * scale), (view, k_, np.abs(got - want).max(), scale)


@pytest.mark.parametrize("L,H,nh,T,K", [(2, 32, 4, 2, 2), (3, 64, 1, 2, 1), (2, 128, 8, 1, 3), (2, 64, 4, 6, 3),
                                        (1, 256, 8, 2, 1), (1, 32, 2, 1, 1), (2, 256, 1, 2, 2), (1, 64, 4, 3, 8)])
def test_sampled_batch_vs_oracle(L, H, nh, T, K):
    """Every head width F = H / nh from 4 (8 heads at 32) to 256 (head_sum's F > 32 branch), one layer (the top
    layer is layer 0: dX0 comes straight from the Set2Set gradient), and GAT_MAXK = 8 LSTM layers."""
    b, views, pos = _batch(4, 12)
    cfg = glayout.make_gat_cfg(num_layers=L, hidden=H, num_heads=nh, set2set_iter=T, set2set_layers=K)
    _check(lib(), cfg, b, views, pos, seed=L * 7 + H)


@pytest.mark.parametrize("production_hub_deg", [False, True])
@pytest.mark.parametrize("short", [False, True])
def test_multigraph_batch_vs_oracle(production_hub_deg, short):
    b, views, pos = _multigraph_batch(short)
    cfg = glayout.make_gat_cfg(num_layers=2, hidden=64, num_heads=4, set2set_iter=2, set2set_layers=2)
    _check(lib(production_hub_deg), cfg, b, views, pos, seed=3)


def test_warp_rows_sampled_batch_vs_oracle():
    b, views, pos = _batch(4, 12)
    cfg = glayout.make_gat_cfg(num_layers=2, hidden=256, num_heads=4, set2set_iter=1, set2set_layers=1)
    _check(lib(production_hub_deg=True), cfg, b, views, pos, seed=9)


def test_hub_rows_above_production_threshold():
    """A star with 300 leaves: its centre row is above the product's hub threshold (256)."""
    n = 301
    rows = [list(range(1, n))] + [[0] for _ in range(1, n)]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    g = dict(subv=np.arange(n), indptr=indptr, indices=np.array(sum(rows, []), np.int64), n=n, m=int(indptr[-1]))
    b = NpBatch.from_subgraphs([[g], [g]])
    pos = np.random.default_rng(2).normal(0, 0.3, (2, b.node_cap, 32)).astype(np.float32)
    assert np.diff(b.indptr[0, :n + 1]).max() > 256
    cfg = glayout.make_gat_cfg(num_layers=2, hidden=32, num_heads=2, set2set_iter=1, set2set_layers=1)
    _check(lib(production_hub_deg=True), cfg, b, [[g], [g]], pos, seed=4)


# launches per call: forward = X0 + 2 per GAT layer (projection, aggregation) + per Set2Set iteration one per LSTM
# layer and one attention + readout; backward = readout + its two weight gradients + per iteration (attention + one
# per LSTM layer) + two weight gradients per LSTM layer + 5 per GAT layer (two softmax passes, split-K weight gradient
# and its reduce, dX) + degree embedding
def _launches(L, T, K):
    return 1 + 2 * L + T * (K + 1) + 1, 3 + T * (K + 1) + 2 * K + 5 * L + 1


def test_launch_counts_per_call():
    Lb = lib()
    b, views, pos = _batch(3, 8)
    for L, T, K in ((5, 6, 3), (2, 2, 1)):
        cfg = glayout.make_gat_cfg(num_layers=L, hidden=32, num_heads=4, set2set_iter=T, set2set_layers=K)
        flat, _, _ = _params(cfg, np.random.default_rng(0))
        n0 = Lb.gccb_launch_count()
        _run(Lb, cfg, b, 0, pos, flat, np.ones((b.B, 32), np.float32))
        fwd, bwd = _launches(L, T, K)
        assert (fwd, bwd) == ({(5, 6, 3): 36, (2, 2, 1): 10}[(L, T, K)], {(5, 6, 3): 59, (2, 2, 1): 20}[(L, T, K)])
        assert Lb.gccb_launch_count() - n0 == fwd + bwd


@pytest.mark.parametrize("L,nh", [(2, 1), (2, 4), (5, 1), (5, 4)])
def test_layout_matches_c(L, nh):
    cfg = glayout.make_gat_cfg(num_layers=L, hidden=64, num_heads=nh, set2set_layers=3)
    lay = glayout.gat_c_layout(lib(), cfg)
    sl, total = glayout.gat_param_slices(cfg)
    assert lay.total == total
    for i in range(L):
        assert lay.fc[i] == sl["gnn.layers.%d.gnn.fc.weight" % i][0]
        assert lay.attn_l[i] == sl["gnn.layers.%d.gnn.attn_l" % i][0]
        assert lay.attn_r[i] == sl["gnn.layers.%d.gnn.attn_r" % i][0]
    assert lay.emb == sl["degree_embedding.weight"][0]
    for k in range(3):
        for f, n in (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh")):
            assert getattr(lay, f)[k] == sl["set2set.lstm.%s_l%d" % (n, k)][0]
    assert (lay.ro0_w, lay.ro0_b, lay.ro2_w, lay.ro2_b) == tuple(
        sl["lin_readout.%s" % k][0] for k in ("0.weight", "0.bias", "2.weight", "2.bias"))


def test_unsupported_configuration_is_refused():
    Lb = lib()
    lay = _capi.GatLayout()
    for kw in (dict(hidden=48), dict(num_heads=3), dict(num_heads=16), dict(num_layers=9), dict(set2set_layers=0)):
        cfg = glayout.make_gat_cfg(**kw)
        assert Lb.gccb_gat_param_layout(C.byref(cfg), C.byref(lay)) == _capi.GCCB_ERR_BADARG, kw
