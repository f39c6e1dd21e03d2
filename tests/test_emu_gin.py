"""CPU: GIN forward / backward, MoCo head and optimiser kernels under the fiber emulator
versus the torch-CPU oracle (which tests/test_oracle_golden.py pins to the real reference).
Kernel LOGIC only; the parity gate proper is tests/test_gpu_*.py on an H100."""
import ctypes as C

import numpy as np
import pytest
import torch

from emu_util import NpBatch, lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets import synthetic
from gcc_b200.models import layout as glayout
from oracle import model as om
from oracle import posenc as opos
from oracle import rwr as orwr


def _batch(B=5, hops=12, seed=3):
    g = synthetic.erdos_renyi(200, 700, seed=seed)
    cdf = orwr.seed_cdf(g.indptr)
    bt = orwr.budget_table(int(np.diff(g.indptr).max()), hops, 0.8)
    rt = orwr.restart_threshold(0.8)
    seeds = orwr.draw_seeds(cdf, 11, range(B))
    subs = orwr.rwr_batch(g.indptr, g.indices, 11, np.arange(B), seeds, bt, rt, int(bt.max()) + 65, 1 << 14)
    views = [[subs[2 * i + v] for i in range(B)] for v in (0, 1)]
    b = NpBatch.from_subgraphs(views)
    pos = np.zeros((2, b.node_cap, 32), np.float32)
    for v in (0, 1):
        for gi, s in enumerate(views[v]):
            a = b.node_off[v, gi]
            pos[v, a:a + s["n"]] = opos.posenc_exact(s["indptr"], s["indices"], s["n"], 32)
    return b, views, pos


def _params(cfg, rng):
    sl, total = glayout.param_slices(cfg)
    flat = np.zeros(total, np.float32)
    sd = {}
    for key, (off, shape) in sl.items():
        n = int(np.prod(shape))
        if key.endswith("weight") and len(shape) == 1:          # BN gamma
            val = rng.uniform(0.5, 1.5, n)
        elif key.endswith("bias"):
            val = rng.normal(0, 0.1, n)
        elif key == "degree_embedding.weight":
            val = rng.normal(0, 1.0, n)
        else:
            val = rng.normal(0, 1.0 / np.sqrt(shape[1]), n)
        flat[off:off + n] = val
        sd[key] = torch.from_numpy(flat[off:off + n].reshape(shape).copy()).double()
    for l in range(cfg.num_layers - 1):
        sd["gnn.ginlayers.%d.eps" % l] = torch.zeros(1, dtype=torch.double)
    return flat, sd, sl


def _oracle_view(b, views, pos, v):
    N = int(b.node_off[v, b.B])
    return dict(indptr=b.indptr[v, :N + 1].astype(np.int64), indices=b.indices[v, :b.edge_off[v, b.B]].astype(np.int64),
                pos=pos[v, :N], seed=(np.arange(N)[:, None] == b.node_off[v, :b.B][None, :]).any(1).astype(np.int64),
                sub_deg=b.sub_deg[v, :N], node_off=b.node_off[v].astype(np.int64))


@pytest.mark.parametrize("L,H,B_,hops", [(3, 32, 5, 12), (5, 64, 5, 12), (3, 64, 14, 28), (3, 128, 5, 12), (5, 256, 6, 16), (5, 128, 24, 64)])
def test_gin_forward_backward_vs_oracle(L, H, B_, hops):
    """(the third case spans several 64-row tiles: graphs straddle tile boundaries in the pooling,
    aggregation and weight-gradient kernels)"""
    rng = np.random.default_rng(L * 100 + H)
    b, views, pos = _batch(B_, hops)
    assert B_ < 10 or int(b.node_off[0, b.B]) > 128
    print("N =", int(b.node_off[0, b.B]))
    _forward_backward_vs_oracle(lib(), L, H, b, views, pos, rng)


def _forward_backward_vs_oracle(Lb, L, H, b, views, pos, rng, kink_flips=0):
    """Both views through gccb_gin_forward / gccb_gin_backward (train mode, dropout on view 0) against the float64
    oracle and its autograd gradients; the running statistics are updated by both forwards.  Gradients: every entry
    within rtol 2e-3 + 2e-4 of the tensor's scale, except at most `kink_flips` entries per tensor, which must still be
    within 5e-3 of the scale (a ReLU pre-activation within fp32 noise of zero lands on the other side of the kink)."""
    cfg = glayout.make_cfg(num_layers=L, hidden=H)
    lay = glayout.c_layout(Lb, cfg)
    flat, sd, sl = _params(cfg, rng)
    assert lay.total == len(flat) and lay.emb == sl["degree_embedding.weight"][0]
    assert lay.w2[1] == sl["gnn.ginlayers.1.apply_func.mlp.linears.1.weight"][0]
    rs, rtotal = glayout.running_slices(cfg)
    assert lay.run_total == rtotal
    running = np.zeros(rtotal, np.float32)
    for key, (off, shape) in rs.items():
        running[off:off + shape[0]] = 1.0 if key.endswith("var") else 0.0
    running0 = running.copy()
    nbt = np.zeros(3 * (L - 1), np.int64)
    acts = np.zeros(Lb.gccb_gin_acts_bytes(C.byref(cfg), b.B, b.node_cap), np.uint8)
    B = b.B
    key, step = 77, 5
    for view, drop_base in ((0, 0), (1, -1)):
        feat = np.zeros((B, H), np.float32)
        pooled = np.zeros((L - 1, B, H), np.float32)
        rc = Lb.gccb_gin_forward(C.byref(cfg), C.byref(b.c), view, ptr(pos), ptr(flat), ptr(running), ptr(nbt), 1,
                                 key, step, drop_base, ptr(acts), acts.nbytes, ptr(feat), ptr(pooled), None)
        assert rc == 0, Lb.gccb_last_error()
        ov = _oracle_view(b, views, pos, view)
        P = {k: v.clone().requires_grad_(not k.endswith("eps")) for k, v in sd.items()}
        keep = None
        if drop_base >= 0:
            keep = [orwr.dropout_mask(key, step, drop_base + i, B * H, 0.5).reshape(B, H) for i in range(L)]
        f_o, outs_o, stats_o = om.gin_encoder_forward(P, ov["indptr"], ov["indices"], torch.from_numpy(ov["pos"]).double(),
                                                      ov["seed"], ov["sub_deg"], ov["node_off"], num_layers=L,
                                                      dropout_keep=keep)
        assert np.allclose(feat, f_o.detach().numpy(), rtol=1e-3, atol=2e-5), np.abs(feat - f_o.detach().numpy()).max()
        for i in range(L - 1):
            assert np.allclose(pooled[i], outs_o[i].detach().numpy(), rtol=1e-3, atol=1e-3)
        # backward: loss = sum(feat * w)
        w = rng.normal(0, 1, (B, H)).astype(np.float32)
        grads = np.zeros_like(flat)
        ws = np.zeros(Lb.gccb_gin_backward_workspace(C.byref(cfg), B, b.node_cap), np.uint8)
        rc = Lb.gccb_gin_backward(C.byref(cfg), C.byref(b.c), view, ptr(flat), ptr(acts), ptr(w), ptr(grads),
                                  key, step, drop_base, ptr(ws), ws.nbytes, None)
        assert rc == 0, Lb.gccb_last_error()
        loss = (f_o * torch.from_numpy(w).double()).sum()
        names = [k for k in sl]
        g_o = torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)
        for k_, go in zip(names, g_o):
            off, shape = sl[k_]
            got = grads[off:off + int(np.prod(shape))].reshape(shape)
            want = go.numpy() if go is not None else np.zeros(shape)
            scale = max(np.abs(want).max(), 1e-3)
            if "mlp.linears" in k_ and k_.endswith("bias"):
                # bias feeding a train-mode BatchNorm: the true gradient is exactly 0; fp32 gives noise
                assert np.abs(got).max() < 1e-5, (view, k_, np.abs(got).max())
                continue
            bad = ~np.isclose(got, want, rtol=2e-3, atol=2e-4 * scale)
            assert bad.sum() <= kink_flips and np.abs(got - want).max() <= 5e-3 * scale, \
                (view, k_, int(bad.sum()), np.abs(got - want).max(), scale)
    # running statistics: both forwards updated the same buffers (two train-mode passes)
    assert np.all(nbt == 2)
    assert not np.allclose(running, running0)


def _spread_degree_batch():
    """Two ego-nets (the same in both views, in swapped order) whose rows have every degree residue mod 8 between 4
    and 300: centre i is joined to leaves 0 .. d_i - 1 of a shared leaf pool, d_i = 4 .. 19, 250 .. 257 and 300, so
    leaf j has degree #{i : d_i > j} and the pool spans the degrees in between."""
    def net(ds, extra):
        n_c, n_l = len(ds), max(ds) + extra
        src = np.concatenate([np.full(d, i) for i, d in enumerate(ds)])
        dst = n_c + np.concatenate([np.arange(d) for d in ds])
        src, dst = np.concatenate([src, dst]), np.concatenate([dst, src])
        order = np.lexsort((dst, src))
        n = n_c + n_l
        indptr = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))])
        return dict(subv=np.arange(n), indptr=indptr, indices=dst[order], n=n, m=len(src))
    g0 = net(list(range(4, 20)) + list(range(250, 258)) + [300], 3)
    g1 = net([5, 13, 21, 29, 37, 45, 53, 61, 120, 201], 2)
    views = [[g0, g1], [g1, g0]]
    b = NpBatch.from_subgraphs(views)
    pos = np.random.default_rng(8).normal(0, 0.3, (2, b.node_cap, 32)).astype(np.float32)
    return b, views, pos


@pytest.mark.parametrize("L,H", [(3, 32), (3, 64), (3, 128)])
def test_gin_warp_gathers_at_production_hub_threshold(L, H):
    """The emulated kernels built with the product's hub threshold (GCCB_HUB_DEG = 256) instead of the tests' 3: rows
    with 4..256 neighbours take the warp gathers (gather_range: eight neighbours per step, then the remainder;
    gather_range4: four, then the remainder), in the forward aggregation and in the backward's dh gathers, and
    every residue of the degree mod 8 occurs; rows with more neighbours still take the CTA-wide hub path."""
    b, views, pos = _spread_degree_batch()
    for v in (0, 1):
        N = int(b.node_off[v, b.B])
        deg = np.diff(b.indptr[v, :N + 1])
        warp = deg[(deg >= 4) & (deg <= 256)]
        assert set(warp % 8) == set(range(8)) and (deg > 256).sum() == 2 and deg.min() <= 3
    # Rows that sum 250..300 neighbours put a few ReLU pre-activations within fp32 noise of zero: with (L, H) = (3, 64)
    # one to four entries of a tensor land on the other side of a kink and differ from the oracle by up to 2.3e-3
    # of the tensor's scale (the warp and hub gathers agree with each other to 5e-6 relative), hence kink_flips
    _forward_backward_vs_oracle(lib(production_hub_deg=True), L, H, b, views, pos, np.random.default_rng(L * 10 + H),
                                kink_flips=4)


def test_stash_layout_locates_the_forward_intermediates(monkeypatch):
    """gccb_gin_stash_layout: the emulator build has no tensor-core path, so every tensor-core field is -1 even
    when the configuration asks for tensor cores; the offsets it reports for z1, z2 and h of a layer hold what
    the oracle computes there."""
    Lb = lib()
    L, H = 3, 32
    b, views, pos = _batch(4, 12)
    for tc_cfg in (glayout.make_cfg(num_layers=4, hidden=128, tensor_cores=1), glayout.make_cfg(num_layers=L, hidden=H)):
        st = _capi.GinStash()
        assert Lb.gccb_gin_stash_layout(C.byref(tc_cfg), b.B, b.node_cap, C.byref(st)) == 0, Lb.gccb_last_error()
        for name in ("a16", "x16", "coef1", "dz16", "tA", "tB", "cap_pad", "splits"):
            assert getattr(st, name) == -1, name
        assert list(st.w16) == [-1] * 8
        nl = tc_cfg.num_layers - 1
        assert all(x >= 0 for x in list(st.z1)[:nl]) and list(st.z1)[nl:] == [-1] * (8 - nl)
        assert st.DW == st.PW == max(tc_cfg.hidden, 64) and st.dz2[1] > st.dz2[0] >= 0
    cfg = glayout.make_cfg(num_layers=L, hidden=H)
    flat, sd, _ = _params(cfg, np.random.default_rng(9))
    running = np.zeros(glayout.running_slices(cfg)[1], np.float32)
    acts = np.zeros(Lb.gccb_gin_acts_bytes(C.byref(cfg), b.B, b.node_cap), np.uint8)
    feat = np.zeros((b.B, H), np.float32)
    rc = Lb.gccb_gin_forward(C.byref(cfg), C.byref(b.c), 0, ptr(pos), ptr(flat), ptr(running), None, 1, 0, 0, -1,
                             ptr(acts), acts.nbytes, ptr(feat), None, None)
    assert rc == 0, Lb.gccb_last_error()
    ov = _oracle_view(b, views, pos, 0)
    seen = []                                    # per GIN layer the oracle normalises z1, z2, then y = relu(bn_a(z2))
    bn = om._bn

    def record(x, *a, **k):
        y = bn(x, *a, **k)
        seen.append((x.detach(), y.detach()))
        return y
    monkeypatch.setattr(om, "_bn", record)
    om.gin_encoder_forward(sd, ov["indptr"], ov["indices"], torch.from_numpy(ov["pos"]).double(), ov["seed"],
                           ov["sub_deg"], ov["node_off"], num_layers=L)
    N, l = int(b.node_off[0, b.B]), 1
    for got_off, want in ((st.z1[l], seen[3 * l][0]), (st.z2[l], seen[3 * l + 1][0]),
                          (st.h[l], torch.relu(seen[3 * l + 2][1]))):
        got = acts[got_off:got_off + N * H * 4].view(np.float32).reshape(N, H)
        assert np.allclose(got, want.numpy(), rtol=1e-4, atol=1e-4 * float(want.abs().max())), \
            np.abs(got - want.numpy()).max()


def test_moco_head_fused_at_d32_and_optimiser_vs_oracle():
    Lb = lib()
    rng = np.random.default_rng(0)
    B, d, K, T = 6, 16, 50, 0.07
    q = rng.normal(size=(B, d)).astype(np.float32); q /= np.linalg.norm(q, axis=1, keepdims=True)
    k = rng.normal(size=(B, d)).astype(np.float32); k /= np.linalg.norm(k, axis=1, keepdims=True)
    mem = rng.uniform(-1, 1, (K, d)).astype(np.float32)
    tq = torch.from_numpy(q).double().requires_grad_(True)
    out_o = om.moco_logits(tq, torch.from_numpy(k).double(), torch.from_numpy(mem).double(), T)
    loss_o = om.nce_softmax_loss(out_o)
    (dq_o,) = torch.autograd.grad(loss_o, tq)
    out = np.zeros((B, K + 1), np.float32)
    assert Lb.gccb_moco_logits(ptr(q), ptr(k), ptr(mem), B, d, K, T, ptr(out), None) == 0
    assert np.allclose(out, out_o.detach().numpy(), rtol=1e-5, atol=1e-5)
    loss = np.zeros(1, np.float32); dout = np.zeros_like(out)
    assert Lb.gccb_nce_loss(ptr(out), B, K + 1, 0, ptr(loss), ptr(dout), None) == 0
    assert np.isclose(loss[0], float(loss_o), rtol=1e-5)
    dq = np.zeros_like(q)
    assert Lb.gccb_moco_logits_backward(ptr(dout), ptr(k), ptr(mem), B, d, K, T, ptr(dq), None) == 0
    assert np.allclose(dq, dq_o.numpy(), rtol=1e-4, atol=1e-6)
    # fused, at the encoder width 32: zero columns appended to q, k and the queue leave the loss and dq unchanged
    dp = 32
    qp, kp, memp = (np.pad(a, ((0, 0), (0, dp - d))) for a in (q, k, mem))
    stats = np.zeros(2, np.float32); dq2 = np.zeros_like(qp)
    ws = np.zeros(Lb.gccb_infonce_workspace(B, dp, K), np.uint8)
    assert Lb.gccb_infonce_fused(ptr(qp), ptr(kp), ptr(memp), B, dp, K, T, ptr(stats), ptr(dq2), ptr(ws), ws.nbytes,
                                 None) == 0
    assert np.isclose(stats[0], float(loss_o), rtol=1e-5)
    assert np.isclose(stats[1], out_o[:, 0].mean().item(), rtol=1e-5)
    assert np.allclose(dq2[:, :d], dq_o.numpy(), rtol=1e-4, atol=1e-6) and not dq2[:, d:].any()
    # label-arange mode + E2E head
    sq = out[:, :B].copy()
    assert Lb.gccb_nce_loss(ptr(sq), B, B, 1, ptr(loss), None, None) == 0
    assert np.isclose(loss[0], float(om.nce_softmax_loss_ns(torch.from_numpy(sq).double())), rtol=1e-5)
    tq2 = torch.from_numpy(q).double().requires_grad_(True); tk2 = torch.from_numpy(k).double().requires_grad_(True)
    lo = om.nce_softmax_loss_ns(tk2 @ tq2.t() / T)
    gq, gk = torch.autograd.grad(lo, [tq2, tk2])
    dq3 = np.zeros_like(q); dk3 = np.zeros_like(k); ws2 = np.zeros(B * B, np.float32)
    assert Lb.gccb_e2e_nce(ptr(q), ptr(k), B, d, T, ptr(stats), ptr(dq3), ptr(dk3), ptr(ws2), ws2.nbytes, None) == 0
    assert np.isclose(stats[0], float(lo), rtol=1e-5)
    assert np.allclose(dq3, gq.numpy(), rtol=1e-4, atol=1e-6) and np.allclose(dk3, gk.numpy(), rtol=1e-4, atol=1e-6)
    # enqueue with wrap-around
    idx = np.array([K - 4], np.int64)
    mem2 = mem.copy(); tm = torch.from_numpy(mem.copy())
    assert Lb.gccb_moco_enqueue(ptr(mem2), ptr(k), B, d, K, ptr(idx), 1, 0, None, 0, None) == 0
    new_idx = om.moco_enqueue(tm, torch.from_numpy(k), K - 4)
    assert idx[0] == new_idx == 2 and np.array_equal(mem2, tm.numpy())
    # a skipped step (batch published empty: overflow bits set in the flag word) leaves queue and pointer alone
    skip = np.array([2], np.int32); mem3 = mem2.copy(); idx3 = idx.copy()
    assert Lb.gccb_moco_enqueue(ptr(mem3), ptr(k), B, d, K, ptr(idx3), 1, 0, ptr(skip), 3, None) == 0
    assert idx3[0] == idx[0] and np.array_equal(mem3, mem2)
    # several ranks' keys from one gathered buffer, in rank order, one launch
    parts, stride = 3, B * d + 7
    gk_ = rng.normal(size=(parts, stride)).astype(np.float32)
    idx4 = np.array([K - 3], np.int64); mem4 = mem.copy(); tm4 = torch.from_numpy(mem.copy()); ii = K - 3
    assert Lb.gccb_moco_enqueue(ptr(mem4), ptr(gk_), B, d, K, ptr(idx4), parts, stride, None, 0, None) == 0
    for r in range(parts):
        ii = om.moco_enqueue(tm4, torch.from_numpy(gk_[r, :B * d].reshape(B, d).copy()), ii)
    assert idx4[0] == ii and np.array_equal(mem4, tm4.numpy())
    # clip + Adam + EMA
    n_live, n_all = 1000, 1300
    p = rng.normal(size=n_all).astype(np.float32); g = rng.normal(size=n_live).astype(np.float32)
    m = rng.normal(size=n_live).astype(np.float32) * 0.1; v = np.abs(rng.normal(size=n_live)).astype(np.float32) * 0.01
    pe = rng.normal(size=n_all).astype(np.float32)
    p_o, g_o, m_o, v_o, pe_o = [x.astype(np.float64) for x in (p, g, m, v, pe)]
    t, lr = 7, 0.004
    gn_o = om.clip_adam_ema(p_o[:n_live], g_o, m_o, v_o, None, t, lr)
    om.ema_update(pe_o, p_o, 0.999)
    hyper = np.array([lr, 1 - 0.9 ** t, np.sqrt(1 - 0.999 ** t), 0], np.float32)
    gn = np.zeros(1, np.float32); wsd = np.zeros(1, np.float64)
    assert Lb.gccb_clip_adam_ema(ptr(p), ptr(g), ptr(m), ptr(v), ptr(pe), n_live, n_all, ptr(hyper), 0.9, 0.999, 1e-8,
                                 1e-5, 1.0, 0.999, 1.0, ptr(gn), ptr(wsd), None, 0, None) == 0
    assert np.isclose(gn[0], gn_o, rtol=1e-5)
    assert np.allclose(p, p_o, rtol=1e-5, atol=1e-6) and np.allclose(m, m_o, rtol=1e-5, atol=1e-7)
    assert np.allclose(v, v_o, rtol=1e-5, atol=1e-9) and np.allclose(pe, pe_o, rtol=1e-5, atol=1e-6)
    gathered = rng.normal(size=(3, 40)).astype(np.float32); outs = np.zeros(32, np.float32)
    anyf = np.array([7], np.int32)
    gathered[:, 35] = 0.0
    assert Lb.gccb_sum_ranks(ptr(gathered), 3, 40, 32, ptr(outs), 35, ptr(anyf), None) == 0
    assert np.allclose(outs, gathered[:, :32].sum(0), rtol=1e-6) and anyf[0] == 0
    gathered[1, 35] = 2.0
    assert Lb.gccb_sum_ranks(ptr(gathered), 3, 40, 32, ptr(outs), 35, ptr(anyf), None) == 0 and anyf[0] == 1
    # the skip word makes the optimiser a no-op
    snap = [x.copy() for x in (p, m, v, pe)]
    assert Lb.gccb_clip_adam_ema(ptr(p), ptr(g), ptr(m), ptr(v), ptr(pe), n_live, n_all, ptr(hyper), 0.9, 0.999, 1e-8,
                                 1e-5, 1.0, 0.999, 1.0, ptr(gn), ptr(wsd), ptr(anyf), -1, None) == 0
    assert all(np.array_equal(a, b) for a, b in zip(snap, (p, m, v, pe)))


@pytest.mark.parametrize("B,d,K", [(37, 32, 300), (5, 64, 129), (33, 128, 64), (9, 256, 200)])
def test_fused_infonce_tiled_kernel_ragged_shapes(B, d, K):
    """The tiled InfoNCE kernel (d in {32, 64, 128, 256}: 32 query rows x 128 / 64 keys per CTA) with
    row counts and queue sizes that are not multiples of its tiles, against memory_moco.py:26-53 +
    criterions.py:12-17 (oracle)."""
    Lb = lib()
    rng = np.random.default_rng(B * 1000 + d)
    T = 0.07
    q = rng.normal(size=(B, d)).astype(np.float32); q /= np.linalg.norm(q, axis=1, keepdims=True)
    k = rng.normal(size=(B, d)).astype(np.float32); k /= np.linalg.norm(k, axis=1, keepdims=True)
    mem = rng.uniform(-1, 1, (K, d)).astype(np.float32); mem /= np.linalg.norm(mem, axis=1, keepdims=True)
    tq = torch.from_numpy(q).double().requires_grad_(True)
    out_o = om.moco_logits(tq, torch.from_numpy(k).double(), torch.from_numpy(mem).double(), T)
    loss_o = om.nce_softmax_loss(out_o)
    (dq_o,) = torch.autograd.grad(loss_o, tq)
    stats = np.zeros(2, np.float32); dq = np.zeros_like(q)
    ws = np.zeros(Lb.gccb_infonce_workspace(B, d, K), np.uint8)
    rc = Lb.gccb_infonce_fused(ptr(q), ptr(k), ptr(mem), B, d, K, T, ptr(stats), ptr(dq), ptr(ws), ws.nbytes, None)
    assert rc == 0, Lb.gccb_last_error()
    assert np.isclose(stats[0], float(loss_o), rtol=2e-5), (stats[0], float(loss_o))
    assert np.isclose(stats[1], out_o[:, 0].mean().item(), rtol=2e-5)
    assert np.allclose(dq, dq_o.numpy(), rtol=2e-4, atol=2e-6), np.abs(dq - dq_o.numpy()).max()


def test_fused_infonce_refuses_other_widths():
    """The fused head has kernels for the encoder widths only: d = 48 is refused with a message and has no
    workspace size.  The unfused logits keep taking it."""
    Lb = lib()
    B, d, K = 4, 48, 40
    q, k = np.ones((B, d), np.float32), np.ones((B, d), np.float32)
    mem = np.ones((K, d), np.float32)
    stats = np.zeros(2, np.float32); dq = np.zeros_like(q); ws = np.zeros(1 << 16, np.uint8)
    assert Lb.gccb_infonce_workspace(B, d, K) == 0
    rc = Lb.gccb_infonce_fused(ptr(q), ptr(k), ptr(mem), B, d, K, 0.07, ptr(stats), ptr(dq), ptr(ws), ws.nbytes, None)
    assert rc == _capi.GCCB_ERR_BADARG
    assert b"d = 48" in Lb.gccb_last_error()
    out = np.zeros((B, K + 1), np.float32)
    assert Lb.gccb_moco_logits(ptr(q), ptr(k), ptr(mem), B, d, K, 0.07, ptr(out), None) == 0
