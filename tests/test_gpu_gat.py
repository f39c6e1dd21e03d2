"""GPU: the GAT encoder (gnn_model="gat", csrc/gat.cu) on an H100 against the float64 restatement
(tests/gat_oracle.py) fed the kernels' own batch and positional features: every layer's output, the embedding and
every parameter gradient at hidden 32 to 256, 1 to 8 heads and 1 / 2 / 5 layers; every stage teacher-forced from the
stored operands on sampled, hub, large, short and C2 batches (bounds derived above test_every_stage_teacher_forced);
one MoCo and one E2E engine step against the oracle's step with the GAT encoder; run-ahead against serial batches;
train.py --moco --model gat, generate.py and --finetune from its checkpoint; the two-GPU replica check with GAT.

Bounds.  The forward is fp32 with float64 in the oracle: a projection row is a K <= 256 term fmaf chain (relative
error <= K u, u = 2^-24), the edge softmax adds an exp and a division per term, the LSTM gates and the readout are
<= 3H-term dot products; over 5 layers and 6 Set2Set iterations the embedding stays within 1e-3 of its scale (the
project's bar).  Gradients compose the same chains backwards and add float atomics of CTA partials in the attention
vectors; each tensor is held to 2e-3 of its own scale, with a floor of 1e-3 of the largest gradient for tensors whose
true gradient nearly cancels.  Weights after one Adam step (lr 0.005): 2e-3 of the tensor's largest weight."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import gat_oracle
from test_gpu_pretrain_downstream import _node_ds, _view, data_root  # noqa: F401
from test_gpu_gin_stages import _batch as _gin_batch, _buffers, _er, _pair, _single, _star
from test_gpu_parity import _fill_batch
from test_gpu_tc_gin import _clique

pytestmark = pytest.mark.gpu


def _mk(H, L, nh=4, T=6, K=3):
    from gcc_b200.models import GraphEncoder
    return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                        node_hidden_dim=H, num_layers=L, num_heads=nh, num_step_set2set=T, num_layer_set2set=K,
                        norm=True, gnn_model="gat", degree_input=True)


def _sampled(B=32, hops=64):
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
    g = synthetic.chung_lu(3000, 20000, seed=0)
    ds = LoadBalanceGraphDataset(rw_hops=hops, restart_prob=0.8, dgl_graphs_file=g, num_samples=4 * B, batch_size=B,
                                 seed=3)
    return ds


def _oracle(sd, v, L, nh, T, K, record=None):
    return gat_oracle.gat_encoder_forward(sd, v["indptr"], v["indices"], torch.as_tensor(v["pos"]), v["seed"],
                                          v["sub_deg"], v["node_off"], L, nh, T, K, record=record)


def _close(got, want, rel, floor=0.0, what=""):
    scale = max(float(np.abs(want).max()), floor, 1e-30)
    err = float(np.abs(got - want).max())
    assert err <= rel * scale, (what, err, scale)
    return err / scale


@pytest.mark.parametrize("L,H,nh", [(L, H, 4) for L in (2, 5) for H in (32, 64, 128)] +
                         [(2, 256, 4), (2, 256, 1), (2, 256, 8), (1, 64, 4), (1, 256, 8)])
def test_forward_backward_vs_float64(L, H, nh):
    from gcc_b200.datasets.data_util import BatchedSubgraphs
    torch.manual_seed(H + L)
    ds = _sampled()
    buf = ds.sample_batch(first_sample=0)
    ds.posenc(buf)
    T, K = 6, 3
    model = _mk(H, L, nh, T, K).cuda()
    worst = {}
    for view in (0, 1):
        g = BatchedSubgraphs(buf, view)
        w = torch.randn(buf.B, H, device="cuda")
        feat = model(g)
        (feat * w).sum().backward()
        torch.cuda.synchronize()
        v = _view(buf, view)
        sd = {k: p.detach().cpu().double().clone().requires_grad_(True) for k, p in model.state_dict().items()}
        rec = {}
        f_o = _oracle(sd, v, L, nh, T, K, rec)
        worst["feat"] = max(worst.get("feat", 0), _close(feat.detach().cpu().numpy(), f_o.detach().numpy(), 1e-3,
                                                         what="feat"))
        (f_o * w.cpu().double()).sum().backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        floor = 1e-3 * max(float(p.grad.abs().max()) for p in sd.values())
        for k, p in sd.items():
            worst[k] = max(worst.get(k, 0), _close(grads[k].cpu().numpy(), p.grad.numpy(), 2e-3, floor, k))
        model.zero_grad()
    print("H=%d heads=%d L=%d N=%d: worst feat %.2e, worst gradient %.2e" % (
        H, nh, L, int(buf.node_off[0, buf.B]), worst["feat"], max(v for k, v in worst.items() if k != "feat")))


def _engine(ds, moco, prefetch, H=64, L=3, K=64):
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.engine import PretrainEngine
    torch.manual_seed(5)
    model, ema = _mk(H, L, T=3, K=2), _mk(H, L, T=3, K=2)
    ema.load_state_dict(model.state_dict())
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).cuda()
    return PretrainEngine(ds, model.cuda(), ema.cuda(), contrast, moco=moco, prefetch=prefetch)


@pytest.mark.parametrize("moco", [True, False])
def test_engine_step_vs_oracle_step(moco):
    """One MoCo / E2E engine step against the oracle's step with the GAT encoder (gat_oracle.train_step, i.e.
    oracle/step.py's head, loss, clip, Adam, EMA and enqueue): loss, pre-clip gradient norm, embeddings, and the
    weights (and EMA weights and queue for MoCo) after the step."""
    ds = _sampled(B=16)
    eng = _engine(ds, moco, prefetch=0)
    L, T, K, nh = 3, 3, 2, 4
    sd0 = {k: v.detach().cpu().double().clone() for k, v in eng.model.state_dict().items()}
    state = dict(params={k: v.clone() for k, v in sd0.items()}, ema={k: v.clone() for k, v in sd0.items()},
                 memory=eng.contrast.memory.detach().cpu().double().clone(), index=0, adam_m={}, adam_v={}, adam_t=0)
    eng.step(lr=0.005)
    s = eng.read_stats()
    buf = eng.cur_buf
    r = gat_oracle.train_step(state, _view(buf, 0), _view(buf, 1), num_layers=L, num_heads=nh, set2set_iter=T,
                              set2set_layers=K, moco=moco, T=eng.T, lr=0.005, alpha=eng.alpha, clip_norm=eng.clip,
                              weight_decay=eng.wd, beta1=eng.betas[0], beta2=eng.betas[1])
    assert np.isclose(s["loss"], r["loss"], rtol=1e-3), (s["loss"], r["loss"])
    assert np.isclose(s["grad_norm"], r["grad_norm"], rtol=2e-3), (s["grad_norm"], r["grad_norm"])
    _close(eng.feat_q.cpu().numpy(), r["feat_q"].numpy(), 1e-3, what="feat_q")
    _close(eng.feat_k.cpu().numpy(), r["feat_k"].numpy(), 1e-3, what="feat_k")
    # Adam divides by sqrt(v): an entry whose gradient is at fp32 noise moves by up to lr either way, so the bar is
    # 2e-3 of the tensor's largest weight, as the project's other one-step checks are
    sd1 = eng.model.state_dict()
    for k, want in state["params"].items():
        _close(sd1[k].cpu().double().numpy(), want.numpy(), 2e-3, what=k)
    if moco:
        sde = eng.model_ema.state_dict()
        for k, want in state["ema"].items():
            _close(sde[k].cpu().double().numpy(), want.numpy(), 2e-3, what="ema " + k)
        _close(eng.contrast.memory.cpu().double().numpy(), state["memory"].numpy(), 1e-3, what="queue")


def test_run_ahead_and_serial_give_the_same_batches():
    ds_a, ds_b = _sampled(B=16), _sampled(B=16)
    a, b = _engine(ds_a, True, prefetch=4), _engine(ds_b, True, prefetch=0)
    for _ in range(3):
        a.step(lr=0.005)
        b.step(lr=0.005)
        torch.cuda.synchronize()
        for v in (0, 1):
            va, vb = _view(a.cur_buf, v), _view(b.cur_buf, v)
            for k in ("indptr", "indices", "node_off", "sub_deg"):
                assert np.array_equal(va[k], vb[k]), k
    sa, sb = a.read_stats(), b.read_stats()
    assert np.isclose(sa["loss"], sb["loss"], rtol=1e-4), (sa["loss"], sb["loss"])


def test_train_generate_finetune_gat(data_root, monkeypatch):  # noqa: F811
    import generate
    import train
    monkeypatch.chdir(data_root)
    args = train.parse_option(["--batch-size", "16", "--epochs", "2", "--nce-k", "64", "--hidden-size", "32",
                               "--num-layer", "2", "--rw-hops", "32", "--print-freq", "2", "--model", "gat",
                               "--set2set-iter", "2", "--set2set-lstm-layer", "1",
                               "--model-path", str(data_root / "gat"), "--tb-path", str(data_root / "tb"),
                               "--dataset", "usa_airport", "--moco"])
    train.main(args)
    ckpt = str(data_root / "gat" / os.path.basename(args.model_folder) / "current.pth")
    c = torch.load(ckpt, map_location="cpu", weights_only=False)
    assert c["opt"].model == "gat" and "gnn.layers.1.gnn.attn_l" in c["model"]
    assert all(torch.isfinite(v).all() for v in c["model"].values())
    emb = generate.main(types.SimpleNamespace(load_path=ckpt, dataset="usa_airport", graph_nodes=0, graph_edges=0,
                                              batch_size=16, gpu=0))
    assert emb.shape[1] == 32 and torch.isfinite(emb).all()
    ft = train.parse_option(["--finetune", "--resume", ckpt, "--dataset", "usa_airport", "--epochs", "1",
                             "--batch-size", "16", "--model-path", str(data_root / "gat_ft"),
                             "--tb-path", str(data_root / "tb"), "--gpu", "0"])
    f1 = train.main_finetune(ft)
    assert 0.0 <= f1 <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# Stage by stage, teacher-forced: every stage is recomputed in float64 from the operands the kernels stored
# (gccb_gat_stash_layout) and held to a bound derived from the kernel's arithmetic.  u = 2^-24.  An fp32 chain of n
# fmaf / adds has |error| <= n u sum|terms| (to first order); a stored fp32 result adds u |result|; expf, the
# leaky_relu add and the multiplication by 1/denominator add at most 8 u relative per term (C_EXP).  So:
#   z = X W^T (K terms)                  (K + 1) u |X| |W|^T
#   el, er (F terms)                     (F + 1) u |z| |attn|
#   softmax max                          3 u |max| (the fp32 add el + er and the multiply by 0.2f each round once;
#                                        0.2f differs from 0.2 by u / 4)
#   denominator (online, deg terms)      (2 deg + C_EXP) u den   (each rescale multiplies by one more rounded exp)
#   out = sum a z (deg terms)            (deg + C_EXP) u sum a |z|, then leaky_relu (exact up to u)
#   LSTM gate pre-activations (3H)       (KI + H + 3) u (|W_ih| |x| + |W_hh| |h| + |b|); sigmoid' <= 1/4, tanh' <= 1,
#                                        plus C_EXP u for the activation itself
#   c = f c' + i g, h = o tanh(c)        C_EXP u (|f c'| + |i g|), C_EXP u |h| + |o| (c error)
#   Set2Set e_i, alpha, r                (H + 1) u |x||q|;  alpha: 2 alpha max|de| + (n + C_EXP) u alpha;  r: (n + 1) u
#                                        sum alpha |x|
#   readout                              (2H + 2) u |W0||q*| + u|b0|;  (H + 2) u |W2||y1| + u|b2|;  normalise (H + C_EXP) u
# Backward: dscore (2H + C_EXP) u (|df| + |s| sum|s df| / n^2) / n;  d1 (H + 1) u |W2|^T |d2|;  the softmax backward
# passes (deg + F + C_EXP) u times the sum of the absolute terms they add; dX = dz W (H + 1) u;  split-K weight
# gradients and the attention-vector and degree-embedding sums (rows + 1) u sum|terms| (a sum of n terms in any order,
# split-K chunks or float atomics, has depth <= n - 1).  Quantities the stage's float64 recomputation takes from
# the kernel (the stored max, denominator, gates) are not re-derived, so each bound covers one stage only.
# Hub rows (deg > HUB_DEG) take another order: warp w of the CTA walks the entries [w c, (w + 1) c), c = ceil(deg / 8),
# and the 8 partials are combined in a fixed order.  The denominator: a lane's online sum over its ceil(c / 32)
# entries (two roundings each), a 5-level warp sum after one rescaling exp, then 8 partials each rescaled by one more
# exp and added in turn: depth 2 ceil(c / 32) + 5 + 8 plus two exps <= 2 deg + C_EXP for any deg > 256.  The
# aggregation and both softmax-backward passes: c sequential fmaf per lane column, then 8 partials added in turn:
# depth c + 8 <= deg, each term with the same exp and 1/denominator as a warp row.  So the bounds above cover the hub
# order unchanged; the weight-gradient sums already allow any order.  The hub rows' attention-vector partials go to a
# per-thread sum of their own, then the shared and global atomics: still a sum of at most N terms.
# Layers above 0, whose backward buffers the next layer down overwrites, are checked against float64 autograd of the
# layers above recomputed from the stored h[l-1], at test_gpu_gin_stages' bar for middle layers (_vs_autograd).
U = 2.0 ** -24
C_EXP = 8
SMS, HUB_DEG, GB = 132, 256, 4       # GCCB_NUM_SMS, GCCB_HUB_DEG, GAT_GB


def _stage(name, got, want, bound, worst):
    got, want, bound = (torch.as_tensor(x).double() for x in (got, want, bound))
    excess = ((got - want).abs() / (bound + 1e-30)).max().item() if got.numel() else 0.0
    worst[name] = max(worst.get(name, 0.0), excess)
    assert excess <= 1.0, (name, excess, float((got - want).abs().max()))


def _vs_autograd(name, got, want, floor, mid, notes):
    """test_gpu_gin_stages' bar for middle layers: 2e-3 |want| + 2e-4 scale.  Entries outside it are counted and
    printed; they may only be isolated leaky_relu-kink flips (an output or logit within rounding of 0 takes the other
    slope): at most 0.1 % of the tensor (one in a tensor of fewer than 1000) outside 5e-3 |want| + 5e-3 scale, none
    beyond 5e-2 of the scale."""
    got, want = got.double().reshape(want.shape), want.double()
    scale = max(float(want.abs().max()), floor, 1e-30)
    err = (got - want).abs()
    r = err / (2e-3 * want.abs() + 2e-4 * scale)
    outside = int((r > 1.0).sum())
    w, o = mid.get(name, (0.0, 0))
    mid[name] = (max(w, float(r.max())), o + outside)
    if outside:
        wide = int((err > 5e-3 * want.abs() + 5e-3 * scale).sum())
        notes.append("%s: %d of %d entries outside the bar (worst %.2f of it), %d outside 5e-3, largest |err| %.2e "
                     "of the scale" % (name, outside, r.numel(), float(r.max()), wide, float(err.max()) / scale))
        assert wide <= max(1, r.numel() // 1000) and float(err.max()) <= 5e-2 * scale, (name, outside, wide)


def _gat_layer(X, Wf, al, ar, row, col, nh, act):
    """One GAT layer in the dtype and on the device of X (autograd through everything but the softmax max)."""
    N, H = X.shape[0], Wf.shape[0]
    z = (X @ Wf.t()).view(N, nh, H // nh)
    el = (z * al.reshape(nh, -1)).sum(-1)
    er = (z * ar.reshape(nh, -1)).sum(-1)
    e = torch.nn.functional.leaky_relu(el[col] + er[row], 0.2)
    mx = e.new_full((N, nh), -torch.inf).scatter_reduce(0, row[:, None].expand(-1, nh), e.detach(), "amax")
    ex = torch.exp(e - mx[row])
    a = ex / e.new_zeros(N, nh).index_add(0, row, ex)[row]
    out = e.new_zeros(N, nh, H // nh).index_add(0, row, a[:, :, None] * z[col]).reshape(N, H)
    return torch.nn.functional.leaky_relu(out, 0.01) if act else out


def _s2s_readout(x, P, gid, B, T, K, pres=None):
    """Set2Set (T iterations of a K-layer LSTM), lin_readout and F.normalize on x's device.  pres (a list) receives
    every cell's pre-activation gates, their gradients retained."""
    H = x.shape[1]
    hk = [x.new_zeros(B, H) for _ in range(K)]
    ck = [x.new_zeros(B, H) for _ in range(K)]
    q_star = x.new_zeros(B, 2 * H)
    for it in range(T):
        inp = q_star
        for k in range(K):
            pre = (inp @ P["set2set.lstm.weight_ih_l%d" % k].t() + hk[k] @ P["set2set.lstm.weight_hh_l%d" % k].t()
                   + P["set2set.lstm.bias_ih_l%d" % k] + P["set2set.lstm.bias_hh_l%d" % k])
            if pres is not None:
                if pre.requires_grad:
                    pre.retain_grad()
                else:                                    # the first cells depend on nothing that needs a gradient
                    pre = pre.detach().requires_grad_(True)
                pres.append(pre)
            i_, f_, g_, o_ = pre.split(H, 1)
            ck[k] = torch.sigmoid(f_) * ck[k] + torch.sigmoid(i_) * torch.tanh(g_)
            hk[k] = torch.sigmoid(o_) * torch.tanh(ck[k])
            inp = hk[k]
        qv = hk[K - 1]
        e_i = (x * qv[gid]).sum(1)
        emx = x.new_zeros(B).scatter_reduce(0, gid, e_i.detach(), "amax", include_self=False)
        ex = torch.exp(e_i - emx[gid])
        al = ex / x.new_zeros(B).index_add(0, gid, ex)[gid]
        q_star = torch.cat([qv, x.new_zeros(B, H).index_add(0, gid, al[:, None] * x)], 1)
    out = torch.relu(q_star @ P["lin_readout.0.weight"].t() + P["lin_readout.0.bias"]) @ P["lin_readout.2.weight"].t() \
        + P["lin_readout.2.bias"]
    return torch.nn.functional.normalize(out, eps=1e-5)


def _row_grid(cap):
    """gat.cu row_grid: CTAs of the row kernels (aggregation, both softmax-backward passes); CTA c takes the groups of
    8 rows c, c + grid, ..."""
    return min(max((cap + 7) // 8, 1), 8 * SMS)


def _tile_grid(cap):
    """gat.cu tile_grid: CTAs of the projection and dX kernels; CTA c takes the 64-row tiles c, c + grid, ..."""
    return min(max((cap + 63) // 64, 1), 4 * SMS)


def _paths(deg, cap, noff):
    """What a view reaches, restated from gat.cu's grids, its hub rule (a row with more than HUB_DEG entries is
    split across the CTA's 8 warps after the warp rows of its group) and the GAT_GB graphs per CTA of the LSTM and
    readout kernels."""
    deg, noff = deg.cpu().numpy(), noff.cpu().numpy()
    N, B = len(deg), len(noff) - 1
    hub = deg > HUB_DEG
    ng, grp = (N + 7) // 8, np.arange(N) // 8
    n_hub = np.bincount(grp, weights=hub, minlength=ng)
    n_rows = np.bincount(grp, minlength=ng)
    rg = _row_grid(cap)
    cta, rnd = np.arange(ng) % rg, np.arange(ng) // rg
    first_hub, last_warp = np.full(rg, np.inf), np.full(rg, -1.0)
    np.minimum.at(first_hub, cta[n_hub > 0], rnd[n_hub > 0])
    np.maximum.at(last_warp, cta[n_hub < n_rows], rnd[n_hub < n_rows])
    return dict(N=N, B=B, hub_rows=int(hub.sum()), all_hub_groups=int((n_hub == 8).sum()),
                mixed_groups=int(((n_hub > 0) & (n_hub < n_rows)).sum()), clamped=int((deg > 512).sum()),
                empty_rows=int((deg == 0).sum()), groups_per_cta=-(-ng // rg),
                hub_then_warp_ctas=int((first_hub < last_warp).sum()),
                tiles_per_cta=-(-((N + 63) // 64) // _tile_grid(cap)), largest_graph=int(np.diff(noff).max()),
                gb_tail=B % GB)


def _stage_batch(kind):
    if kind == "sampled":
        ds = _sampled()
        buf = ds.sample_batch(first_sample=0)
        ds.posenc(buf)
        return buf
    if kind == "hub":
        # cliques of 300 and 290 (groups of 8 hub rows), a 600-leaf star (a hub row among warp rows, its degree above
        # 512: the embedding index is clamped), a single vertex (a row without entries, a one-node Set2Set graph), a
        # pair, and random graphs past 8,448 rows: a clique's groups and then warp-row groups in the same CTA, in both
        # views (view 1 lists the graphs in reverse).  13 graphs: B is not a multiple of GAT_GB
        return _buffers([_clique(300), _star(600), _single(), _pair()] +
                        [_er(1000, 3000 + 41 * i, seed=20 + i) for i in range(8)] + [_clique(290)])
    return _gin_batch(kind)          # "large": 36 random graphs of 1,000 vertices; "c2": a C2 batch (B 256, rw_hops 256)


# (kind, H, heads, L, Set2Set iterations, LSTM layers)
CASES = [("sampled", H, 4, L, 6, 3) for L in (2, 5) for H in (32, 64, 128)] + [
    ("sampled", 256, 4, 2, 6, 3), ("sampled", 256, 8, 2, 6, 3), ("sampled", 64, 1, 2, 6, 3),
    ("sampled", 128, 2, 3, 6, 3), ("sampled", 32, 8, 2, 6, 3), ("sampled", 64, 4, 1, 6, 3),
    ("sampled", 256, 1, 1, 1, 1), ("sampled", 64, 4, 2, 2, 8),
    ("hub", 64, 1, 2, 2, 2), ("hub", 64, 4, 2, 2, 2), ("hub", 256, 1, 2, 2, 2), ("hub", 256, 4, 2, 2, 2),
    ("large", 32, 4, 2, 2, 1), ("large", 128, 4, 2, 2, 1),
    ("short", 64, 4, 2, 3, 2),
    ("c2", 64, 4, 5, 6, 3)]


@pytest.mark.parametrize("kind,H,nh,L,T,K", CASES)
def test_every_stage_teacher_forced(kind, H, nh, L, T, K):
    """Every stage of both views against its float64 recomputation from the stored operands (bounds above), the BPTT
    gate gradients and (at L = 1) the Set2Set gradient into x against float64 autograd of the Set2Set from the stored
    x, and the layers above 0 against float64 autograd from the stored h[l-1].  The references run on the GPU.
    Batches: sampled ego-nets; hub rows; N > 33,792 with 1,000-node Set2Set graphs; a narrowed batch over the stale
    rows of a larger one; a C2 batch.  Each asserts the paths it is named for."""
    from gcc_b200 import _capi, _lib
    from gcc_b200.models import layout as glayout
    dev = "cuda"
    torch.manual_seed(100 + H + L)
    F_ = H // nh
    model = _mk(H, L, nh, T, K).cuda()
    cfg, lib = model.cfg, _lib.get()

    def run(b, view, dfeat, grads):
        _lib.check(lib.gccb_gat_forward(C.byref(cfg), C.byref(b.c), view, _lib.dptr(b.pos), _lib.dptr(model.flat_params),
                                        _lib.dptr(acts), acts.numel(), _lib.dptr(feat), _lib.stream_ptr()), "fwd")
        _lib.check(lib.gccb_gat_backward(C.byref(cfg), C.byref(b.c), view, _lib.dptr(model.flat_params),
                                         _lib.dptr(acts), _lib.dptr(dfeat), _lib.dptr(grads), _lib.dptr(ws), ws.numel(),
                                         _lib.stream_ptr()), "bwd")

    if kind == "short":
        # GIN's recipe: both views of a 12-graph batch leave their activations and gradients behind, then 7 other
        # graphs are checked in the same buffers narrowed to B = 7
        full = _buffers([_er(200 + 13 * i, 700, seed=30 + i) for i in range(12)], pos_seed=9)
        acts = torch.zeros(model.acts_bytes(full.B, full.node_cap), dtype=torch.uint8, device=dev)
        ws = torch.zeros(model.backward_workspace_bytes(full.B, full.node_cap), dtype=torch.uint8, device=dev)
        feat = torch.zeros(full.B, H, device=dev)
        for view in (0, 1):
            run(full, view, torch.ones(full.B, H, device=dev), torch.zeros(model.n_live, device=dev))
        torch.cuda.synchronize()
        n_full = int(full.node_off[0, full.B])
        buf = full.narrow(7)
        graphs = [_er(150 + 11 * i, 500, seed=60 + i) for i in range(7)]
        _fill_batch(buf, [graphs, graphs[::-1]])
        n7 = int(buf.node_off[0, 7])
        buf.pos[:, :n7].copy_(0.3 * torch.randn(2, n7, 32, device=dev))
    else:
        buf = _stage_batch(kind)
        acts = torch.zeros(model.acts_bytes(buf.B, buf.node_cap), dtype=torch.uint8, device=dev)
        ws = torch.zeros(model.backward_workspace_bytes(buf.B, buf.node_cap), dtype=torch.uint8, device=dev)
    B, cap = buf.B, buf.node_cap
    st = _capi.GatStash()
    assert lib.gccb_gat_stash_layout(C.byref(cfg), B, cap, C.byref(st)) == 0
    sl, _ = glayout.gat_param_slices(cfg)
    P = {k: model.flat_params[o:o + torch.Size(s).numel()].view(s).detach().double() for k, (o, s) in sl.items()}
    Pa = {k: v.abs() for k, v in P.items()}
    worst, mid, notes, paths = {}, {}, [], []
    for view in (0, 1):
        feat = torch.zeros(B, H, device=dev)
        dfeat = torch.randn(B, H, device=dev)
        grads = torch.zeros(model.n_live, device=dev)
        run(buf, view, dfeat, grads)
        torch.cuda.synchronize()
        A, W_ = acts, ws
        G = grads.double()
        floor = 1e-3 * float(G.abs().max())

        def T_(buf_, off, *shape):
            n = int(np.prod(shape))
            return buf_[off:off + 4 * n].view(torch.float32).reshape(shape).double()

        def grad(k):
            o, s = sl[k]
            return G[o:o + torch.Size(s).numel()].view(s)

        noff = buf.node_off[view, :B + 1].long()
        N = int(noff[B])
        indptr = buf.indptr[view, :N + 1].long()
        deg_i = indptr[1:] - indptr[:-1]
        row = torch.repeat_interleave(torch.arange(N, device=dev), deg_i)
        col = buf.indices[view, :int(indptr[N])].long()
        deg = deg_i.double()
        gid = torch.repeat_interleave(torch.arange(B, device=dev), noff[1:] - noff[:-1])
        cnt = (noff[1:] - noff[:-1]).double()
        sub_deg = buf.sub_deg[view, :N].long()
        # ---- what the batch reaches
        p = _paths(deg_i, cap, noff)
        paths.append("view %d: %s" % (view, ", ".join("%s %s" % kv for kv in p.items())))
        if kind == "sampled":
            assert p["hub_rows"] == 0                                     # one warp per row throughout
        if kind == "hub":
            assert p["hub_rows"] >= 591 and p["all_hub_groups"] >= 70 and p["mixed_groups"] >= 1
            assert p["clamped"] >= 1 and p["empty_rows"] >= 1 and p["N"] > 8 * 8 * SMS and p["gb_tail"] != 0
            assert p["hub_then_warp_ctas"] >= 1 and p["groups_per_cta"] >= 2
        if kind == "large":
            assert p["N"] > 64 * 4 * SMS and p["tiles_per_cta"] >= 2 and p["groups_per_cta"] >= 2
            assert p["largest_graph"] >= 1000
        if kind == "short":
            assert p["N"] < n_full and p["B"] == 7 and p["gb_tail"] != 0
        if kind == "c2":
            assert p["B"] == 256 and (L, H, nh, T, K) == (5, 64, 4, 6, 3)
        # ---- X0 (the GIN path's kernel): bit-exact
        x0 = T_(A, st.x0, cap, 64)[:N]
        emb = P["degree_embedding.weight"]
        seed = (torch.arange(N, device=dev) == noff[gid]).double()
        want = torch.cat([buf.pos[view, :N].double(), emb[sub_deg.clamp(0, 512)], seed[:, None],
                          torch.zeros(N, 64 - 49, dtype=torch.float64, device=dev)], 1)
        _stage("x0", x0, want, torch.zeros_like(want), worst)
        X = x0[:, :49]
        for l in range(L):
            pf = "gnn.layers.%d.gnn." % l
            Wf, Kin = P[pf + "fc.weight"], X.shape[1]
            z = T_(A, st.z[l], cap, H)[:N]
            _stage("z", z, X @ Wf.t(), (Kin + 1) * U * (X.abs() @ Pa[pf + "fc.weight"].t()), worst)
            att = T_(A, st.att[l], 4, cap, nh)[:, :N]
            z3 = z.view(N, nh, F_)
            for j, a_ in ((0, "attn_l"), (1, "attn_r")):
                _stage("el/er", att[j], (z3 * P[pf + a_]).sum(-1), (F_ + 1) * U * (z3.abs() * Pa[pf + a_]).sum(-1),
                       worst)
            el, er, mx, den = att
            e = torch.nn.functional.leaky_relu(el[col] + er[row], 0.2)
            mx_w = torch.zeros(N, nh, dtype=torch.float64, device=dev).scatter_reduce(
                0, row[:, None].expand(-1, nh), e, "amax", include_self=False)
            _stage("softmax max", mx, mx_w, 3 * U * mx_w.abs(), worst)
            ex = torch.exp(e - mx[row])
            den_w = torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(0, row, ex)
            _stage("softmax denominator", den, den_w, (2 * deg[:, None] + C_EXP) * U * den_w, worst)
            a = ex / den[row].clamp_min(1e-300)
            out = torch.zeros(N, nh, F_, dtype=torch.float64, device=dev).index_add(
                0, row, a[:, :, None] * z3[col]).reshape(N, H)
            bnd = (deg[:, None] + C_EXP) * U * torch.zeros(N, nh, F_, dtype=torch.float64, device=dev).index_add(
                0, row, a[:, :, None] * z3[col].abs()).reshape(N, H) + U * out.abs()
            act = l < L - 1
            h = T_(A, st.h[l], cap, H)[:N]
            _stage("aggregation", h, torch.nn.functional.leaky_relu(out, 0.01) if act else out, bnd, worst)
            X = h
            del e, ex, a, out, bnd
        # ---- Set2Set, every cell and attention from the stored operands
        x, xa = X, X.abs()
        qstar = T_(A, st.qstar, T + 1, B, 2 * H)
        hs, cs = T_(A, st.hs, T + 1, K, B, H), T_(A, st.cs, T + 1, K, B, H)
        gates = T_(A, st.gates, T, K, B, 4 * H)
        alpha = T_(A, st.alpha, T, cap)[:, :N]
        for it in range(T):
            for k in range(K):
                inp = qstar[it] if k == 0 else hs[it + 1, k - 1]
                wih, whh = P["set2set.lstm.weight_ih_l%d" % k], P["set2set.lstm.weight_hh_l%d" % k]
                bsum = P["set2set.lstm.bias_ih_l%d" % k] + P["set2set.lstm.bias_hh_l%d" % k]
                pre = inp @ wih.t() + hs[it, k] @ whh.t() + bsum
                pb = (inp.shape[1] + H + 3) * U * (inp.abs() @ wih.abs().t() + hs[it, k].abs() @ whh.abs().t() +
                                                   bsum.abs())
                sg = torch.sigmoid(pre)
                g_w = torch.cat([sg[:, :2 * H], torch.tanh(pre[:, 2 * H:3 * H]), sg[:, 3 * H:]], 1)
                slope = torch.cat([torch.full_like(pb[:, :2 * H], 0.25), torch.ones_like(pb[:, :H]),
                                   torch.full_like(pb[:, :H], 0.25)], 1)
                _stage("lstm gates", gates[it, k], g_w, slope * pb + C_EXP * U * g_w.abs(), worst)
                gi, gf, gg, go = gates[it, k].split(H, 1)
                c_w = gf * cs[it, k] + gi * gg
                _stage("lstm c", cs[it + 1, k], c_w, C_EXP * U * ((gf * cs[it, k]).abs() + (gi * gg).abs()), worst)
                h_w = go * torch.tanh(cs[it + 1, k])
                _stage("lstm h", hs[it + 1, k], h_w, C_EXP * U * (h_w.abs() + go.abs() * U), worst)
            q = hs[it + 1, K - 1]
            e_i = (x * q[gid]).sum(1)
            e_b = (H + 1) * U * (xa * q[gid].abs()).sum(1)
            emax = torch.zeros(B, dtype=torch.float64, device=dev).scatter_reduce(0, gid, e_i, "amax",
                                                                                   include_self=False)
            ex = torch.exp(e_i - emax[gid])
            al_w = ex / torch.zeros(B, dtype=torch.float64, device=dev).index_add(0, gid, ex)[gid]
            demax = torch.zeros(B, dtype=torch.float64, device=dev).scatter_reduce(0, gid, e_b, "amax",
                                                                                    include_self=False)
            _stage("set2set alpha", alpha[it], al_w, 2 * al_w * demax[gid] + (cnt[gid] + C_EXP) * U * al_w, worst)
            r_w = torch.zeros(B, H, dtype=torch.float64, device=dev).index_add(0, gid, alpha[it][:, None] * x)
            r_b = (cnt[:, None] + 1) * U * torch.zeros(B, H, dtype=torch.float64, device=dev).index_add(
                0, gid, alpha[it][:, None] * xa)
            _stage("set2set r", qstar[it + 1, :, H:], r_w, r_b, worst)
            _stage("set2set q", qstar[it + 1, :, :H], q, torch.zeros_like(q), worst)
        # ---- readout
        qs_, w0, w2 = qstar[T], P["lin_readout.0.weight"], P["lin_readout.2.weight"]
        y1 = T_(A, st.y1, B, H)
        pre1 = qs_ @ w0.t() + P["lin_readout.0.bias"]
        _stage("readout 0", y1, pre1.clamp_min(0), (2 * H + 2) * U * (qs_.abs() @ w0.abs().t() +
                                                                      P["lin_readout.0.bias"].abs()), worst)
        score = T_(A, st.score, B, H)
        s_w = y1 @ w2.t() + P["lin_readout.2.bias"]
        _stage("readout 2", score, s_w, (H + 2) * U * (y1 @ w2.abs().t() + P["lin_readout.2.bias"].abs()), worst)
        n = score.norm(dim=1, keepdim=True)
        f_w = score / n.clamp_min(1e-5)
        _stage("normalise", feat.double(), f_w, (H + C_EXP) * U * f_w.abs() + U * 1e-30, worst)
        # ---- backward: readout
        df = dfeat.double()
        dot = (score * df).sum(1, keepdim=True)
        d2_w = (df - score * dot / n ** 2) / n
        dy = T_(W_, st.dy, B, 2, H)
        d2, d1 = dy[:, 1], dy[:, 0]
        _stage("dscore", d2, d2_w, (2 * H + C_EXP) * U * (df.abs() + score.abs() * (score * df).abs().sum(1, keepdim=True)
                                                      / n ** 2) / n, worst)
        d1_w = (d2 @ w2) * (y1 > 0)
        _stage("d lin_readout.0", d1, d1_w, (H + 1) * U * (d2.abs() @ w2.abs()) * (y1 > 0), worst)
        # readout and LSTM weight gradients from the stored output gradients and inputs (fixed-order row sums)
        _stage("grad lin_readout.2.weight", grad("lin_readout.2.weight"), d2.t() @ y1, (B + 1) * U * (d2.abs().t() @ y1),
               worst)
        _stage("grad lin_readout.0.weight", grad("lin_readout.0.weight"), d1.t() @ qs_,
               (B + 1) * U * (d1.abs().t() @ qs_.abs()), worst)
        dg = T_(W_, st.dgates, T, K, B, 4 * H)
        for k in range(K):
            inp = qstar[:T] if k == 0 else hs[1:, k - 1]
            d = dg[:, k].reshape(T * B, 4 * H)
            i2 = inp.reshape(T * B, -1)
            _stage("grad weight_ih", grad("set2set.lstm.weight_ih_l%d" % k), d.t() @ i2,
                   (T * B + 1) * U * (d.abs().t() @ i2.abs()), worst)
            h2 = hs[:T, k].reshape(T * B, H)
            _stage("grad weight_hh", grad("set2set.lstm.weight_hh_l%d" % k), d.t() @ h2,
                   (T * B + 1) * U * (d.abs().t() @ h2.abs()), worst)
            for bn in ("bias_ih", "bias_hh"):
                _stage("grad " + bn, grad("set2set.lstm.%s_l%d" % (bn, k)), d.sum(0), (T * B + 1) * U * d.abs().sum(0),
                       worst)
        # BPTT: the stored pre-activation gate gradients against float64 autograd of the Set2Set + readout recomputed
        # from the stored top-layer output x (a composition of T x K cells: held to 2e-3 of each cell's scale)
        dh = T_(W_, st.dh, cap, H)[:N]        # the gradient of layer 0's output: layer 1's dX, or at L = 1 Set2Set's
        xs = x.clone().requires_grad_(True)
        pres = []
        (_s2s_readout(xs, P, gid, B, T, K, pres) * df).sum().backward()
        for idx, pre in enumerate(pres):
            it, k = divmod(idx, K)
            sc = max(float(pre.grad.abs().max()), 1e-30)
            _stage("lstm dgates (BPTT)", dg[it, k], pre.grad, torch.full_like(pre.grad, 2e-3 * sc), worst)
        if L == 1:
            # the top layer is layer 0: its output gradient is the Set2Set attention backward's dx alone
            sc = max(float(xs.grad.abs().max()), 1e-30)
            _stage("dh = Set2Set gradient into x (L = 1)", dh, xs.grad, torch.full_like(xs.grad, 2e-3 * sc), worst)
        del xs, pres
        # ---- backward of layers 1 .. L-1: float64 autograd of layers l .. L-1, the Set2Set and the readout from the
        # stored h[l-1]: fc / attention gradients of layer l, and at l = 1 the dh that reaches layer 0
        for l in range(1, L):
            hin = T_(A, st.h[l - 1], cap, H)[:N].requires_grad_(l == 1)
            y = hin
            leaves = {}
            for m in range(l, L):
                pf = "gnn.layers.%d.gnn." % m
                prm = {k_: P[pf + k_].clone().requires_grad_(m == l) for k_ in ("fc.weight", "attn_l", "attn_r")}
                if m == l:
                    leaves = prm
                y = _gat_layer(y, prm["fc.weight"], prm["attn_l"], prm["attn_r"], row, col, nh, m < L - 1)
            (_s2s_readout(y, P, gid, B, T, K) * df).sum().backward()
            for k_, t in leaves.items():
                _vs_autograd("grad %s (layer %d)" % (k_, l), grad("gnn.layers.%d.gnn.%s" % (l, k_)), t.grad, floor, mid,
                             notes)
            if l == 1:
                _vs_autograd("dh into layer 0", dh, hin.grad, 0.0, mid, notes)
            del y, hin, leaves
        # ---- backward: layer 0's edge softmax, dX, fc / attention / embedding gradients from the stored operands
        h0 = T_(A, st.h[0], cap, H)[:N]
        dout = T_(W_, st.dout, cap, H)[:N]
        dout_w = dh * torch.where(h0 > 0, 1.0, 0.01) if L > 1 else dh
        _stage("dout", dout, dout_w, U * dout_w.abs(), worst)
        z = T_(A, st.z[0], cap, H)[:N]
        z3, d3 = z.view(N, nh, F_), dout.view(N, nh, F_)
        el, er, mx, den = T_(A, st.att[0], 4, cap, nh)[:, :N]
        pre = el[col] + er[row]
        a = torch.exp(torch.nn.functional.leaky_relu(pre, 0.2) - mx[row]) / den[row]
        slope = torch.where(pre > 0, 1.0, 0.2)
        da = (d3[row] * z3[col]).sum(-1)
        da_abs = (d3[row].abs() * z3[col].abs()).sum(-1)
        sv = T_(W_, st.sv, 2, cap, nh)[:, :N]
        cb = (deg[:, None] + F_ + C_EXP) * U
        S_w = torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(0, row, a * da)
        _stage("softmax bwd S", sv[0], S_w,
               cb * torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(0, row, a * da_abs), worst)
        der_w = torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(0, row, a * (da - sv[0][row]) * slope)
        der_b = cb * torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(
            0, row, a * (2 * da_abs + sv[0][row].abs()))
        _stage("softmax bwd der", sv[1], der_w, der_b, worst)
        dpre = a * (da - sv[0][row]) * slope                 # edge u -> v, summed at the source u
        del_w = torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(0, col, dpre)
        del_b = (deg[:, None] + F_ + C_EXP) * U * torch.zeros(N, nh, dtype=torch.float64, device=dev).index_add(
            0, col, a * (da_abs + sv[0][row].abs()))
        al_, ar_ = P["gnn.layers.0.gnn.attn_l"].view(nh, F_), P["gnn.layers.0.gnn.attn_r"].view(nh, F_)
        agg = torch.zeros(N, nh, F_, dtype=torch.float64, device=dev).index_add(0, col, a[:, :, None] * d3[row])
        agg_b = torch.zeros(N, nh, F_, dtype=torch.float64, device=dev).index_add(0, col, a[:, :, None] * d3[row].abs())
        dz_w = (agg + del_w[:, :, None] * al_ + sv[1][:, :, None] * ar_).reshape(N, H)
        dz_b = ((deg[:, None, None] + F_ + C_EXP) * U * agg_b + del_b[:, :, None] * al_.abs() +
                del_w.abs()[:, :, None] * al_.abs() * U + U * (sv[1].abs()[:, :, None] * ar_.abs())).reshape(N, H)
        dz = T_(W_, st.dz, cap, H)[:N]
        _stage("dz", dz, dz_w, dz_b + U * dz_w.abs(), worst)
        del pre, a, slope, da, da_abs, dpre, agg, agg_b
        Wf = P["gnn.layers.0.gnn.fc.weight"]
        dx0 = T_(W_, st.dx0, cap, 64)[:N]
        _stage("dX0", dx0[:, :49], dz @ Wf, (H + 1) * U * (dz.abs() @ Wf.abs()), worst)
        _stage("grad fc.weight (layer 0)", grad("gnn.layers.0.gnn.fc.weight"), dz.t() @ x0[:, :49],
               (N + 1) * U * (dz.abs().t() @ x0[:, :49].abs()), worst)
        gl_w = (del_w[:, :, None] * z3).sum(0).view(1, nh, F_)
        gl_b = ((N + 1) * U * (del_w.abs()[:, :, None] * z3.abs()).sum(0) + (del_b[:, :, None] * z3.abs()).sum(0))
        _stage("grad attn_l (layer 0)", grad("gnn.layers.0.gnn.attn_l"), gl_w, gl_b.view(1, nh, F_), worst)
        gr_w = (sv[1][:, :, None] * z3).sum(0).view(1, nh, F_)
        _stage("grad attn_r (layer 0)", grad("gnn.layers.0.gnn.attn_r"), gr_w,
               ((N + 1) * U * (sv[1].abs()[:, :, None] * z3.abs()).sum(0)).view(1, nh, F_), worst)
        dg_ = sub_deg.clamp(0, 512)
        gemb_w = torch.zeros(513, 16, dtype=torch.float64, device=dev).index_add(0, dg_, dx0[:, 32:48])
        gemb_b = (N + 1) * U * torch.zeros(513, 16, dtype=torch.float64, device=dev).index_add(
            0, dg_, dx0[:, 32:48].abs())
        _stage("grad degree_embedding", grad("degree_embedding.weight"), gemb_w, gemb_b, worst)
    print("%s H=%d heads=%d L=%d T=%d K=%d\n  %s\n  largest |error| / bound per stage: %s" % (
        kind, H, nh, L, T, K, "\n  ".join(paths),
        ", ".join("%s %.2f" % kv for kv in sorted(worst.items(), key=lambda kv: -kv[1]))))
    if mid:
        print("  vs float64 autograd of the layers above (worst / bar, entries outside): %s" % ", ".join(
            "%s %.2f (%d)" % (k_, w, o) for k_, (w, o) in sorted(mid.items())))
    for s in notes:
        print("  " + s)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_replicas_stay_identical_gat():
    """tests/dist_replica_check.py with the GAT encoder (tests/dist_replica_check_gat.py), over NCCL on 2 GPUs."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29519",
                        os.path.join(root, "tests", "dist_replica_check_gat.py")], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "REPLICAS IDENTICAL" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
