"""GPU (H100): every stage of the tensor-core GIN forward and backward (gin_fwd.cu / gin_bwd.cu, hidden >= 128)
against float64, teacher-forced: each stage's reference is computed from the inputs the kernels themselves stored
(located with gccb_gin_stash_layout), so bf16 rounding-boundary flips upstream cannot amplify and every check is an
elementwise bound on fp32-versus-fp64 arithmetic.

Bounds (U = 2^-24, the fp32 unit roundoff):
  GEMM (bf16 operands, fp32 accumulation over K products):  |got - ref| <= C_DOT * K * U * (|A| . |B|^T) + U |bias|,
    the standard dot-product bound with the absolute products summed in fp64.  C_DOT = 4 allows for the tensor
    core's accumulator not rounding to nearest.
  Column reductions (BatchNorm statistics, BatchNorm-backward means): fp32 partial sums of at most
    depth(N) = 64 + N / 1024 additions per term before the float64 atomics, so |error| <= depth * U * sum |terms|
    (the reduction kernels give a thread at most max(16, N / 2112) rows and then add at most 16 partials).
  Elementwise chains (BatchNorm affine, its backward): 8 U of the sum of the magnitudes of the chain's terms, which
    also covers the kernels deriving their BatchNorm coefficients in fp32 from the float64 sums.
  Two ReLU masks of the backward (BN_a, BN_b pre-activations) use fp32 coefficients the kernels do not store; elements
    whose fp64 pre-activation lies within 1e-6 of the column scale of zero are excluded from the elementwise dz2 check
    (their count is printed) and their largest possible effect on the column means is added to every bound.  The
    BatchNorm-1 mask of the backward uses the stored coefficients, so its sign is exact.
The worst error / bound ratio of every stage is printed (-s).  On an H100 80GB HBM3 (400 W power limit) the
forward / input-gradient GEMM stages reached at most 0.06 of their bound with C_DOT = 4, so the tensor core's
accumulation stays well inside the round-to-nearest bound; the split-K weight gradients reached 0.84 (the hub batch,
where whole cliques share identical rows), every other stage at most 0.27."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_emu_gin import _params
from test_gpu_parity import _dataset, _fill_batch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_DOT = 4.0
PRE_EXCL = 1e-6


def _depth(N):
    return 64 + N // 1024


def _bf(x):
    """bf16 round-to-nearest-even of an fp32 tensor (what __float2bfloat16_rn does), as float64."""
    return x.float().to(torch.bfloat16).double()


def _fma32(x, s, t):
    """fmaf(x, s, t) for fp32 tensors, exactly: the product is exact in fp64, TwoSum recovers the rounding error of
    the fp64 sum, and that error decides the one case where rounding the fp64 sum to fp32 differs from rounding the
    exact value: an fp64 sum exactly halfway between two fp32 neighbours."""
    p = x.double() * s.double()
    t = t.double().expand_as(p)
    hi = p + t
    bb = hi - p
    lo = (p - (hi - bb)) + (t - bb)
    r = hi.float()
    rd = r.double()
    inf = torch.full_like(r, float("inf"))
    nxt = torch.nextafter(r, torch.where(hi > rd, inf, -inf))
    tie = (hi != rd) & (hi == (rd + nxt.double()) / 2) & (lo != 0)
    away = torch.sign(lo) == torch.sign(hi - rd)
    return torch.where(tie & away, nxt, r)


class _Report:
    def __init__(self, tag):
        self.tag, self.worst, self.notes = tag, {}, []

    def check(self, stage, got, want, bound, keep=None):
        err = (got.double() - want).abs()
        bound = bound.expand_as(err)
        if keep is not None:
            err, bound = err[keep], bound[keep]
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        worst = float(ratio.max()) if ratio.numel() else 0.0
        self.worst[stage] = max(self.worst.get(stage, 0.0), worst)
        if not worst <= 1.0:                                      # NaN fails too
            i = int(ratio.argmax())
            raise AssertionError("%s %s: error / bound %.3g at flat index %d (|err| %.3e, bound %.3e)" % (
                self.tag, stage, worst, i, float(err.flatten()[i]), float(bound.flatten()[i])))

    def exact(self, stage, got, want):
        assert torch.equal(got, want), (self.tag, stage, int((got != want).sum()))
        self.worst.setdefault(stage + " (bit-exact)", 0.0)

    def show(self):
        print("\n[%s] worst |error| / bound per stage" % self.tag)
        for k, v in self.worst.items():
            print("  %-34s %.3f" % (k, v))
        for n in self.notes:
            print("  " + n)


def _clique(n):
    return dict(indptr=np.arange(n + 1) * (n - 1),
                indices=np.concatenate([np.delete(np.arange(n), i) for i in range(n)]))


def _hub_buffers():
    """Disjoint 290- and 300-vertex cliques (every row a hub: more than 256 neighbours), a 400-vertex star (one hub
    row) and a small random graph; more hub rows per CTA than the per-CTA hub queue holds."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import BatchBuffers
    star, er = synthetic.star_graph(400), synthetic.erdos_renyi(60, 150, seed=1)
    graphs = [_clique(300), dict(indptr=er.indptr, indices=er.indices), dict(indptr=star.indptr, indices=star.indices),
              _clique(290)]
    views = [graphs, graphs[::-1]]
    n = sum(len(g["indptr"]) - 1 for g in graphs)
    m = sum(len(g["indices"]) for g in graphs)
    buf = BatchBuffers(len(graphs), n + 100, m + 100, 32, 64, "cuda")
    _fill_batch(buf, views)
    gen = torch.Generator(device="cuda").manual_seed(4)
    buf.pos.copy_(0.3 * torch.randn(buf.pos.shape, device="cuda", generator=gen))
    return buf


def _batch(kind):
    from gcc_b200.datasets import synthetic
    if kind == "hub":
        return _hub_buffers()
    g = synthetic.chung_lu(4000, 30000, seed=6)
    kw = {}
    if kind == "large":       # more 128-row tiles than SMs: the resident-weight GEMM, with N far below node_cap
        kw["node_cap"] = 128 * torch.cuda.get_device_properties(0).multi_processor_count + 640
    ds = _dataset(g, 24, 64, seed=3, **kw)
    buf = ds.sample_batch(first_sample=0)
    torch.cuda.synchronize()
    buf.check_flags()
    return buf


def _coef(S, N, gamma, beta, eps):
    mean = S[0] / N
    var = (S[1] / N - mean * mean).clamp_min(0.0)
    inv = 1.0 / torch.sqrt(var + eps)
    sc = gamma * inv
    return mean, inv, sc, beta - mean * sc


def _rows_mean(x):
    return x.mean(0)


@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("kind", ["sampled", "hub", "large"])
@pytest.mark.parametrize("H", [128, 256])
def test_tc_gin_stages_vs_float64(H, kind, L):
    from gcc_b200 import _capi, _lib
    from gcc_b200.models import layout as glayout
    lib = _lib.get()
    _lib.require_device()
    rep = _Report("H=%d %s L=%d" % (H, kind, L))
    buf = _batch(kind)
    B, cap = buf.B, buf.node_cap
    cfg = glayout.make_cfg(num_layers=L, hidden=H, tensor_cores=1)
    lay = glayout.c_layout(lib, cfg)
    st = _capi.GinStash()
    _lib.check(lib.gccb_gin_stash_layout(C.byref(cfg), B, cap, C.byref(st)), "gccb_gin_stash_layout")
    assert st.cap_pad == (cap + 63) // 64 * 64 and st.splits >= 1 and st.a16 >= 0 and st.DW == H
    flat, _, _ = _params(cfg, np.random.default_rng(L * 1000 + H))
    lt = L - 2                                                    # top GIN layer
    flat[lay.b1[lt]:lay.b1[lt] + H] += 200.0                       # its z1 columns: |mean| >> std
    params = torch.from_numpy(flat).cuda()
    running = torch.zeros(lay.run_total, device="cuda")
    acts = torch.zeros(lib.gccb_gin_acts_bytes(C.byref(cfg), B, cap), dtype=torch.uint8, device="cuda")
    ws = torch.zeros(lib.gccb_gin_backward_workspace(C.byref(cfg), B, cap), dtype=torch.uint8, device="cuda")
    grads = torch.zeros_like(params)
    feat = torch.zeros(B, H, device="cuda")
    eps = float(np.float32(cfg.bn_eps))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (cap + 127) // 128 > sms if kind == "large" else True

    def P(off, *shape):
        n = int(np.prod(shape))
        return params[off:off + n].view(*shape).double()

    def T(base, off, dtype, *shape):
        n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
        assert off >= 0
        return base[off:off + n].view(dtype).view(*shape)

    gen = torch.Generator(device="cuda").manual_seed(H + L)
    for view in (0, 1):
        dfeat = torch.randn(B, H, device="cuda", generator=gen)
        g_before = grads.clone()
        _lib.check(lib.gccb_gin_forward(C.byref(cfg), C.byref(buf.c), view, _lib.dptr(buf.pos), _lib.dptr(params),
                                        _lib.dptr(running), None, 1, 0, 0, -1, _lib.dptr(acts), acts.numel(),
                                        _lib.dptr(feat), None, _lib.stream_ptr()), "gccb_gin_forward")
        _lib.check(lib.gccb_gin_backward(C.byref(cfg), C.byref(buf.c), view, _lib.dptr(params), _lib.dptr(acts),
                                         _lib.dptr(dfeat), _lib.dptr(grads), 0, 0, -1, _lib.dptr(ws), ws.numel(),
                                         _lib.stream_ptr()), "gccb_gin_backward")
        torch.cuda.synchronize()
        N = int(buf.node_off[view, B])
        D = _depth(N)
        indptr = buf.indptr[view, :N + 1].long()
        deg = (indptr[1:] - indptr[:-1])
        row = torch.repeat_interleave(torch.arange(N, device="cuda"), deg)
        col = buf.indices[view, :int(indptr[-1])].long()
        gid = buf.graph_id[view, :N].long()
        if kind == "hub":
            assert int(deg.max()) > 256
        if view == 0:
            rep.notes.append("N = %d, node_cap = %d, hub rows = %d" % (N, cap, int((deg > 256).sum())))

        def agg(x):                                               # x + sum_nbr x, and the same of |x|
            return x.index_add(0, row, x[col]), x.abs().index_add(0, row, x[col].abs())

        stats = T(acts, st.stats, torch.float64, L - 1, 3, 2, H)
        coef1 = T(ws, st.coef1, torch.float32, L - 1, 2, H)
        G = grads.double() - g_before.double()                    # this view's contribution (exact in fp64)
        Gslack = U * grads.double().abs()                          # rounding of the accumulation into grads

        def gslice(off, *shape):
            n = int(np.prod(shape))
            return G[off:off + n].view(*shape), Gslack[off:off + n].view(*shape)

        fwd = {}
        for l in range(L - 1):
            inf, KW = (cfg.pos_dim + cfg.deg_dim + 1, 64) if l == 0 else (H, H)
            W1, W2 = P(lay.w1[l], H, inf), P(lay.w2[l], H, H)
            W1f = torch.zeros(H, KW, device="cuda", dtype=torch.float64)
            W1f[:, :inf] = W1
            b1, b2 = P(lay.b1[l], H), P(lay.b2[l], H)
            # bf16 weight copies: W1 [H][KW] (zero padded), W2, W1^T, W2^T
            w16 = T(acts, st.w16[l], torch.bfloat16, 2 * H * KW + 2 * H * H)
            parts = torch.split(w16, [H * KW, H * H, KW * H, H * H])
            rep.exact("w16", parts[0].view(H, KW), W1f.float().to(torch.bfloat16))
            assert not parts[0].view(H, KW)[:, inf:].any() and not parts[2].view(KW, H)[inf:].any()
            rep.exact("w16", parts[1].view(H, H), W2.float().to(torch.bfloat16))
            rep.exact("w16", parts[2].view(KW, H), W1f.t().float().to(torch.bfloat16))
            rep.exact("w16", parts[3].view(H, H), W2.t().float().to(torch.bfloat16))
            # aggregation a = h + sum_nbr h from the stored h of the layer below
            hin = T(acts, st.x0, torch.float32, cap, 64)[:N] if l == 0 else T(acts, st.h[l - 1], torch.float32, cap, H)[:N]
            a = T(acts, st.a[l], torch.float32, cap, KW)[:N]
            ref, mag = agg(hin.double())
            rep.check("a = h + sum_nbr h", a, ref, (deg + 9).double()[:, None] * U * mag)
            if l == L - 2:
                rep.exact("a16 = bf16(a)", T(acts, st.a16, torch.bfloat16, cap, KW)[:N], a.to(torch.bfloat16))
            # z1 = bf16(a) bf16(W1)^T + b1
            z1 = T(acts, st.z1[l], torch.float32, cap, H)[:N]
            A, Bw = _bf(a), _bf(W1f.float())
            rep.check("z1 GEMM", z1, A @ Bw.t() + b1, C_DOT * KW * U * (A.abs() @ Bw.abs().t()) + U * b1.abs())
            # x1 = bf16(relu(fma(z1, sc, sh))) with the kernels' own BatchNorm-1 coefficients
            sc1, sh1 = coef1[l, 0], coef1[l, 1]
            x1 = _fma32(z1, sc1, sh1).clamp_min(0.0).to(torch.bfloat16)
            if l == L - 2:
                rep.exact("x16 = bf16(relu(bn1(z1)))", T(acts, st.x16, torch.bfloat16, cap, H)[:N], x1)
            z2 = T(acts, st.z2[l], torch.float32, cap, H)[:N]
            X, Bw2 = x1.double(), _bf(W2.float())
            rep.check("z2 GEMM", z2, X @ Bw2.t() + b2, C_DOT * H * U * (X.abs() @ Bw2.abs().t()) + U * b2.abs())
            # BatchNorm statistics of z1 and z2 and the variance derived from them
            for which, z in ((0, z1), (1, z2)):
                S = stats[l, which]
                zd = z.double()
                s1b, s2b = D * U * zd.abs().sum(0), (D + 1) * U * (zd * zd).sum(0)
                rep.check("stats sum", S[0], zd.sum(0), s1b)
                rep.check("stats sum of squares", S[1], (zd * zd).sum(0), s2b)
                m = S[0] / N
                var = S[1] / N - m * m
                rep.check("stats variance", var, zd.var(0, unbiased=False),
                          s2b / N + 2 * m.abs() * s1b / N + (s1b / N) ** 2 + 1e-15 * (S[1] / N + m * m))
            if l == lt:
                cm = float((z1.double().mean(0).abs() / z1.double().std(0)).min())
                rep.notes.append("view %d: top layer z1 columns, smallest |mean| / std = %.1f" % (view, cm))
                assert cm > 10 or kind == "hub"                   # the cancellation case is really exercised
            # BN_a -> ReLU -> (statistics of y) -> BN_b -> ReLU
            mA, iA, scA, shA = _coef(stats[l, 1], N, P(lay.bna_w[l], H), P(lay.bna_b[l], H), eps)
            z2d = z2.double()
            ya = z2d * scA + shA
            y = ya.clamp_min(0.0)
            e_y = 8 * U * ((z2d * scA).abs() + shA.abs() + (mA * scA).abs())
            Sb = stats[l, 2]
            rep.check("stats of y", Sb[0], y.sum(0), e_y.sum(0) + D * U * y.sum(0))
            rep.check("stats of y", Sb[1], (y * y).sum(0), (2 * y * e_y + e_y * e_y).sum(0) + (D + 1) * U * (y * y).sum(0))
            mB, iB, scB, shB = _coef(Sb, N, P(lay.bnb_w[l], H), P(lay.bnb_b[l], H), eps)
            hb = y * scB + shB
            hout = T(acts, st.h[l], torch.float32, cap, H)[:N]
            rep.check("h = BN/ReLU tail", hout, hb.clamp_min(0.0),
                      scB.abs() * e_y + 8 * U * ((y * scB).abs() + shB.abs() + (mB * scB).abs()))
            fwd[l] = dict(a=a, z1=z1, z2=z2, x1=x1, W1f=W1f, W2=W2, inf=inf, KW=KW, ya=ya, y=y, hb=hb, e_y=e_y,
                          A=(mA, iA, scA, shA), Bc=(mB, iB, scB, shB))

        # ---------------- backward ----------------
        dpool = T(ws, st.dpool, torch.float32, L, B, H)
        for l in range(L - 1):
            f = fwd[l]
            dz2k = T(ws, st.dz2[l & 1], torch.float32, cap, H)[:N]
            dz1k = T(ws, st.g1[l & 1], torch.float32, cap, H)[:N]
            z1d, z2d = f["z1"].double(), f["z2"].double()
            if l == lt:
                # the top layer's dh is dpool[L-1] broadcast by graph: its whole chain is reconstructed
                mA, iA, scA, shA = f["A"]
                mB, iB, scB, shB = f["Bc"]
                ya, y, hb, e_ya = f["ya"], f["y"], f["hb"], f["e_y"]
                dh = dpool[L - 1].double()[gid]
                scaleA = ((z2d * scA).abs() + shA.abs() + (mA * scA).abs()).max(0).values
                scaleB = ((y * scB).abs() + shB.abs() + (mB * scB).abs()).max(0).values
                riskA, riskB = ya.abs() <= PRE_EXCL * scaleA, hb.abs() <= PRE_EXCL * scaleB
                yhat = (y - mB) * iB
                e_yhat = iB * (e_ya + 8 * U * (y.abs() + mB.abs()))
                g4 = (hb > 0) * dh
                mB1, mB2 = _rows_mean(g4), _rows_mean(g4 * yhat)
                dy = scB * (g4 - mB1 - yhat * mB2)
                g3 = (ya > 0) * dy
                z2hat = (z2d - mA) * iA
                mA1, mA2 = _rows_mean(g3), _rows_mean(g3 * z2hat)
                dz2 = scA * (g3 - mA1 - z2hat * mA2)
                dB1 = (riskB * dh.abs()).sum(0) / N + D * U * _rows_mean(g4.abs())
                dB2 = (riskB * (dh * yhat).abs()).sum(0) / N + D * U * _rows_mean((g4 * yhat).abs()) + \
                    _rows_mean(g4.abs() * e_yhat)
                ddy = scB.abs() * (dB1 + yhat.abs() * dB2 + mB2.abs() * e_yhat) + \
                    8 * U * scB.abs() * (g4.abs() + mB1.abs() + (yhat * mB2).abs())
                e_z2hat = iA * 8 * U * (z2d.abs() + mA.abs())
                mask_a = (ya > 0).double()
                dA1 = (riskA * dy.abs()).sum(0) / N + _rows_mean(mask_a * ddy) + D * U * _rows_mean(g3.abs())
                dA2 = (riskA * (dy * z2hat).abs()).sum(0) / N + _rows_mean(mask_a * ddy * z2hat.abs()) + \
                    _rows_mean(g3.abs() * e_z2hat) + D * U * _rows_mean((g3 * z2hat).abs())
                bound = scA.abs() * (mask_a * ddy + dA1 + z2hat.abs() * dA2 + mA2.abs() * e_z2hat) + \
                    8 * U * scA.abs() * (g3.abs() + mA1.abs() + (z2hat * mA2).abs())
                keep = ~(riskA | riskB)
                rep.notes.append("view %d: dz2 elements excluded near a BN_a / BN_b ReLU kink: %d of %d" % (
                    view, int((~keep).sum()), keep.numel()))
                rep.check("dz2 (BN_b, BN_a backward)", dz2k, dz2, bound, keep)
                for off, val, err in ((lay.bnb_w[l], N * mB2, N * dB2), (lay.bnb_b[l], N * mB1, N * dB1),
                                      (lay.bna_w[l], N * mA2, N * dA2), (lay.bna_b[l], N * mA1, N * dA1)):
                    got, slack = gslice(off, H)
                    rep.check("BN_a / BN_b gamma, beta grads", got, val, err + U * val.abs() + slack)
            # g1 ends as dz1 = BN1^T(mask . (bf16(dz2) bf16(W2))), from the kernels' own dz2
            A2, W2b = _bf(dz2k), _bf(f["W2"].float())
            dx1 = A2 @ W2b
            e_dx1 = C_DOT * H * U * (A2.abs() @ W2b.abs())
            sc1k, sh1k = coef1[l, 0].double(), coef1[l, 1].double()
            mask1 = (z1d * sc1k + sh1k > 0).double()              # exact sign of the kernels' fp32 fma
            m1, i1, sc1, _ = _coef(stats[l, 0], N, P(lay.bn1_w[l], H), P(lay.bn1_b[l], H), eps)
            g = mask1 * dx1
            zhat = (z1d - m1) * i1
            e_zhat = i1 * 8 * U * (z1d.abs() + m1.abs())
            n1, n2 = _rows_mean(g), _rows_mean(g * zhat)
            dg = mask1 * e_dx1
            d1 = _rows_mean(dg) + D * U * _rows_mean(g.abs())
            d2 = _rows_mean(dg * zhat.abs()) + _rows_mean(g.abs() * e_zhat) + D * U * _rows_mean((g * zhat).abs())
            rep.check("dz1 (BN1 backward)", dz1k, sc1 * (g - n1 - zhat * n2),
                      sc1.abs() * (dg + d1 + zhat.abs() * d2 + n2.abs() * e_zhat) +
                      8 * U * sc1.abs() * (g.abs() + n1.abs() + (zhat * n2).abs()))
            for off, val, err in ((lay.bn1_w[l], N * n2, N * d2), (lay.bn1_b[l], N * n1, N * d1)):
                got, slack = gslice(off, H)
                rep.check("BN1 gamma, beta grads", got, val, err + U * val.abs() + slack)
            # weight gradients: dW2 = bf16(dz2)^T x1, dW1 = bf16(dz1)^T bf16(a), split-K over the rows
            X1 = f["x1"].double()
            got, slack = gslice(lay.w2[l], H, H)
            rep.check("dW2 GEMM (split-K, accumulate)", got, A2.t() @ X1,
                      C_DOT * N * U * (A2.abs().t() @ X1.abs()) + slack)
            A1, Aa = _bf(dz1k), _bf(f["a"])
            inf, KW = f["inf"], f["KW"]
            got, slack = gslice(lay.w1[l], H, inf)                 # row pitch in_features (49 for layer 0)
            rep.check("dW1 GEMM (split-K, accumulate)", got, (A1.t() @ Aa)[:, :inf],
                      (C_DOT * N * U * (A1.abs().t() @ Aa.abs()))[:, :inf] + slack)
            for off in (lay.b1[l], lay.b2[l]):                     # Linear biases feeding a train-mode BatchNorm
                assert not grads[off:off + H].any(), (rep.tag, "bias gradient", l)
            if l == 0:
                rep.exact("dz16 = bf16(dz1)", T(ws, st.dz16, torch.bfloat16, cap, H)[:N], dz1k.to(torch.bfloat16))
                tA = T(ws, st.tA, torch.bfloat16, H, st.cap_pad)
                tB = T(ws, st.tB, torch.bfloat16, KW, st.cap_pad)
                rep.exact("tA = bf16(dz1)^T", tA[:, :N], dz1k.t().to(torch.bfloat16))
                rep.exact("tB = bf16(a)^T", tB[:, :N], f["a"].t().to(torch.bfloat16))
                assert not tA[:, N:].any() and not tB[:, N:].any()
                W1b = _bf(f["W1f"].float())
                da = T(ws, st.da, torch.float32, cap, KW)[:N]
                rep.check("da GEMM", da, A1 @ W1b, C_DOT * H * U * (A1.abs() @ W1b.abs()))
                assert not da[:, inf:].any()
                # layer-0 input gradient: dpool[0] broadcast + (I + A) da, hub rows included
                dh0 = T(ws, st.dh, torch.float32, cap, 64)[:N]
                s, mag = agg(da.double())
                dp = dpool[0].double()[gid][:, :64]
                rep.check("dh = dpool + (I + A) da", dh0, dp + s, (deg + 10).double()[:, None] * U * (mag + dp.abs()))
        assert not grads[lay.b1[0]:lay.b1[0] + H].any()             # dW1 of layer 0 (49 of 64 columns) stops at b1[0]
    rep.show()
