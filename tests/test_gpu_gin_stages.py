"""GPU (H100): every stage of the fp32 SIMT GIN forward and backward (gin_fwd.cu / gin_bwd.cu with tensor_cores = 0,
the path of the config-2 training step) against float64, teacher-forced: each stage's reference is computed from the
operands the kernels themselves stored (located with gccb_gin_stash_layout), so upstream rounding cannot amplify.

Bounds (U = 2^-24, the fp32 unit roundoff).  Each one is the summation depth of the kernel's own order times U times
the sum of the magnitudes of the terms, plus the propagated error of any operand the kernel recomputes in fp32:
  GEMM (tile_gemm: acc = 0, then K sequential fmaf, then + bias):  (K + 2) U (|A| |B|^T) + U |bias|.
  Aggregation a = h + sum_nbr h: a warp row adds groups of 8 neighbours as a pairwise tree (3 levels) to its
    accumulator and the rest one by one; a hub row (> 256 neighbours) adds 8 warps' partial sums and then h: no term
    passes through more than deg + 9 additions:  (deg + 9) U (|h| + sum_nbr |h|).
  BatchNorm statistics of z1 / z2 (tile_colstats): 4 rows per thread, then 16 thread partials, one float64 atomic
    per tile:  depth 20 (+1 for the float64 atomics).  Statistics of y (gin_bn_tail_kernel mode 0): a thread adds
    every (grid * RP)-th row, RP = 1024 / H, then RP partials:  depth ceil(N / (grid RP)) + RP.
  Elementwise BatchNorm chains: 8 U of the sum of the magnitudes of the chain's terms; this also covers the kernels
    deriving their coefficients in fp32 from the stored float64 sums (at most 6 roundings on the way).
  Pooling (gin_pool_kernel): runs of at most W / 4 rows (W = 64 or 32; 8 rows of float4 at W = 128) in fp32, then
    float64 atomics and one rounding to fp32:  (run + 2) U sum |h|.
  Heads (gin_pool_predict_kernel): four lanes per output, ceil(in / 4) fmaf each, two shuffles, bias:
    (ceil(in / 4) + 3) U (|pooled| |Wp|^T) + U |bp|, doubled by the dropout scale; the L layers add into score:
    + L U sum_l |s_l|.  Normalisation: ||x||^2 over H / 32 fmaf per lane and a 5-level warp sum (depth H / 32 + 5);
    the square root and the division add (depth / 2 + 3) U relative.
  Backward column reductions before their float64 atomics:  BN_b in gin_bwd_dh_kernel: a lane adds every
    (grid_dh 8 RPW)-th row (RPW = rows per warp pass), log2(RPW) shuffles, 9 partials and the CTA's hub rows;
    BN_a in gin_bwd_reduce_kernel: as the statistics of y;  BN1 in gin_bwd_gemm2_kernel (tile_colstats2): 20.
  Split-K weight gradients (gin_wgrad_kernel): a chunk is ceil(tiles / 132) 64-row tiles of sequential fmaf;
    gin_wgrad_reduce_kernel adds the 132 chunks as four strided runs of 33 and a pairwise sum (35) for the weights,
    sequentially (132) for the biases:  (64 ceil(tiles / 132) + 35 or 132 + 1) U (|P|^T |Q|).
  Head gradients: dpool = dS Wp over H sequential fmaf, dWp and dbp over the B graphs sequentially.
  Degree-embedding gradient: float atomics in arbitrary order into a per-CTA shared histogram (64 CTAs), then
    global atomics:  (rows sharing that degree + 64) U sum |terms|.
  Accumulation into `grads` (both views add to it): + U |grads| per addition (64 for the embedding histogram).
ReLU masks: the backward recomputes its BN1, BN_a and BN_b coefficients in fp32 and does not store them, so an
element whose float64 pre-activation lies within PRE_EXCL of zero, relative to its column's scale, may take either
side.  Such elements are excluded from elementwise checks (their count is printed), and their largest possible effect
(the whole gradient they pass or block) is added to every column mean, and so to every bound, that depends on them.

Only layers 0 and 1 keep their backward buffers (g1 / dz2 alternate between two buffers by layer parity); the top
layer's chain is reconstructed from dpool[L-1].  At L = 5 the top layer (3) is therefore checked against that
reconstruction (its weight gradients are read from buffers layer 1 later overwrites: a missing side-stream wait would
show), layer 2 against the float64 oracle's autograd gradients at the emulator tests' bar, layers 1 and 0
teacher-forced.  The Linear biases b1 / b2 feed a train-mode BatchNorm: their true gradient is zero, and the SIMT
path adds the fp32 column sums of dz1 / dz2 (as the reference's autograd does), checked against their bound.

Every batch kind asserts that it reaches the path it is named for, restating the kernels' grids and row dealing.

Measured on an H100 80GB HBM3 (worst error / bound over all cases): the running statistics 0.99 (one rounding of a
float64 value to fp32, whose worst case is the bound itself), the BN1 gradients 0.99 and dz1 0.97 (sampled, H = 64,
L = 2), the top BN_a / BN_b gradients 0.94, dW2 0.90, the head gradients 0.85, every other stage at most 0.8.  At
L = 5 layer 2 stayed within the emulator bar on the sampled and C2 batches (at most 0.62 of it); on the short batch
(H = 64) 1 to 24 entries of five tensors exceeded it by up to 2.7x, all within 1.3e-3 of their tensor's scale."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_emu_gin import _params
from test_gpu_parity import _dataset, _fill_batch
from test_gpu_tc_gin import _clique, _coef, _Report

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
PRE_EXCL = 1e-6
SMS = 132                      # GCCB_NUM_SMS: the split-K chunks of the weight gradients
HUB_DEG, HUB_QUEUE = 256, 64   # GCCB_HUB_DEG, GCCB_HUB_QUEUE
DH_GRID = 1184                 # grid cap of gin_bwd_dh_kernel


def _gemm_grid(cap):
    return min((cap + 63) // 64, 4 * SMS)


def _dh_grid(cap):
    return min((cap + 63) // 64, DH_GRID)


def _rpw(W):
    return 32 // min(W // 4, 32)


def _dh_cta(rows, W, cap):
    """CTA of gin_bwd_dh_kernel<W> that finishes each row: warp passes of RPW rows dealt round-robin."""
    return (rows // _rpw(W)) // 8 % _dh_grid(cap)


# ------------------------------------------------------------------------------------------------ batches
def _graph(indptr, indices):
    return dict(indptr=np.asarray(indptr, np.int64), indices=np.asarray(indices, np.int64))


def _er(n, m, seed):
    from gcc_b200.datasets import synthetic
    g = synthetic.erdos_renyi(n, m, seed=seed)
    return _graph(g.indptr, g.indices)


def _star(leaves):
    """Centre first (row 0, degree = leaves), leaves of degree 1."""
    ip = np.concatenate([[0, leaves], leaves + np.arange(1, leaves + 1)])
    ix = np.concatenate([np.arange(1, leaves + 1), np.zeros(leaves, np.int64)])
    return _graph(ip, ix)


def _path(n):
    src = np.concatenate([np.arange(n - 1), np.arange(1, n)])
    dst = np.concatenate([np.arange(1, n), np.arange(n - 1)])
    o = np.lexsort((dst, src))
    return _graph(np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]), dst[o])


def _biclique(a, b):
    """K_{a,b}, the a side first: rows 0..a-1 have b neighbours."""
    n = a + b
    src = np.concatenate([np.repeat(np.arange(a), b), np.tile(np.arange(a, n), a)])
    dst = np.concatenate([np.tile(np.arange(a, n), a), np.repeat(np.arange(a), b)])
    o = np.lexsort((dst, src))
    return _graph(np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]), dst[o])


def _single():
    return _graph([0, 0], [])


def _pair():
    return _graph([0, 1, 2], [1, 0])


def _buffers(graphs, node_cap=None, pos_seed=4, swap=True):
    from gcc_b200.datasets.graph_dataset import BatchBuffers
    views = [graphs, graphs[::-1] if swap else graphs]
    n = sum(len(g["indptr"]) - 1 for g in graphs)
    m = sum(len(g["indices"]) for g in graphs)
    buf = BatchBuffers(len(graphs), node_cap or n + 100, m + 100, 32, 64, "cuda")
    _fill_batch(buf, views)
    gen = torch.Generator(device="cuda").manual_seed(pos_seed)
    buf.pos.copy_(0.3 * torch.randn(buf.pos.shape, device="cuda", generator=gen))
    return buf


def _queue_graphs():
    """Blocks of K_{16,257} whose 16 hub rows fall on rows k * 37888 .. + 15, k = 0..4: CTA 0 of gin_bwd_dh_kernel
    finishes rows (8b + w) RPW + k 1184 8 RPW for b = 0 (RPW = 2 at width 64, 4 at width 32; 37888 = 1184 * 8 * 4), so
    its 64-entry hub queue receives 80 rows.  Paths fill the rows in between."""
    graphs, row = [], 0
    for k in range(5):
        target = k * DH_GRID * 8 * 4
        while row < target:
            n = min(1000, target - row)
            graphs.append(_path(n) if n > 1 else _single())
            row += n
        graphs.append(_biclique(16, 257))
        row += 16 + 257
    graphs.append(_er(300, 900, seed=2))
    return graphs


def _batch(kind):
    from gcc_b200.datasets import synthetic
    if kind == "hub":
        # cliques of 290 and 300 (every row a hub), a 600-leaf star (degree > 512: the embedding index is clamped),
        # a single vertex, a pair, a random graph; odd total row count
        return _buffers([_clique(300), _er(61, 150, seed=1), _star(600), _single(), _pair(), _clique(290)])
    if kind == "large":
        return _buffers([_er(1000, 3000 + 37 * i, seed=10 + i) for i in range(36)])
    if kind == "queue":
        graphs = _queue_graphs()
        n = sum(len(g["indptr"]) - 1 for g in graphs)
        return _buffers(graphs, node_cap=max(n + 100, 64 * DH_GRID + 1), swap=False)     # rows placed for CTA 0
    if kind == "c2":
        from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
        g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
        ds = LoadBalanceGraphDataset(rw_hops=256, restart_prob=0.8, positional_embedding_size=32, dgl_graphs_file=g,
                                     num_samples=2000, num_workers=12, num_copies=6, batch_size=256, seed=0)
    else:
        ds = _dataset(synthetic.chung_lu(4000, 30000, seed=6), 24, 64, seed=3)
    buf = ds.sample_batch(first_sample=0)
    torch.cuda.synchronize()
    buf.check_flags()
    return buf


# ------------------------------------------------------------------------------------------------ helpers
def _mm_bound(A, B, depth):
    """Bound of an fp32 sum-of-products over `depth` sequential steps: depth U (|A| |B|)."""
    return depth * U * (A.abs() @ B.abs())


class _Stages:
    """One GIN configuration and its buffers; forward / backward of one view and their float64 checks."""

    def __init__(self, rep, buf, H, L, seed):
        from gcc_b200 import _capi, _lib
        from gcc_b200.models import layout as glayout
        self.lib, self._lib, self.rep = _lib.get(), _lib, rep
        _lib.require_device()
        self.H, self.L = H, L
        self.cfg = glayout.make_cfg(num_layers=L, hidden=H, tensor_cores=0)
        self.lay = glayout.c_layout(self.lib, self.cfg)
        self.flat, self.sd, self.sl = _params(self.cfg, np.random.default_rng(seed))
        o = self.lay.b1[L - 2]
        self.flat[o:o + H] += 200.0                                     # top z1 columns: |mean| >> std
        self.sd["gnn.ginlayers.%d.apply_func.mlp.linears.0.bias" % (L - 2)] = torch.from_numpy(
            self.flat[o:o + H].copy()).double()
        self.params = torch.from_numpy(self.flat).cuda()
        rs, rtotal = glayout.running_slices(self.cfg)
        run = np.zeros(rtotal, np.float32)
        for key, (off, shape) in rs.items():
            run[off:off + shape[0]] = 1.0 if key.endswith("var") else 0.0
        self.running = torch.from_numpy(run).cuda()
        self.nbt = torch.zeros(3 * (L - 1), dtype=torch.int64, device="cuda")
        self.grads = torch.zeros_like(self.params)
        self.eps = float(np.float32(self.cfg.bn_eps))
        self.mom = float(np.float32(self.cfg.bn_momentum))
        self.alloc(buf)
        self.GinStash = _capi.GinStash

    def alloc(self, buf):
        lib, cfg = self.lib, self.cfg
        self.acts = torch.zeros(lib.gccb_gin_acts_bytes(C.byref(cfg), buf.B, buf.node_cap), dtype=torch.uint8,
                                device="cuda")
        self.ws = torch.zeros(lib.gccb_gin_backward_workspace(C.byref(cfg), buf.B, buf.node_cap), dtype=torch.uint8,
                              device="cuda")

    def P(self, off, *shape):
        n = int(np.prod(shape))
        return self.params[off:off + n].view(*shape).double()

    @staticmethod
    def T(base, off, dtype, *shape):
        n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
        assert off >= 0
        return base[off:off + n].view(dtype).view(*shape)

    def forward(self, buf, view, train, drop_base, key=77, step=5):
        _lib = self._lib
        self.feat = torch.zeros(buf.B, self.H, device="cuda")
        _lib.check(self.lib.gccb_gin_forward(
            C.byref(self.cfg), C.byref(buf.c), view, _lib.dptr(buf.pos), _lib.dptr(self.params),
            _lib.dptr(self.running), _lib.dptr(self.nbt), int(train), key, step, drop_base, _lib.dptr(self.acts),
            self.acts.numel(), _lib.dptr(self.feat), None, _lib.stream_ptr()), "gccb_gin_forward")

    def backward(self, buf, view, dfeat, drop_base, key=77, step=5):
        _lib = self._lib
        _lib.check(self.lib.gccb_gin_backward(
            C.byref(self.cfg), C.byref(buf.c), view, _lib.dptr(self.params), _lib.dptr(self.acts), _lib.dptr(dfeat),
            _lib.dptr(self.grads), key, step, drop_base, _lib.dptr(self.ws), self.ws.numel(), _lib.stream_ptr()),
            "gccb_gin_backward")

    def stash(self, buf):
        st = self.GinStash()
        self._lib.check(self.lib.gccb_gin_stash_layout(C.byref(self.cfg), buf.B, buf.node_cap, C.byref(st)),
                        "gccb_gin_stash_layout")
        return st


def _graph_view(buf, view):
    B, cap = buf.B, buf.node_cap
    N = int(buf.node_off[view, B])
    indptr = buf.indptr[view, :N + 1].long()
    deg = indptr[1:] - indptr[:-1]
    E = int(indptr[-1])
    col = buf.indices[view, :E].long()
    A = torch.sparse_csr_tensor(indptr, col, torch.ones(E, dtype=torch.float64, device="cuda"), (N, N))
    gid = buf.graph_id[view, :N].long()
    return dict(N=N, cap=cap, B=B, deg=deg, A=A, gid=gid, col=col, indptr=indptr)


def _paths(g, H, L):
    """What the batch reaches, restated from the kernels' grids and row dealing."""
    N, cap, deg = g["N"], g["cap"], g["deg"]
    rows = torch.arange(N, device="cuda")
    hub = deg > HUB_DEG
    out = dict(N=N, cap=cap, hub_rows=int(hub.sum()), clamped=int((deg > 512).sum()),
               tiles_per_cta=-(-((N + 63) // 64) // _gemm_grid(cap)))
    warp = deg[~hub & (deg > 0)]
    out["warp_deg_mod8"] = len(set((warp % 8).tolist()))
    for W in sorted({H, 64}):
        c = _dh_cta(rows[hub], W, cap)
        out["dh%d_hub_rows_per_cta" % W] = int(torch.bincount(c).max()) if c.numel() else 0
    return out


# ------------------------------------------------------------------------------------------------ the checks
def _check_forward(S, buf, view, g, st, fwd_running0, train):
    """Forward stages of one view; returns the float64 quantities the backward checks reuse."""
    rep, H, L, lay, cfg = S.rep, S.H, S.L, S.lay, S.cfg
    N, cap, B, deg, A, gid = g["N"], g["cap"], g["B"], g["deg"], g["A"], g["gid"]
    acts, T, P = S.acts, S.T, S.P
    grid = _gemm_grid(cap)
    RP = 1024 // H
    D_T = 21                                                     # tile_colstats depth + the float64 atomics
    D_Y = -(-N // (grid * RP)) + RP + 1
    stats = T(acts, st.stats, torch.float64, L - 1, 3, 2, H)

    def agg(x):
        return x + A @ x, x.abs() + A @ x.abs()

    # X0 = [pos | emb(clamp(deg, 0, 512)) | seed | 0]
    x0 = T(acts, st.x0, torch.float32, cap, 64)[:N]
    sub_deg = buf.sub_deg[view, :N].long().clamp(0, cfg.max_degree)
    want = torch.zeros(N, 64, device="cuda")
    want[:, :cfg.pos_dim] = buf.pos[view, :N]
    want[:, cfg.pos_dim:cfg.pos_dim + cfg.deg_dim] = S.params[lay.emb:lay.emb + (cfg.max_degree + 1) * cfg.deg_dim].view(
        -1, cfg.deg_dim)[sub_deg]
    want[:, cfg.pos_dim + cfg.deg_dim] = (torch.arange(N, device="cuda") == buf.node_off[view, gid].long()).float()
    rep.exact("X0", x0, want)
    fwd = dict(x0=x0)
    hs = [x0]
    for l in range(L - 1):
        inf, KW = (cfg.pos_dim + cfg.deg_dim + 1, 64) if l == 0 else (H, H)
        W1, W2 = P(lay.w1[l], H, inf), P(lay.w2[l], H, H)
        W1f = torch.zeros(H, KW, device="cuda", dtype=torch.float64)
        W1f[:, :inf] = W1
        b1, b2 = P(lay.b1[l], H), P(lay.b2[l], H)
        hin = hs[-1].double()
        a = T(acts, st.a[l], torch.float32, cap, KW)[:N]
        ref, mag = agg(hin)
        rep.check("a = h + sum_nbr h", a, ref, (deg + 9).double()[:, None] * U * mag)
        z1 = T(acts, st.z1[l], torch.float32, cap, H)[:N]
        ad = a.double()
        rep.check("z1 GEMM", z1, ad @ W1f.t() + b1, _mm_bound(ad, W1f.t(), KW + 2) + U * b1.abs())
        if train:
            S1 = stats[l, 0]
            m1, i1, sc1, sh1 = _coef(S1, N, P(lay.bn1_w[l], H), P(lay.bn1_b[l], H), S.eps)
        else:
            r = S.running[(l * 3) * 2 * H:(l * 3 + 1) * 2 * H].double()
            m1, i1 = r[:H], 1.0 / torch.sqrt(r[H:] + S.eps)
            sc1 = P(lay.bn1_w[l], H) * i1
            sh1 = P(lay.bn1_b[l], H) - m1 * sc1
        z1d = z1.double()
        pre1 = z1d * sc1 + sh1
        x1 = pre1.clamp_min(0.0)
        e_x1 = 8 * U * ((z1d * sc1).abs() + sh1.abs() + (m1 * sc1).abs())
        z2 = T(acts, st.z2[l], torch.float32, cap, H)[:N]
        rep.check("z2 GEMM", z2, x1 @ W2.t() + b2,
                  _mm_bound(x1, W2.t(), H + 2) + e_x1 @ W2.abs().t() + U * b2.abs())
        z2d = z2.double()
        if train:
            for which, z in ((0, z1d), (1, z2d)):
                Sx = stats[l, which]
                s1b, s2b = D_T * U * z.abs().sum(0), (D_T + 1) * U * (z * z).sum(0)
                rep.check("stats of z1, z2: sum", Sx[0], z.sum(0), s1b)
                rep.check("stats of z1, z2: sum of squares", Sx[1], (z * z).sum(0), s2b)
            mA, iA, scA, shA = _coef(stats[l, 1], N, P(lay.bna_w[l], H), P(lay.bna_b[l], H), S.eps)
        else:
            r = S.running[(l * 3 + 1) * 2 * H:(l * 3 + 2) * 2 * H].double()
            mA, iA = r[:H], 1.0 / torch.sqrt(r[H:] + S.eps)
            scA = P(lay.bna_w[l], H) * iA
            shA = P(lay.bna_b[l], H) - mA * scA
        ya = z2d * scA + shA
        y = ya.clamp_min(0.0)
        e_y = 8 * U * ((z2d * scA).abs() + shA.abs() + (mA * scA).abs())
        if train:
            Sb = stats[l, 2]
            rep.check("stats of y", Sb[0], y.sum(0), e_y.sum(0) + D_Y * U * y.sum(0))
            rep.check("stats of y", Sb[1], (y * y).sum(0),
                      (2 * y * e_y + e_y * e_y).sum(0) + (D_Y + 1) * U * (y * y).sum(0))
            mB, iB, scB, shB = _coef(Sb, N, P(lay.bnb_w[l], H), P(lay.bnb_b[l], H), S.eps)
        else:
            r = S.running[(l * 3 + 2) * 2 * H:(l * 3 + 3) * 2 * H].double()
            mB, iB = r[:H], 1.0 / torch.sqrt(r[H:] + S.eps)
            scB = P(lay.bnb_w[l], H) * iB
            shB = P(lay.bnb_b[l], H) - mB * scB
        hb = y * scB + shB
        h = T(acts, st.h[l], torch.float32, cap, H)[:N]
        rep.check("h (next gather / pooling)" if train else "h (eval, running statistics)", h, hb.clamp_min(0.0),
                  scB.abs() * e_y + 8 * U * ((y * scB).abs() + shB.abs() + (mB * scB).abs()))
        hs.append(h)
        fwd[l] = dict(a=a, z1=z1, z2=z2, x1=x1, e_x1=e_x1, pre1=pre1, W1f=W1f, W2=W2, inf=inf, KW=KW, ya=ya, y=y,
                      hb=hb, e_y=e_y, m1=m1, i1=i1, sc1=sc1, sh1=sh1, A=(mA, iA, scA, shA), Bc=(mB, iB, scB, shB))
    if not train:
        return fwd
    # running statistics (block 0 of the kernel reading each BatchNorm's coefficients), num_batches_tracked
    n = float(N)
    for l in range(L - 1):
        for k in range(3):
            Sx = stats[l, k]
            mean = Sx[0] / n
            var = (Sx[1] / n - mean * mean).clamp_min(0.0) * n / (n - 1)
            o = (l * 3 + k) * 2 * H
            old = fwd_running0[o:o + 2 * H].double()
            want = torch.cat([(1 - S.mom) * old[:H] + S.mom * mean, (1 - S.mom) * old[H:] + S.mom * var])
            rep.check("running mean / unbiased var", S.running[o:o + 2 * H], want,
                      U * want.abs() + 2.0 ** -50 * (old.abs() + torch.cat([mean.abs(), Sx[1].abs() / n + mean * mean])))
    # pooled sums per graph and layer, from the stored h
    PW = st.PW
    pooled = T(acts, st.pooled, torch.float32, L, B, PW)
    for l, hh in enumerate(hs):
        W = hh.shape[1]
        run = W // 4 if W < 128 else 8
        hd = hh.double()
        want = torch.zeros(B, W, dtype=torch.float64, device="cuda").index_add_(0, gid, hd)
        mag = torch.zeros(B, W, dtype=torch.float64, device="cuda").index_add_(0, gid, hd.abs())
        rep.check("pooled sums", pooled[l, :, :W], want, (run + 2) * U * mag)
    fwd["pooled"] = pooled
    return fwd


def _check_heads(S, g, st, fwd, dfeat, drop_base, key=77, step=5):
    """score, feat, and the backward of the normalisation and the heads: dS, dpool, dWp, dbp."""
    from oracle import rwr as orwr
    rep, H, L, lay, cfg = S.rep, S.H, S.L, S.lay, S.cfg
    B = g["B"]
    pooled = fwd["pooled"]
    # score follows pooled in the stash (make_acts_layout: 256-byte aligned regions)
    score = S.T(S.acts, st.pooled + (L * B * st.PW * 4 + 255) // 256 * 256, torch.float32, B, H)
    keep = [torch.from_numpy(orwr.dropout_mask(key, step, drop_base + l, B * H, cfg.dropout_p).reshape(B, H)).cuda()
            if drop_base >= 0 else torch.ones(B, H, dtype=torch.bool, device="cuda") for l in range(L)]
    scale = 1.0 / (1.0 - cfg.dropout_p) if drop_base >= 0 else 1.0
    want = torch.zeros(B, H, dtype=torch.float64, device="cuda")
    err = torch.zeros_like(want)
    s_abs = torch.zeros_like(want)
    for l in range(L):
        inf = cfg.pos_dim + cfg.deg_dim + 1 if l == 0 else H
        Wp, bp = S.P(lay.wp[l], H, inf), S.P(lay.bp[l], H)
        pl = pooled[l, :, :inf].double()
        k = keep[l].double() * scale
        s = (pl @ Wp.t() + bp) * k
        want += s
        s_abs += s.abs()
        err += k * (_mm_bound(pl, Wp.t(), -(-inf // 4) + 3) + U * bp.abs())
    err += L * U * s_abs
    rep.check("score (heads, dropout, layer sum)", score, want, err)
    x = score.double()
    dn = H // 32 + 5
    nrm = x.norm(dim=1, keepdim=True)
    fref = x / nrm
    rep.check("feat (L2 normalisation)", S.feat, fref, (dn / 2 + 3) * U * fref.abs())
    # backward of the normalisation from the stored score, then the dropout scale
    gy = dfeat.double()
    dot = (x * gy).sum(1, keepdim=True)
    q = dot / (nrm * nrm)
    e_q = dn * U * (x * gy).abs().sum(1, keepdim=True) / (nrm * nrm) + q.abs() * (dn + 4) * U
    dx = (gy - x * q) / nrm
    e_dx = (x.abs() * e_q + (dn / 2 + 4) * U * (gy.abs() + (x * q).abs())) / nrm
    dpool = S.T(S.ws, st.dpool, torch.float32, L, B, st.DW)
    G, slack = S.G, S.Gslack
    for l in range(L):
        inf = cfg.pos_dim + cfg.deg_dim + 1 if l == 0 else H
        Wp = S.P(lay.wp[l], H, inf)
        k = keep[l].double() * scale
        dS, e_dS = dx * k, e_dx * k
        pl = pooled[l, :, :inf].double()
        rep.check("dpool = dS Wp", dpool[l, :, :inf], dS @ Wp, _mm_bound(dS, Wp, H + 1) + e_dS @ Wp.abs())
        assert not dpool[l, :, inf:].any()
        o = lay.wp[l]
        rep.check("dWp, dbp", G[o:o + H * inf].view(H, inf), dS.t() @ pl,
                  _mm_bound(dS.t(), pl, B + 1) + e_dS.t() @ pl.abs() + slack[o:o + H * inf].view(H, inf))
        o = lay.bp[l]
        rep.check("dWp, dbp", G[o:o + H], dS.sum(0), (B + 1) * U * dS.abs().sum(0) + e_dS.sum(0) + slack[o:o + H])
    return dpool


def _check_backward(S, buf, view, g, st, fwd, dpool, oracle_grads):
    rep, H, L, lay, cfg = S.rep, S.H, S.L, S.lay, S.cfg
    N, cap, B, deg, A, gid = g["N"], g["cap"], g["B"], g["deg"], g["A"], g["gid"]
    T, P, ws = S.T, S.P, S.ws
    G, slack = S.G, S.Gslack
    grid = _gemm_grid(cap)
    RP = 1024 // H
    D_A = -(-N // (grid * RP)) + RP + 1
    rows = torch.arange(N, device="cuda")
    hub = deg > HUB_DEG
    hub_cta = int(torch.bincount(_dh_cta(rows[hub], H, cap)).max()) if hub.any() else 0
    RPW = _rpw(H)
    D_B = -(-N // (_dh_grid(cap) * 8 * RPW)) + int(math.log2(RPW)) + 9 + hub_cta + 1
    D_1 = 21
    per = -(-((N + 63) // 64) // SMS)
    D_W, D_Wb = 64 * per + 35 + 1, 64 * per + SMS + 1

    def gsl(off, *shape):
        n = int(np.prod(shape))
        return G[off:off + n].view(*shape), slack[off:off + n].view(*shape)

    def mean(x):
        return x.mean(0)

    lt = L - 2
    for l in range(L - 1):
        f = fwd[l]
        z1d, z2d = f["z1"].double(), f["z2"].double()
        survives = l <= 1
        if l == lt:
            # the top layer's dh is dpool[L-1] broadcast by graph: its whole BN_b / BN_a chain is reconstructed
            mA, iA, scA, shA = f["A"]
            mB, iB, scB, shB = f["Bc"]
            ya, y, hb, e_ya = f["ya"], f["y"], f["hb"], f["e_y"]
            dh = dpool[L - 1, :, :H].double()[gid]
            scaleA = ((z2d * scA).abs() + shA.abs() + (mA * scA).abs()).max(0).values
            scaleB = ((y * scB).abs() + shB.abs() + (mB * scB).abs()).max(0).values
            riskA, riskB = ya.abs() <= PRE_EXCL * scaleA, hb.abs() <= PRE_EXCL * scaleB
            yhat = (y - mB) * iB
            e_yhat = iB * (e_ya + 8 * U * (y.abs() + mB.abs()))
            g4 = (hb > 0) * dh
            mB1, mB2 = mean(g4), mean(g4 * yhat)
            dy = scB * (g4 - mB1 - yhat * mB2)
            g3 = (ya > 0) * dy
            z2hat = (z2d - mA) * iA
            mA1, mA2 = mean(g3), mean(g3 * z2hat)
            dz2 = scA * (g3 - mA1 - z2hat * mA2)
            dB1 = (riskB * dh.abs()).sum(0) / N + D_B * U * mean(g4.abs())
            dB2 = (riskB * (dh * yhat).abs()).sum(0) / N + D_B * U * mean((g4 * yhat).abs()) + mean(g4.abs() * e_yhat)
            ddy = scB.abs() * (dB1 + yhat.abs() * dB2 + mB2.abs() * e_yhat) + \
                8 * U * scB.abs() * (g4.abs() + mB1.abs() + (yhat * mB2).abs())
            e_z2hat = iA * 8 * U * (z2d.abs() + mA.abs())
            mask_a = (ya > 0).double()
            dA1 = (riskA * dy.abs()).sum(0) / N + mean(mask_a * ddy) + D_A * U * mean(g3.abs())
            dA2 = (riskA * (dy * z2hat).abs()).sum(0) / N + mean(mask_a * ddy * z2hat.abs()) + \
                mean(g3.abs() * e_z2hat) + D_A * U * mean((g3 * z2hat).abs())
            e_dz2 = scA.abs() * (mask_a * ddy + dA1 + z2hat.abs() * dA2 + mA2.abs() * e_z2hat) + \
                8 * U * scA.abs() * (g3.abs() + mA1.abs() + (z2hat * mA2).abs())
            keep = ~(riskA | riskB)
            rep.notes.append("view %d layer %d: dz2 elements excluded near a BN_a / BN_b ReLU kink: %d of %d" % (
                view, l, int((~keep).sum()), keep.numel()))
            for off, val, err in ((lay.bnb_w[l], N * mB2, N * dB2), (lay.bnb_b[l], N * mB1, N * dB1),
                                  (lay.bna_w[l], N * mA2, N * dA2), (lay.bna_b[l], N * mA1, N * dA1)):
                got, sl = gsl(off, H)
                rep.check("BN_a / BN_b gamma, beta grads (top)", got, val, err + U * val.abs() + sl)
            if survives:
                dz2k = T(ws, st.dz2[l & 1], torch.float32, cap, H)[:N]
                rep.check("dz2 (BN_b, BN_a backward, top)", dz2k, dz2, e_dz2, keep)
                src, e_src = dz2k.double(), torch.zeros_like(dz2)
            else:
                # excluded elements may pass or block their whole gradient
                src = dz2
                e_src = e_dz2 + (~keep) * scA.abs() * (riskA * dy.abs() + riskB * (scB * dh).abs())
        elif survives:
            src = T(ws, st.dz2[l & 1], torch.float32, cap, H)[:N].double()
            e_src = torch.zeros_like(src)
        else:
            # layer 2 at L = 5: its buffers were reused by layer 0; the float64 oracle's autograd gradients
            _check_vs_oracle(S, l, oracle_grads)
            continue
        tag = "" if survives else " (top, reconstructed)"
        # g1 = [bn1(z1) > 0] (dz2 W2), then dz1 = BN1 backward (in place in g1)
        W2 = f["W2"]
        dx1 = src @ W2
        e_dx1 = _mm_bound(src, W2, H + 2) + e_src @ W2.abs()
        m1, i1, sc1, sh1, pre1 = f["m1"], f["i1"], f["sc1"], f["sh1"], f["pre1"]
        scale1 = ((z1d * sc1).abs() + sh1.abs() + (m1 * sc1).abs()).max(0).values
        risk1 = pre1.abs() <= PRE_EXCL * scale1
        mask1 = (pre1 > 0).double()
        gg = mask1 * dx1
        zhat = (z1d - m1) * i1
        e_zhat = i1 * 8 * U * (z1d.abs() + m1.abs())
        n1, n2 = mean(gg), mean(gg * zhat)
        dg = mask1 * e_dx1
        d1 = mean(dg) + (risk1 * dx1.abs()).sum(0) / N + D_1 * U * mean(gg.abs())
        d2 = mean(dg * zhat.abs()) + (risk1 * (dx1 * zhat).abs()).sum(0) / N + mean(gg.abs() * e_zhat) + \
            D_1 * U * mean((gg * zhat).abs())
        dz1 = sc1 * (gg - n1 - zhat * n2)
        e_dz1 = sc1.abs() * (dg + d1 + zhat.abs() * d2 + n2.abs() * e_zhat) + \
            8 * U * sc1.abs() * (gg.abs() + n1.abs() + (zhat * n2).abs())
        keep1 = ~risk1
        rep.notes.append("view %d layer %d: dz1 elements excluded near the BN1 ReLU kink: %d of %d" % (
            view, l, int(risk1.sum()), risk1.numel()))
        if survives:
            dz1k = T(ws, st.g1[l & 1], torch.float32, cap, H)[:N]
            rep.check("dz1 (BN1 backward)", dz1k, dz1, e_dz1, keep1)
            dsrc, e_dsrc = dz1k.double(), torch.zeros_like(dz1)
        else:
            dsrc, e_dsrc = dz1, e_dz1 + risk1 * (sc1 * dx1).abs() * 2
        for off, val, err in ((lay.bn1_w[l], N * n2, N * d2), (lay.bn1_b[l], N * n1, N * d1)):
            got, sl = gsl(off, H)
            rep.check("BN1 gamma, beta grads" + tag, got, val, err + U * val.abs() + sl)
        # weight gradients: dW2 = dz2^T x1, db2 = sum dz2, dW1 = dz1^T a, db1 = sum dz1 (split-K)
        x1, e_x1 = f["x1"], f["e_x1"]
        got, sl = gsl(lay.w2[l], H, H)
        rep.check("dW2 (split-K)" + tag, got, src.t() @ x1,
                  _mm_bound(src.t(), x1, D_W) + src.abs().t() @ e_x1 + e_src.t() @ x1.abs() + sl)
        got, sl = gsl(lay.b2[l], H)
        rep.check("db2 = column sums of dz2" + tag, got, src.sum(0), D_Wb * U * src.abs().sum(0) + e_src.sum(0) + sl)
        ad = f["a"].double()
        inf = f["inf"]
        got, sl = gsl(lay.w1[l], H, inf)
        rep.check("dW1 (split-K)" + tag, got, (dsrc.t() @ ad)[:, :inf],
                  (_mm_bound(dsrc.t(), ad, D_W) + e_dsrc.t() @ ad.abs())[:, :inf] + sl)
        got, sl = gsl(lay.b1[l], H)
        rep.check("db1 = column sums of dz1" + tag, got, dsrc.sum(0), D_Wb * U * dsrc.abs().sum(0) + e_dsrc.sum(0) + sl)
        if l == 0:
            W1f = f["W1f"]
            da = T(ws, st.da, torch.float32, cap, 64)[:N]
            rep.check("da = dz1 W1", da, dsrc @ W1f, _mm_bound(dsrc, W1f, H + 2))
            assert not da[:, inf:].any()
            dh0 = T(ws, st.dh, torch.float32, cap, 64)[:N]
            dad = da.double()
            dp = dpool[0].double()[gid][:, :64]
            rep.check("dh0 = dpool[0] + (I + A) da", dh0, dp + dad + A @ dad,
                      (deg + 10).double()[:, None] * U * (dad.abs() + A @ dad.abs() + dp.abs()))
            # degree-embedding gradient: histogram of dh0's embedding columns by clamp(sub_deg, 0, 512)
            D, P0 = cfg.deg_dim, cfg.pos_dim
            sd = buf.sub_deg[view, :N].long().clamp(0, cfg.max_degree)
            terms = dh0[:, P0:P0 + D].double()
            want = torch.zeros(cfg.max_degree + 1, D, dtype=torch.float64, device="cuda").index_add_(0, sd, terms)
            mag = torch.zeros_like(want).index_add_(0, sd, terms.abs())
            cnt = torch.bincount(sd, minlength=cfg.max_degree + 1).double()[:, None]
            got, sl = gsl(lay.emb, cfg.max_degree + 1, D)           # up to 64 CTA partials added into grads
            rep.check("degree-embedding gradient", got, want, (cnt + 64) * U * mag + 64 * sl)


def _oracle_grads(S, buf, view, dfeat, drop_base, key=77, step=5):
    """float64 autograd gradients of sum(feat * dfeat) through oracle.model.gin_encoder_forward (CPU)."""
    from oracle import model as om
    from oracle import rwr as orwr
    B, L, H = buf.B, S.L, S.H
    N, E = int(buf.node_off[view, B]), int(buf.edge_off[view, B])
    noff = buf.node_off[view].cpu().numpy().astype(np.int64)
    seed = np.zeros(N, np.int64)
    seed[noff[:B]] = 1
    Pd = {k: v.clone().requires_grad_(not k.endswith("eps")) for k, v in S.sd.items()}
    keep = [orwr.dropout_mask(key, step, drop_base + i, B * H, 0.5).reshape(B, H) for i in range(L)] \
        if drop_base >= 0 else None
    f, _, _ = om.gin_encoder_forward(Pd, buf.indptr[view, :N + 1].cpu().numpy().astype(np.int64),
                                     buf.indices[view, :E].cpu().numpy().astype(np.int64),
                                     buf.pos[view, :N].cpu().double(), seed, buf.sub_deg[view, :N].cpu().numpy(),
                                     noff, num_layers=L, dropout_keep=keep)
    names = [k for k in S.sl]
    gr = torch.autograd.grad((f * dfeat.cpu().double()).sum(), [Pd[k] for k in names], allow_unused=True)
    return {k: gv for k, gv in zip(names, gr)}


def _check_vs_oracle(S, l, og):
    """Layer l's gradients against the oracle's, per tensor: rtol 2e-3, atol 2e-4 of the tensor's scale (the emulator
    tests' bar).  Entries outside it are counted and printed; they must be isolated ReLU-kink flips, held to the wide
    SIMT test's rule: at least 99.9 % of a tensor's entries (all but one in a tensor of fewer than 1000) within
    5e-3 |want| + 5e-3 scale, none beyond 5e-2 of the scale."""
    worst = 0.0
    for k, (off, shape) in S.sl.items():
        if not k.startswith("gnn.ginlayers.%d." % l) or k.endswith("eps"):
            continue
        n = int(np.prod(shape))
        got = S.G[off:off + n].view(*shape).cpu()
        if "mlp.linears" in k and k.endswith("bias"):
            continue                                           # checked against its bound where the buffers survive
        want = og[k]
        scale = max(float(want.abs().max()), 1e-3)
        err = (got - want).abs()
        r = err / (2e-3 * want.abs() + 2e-4 * scale)
        worst = max(worst, float(r.max()))
        outside = int((r > 1.0).sum())
        if outside:
            wide = int((err > 5e-3 * want.abs() + 5e-3 * scale).sum())
            S.rep.notes.append("layer %d %s: %d of %d entries outside the emulator bar (worst %.2f of it), %d outside "
                               "5e-3, largest |err| %.2e of the scale" % (l, k, outside, r.numel(), float(r.max()),
                                                                          wide, float(err.max()) / scale))
            assert wide <= max(1, r.numel() // 1000) and float(err.max()) <= 5e-2 * scale, (S.rep.tag, k, wide)
    S.rep.notes.append("layer %d vs the float64 oracle's autograd: worst |err| / (2e-3 |want| + 2e-4 scale) = %.3f" % (
        l, worst))


def _run_views(S, buf, st, g_views, eval_after=True):
    rep, L, H = S.rep, S.L, S.H
    gen = torch.Generator(device="cuda").manual_seed(H + L)
    for view in (0, 1):
        drop_base = 0 if view == 0 else L            # distinct dropout masks per view
        g = g_views[view]
        dfeat = torch.randn(buf.B, H, device="cuda", generator=gen)
        run0 = S.running.clone()
        nbt0 = S.nbt.clone()
        g_before = S.grads.clone()
        S.forward(buf, view, True, drop_base)
        S.backward(buf, view, dfeat, drop_base)
        torch.cuda.synchronize()
        assert torch.equal(S.nbt, nbt0 + 1)
        S.G = S.grads.double() - g_before.double()
        S.Gslack = U * S.grads.double().abs()
        fwd = _check_forward(S, buf, view, g, st, run0, True)
        dpool = _check_heads(S, g, st, fwd, dfeat, drop_base)
        og = _oracle_grads(S, buf, view, dfeat, drop_base) if L == 5 else None
        _check_backward(S, buf, view, g, st, fwd, dpool, og)
    if eval_after:
        # eval mode (what generate.py runs): h from the running statistics; running buffers and counters untouched
        run0, nbt0 = S.running.clone(), S.nbt.clone()
        S.forward(buf, 0, False, -1)
        torch.cuda.synchronize()
        _check_forward(S, buf, 0, g_views[0], st, None, False)
        rep.exact("running statistics after eval", S.running, run0)
        assert torch.equal(S.nbt, nbt0)


CASES = [("sampled", 32, 2), ("sampled", 64, 2), ("sampled", 32, 3), ("sampled", 64, 3), ("sampled", 32, 5),
         ("sampled", 64, 5), ("sampled", 128, 3), ("c2", 64, 5), ("hub", 32, 3), ("hub", 64, 3), ("large", 32, 2),
         ("large", 64, 3), ("queue", 32, 3), ("queue", 64, 3), ("short", 32, 3), ("short", 64, 5)]


@pytest.mark.parametrize("kind,H,L", CASES)
def test_simt_gin_stages_vs_float64(kind, H, L):
    rep = _Report("H=%d %s L=%d" % (H, kind, L))
    if kind == "short":
        full = _buffers([_er(200 + 13 * i, 700, seed=30 + i) for i in range(12)], pos_seed=9)
        S = _Stages(rep, full, H, L, seed=L * 1000 + H)
        for view in (0, 1):                                          # leave stale activations and gradients behind
            S.forward(full, view, True, -1)
            S.backward(full, view, torch.ones(full.B, H, device="cuda"), -1)
        torch.cuda.synchronize()
        n_full = int(full.node_off[0, full.B])
        buf = full.narrow(7)
        graphs = [_er(150 + 11 * i, 500, seed=60 + i) for i in range(7)]
        _fill_batch(buf, [graphs, graphs[::-1]])
        buf.pos[:, :int(buf.node_off[0, 7])].copy_(0.3 * torch.randn(2, int(buf.node_off[0, 7]), 32, device="cuda"))
        S.grads.zero_()
    else:
        buf = _batch(kind)
        S = _Stages(rep, buf, H, L, seed=L * 1000 + H)
    st = S.stash(buf)
    assert st.a16 == -1 and st.coef1 == -1 and st.DW == max(H, 64)     # the SIMT path, whatever H
    gv = [_graph_view(buf, v) for v in (0, 1)]
    for v in (0, 1):
        p = _paths(gv[v], H, L)
        rep.notes.append("view %d: %s" % (v, ", ".join("%s %s" % kv for kv in p.items())))
        if kind in ("sampled", "c2"):
            assert p["warp_deg_mod8"] == 8
        if kind == "hub":
            assert p["hub_rows"] >= 590 and p["clamped"] >= 1 and p["N"] % 2 == 1
            assert int((gv[v]["deg"] == 0).sum()) >= 1 and int((gv[v]["deg"] == 1).sum()) >= 602
        if kind == "large":
            assert p["tiles_per_cta"] >= 2
        if kind == "queue":
            assert p["cap"] > 64 * DH_GRID and all(p["dh%d_hub_rows_per_cta" % W] > HUB_QUEUE for W in {H, 64})
        if kind == "short":
            assert p["N"] < n_full
    _run_views(S, buf, st, gv)
    rep.show()
