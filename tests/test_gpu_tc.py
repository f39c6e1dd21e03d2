"""GPU (H100): the wgmma / TMA contraction kernel (csrc/tc_gemm.cu) through the C ABI against float64
products of the same bf16-rounded operands.  The kernel accumulates in fp32, so every output element is held to
the dot-product bound  |got - want| <= C_DOT * K * 2^-24 * |alpha| * (|A| . |B|^T) + 2^-24 * (|alpha| |A| . |B|^T + |bias|)
(the absolute products summed in float64; the second term is the rounding of the epilogue's alpha * acc + bias).
C_DOT = 4 allows for the tensor core's accumulator not rounding to nearest."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C_DOT = 4.0


def _gemm(A, Bm, m_valid=None, bias=None, alpha=1.0, want_bf16=False, stats=False, splits=1, ldo=None):
    from gcc_b200 import _lib
    lib = _lib.get()
    M, K = A.shape
    N = Bm.shape[0]
    ldo = ldo or N
    out = torch.full((M, ldo), float("nan"), device="cuda")
    outb = torch.zeros(M, ldo, dtype=torch.bfloat16, device="cuda") if want_bf16 else None
    cs = torch.zeros(2, N, dtype=torch.float64, device="cuda") if stats else None
    md = torch.tensor([m_valid], dtype=torch.int32, device="cuda") if m_valid is not None else None
    scratch = torch.empty(splits * M * N, device="cuda") if splits > 1 or ldo % 8 else None
    _lib.check(lib.gccb_tc_gemm_bf16(_lib.dptr(A), _lib.dptr(Bm), M, N, K, _lib.dptr(md), _lib.dptr(bias), alpha,
                                     _lib.dptr(out), _lib.dptr(outb), ldo, _lib.dptr(cs), splits, _lib.dptr(scratch),
                                     _lib.stream_ptr()), "gccb_tc_gemm_bf16")
    torch.cuda.synchronize()
    return out, outb, cs


_ROWS = [
    (128, 64, 64, None, None), (300, 256, 256, None, None), (1000, 128, 64, None, None), (4096, 256, 256, None, None),
    (257, 32, 128, None, None), (40000, 256, 256, None, None),
    (20000, 128, 128, 19990, None),     # more row tiles than SMs, N = 128: the resident-B variant BRES<128>
    (20000, 256, 64, 19990, None),      # resident B with a single k-block (layer 0's K)
    (300, 64, 128, 290, 67),            # row pitch > N and not a multiple of 8: via scratch, bias / alpha in the reduce
    (600, 768, 128, 555, None),         # N > 512: the bias is read from global memory, three column tiles
    (1000, 128, 64, 0, None),           # no valid row: nothing written, statistics stay zero
    (500, 256, 128, 10 ** 6, None),     # more valid rows than M_cap: clamped to M_cap
    (1000, 256, 448, None, None),       # 7 k-blocks: the 4-stage ring wraps inside a tile
    (300, 128, 320, None, None)]        # 5 k-blocks


@pytest.mark.parametrize("M,N,K,mv,ldo", _ROWS, ids=["-".join(str(x) for x in r if x is not None) for r in _ROWS])
def test_tc_gemm_matches_fp32_matmul(M, N, K, mv, ldo):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    Bm = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    if mv is None:
        mv = M - 37 if M > 200 else M
    stats = N <= 256 and not ldo                           # fused statistics need one column tile and a direct store
    out, outb, cs = _gemm(A, Bm, m_valid=mv, bias=bias, alpha=0.5, want_bf16=True, stats=stats, ldo=ldo)
    mv = min(mv, M)
    A64, B64 = A.double(), Bm.double()
    prod = A64.abs() @ B64.abs().t()
    want = 0.5 * (A64 @ B64.t()) + bias.double()
    bound = C_DOT * K * U * 0.5 * prod + U * (0.5 * prod + bias.double().abs())
    err = (out[:mv, :N].double() - want[:mv]).abs()
    ratio = float((err / bound[:mv]).max()) if mv else 0.0
    print("tc_gemm M=%d N=%d K=%d valid=%d ldo=%s: worst |err| / bound = %.3f" % (M, N, K, mv, ldo, ratio))
    assert ratio <= 1.0, ratio
    assert torch.isnan(out[mv:]).all()                     # rows beyond the device-side row count stay untouched
    assert torch.isnan(out[:, N:]).all()                   # and so do the columns between N and the row pitch
    assert torch.equal(outb[:mv, :N], out[:mv, :N].to(torch.bfloat16))   # bf16 copy = RNE of the fp32 result
    if not stats:
        return
    if mv == 0:
        assert not cs.any()
        return
    scale = float(want[:mv].abs().max())
    w64 = want[:mv].double()
    assert torch.allclose(cs[0], w64.sum(0), atol=1e-3 * scale * mv ** 0.5 + 1e-6)
    assert torch.allclose(cs[1], (w64 * w64).sum(0), rtol=5e-3)
    # against the stored values themselves: fp32 partial sums (2 rows, 3 shuffle levels, the CTA's tiles, 8 warps)
    o64 = out[:mv, :N].double()
    depth = 16 + (mv + 127) // 128
    assert ((cs[0] - o64.sum(0)).abs() <= depth * U * o64.abs().sum(0)).all()
    assert ((cs[1] - (o64 * o64).sum(0)).abs() <= (depth + 1) * U * (o64 * o64).sum(0)).all()


def test_tc_gemm_split_k_and_transposed_cast():
    """The weight-gradient shape: dW[256 x 256] = dZ^T . X over ~20k rows, operands transposed by
    gccb_cast_bf16, split-K partials reduced in a fixed order (bit-identical run to run)."""
    from gcc_b200 import _lib
    lib = _lib.get()
    g = torch.Generator(device="cuda").manual_seed(5)
    rows, H, cap = 20000, 256, 20480
    dz = torch.randn(cap, H, device="cuda", generator=g)
    x = torch.randn(cap, H, device="cuda", generator=g)
    nd = torch.tensor([rows], dtype=torch.int32, device="cuda")
    dzT = torch.empty(H, cap, dtype=torch.bfloat16, device="cuda")
    xT = torch.empty(H, cap, dtype=torch.bfloat16, device="cuda")
    for src, dst in ((dz, dzT), (x, xT)):
        _lib.check(lib.gccb_cast_bf16(_lib.dptr(src), cap, H, H, _lib.dptr(dst), cap, H, 1, _lib.dptr(nd),
                                      _lib.stream_ptr()), "gccb_cast_bf16")
    torch.cuda.synchronize()
    assert torch.equal(dzT[:, :rows], dz[:rows].to(torch.bfloat16).t()) and not dzT[:, rows:].any()
    outs = []
    for _ in range(2):
        out, _, _ = _gemm(dzT, xT, splits=37)
        outs.append(out)
    want = dzT.float() @ xT.float().t()
    scale = float(want.abs().max())
    assert torch.allclose(outs[0], want, atol=2e-3 * scale, rtol=0), float((outs[0] - want).abs().max())
    assert torch.equal(outs[0], outs[1])
