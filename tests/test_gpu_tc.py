"""GPU (H100): the wgmma / TMA contraction kernel (csrc/tc_gemm.cu) through the C ABI against
torch fp32 matmul of the same bf16-rounded operands (fp32 accumulate on both sides: the only difference
is summation order, so the bar is 2e-3 of the output scale)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _gemm(A, Bm, m_valid=None, bias=None, alpha=1.0, want_bf16=False, stats=False, splits=1):
    from gcc_b200 import _lib
    lib = _lib.get()
    M, K = A.shape
    N = Bm.shape[0]
    out = torch.full((M, N), float("nan"), device="cuda")
    outb = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda") if want_bf16 else None
    cs = torch.zeros(2, N, dtype=torch.float64, device="cuda") if stats else None
    md = torch.tensor([m_valid], dtype=torch.int32, device="cuda") if m_valid is not None else None
    scratch = torch.empty(splits * M * N, device="cuda") if splits > 1 else None
    _lib.check(lib.gccb_tc_gemm_bf16(_lib.dptr(A), _lib.dptr(Bm), M, N, K, _lib.dptr(md), _lib.dptr(bias), alpha,
                                     _lib.dptr(out), _lib.dptr(outb), N, _lib.dptr(cs), splits, _lib.dptr(scratch),
                                     _lib.stream_ptr()), "gccb_tc_gemm_bf16")
    torch.cuda.synchronize()
    return out, outb, cs


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (300, 256, 256), (1000, 128, 64), (4096, 256, 256),
                                   (257, 32, 128), (40000, 256, 256)])
def test_tc_gemm_matches_fp32_matmul(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    Bm = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    mv = M - 37 if M > 200 else M
    out, outb, cs = _gemm(A, Bm, m_valid=mv, bias=bias, alpha=0.5, want_bf16=True, stats=True)
    want = 0.5 * (A.float() @ Bm.float().t()) + bias
    scale = float(want.abs().max())
    err = float((out[:mv] - want[:mv]).abs().max()) / scale
    print("tc_gemm M=%d N=%d K=%d: max |err| / max |out| = %.2e" % (M, N, K, err))
    assert err < 2e-3, err
    assert torch.isnan(out[mv:]).all()                     # rows beyond the device-side row count stay untouched
    assert torch.allclose(outb[:mv].float(), want[:mv], atol=1e-2 * scale, rtol=1e-2)
    w64 = want[:mv].double()
    assert torch.allclose(cs[0], w64.sum(0), atol=1e-3 * scale * mv ** 0.5 + 1e-6)
    assert torch.allclose(cs[1], (w64 * w64).sum(0), rtol=5e-3)


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
