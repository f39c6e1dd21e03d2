"""GPU (H100): the contrastive head (csrc/moco.cu) against float64 computed in torch on the GPU, element by element:
gccb_infonce_fused on both its paths, gccb_e2e_nce, the module API (gccb_moco_logits, gccb_nce_loss,
gccb_moco_logits_backward) and gccb_moco_enqueue.  Every float output is held to |got - ref| <= bound, the bound
derived from the kernel's own order of operations (tests/contrastive_bounds.py computes them); `-s` prints the worst
error / bound of each check and case, and a table of the worst over all cases at the end.

Bounds (U = 2^-24; expf costs 4 U (2 ulp), logf 2 U, each other operation U):
  Logits.  SIMT: a d-term fmaf chain, times the fp32 1 / T:  lb = (d + 2) U sum_c |q_c m_c| / T.  The positive logit
    of the merge: ceil(d / 128) fmaf per thread, 5 shuffle levels, 3 adds of the warp partials:  depth ceil(d / 128)
    + 10; of nce_tc_softmax_kernel: ceil(d / 256) + 15.  Tensor cores: the reference takes the bf16-rounded q and queue
    (what the GEMM consumes), lb = (C_DOT d + 2) U (|q16| . |m16|^T) / T, C_DOT = 4 as in test_gpu_tc.py.
  Softmax.  With logit errors e_j, |e_j| <= lb_j, p'_j / p_j = exp(e_j) / sum_k p_k exp(e_k), so
    |log(p'_j / p_j)| <= lb_j + Lr,  Lr = log sum_k p_k exp(lb_k)  (the issue's lb_j + sum_k p_k lb_k, to all orders).
    The fp32 evaluation adds c U, c = the normaliser's summation depth (SIMT: KPT terms per lane, 5 shuffle levels,
    lpos and the nch chunk sums in sequence; tensor cores: ceil(K / 1024) float4 groups per thread + 2, 5 levels,
    9 sequential adds) plus the exps (4 U each, two on the SIMT path), products and divisions, plus |l_j - max| U for
    each exp's rounded argument.  Relative bound: rel_j = expm1(lb_j + Lr + c U + |l_j - max| U).
  Loss per row, -log p_pos = logf(S) + M - l_pos:  lb_pos + Lr + c U + 3 U |log S| + U (|M| + 3 |loss|).  Its mean
    over B rows goes through float atomics in any order:  + (B + 1) U mean |loss_i|.  The mean positive logit: the
    mean of lb_pos + (B + 1) U mean |l_pos|.  Both are absolute: the saturated regime drives the loss to 0.
  dq = ((p_pos - 1) k + sum_j p_j key_j) / (T B):  sum_j rel_j p_j |key_j| + rel_pos p_pos |k|, plus the
    accumulation: SIMT, a chain of up to CK keys in a chunk then nch + 1 merge fmaf (CK + nch + 2) U; tensor cores,
    P rounded to bf16 ((1 + rel)(1 + 2^-8) - 1 relative; bf16 has 8 significant bits, so its unit roundoff is 2^-8,
    not 2^-9) and the dq GEMM over K keys with its split-K reduce (C_DOT K + splits + 2) U, all times the magnitudes
    sum_j p_j |key_j| and |1 - p_pos| |k|; 3 U more for the final scale.
  Teacher-forced, SIMT: the records {m, s, acc[d]} at part + (ch B + i)(d + 2) are checked against float64 with
    the stored m as the shift (m within the chunk's max lb of the exact maximum; s: one exp and KPT + 5 additions per
    term; acc: one exp and up to CK fmaf), then the merge against float64 from the stored records with only the
    positive logit's error and the merge's own exps, products and nch + 1 sums, so an error in the partials is
    counted once.  Tensor cores (workspace of nce_tc_layout, restated in contrastive_bounds.tc_layout): the stored
    logits against q16 . m16^T / T; the stored bf16 P against the float64 softmax of the stored logits (the
    positive logit's error and the exps, then 2^-8); dq against the stored P and p_pos, (C_DOT K + splits + 3) U.
  E2E: logits k_i . q_j / T as d-term chains; dout = (p - I) / B (stored in the workspace): rel_ij p_ij + 3 U |p - I|;
    dk and dq are B-term fmaf chains over dout:  sum_j |ddout_ij| |q_j| / T + (B + 2) U sum_j |dout_ij| |q_j| / T, and
    teacher-forced from the stored dout with the chain alone.
  Module API: moco_logits, (d + 2) U |q| |m| / T; nce_loss from the stored logits (exps, ceil(C / 256) + 13 sums);
    moco_logits_bwd from the stored dout: groups = max(1, 256 / d) strided chains of ceil(K / groups) fmaf, then
    dout_0 k and the groups in sequence:  (ceil(K / groups) + groups + 3) U (|dout_0| |k| + sum_j |dout_j| |m_j|) / T.

Bits: dq is the same bit for bit from run to run, with a dirty workspace, and for a permutation of the batch rows;
only the two statistics go through atomics.  On the tensor-core path the permutation claim relies on a wgmma element
not depending on its row within the tile; it held on the H100.  A b-row call into the engine's [B][d] buffers matches a
call on compact copies of the b rows: dq is the mean over the call's own b rows, so it is not the first b rows of a
B-row call (those carry 1 / B).

Measured on an H100 80GB HBM3, worst error / bound over all cases of each check: tc.p16 1.00 (a single bf16 rounding,
whose worst case is the bound), dq tc 0.74, e2e.dout 0.50, merge.dq 0.43, e2e.dk / e2e.dq from the stored dout 0.42 /
0.37, rec.m 0.21, mean lpos 0.18, merge.loss 0.17, api.dout 0.17, rec.s / rec.acc 0.15, dq simt 0.14, tc.ppos 0.13,
loss 0.12, e2e.loss 0.09, api.logits 0.08, e2e.dk / e2e.dq 0.06, e2e.ldiag 0.04, api.loss 0.03, tc.logits 0.012.
Two chain bounds stay below 1e-2: tc.dq 0.009 (the dq GEMM teacher-forced, depth C_DOT K) and api.dq 0.003
(moco_logits_bwd, depth ceil(K / groups) = 4096 to 16384).  Both are worst-case sums over thousands of roundings that
on random data add with random signs, about sqrt(depth) of them; the kernels' end-to-end dq is held to the tighter
softmax-dominated bounds above, which the mutated kernels (a dropped chunk, a padded key, a bf16 positive logit, the
previous row's p_pos) all exceed."""
import math

import numpy as np
import pytest
import torch

import contrastive_bounds as cb

pytestmark = pytest.mark.gpu

F = torch.nn.functional
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst error / bound over all cases:")
    for name in sorted(_WORST):
        ratio, case = _WORST[name]
        print("  %-22s %.3g   (%s)" % (name, ratio, case))


def _check(case, name, got, want, bound):
    got = torch.as_tensor(got, device=want.device).double()
    assert torch.isfinite(got).all(), (case, name, "non-finite output")
    err = (got - want).abs()
    ratio = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print("%s %-14s worst |err| / bound = %.3g" % (case, name, worst))
    if worst > _WORST.get(name, (-1.0, ""))[0]:
        _WORST[name] = (worst, case)
    if worst > 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError("%s %s: %d of %d elements exceed their bound; worst at flat index %d: got %r want %r "
                             "bound %r" % (case, name, int((ratio > 1).sum()), ratio.numel(), i,
                                           float(got.reshape(-1)[i]), float(want.reshape(-1)[i]),
                                           float(bound.reshape(-1)[i])))


def _lib():
    from gcc_b200 import _lib
    return _lib, _lib.get()


def _inputs(B, K, d, regime, seed):
    """q, k, queue for one logit regime: rand (k a noisy q), half (a half-initialised queue: uniform stdv rows next to
    normalised keys), sat (q = k, the queue orthogonal to q: exact zero negatives), flat (every logit equal), dom (q
    itself among the last keys, so in the last chunk of the SIMT path), dup (every key repeated)."""
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rn(*s):
        return torch.randn(*s, device="cuda", generator=g)

    if regime == "sat":
        h = d // 2
        q = torch.zeros(B, d, device="cuda")
        q[:, :h] = F.normalize(rn(B, h), dim=1)
        mem = torch.zeros(K, d, device="cuda")
        mem[:, h:] = F.normalize(rn(K, d - h), dim=1)
        return q, q.clone(), mem
    if regime == "flat":
        m = F.normalize(rn(d), dim=0)
        return F.normalize(rn(B, d), dim=1), m.expand(B, d).contiguous(), m.expand(K, d).contiguous()
    q = F.normalize(rn(B, d), dim=1)
    k = F.normalize(q + 0.3 * rn(B, d), dim=1)
    mem = F.normalize(rn(K, d), dim=1)
    if regime == "half":
        stdv = 1.0 / (d / 3) ** 0.5
        mem = torch.rand(K, d, device="cuda", generator=g) * 2 * stdv - stdv
        mem[:K // 2] = F.normalize(mem[:K // 2], dim=1)
    elif regime == "dup":
        mem = mem[torch.randint(0, max(1, K // 4), (K,), device="cuda", generator=g)].contiguous()
    elif regime == "dom":
        ck = cb.nce_ck(d)
        n = min(B, K - (cb.cdiv(K, ck) - 1) * ck)
        mem[K - n:] = q[:n]
    return q.contiguous(), k.contiguous(), mem.contiguous()


CANARY = 4096


def _workspace(B, d, K, fill=0):
    """The bytes gccb_infonce_workspace asks for, then CANARY bytes of 0xA5 that no call may touch."""
    _l, lib = _lib()
    n = lib.gccb_infonce_workspace(B, d, K)
    ws = torch.full((n + CANARY,), fill, dtype=torch.uint8, device="cuda")
    ws[n:] = 0xA5
    return ws, n


def _fused(q, k, mem, T, ws, n, B=None, stats=None, dq=None):
    _l, lib = _lib()
    B = q.shape[0] if B is None else B
    d, K = q.shape[1], mem.shape[0]
    stats = torch.full((4,), math.nan, device="cuda") if stats is None else stats
    dq = torch.full((q.shape[0], d), math.nan, device="cuda") if dq is None else dq
    _l.check(lib.gccb_infonce_fused(_l.dptr(q), _l.dptr(k), _l.dptr(mem), B, d, K, T, _l.dptr(stats), _l.dptr(dq),
                                    _l.dptr(ws), n, _l.stream_ptr()), "gccb_infonce_fused")
    return stats, dq


# (B, K, d, T, regime, path): every (d, path) pair nce_use_tc produces, the recipe shapes, the short batches, both
# sides of the 32-row tile, the 128-row tensor-core tile, the key chunk and K % 64, split counts at their cap K / 64,
# at the SM count and uneven.
_CASES = [
    # d = 32 (SIMT only)
    (1, 1, 32, 0.07, "rand", "simt"), (31, 63, 32, 0.2, "flat", "simt"), (32, 64, 32, 0.07, "sat", "simt"),
    (33, 129, 32, 1.0, "dom", "simt"), (256, 16384, 32, 0.07, "half", "simt"), (1024, 65536, 32, 0.07, "rand", "simt"),
    (129, 127, 32, 0.2, "dup", "simt"),
    # d = 64 (SIMT only; the hidden-64 recipe)
    (256, 16384, 64, 0.07, "half", "simt"), (32, 65, 64, 0.07, "dup", "simt"), (127, 128, 64, 0.2, "flat", "simt"),
    (1, 16383, 64, 0.07, "sat", "simt"), (200, 127, 64, 1.0, "rand", "simt"), (1000, 64, 64, 0.07, "dom", "simt"),
    (33, 65536, 64, 0.07, "dom", "simt"),
    # d = 128
    (127, 16384, 128, 0.07, "rand", "simt"), (31, 1, 128, 0.07, "sat", "simt"), (1, 65, 128, 1.0, "dom", "simt"),
    (128, 65, 128, 0.2, "dom", "simt"), (1024, 16383, 128, 0.07, "half", "simt"), (32, 129, 128, 1.0, "flat", "simt"),
    (256, 16384, 128, 0.07, "half", "tc"), (128, 64, 128, 0.07, "rand", "tc"), (129, 128, 128, 0.2, "dom", "tc"),
    (200, 16384, 128, 1.0, "flat", "tc"), (1000, 65536, 128, 0.07, "dup", "tc"), (1024, 65536, 128, 0.07, "sat", "tc"),
    (128, 128, 128, 1.0, "rand", "tc"),
    # d = 256
    (127, 16384, 256, 0.07, "half", "simt"), (33, 65536, 256, 0.07, "dom", "simt"), (1, 129, 256, 0.2, "rand", "simt"),
    (256, 16383, 256, 0.07, "rand", "simt"), (1024, 63, 256, 0.07, "dup", "simt"), (129, 1, 256, 1.0, "sat", "simt"),
    (32, 64, 256, 0.2, "flat", "simt"), (31, 127, 256, 1.0, "dom", "simt"),
    (1024, 65536, 256, 0.07, "half", "tc"), (128, 16384, 256, 0.07, "rand", "tc"), (129, 65536, 256, 0.07, "dom", "tc"),
    (200, 128, 256, 0.2, "dup", "tc"), (256, 64, 256, 1.0, "flat", "tc"), (1000, 16384, 256, 0.07, "sat", "tc"),
    (1024, 65536, 256, 0.07, "dom", "tc"), (384, 16384, 256, 0.2, "rand", "tc"), (128, 16832, 256, 1.0, "rand", "tc"),
    (200, 640, 256, 0.07, "half", "tc"), (256, 16384, 256, 0.07, "rand", "tc"),
]


def test_case_list_covers_the_dispatch():
    """The coverage claims of _CASES: every (d, path) pair nce_use_tc can produce, the recipe shapes, short batches
    on both paths, K % 64 != 0 with B >= 128 at d >= 128, and tensor-core split counts capped at K / 64, at the SM
    count and uneven."""
    pairs = {(c[2], c[5]) for c in _CASES}
    assert pairs == {(32, "simt"), (64, "simt"), (128, "simt"), (128, "tc"), (256, "simt"), (256, "tc")}
    shapes = {c[:3] for c in _CASES}
    assert {(256, 16384, 64), (256, 16384, 128), (1024, 65536, 256)} <= shapes
    assert any(c[5] == "simt" and c[2] == 256 and c[0] < 128 for c in _CASES)
    assert any(c[5] == "simt" and c[2] >= 128 and c[0] >= 128 and c[1] % 64 for c in _CASES)
    assert any(c[5] == "tc" and c[0] % 128 for c in _CASES)
    lay = [cb.tc_layout(c[0], c[2], c[1]) for c in _CASES if c[5] == "tc"]
    assert any(L["alloc_splits"] == L["kb"] for L in lay)                       # capped at K / 64
    assert any(L["splits"] == cb.SMS for L in lay)                             # one split per SM
    assert any(L["kb"] % L["per"] for L in lay)                                # a short last split
    assert len(_CASES) <= 60
    for B, K, d, T, regime, path in _CASES:
        assert cb.nce_use_tc(B, d, K) == (path == "tc"), (B, K, d)
        if regime == "dom" and path == "simt":                                 # q lands in the last key chunk
            assert K - 1 >= (cb.cdiv(K, cb.nce_ck(d)) - 1) * cb.nce_ck(d)


def _tc_teacher_forced(case, q, k, mem, T, ws):
    """The tensor-core path's stored intermediates (nce_tc_layout): logits, P in bf16, p_pos, then dq from them."""
    B, d = q.shape
    K = mem.shape[0]
    L = cb.tc_layout(B, d, K)
    q16, m16 = q.to(torch.bfloat16).double(), mem.to(torch.bfloat16).double()
    logits = ws[L["logits"]:L["logits"] + B * K * 4].view(torch.float32).view(B, K)
    p16 = ws[L["p16"]:L["p16"] + B * K * 2].view(torch.bfloat16).view(B, K)
    ppos = ws[L["ppos"]:L["ppos"] + B * 4].view(torch.float32)
    want = q16 @ m16.t() / T
    _check(case, "tc.logits", logits, want, cb.chain_bound(q16, m16, cb.C_DOT * d + 2, T))
    q64, k64 = q.double(), k.double()
    lpos = (q64 * k64).sum(1) / T
    lb_pos = cb.tc_pos_depth(d) * cb.U * (q64 * k64).abs().sum(1) / T
    lg = torch.cat([lpos[:, None], logits.double()], 1)
    lb = torch.cat([lb_pos[:, None], torch.zeros_like(logits, dtype=torch.float64)], 1)
    c_row = torch.full((B, 1), float(cb.cdiv(K, 1024) + 2 + 5 + 9 + 4 + 2), dtype=torch.float64, device="cuda")
    sm = cb.softmax_rel(lg, lb, c_row)
    p, rel = sm["p"], sm["rel"]
    _check(case, "tc.p16", p16, p[:, 1:], ((1 + rel[:, 1:]) * (1 + cb.UB) - 1) * p[:, 1:] + 2.0 ** -133)
    _check(case, "tc.ppos", ppos, p[:, 0], rel[:, 0] * p[:, 0] + cb.TINY)
    P, pp = p16.double(), ppos.double()[:, None]
    dqw = ((pp - 1) * k64 + P @ m16) / (T * B)
    mag = ((1 - pp).abs() * k64.abs() + P @ m16.abs())
    return dqw, (cb.C_DOT * K + L["splits"] + 3) * cb.U * mag / (T * B) + 3 * cb.U * mag / (T * B)


@pytest.mark.parametrize("B,K,d,T,regime,path", _CASES, ids=["-".join(str(x) for x in c) for c in _CASES])
def test_fused_head_matches_float64(B, K, d, T, regime, path):
    """gccb_infonce_fused: loss, mean positive logit and dq against float64 within their bounds, the intermediates
    teacher-forced, NaN-filled outputs fully overwritten, nothing written past the workspace, bit-identical dq from
    run to run and with a dirty workspace."""
    case = "nce B=%d K=%d d=%d T=%g %s %s" % (B, K, d, T, regime, path)
    q, k, mem = _inputs(B, K, d, regime, B * 7 + K + d)
    ws, n = _workspace(B, d, K)
    stats, dq = _fused(q, k, mem, T, ws, n)
    torch.cuda.synchronize()
    assert torch.isnan(stats[2:]).all(), "stats written past its two entries"
    assert (ws[n:] == 0xA5).all(), "workspace written past gccb_infonce_workspace bytes"
    ex = (cb.tc_expected if path == "tc" else cb.simt_expected)(q, k, mem, T)
    loss, lossb = cb.mean_bound(ex["loss"], ex["lossb"])
    lpos, lposb = cb.mean_bound(ex["lpos"], ex["lposb"])
    _check(case, "loss", stats[0], loss, lossb)
    _check(case, "mean lpos", stats[1], lpos, lposb)
    _check(case, "dq " + path, dq, ex["dq"], ex["dqb"])
    del ex
    if path == "simt":
        nch = cb.cdiv(K, cb.nce_ck(d))
        rec = ws[:nch * B * (d + 2) * 4].view(torch.float32).view(nch, B, d + 2)
        for name, got, want, bound in cb.simt_records_check(q, mem, T, rec):
            _check(case, name, got, want, bound)
        mg = cb.simt_merge_expected(q, k, rec, T)
        _check(case, "merge.loss", stats[0], *cb.mean_bound(mg["loss"], mg["lossb"]))
        _check(case, "merge.dq", dq, mg["dq"], mg["dqb"])
    else:
        dqw, dqb = _tc_teacher_forced(case, q, k, mem, T, ws)
        _check(case, "tc.dq", dq, dqw, dqb)
    # the same bits again, and with a workspace full of garbage (NaN / huge floats)
    again = _fused(q, k, mem, T, ws, n)[1]
    ws2, _ = _workspace(B, d, K, fill=0xFF)
    dirty = _fused(q, k, mem, T, ws2, n)[1]
    ws3, _ = _workspace(B, d, K, fill=0x7F)
    dirty2 = _fused(q, k, mem, T, ws3, n)[1]
    torch.cuda.synchronize()
    assert torch.equal(again, dq) and torch.equal(dirty, dq) and torch.equal(dirty2, dq)
    assert (ws2[n:] == 0xA5).all() and (ws3[n:] == 0xA5).all()


# one case per (d, path) pair and a short batch on each: (B, K, d, b) with b the rows of the call
_STATE = [(64, 200, 32, 33), (256, 16384, 64, 200), (256, 16383, 128, 127), (1024, 65536, 128, 1000),
          (256, 16384, 256, 100), (1024, 65536, 256, 129)]


@pytest.mark.parametrize("B,K,d,b", _STATE, ids=["-".join(str(x) for x in c) for c in _STATE])
def test_fused_head_state_and_row_placement(B, K, d, b):
    """No state survives between calls: two back-to-back calls on one stream with different T into the same
    workspace each give the bits of an isolated call.  Permuting the batch rows permutes dq bit for bit.  A b-row call
    into a [B][d] dq (the engine's short last batch) leaves rows b..B untouched, writes nothing past
    gccb_infonce_workspace(b, d, K), and gives the bits of a call on compact copies of the b rows whatever rows
    b..B of q and k hold."""
    _l, lib = _lib()
    q, k, mem = _inputs(B, K, d, "half", B + d)
    ws, n = _workspace(B, d, K)
    iso = [_fused(q, k, mem, T, ws, n) for T in (0.07, 0.2)]
    torch.cuda.synchronize()
    pair = [_fused(q, k, mem, T, ws, n) for T in (0.07, 0.2)]               # back to back, no sync in between
    torch.cuda.synchronize()
    for (s0, d0), (s1, d1) in zip(iso, pair):
        assert torch.equal(d0, d1)
        assert torch.allclose(s0[:2], s1[:2], rtol=1e-5, atol=1e-6)           # the atomics' order may differ
    assert not torch.equal(iso[0][1], iso[1][1])
    g = torch.Generator(device="cuda").manual_seed(d)
    perm = torch.randperm(B, device="cuda", generator=g)
    dperm = _fused(q[perm].contiguous(), k[perm].contiguous(), mem, 0.07, ws, n)[1]
    torch.cuda.synchronize()
    assert torch.equal(dperm, iso[0][1][perm])
    # short batch: b rows in the engine's [B][d] buffers, rows b..B of q and k stale (NaN here); dq is the mean over
    # the b rows, so it matches a call on compact [b][d] copies bit for bit
    qB, kB = q.clone(), k.clone()
    qB[b:], kB[b:] = math.nan, math.nan
    wsb, nb = _workspace(b, d, K, fill=0xFF)
    dqB = torch.full((B, d), math.nan, device="cuda")
    stats = torch.full((4,), math.nan, device="cuda")
    _fused(qB, kB, mem, 0.07, wsb, nb, B=b, stats=stats, dq=dqB)
    compact = _fused(q[:b].contiguous(), k[:b].contiguous(), mem, 0.07, *_workspace(b, d, K))[1]
    torch.cuda.synchronize()
    assert torch.isnan(dqB[b:]).all() and torch.isfinite(dqB[:b]).all()
    assert (wsb[nb:] == 0xA5).all() and torch.isnan(stats[2:]).all()
    assert torch.equal(dqB[:b], compact)
    tc = cb.nce_use_tc(b, d, K)
    ex = (cb.tc_expected if tc else cb.simt_expected)(q[:b], k[:b], mem, 0.07)
    case = "short B=%d b=%d K=%d d=%d %s" % (B, b, K, d, "tc" if tc else "simt")
    _check(case, "dq " + ("tc" if tc else "simt"), dqB[:b], ex["dq"], ex["dqb"])
    _check(case, "loss", stats[0], *cb.mean_bound(ex["loss"], ex["lossb"]))


# ---- E2E head ----------------------------------------------------------------------------------------------------
_E2E = [(1, 32, "rand"), (2, 64, "rand"), (31, 128, "sat"), (255, 256, "rand"), (256, 32, "flat"), (257, 64, "rand"),
        (1024, 128, "rand"), (1024, 256, "flat"), (256, 256, "sat"), (12288, 256, "rand"), (12288, 32, "rand"),
        (31, 256, "flat")]


def _e2e_inputs(B, d, regime, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if regime == "sat":                                    # k_i = q_i = e_i: the diagonal logit 1 / T, the rest 0
        q = torch.eye(B, d, device="cuda")
        return q, q.clone()
    if regime == "flat":
        m = F.normalize(torch.randn(d, device="cuda", generator=g), dim=0)
        return m.expand(B, d).contiguous(), m.expand(B, d).contiguous()
    q = F.normalize(torch.randn(B, d, device="cuda", generator=g), dim=1)
    k = F.normalize(q + 0.5 * torch.randn(B, d, device="cuda", generator=g), dim=1)
    return q, k


@pytest.mark.parametrize("B,d,regime", _E2E, ids=["-".join(str(x) for x in c) for c in _E2E])
def test_e2e_head_matches_float64(B, d, regime):
    """gccb_e2e_nce: loss, mean diagonal logit, the stored dout, dq and dk against float64 (end to end, and the
    gradients teacher-forced from the stored dout); dq and dk bit-identical from run to run.  B = 12288 at d = 256
    takes (d + B) 4 = 50,176 bytes of dynamic shared memory, past the 48 KB default."""
    _l, lib = _lib()
    T = 0.07 if regime != "flat" else 0.2
    case = "e2e B=%d d=%d %s" % (B, d, regime)
    q, k = _e2e_inputs(B, d, regime, B + d)
    out = []
    for _ in range(2):
        stats = torch.full((4,), math.nan, device="cuda")
        dq = torch.full((B, d), math.nan, device="cuda")
        dk = torch.full((B, d), math.nan, device="cuda")
        ws = torch.full((B * B + CANARY // 4,), math.nan, device="cuda")
        _l.check(lib.gccb_e2e_nce(_l.dptr(q), _l.dptr(k), B, d, T, _l.dptr(stats), _l.dptr(dq), _l.dptr(dk),
                                  _l.dptr(ws), B * B * 4, _l.stream_ptr()), "gccb_e2e_nce")
        out.append((stats, dq, dk, ws))
    torch.cuda.synchronize()
    stats, dq, dk, ws = out[0]
    assert torch.equal(out[1][1], dq) and torch.equal(out[1][2], dk)
    assert torch.isnan(stats[2:]).all() and torch.isnan(ws[B * B:]).all()
    ex = cb.e2e_expected(q, k, T)
    _check(case, "e2e.loss", stats[0], *cb.mean_bound(ex["loss"], ex["lossb"]))
    _check(case, "e2e.ldiag", stats[1], *cb.mean_bound(ex["ldiag"], ex["ldiagb"]))
    dout = ws[:B * B].view(B, B)
    _check(case, "e2e.dout", dout, ex["dout"], ex["doutb"])
    _check(case, "e2e.dk", dk, ex["dk"], ex["dkb"])
    _check(case, "e2e.dq", dq, ex["dq"], ex["dqb"])
    del ex
    dkw, dkb, dqw, dqb = cb.e2e_grads_from_dout(q, k, dout, T)
    _check(case, "e2e.dk (dout)", dk, dkw, dkb)
    _check(case, "e2e.dq (dout)", dq, dqw, dqb)


# ---- module API --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 256, 100, 96])
def test_module_api_matches_float64(d):
    """gccb_moco_logits, gccb_nce_loss (labels 0 and i, C = K + 1 = 16385) and gccb_moco_logits_backward at the recipe
    size B = 256, K = 16384: each against float64 from its own stored inputs.  At d = 100 and 96, 256 % d != 0 and
    the backward's last threads have no group.  The loss is re-zeroed by every call."""
    _l, lib = _lib()
    B, K, T = 256, 16384, 0.07
    case = "api d=%d" % d
    q, k, mem = _inputs(B, K, d, "half", d)
    out = torch.full((B, K + 1), math.nan, device="cuda")
    _l.check(lib.gccb_moco_logits(_l.dptr(q), _l.dptr(k), _l.dptr(mem), B, d, K, T, _l.dptr(out), _l.stream_ptr()))
    torch.cuda.synchronize()
    want = cb.logits_exact(q, k, mem, T)
    lb = torch.cat([cb.chain_bound(q, k, d + 2, T).diagonal()[:, None], cb.chain_bound(q, mem, d + 2, T)], 1)
    _check(case, "api.logits", out, want, lb)
    C = K + 1
    for mode in (0, 1):
        loss = torch.full((2,), math.nan, device="cuda")
        dout = torch.full((B, C), math.nan, device="cuda")
        for call in range(2):                               # the second call must not add to the first
            _l.check(lib.gccb_nce_loss(_l.dptr(out), B, C, mode, _l.dptr(loss), _l.dptr(dout), _l.stream_ptr()))
            torch.cuda.synchronize()
            if call == 0:
                first = loss.clone()
        # the per-row atomics may add in another order: the two values agree within twice their rounding
        assert abs(float(loss[0]) - float(first[0])) <= 2 * (B + 1) * cb.U * abs(float(first[0]))
        assert torch.isnan(loss[1])
        lg = out.double()
        lab = torch.arange(B, device="cuda") if mode else torch.zeros(B, dtype=torch.long, device="cuda")
        # the labelled column first (softmax_rel is order-free); no logit error: the input is the stored logits
        order = (lab[:, None] + torch.arange(C, device="cuda")[None]) % C
        lo = lg.gather(1, order)
        c_row = torch.full((B, 1), float(cb.cdiv(C, 256) + 13 + 4 + 1), dtype=torch.float64, device="cuda")
        sm = cb.softmax_rel(lo, torch.zeros_like(lo), c_row)
        li, lossb = cb.loss_bound(sm, torch.zeros(B, dtype=torch.float64, device="cuda"), c_row)
        _check(case, "api.loss%d" % mode, loss[0], *cb.mean_bound(li, lossb))
        p = torch.exp(lg - sm["M"]) / sm["S"]
        rel = torch.expm1((c_row + sm["amax"] + (sm["M"] - lg)) * cb.U)
        onehot = F.one_hot(lab, C).double()
        _check(case, "api.dout%d" % mode, dout, (p - onehot) / B,
               (rel * p + cb.TINY + 3 * cb.U * (p - onehot).abs()) / B)
    # backward from the stored dout of label mode 0
    dq = torch.full((B, d), math.nan, device="cuda")
    _l.check(lib.gccb_nce_loss(_l.dptr(out), B, C, 0, _l.dptr(loss), _l.dptr(dout), _l.stream_ptr()))
    _l.check(lib.gccb_moco_logits_backward(_l.dptr(dout), _l.dptr(k), _l.dptr(mem), B, d, K, T, _l.dptr(dq),
                                           _l.stream_ptr()))
    torch.cuda.synchronize()
    d64, k64, m64 = dout.double(), k.double(), mem.double()
    groups = max(1, 256 // d)
    want = (d64[:, :1] * k64 + d64[:, 1:] @ m64) / T
    mag = (d64[:, :1].abs() * k64.abs() + d64[:, 1:].abs() @ m64.abs()) / T
    _check(case, "api.dq", dq, want, (cb.cdiv(K, groups) + groups + 3) * cb.U * mag)


# ---- enqueue -----------------------------------------------------------------------------------------------------
_ENQ = [(16384, 64, 256, 1, 5000, None), (65536, 256, 1024, 1, 65536 - 1024, None),
        (16384, 64, 256, 1, 16383, None),                          # one row before the wrap
        (16384, 64, 100, 1, 16300, None),                          # b does not divide K, wraps
        (16384, 64, 256, 2, 16000, 256 * 64 + 96), (65536, 256, 128, 8, 65000, 128 * 256 + 512),
        (16384, 64, 256, 8, 3, 256 * 64 * 2)]


@pytest.mark.parametrize("K,d,b,parts,index,stride", _ENQ, ids=["-".join(str(x) for x in c) for c in _ENQ])
@pytest.mark.parametrize("skip", [False, True], ids=["run", "skip"])
def test_enqueue_matches_fmod_restatement(K, d, b, parts, index, stride, skip):
    """gccb_moco_enqueue against torch: row (index + r b + i) mod K of the queue takes key i of part r (torch.fmod(
    arange(parts b) + index, K)), the rest of the queue is untouched, the index advances by parts b mod K.  With the
    skip word's bit set the queue and the index stay bit-identical."""
    _l, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(K + b + parts)
    mem = torch.randn(K, d, device="cuda", generator=g)
    stride = stride or b * d
    payload = torch.randn(parts * stride, device="cuda", generator=g)
    idx = torch.tensor([index], dtype=torch.int64, device="cuda")
    word = torch.tensor([0x6 if skip else 0x1], dtype=torch.int32, device="cuda")
    before = mem.clone()
    _l.check(lib.gccb_moco_enqueue(_l.dptr(mem), _l.dptr(payload), b, d, K, _l.dptr(idx), parts, stride,
                                   _l.dptr(word), 0x2, _l.stream_ptr()), "gccb_moco_enqueue")
    torch.cuda.synchronize()
    if skip:
        assert torch.equal(mem, before) and int(idx) == index
        return
    keys = payload.view(parts, stride)[:, :b * d].reshape(parts * b, d)
    rows = torch.fmod(torch.arange(parts * b, device="cuda") + index, K)
    want = before.clone()
    want[rows] = keys
    assert torch.equal(mem, want)
    assert int(idx) == (index + parts * b) % K
