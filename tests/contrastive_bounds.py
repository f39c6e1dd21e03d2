"""Float64 references of the contrastive head (csrc/moco.cu) and per-element bounds on the kernels' error,
shared by the H100 tests (test_gpu_contrastive_head.py, whose docstring derives every bound) and their host-side
self-check (test_contrastive_bounds_host.py).  Everything here is torch float64 and runs on any device.

Notation: l [B, 1 + K] exact logits of a row (column 0 the positive), lb [B, 1 + K] bounds on the error of the
kernel's fp32 logits, U = 2^-24.  A bound is a tensor the size of the output it bounds."""
import math

import torch

U = 2.0 ** -24
UB = 2.0 ** -8          # bf16 unit roundoff: 8 significant bits
C_DOT = 4.0             # tensor-core dot products, as in test_gpu_tc.py
TINY = 2.0 ** -125      # absolute slack per probability for exp results near or in the fp32 subnormal range
SMS = 132               # GCCB_NUM_SMS


def cdiv(a, b):
    return -(-a // b)


# ---- dispatch of gccb_infonce_fused, restated --------------------------------------------------------------------
def nce_use_tc(B, d, K):
    return d >= 128 and K % 64 == 0 and B >= 128


def nce_ck(d):
    """Keys per CTA of infonce_partial_tiled_kernel (infonce_ck)."""
    return 128 if d <= 128 else 64


def nce_kpt(d):
    return nce_ck(d) // 32


def tc_layout(B, d, K):
    """nce_tc_layout: byte offsets of the tensor-core workspace and the split count it sizes `splitk` for; `splits`
    is the count tc::gemm_bf16 then runs (no empty split) and `per` the k-blocks of each but the last."""
    off, L = 0, {}
    for name, nbytes in (("q16", B * d * 2), ("m16", K * d * 2), ("mt16", d * K * 2), ("logits", B * K * 4),
                         ("p16", B * K * 2), ("ppos", B * 4), ("dqn", B * d * 4)):
        L[name] = off
        off += (nbytes + 255) & ~255
    s = max(1, SMS // cdiv(B, 128))
    s = min(s, K // 64)
    L["splitk"], L["alloc_splits"] = off, s
    kb = K // 64
    per = cdiv(kb, s)
    L["splits"], L["per"], L["kb"] = cdiv(kb, per), per, kb
    return L


# ---- softmax with perturbed logits -------------------------------------------------------------------------------
def softmax_rel(l, lb, c_row):
    """p = softmax(l) per row and a bound on |p_kernel / p - 1| for every element, when each logit carries an error
    of at most lb and the fp32 evaluation of exp(l - max) / S costs c_row U (exps, divisions, the normaliser's
    summation) plus the rounding of each exp's argument, |l - max| U.  With perturbed logits l + e, |e| <= lb,
    p' / p = exp(e_j) / sum_k p_k exp(e_k), so |log(p' / p)| <= lb_j + log(sum_k p_k exp(lb_k)) = lb_j + Lr."""
    M = l.max(1, keepdim=True).values
    e = torch.exp(l - M)
    S = e.sum(1, keepdim=True)
    p = e / S
    Lr = torch.log((p * torch.exp(lb)).sum(1, keepdim=True))
    a = (M - l) + 2 * lb.max(1, keepdim=True).values
    amax = a.max(1, keepdim=True).values
    rel = torch.expm1(lb + Lr + (c_row + amax + a) * U)
    return dict(p=p, rel=rel, Lr=Lr, M=M, S=S, amax=amax)


def loss_bound(sm, lb_pos, c_row):
    """-log p_pos as logf(S) + M - l_pos: the perturbation lb_pos + Lr, the normaliser's rounding, logf (1 ulp)
    and the two additions."""
    M, S = sm["M"][:, 0], sm["S"][:, 0]
    loss = -torch.log(sm["p"][:, 0])
    logS = torch.log(S)
    return loss, (lb_pos + sm["Lr"][:, 0] + (c_row[:, 0] + sm["amax"][:, 0]) * U + 3 * U * logS.abs()
                  + U * (M.abs() + loss.abs()) + 2 * U * loss.abs())


def mean_bound(x, xb):
    """Mean of B per-row values added as x_i / B with float atomics in any order: (B - 1) U sum |x_i / B|, plus the
    division of each term."""
    B = x.numel()
    return x.mean(), xb.mean() + (B + 1) * U * x.abs().mean()


def dq_bound(sm, kpos, keys, T, chain, pos_chain, p_round=0.0):
    """dq = ((p_pos - 1) k + sum_j p_j key_j) / (T B) and its bound: each probability's relative error (times the
    bf16 rounding p_round of P before the dq product), `chain` U of the accumulated magnitudes for the key sum,
    `pos_chain` U for the positive term (p_pos - 1 and the roundings it goes through), 3 U for the final scale."""
    p, rel = sm["p"], sm["rel"]
    B = p.shape[0]
    ppos, pn = p[:, :1], p[:, 1:]
    rn = (1 + rel[:, 1:]) * (1 + p_round) - 1
    ak, am = kpos.abs(), keys.abs()
    want = ((ppos - 1) * kpos + pn @ keys) / (T * B)
    mag_n = (pn * (1 + rn)) @ am + TINY * am.sum(0, keepdim=True)
    mag_p = ((1 - ppos).abs() + rel[:, :1] * ppos) * ak
    err = (rel[:, :1] * ppos + TINY) * ak + (pn * rn) @ am + TINY * am.sum(0, keepdim=True)
    err = err + chain * U * mag_n + pos_chain * U * mag_p + 3 * U * (mag_n + mag_p)
    return want, err / (T * B)


# ---- logits ------------------------------------------------------------------------------------------------------
def logits_exact(q, k, mem, T):
    q, k, mem = q.double(), k.double(), mem.double()
    return torch.cat([(q * k).sum(1, keepdim=True), q @ mem.t()], 1) / T


def chain_bound(a, b, depth, T):
    """|a| . |b|^T / T times depth U: a dot product whose every term passes through at most `depth` roundings
    (additions, the multiply by the fp32 1 / T and that reciprocal's own rounding)."""
    return depth * U * (a.double().abs() @ b.double().abs().t()) / T


def simt_pos_depth(d):
    """infonce_merge_kernel: ceil(d / 128) fmaf per thread, 5 shuffle levels, 3 sequential adds of the 4 warps,
    times 1 / T and its rounding."""
    return cdiv(d, 128) + 5 + 3 + 2


def tc_pos_depth(d):
    """nce_tc_softmax_kernel: ceil(d / 256) fmaf per thread, 5 shuffle levels, 8 sequential adds, times 1 / T."""
    return cdiv(d, 256) + 5 + 8 + 2


def simt_expected(q, k, mem, T):
    """The fused head on the SIMT path: logits, loss, mean positive logit and dq with their bounds."""
    B, d = q.shape
    K = mem.shape[0]
    nch, kpt = cdiv(K, nce_ck(d)), nce_kpt(d)
    l = logits_exact(q, k, mem, T)
    q64, k64 = q.double(), k.double()
    lb_pos = simt_pos_depth(d) * U * (q64 * k64).abs().sum(1) / T
    lb = torch.cat([lb_pos[:, None], chain_bound(q, mem, d + 2, T)], 1)
    # normaliser: kpt terms per lane, 5 shuffle levels, then lpos and nch rescaled chunk sums in sequence; two exps
    # (4 U each) and the rescale product per term; the division by S
    c_row = torch.full((B, 1), float(kpt + 5 + nch + 2 + 8 + 1 + 1), dtype=torch.float64, device=l.device)
    sm = softmax_rel(l, lb, c_row)
    loss, lossb = loss_bound(sm, lb_pos, c_row)
    lpos = l[:, 0]
    lposb = lb_pos
    dq, dqb = dq_bound(sm, k64, mem.double(), T, chain=nce_ck(d) + nch + 2, pos_chain=nch + 3)
    return dict(l=l, lb=lb, sm=sm, loss=loss, lossb=lossb, lpos=lpos, lposb=lposb, dq=dq, dqb=dqb)


def tc_expected(q, k, mem, T):
    """The fused head on the tensor-core path: the negatives' logits from the bf16-rounded q and queue, the positive
    in fp32, P rounded to bf16 before the dq product."""
    B, d = q.shape
    K = mem.shape[0]
    q16, m16 = q.to(torch.bfloat16).double(), mem.to(torch.bfloat16).double()
    q64, k64 = q.double(), k.double()
    l = torch.cat([(q64 * k64).sum(1, keepdim=True), q16 @ m16.t()], 1) / T
    lb_pos = tc_pos_depth(d) * U * (q64 * k64).abs().sum(1) / T
    lb = torch.cat([lb_pos[:, None], chain_bound(q16, m16, C_DOT * d + 2, T)], 1)
    # normaliser: ceil(K / 1024) float4 groups per thread (a 2-level pair sum each), 5 shuffle levels, exp(lpos) and
    # 8 warp sums in sequence; one exp (4 U), the multiply by 1 / S and that reciprocal
    c_row = torch.full((B, 1), float(cdiv(K, 1024) + 2 + 5 + 9 + 4 + 2), dtype=torch.float64, device=l.device)
    sm = softmax_rel(l, lb, c_row)
    loss, lossb = loss_bound(sm, lb_pos, c_row)
    L = tc_layout(B, d, K)
    # dq GEMM over K keys in fp32 on the tensor cores, the split-K partials added in sequence, the finishing fmaf
    dq, dqb = dq_bound(sm, k64, m16, T, chain=C_DOT * K + L["splits"] + 2, pos_chain=3, p_round=UB)
    return dict(l=l, lb=lb, sm=sm, loss=loss, lossb=lossb, lpos=l[:, 0], lposb=lb_pos, dq=dq, dqb=dqb,
                q16=q16, m16=m16)


# ---- SIMT partial records, teacher-forced ------------------------------------------------------------------------
def simt_records_check(q, mem, T, rec):
    """rec [nch, B, d + 2] as infonce_partial_tiled_kernel stores it: {m, s, acc[d]} of each (chunk, row).  Each
    record is compared with float64 computed with the stored m as the shift (the record is exact relative to its
    own m): m against the chunk's exact maximum, s and acc against sum_j exp(l_j - m) (m_j).  Returns
    [(name, got, want, bound)]."""
    B, d = q.shape
    K = mem.shape[0]
    ck, kpt = nce_ck(d), nce_kpt(d)
    nch = cdiv(K, ck)
    q64, m64 = q.double(), mem.double()
    l = (q64 @ m64.t()) / T
    lb = chain_bound(q, mem, d + 2, T)
    pad = nch * ck - K
    lpad = torch.nn.functional.pad(l, (0, pad), value=-math.inf).view(B, nch, ck).transpose(0, 1)   # [nch, B, ck]
    lbp = torch.nn.functional.pad(lb, (0, pad)).view(B, nch, ck).transpose(0, 1)
    mp = torch.nn.functional.pad(m64, (0, 0, 0, pad)).view(nch, ck, d)
    rm, rs, racc = rec[:, :, 0].double(), rec[:, :, 1].double(), rec[:, :, 2:].double()
    out = []
    out.append(("rec.m", rm, lpad.max(2).values, lbp.max(2).values + U * lpad.max(2).values.abs()))
    valid = torch.isfinite(lpad)
    a = torch.where(valid, rm[..., None] - lpad, torch.zeros_like(lpad)).abs()
    e = torch.where(valid, torch.exp(lpad - rm[..., None]), torch.zeros_like(lpad))
    # one exp (4 U) and its argument; s: kpt terms per lane and 5 shuffle levels; acc: a chain of up to ck fmaf
    rel_s = torch.expm1(lbp + (4 + a + kpt + 5) * U)
    out.append(("rec.s", rs, e.sum(2), (e * rel_s).sum(2) + TINY * ck))
    rel_a = torch.expm1(lbp + (4 + a) * U)
    am = mp.abs()
    accb = torch.bmm(e * rel_a, am) + ck * U * torch.bmm(e * (1 + rel_a), am) + TINY * am.sum(1, keepdim=True)
    out.append(("rec.acc", racc, torch.bmm(e, mp), accb))
    return out


def simt_merge_expected(q, k, rec, T):
    """infonce_merge_kernel from the stored records: the loss and dq of each row in float64 with the positive logit
    exact, and their bounds (the positive logit's error, the merge's exps, products and sums)."""
    B, d = q.shape
    nch = rec.shape[0]
    q64, k64 = q.double(), k.double()
    lpos = (q64 * k64).sum(1) / T
    lb_pos = simt_pos_depth(d) * U * (q64 * k64).abs().sum(1) / T
    rm, rs, racc = rec[:, :, 0].double().t(), rec[:, :, 1].double().t(), rec[:, :, 2:].double().transpose(0, 1)
    M = torch.maximum(lpos, rm.max(1).values)
    w = rs * torch.exp(rm - M[:, None])                    # [B, nch] each chunk's mass at the row's shift
    epos = torch.exp(lpos - M)
    S = epos + w.sum(1)
    ppos = epos / S
    Lr = torch.log(1 - ppos + ppos * torch.exp(lb_pos))
    a = (M[:, None] - rm).abs()
    amax = torch.maximum(a.max(1).values, (M - lpos).abs())
    cS = (nch + 1) + 4 + 1 + amax                          # sum of nch + 1 terms, exp, product, argument
    loss = torch.log(S) + M - lpos
    lossb = lb_pos + Lr + cS * U + 3 * U * torch.log(S).abs() + U * (M.abs() + 3 * loss.abs())
    rel_pos = torch.expm1(lb_pos + Lr + (cS + 4 + 1 + amax) * U)
    rel_w = torch.expm1(Lr[:, None] + (cS[:, None] + 4 + 1 + a) * U)
    wc = torch.exp(rm - M[:, None]) / S[:, None]           # merge weight of each chunk
    want = ((ppos - 1)[:, None] * k64 + torch.einsum("bc,bcd->bd", wc, racc)) / (T * B)
    mag_n = torch.einsum("bc,bcd->bd", wc * (1 + rel_w), racc.abs())
    mag_p = ((1 - ppos).abs() + rel_pos * ppos)[:, None] * k64.abs()
    err = (rel_pos * ppos)[:, None] * k64.abs() + torch.einsum("bc,bcd->bd", wc * rel_w, racc.abs())
    err = err + (nch + 3) * U * (mag_n + mag_p) + 3 * U * (mag_n + mag_p) + TINY * (nch + 1)
    return dict(loss=loss, lossb=lossb, lpos=lpos, lposb=lb_pos, dq=want, dqb=err / (T * B))


# ---- E2E head ----------------------------------------------------------------------------------------------------
def e2e_expected(q, k, T):
    """gccb_e2e_nce: logits l_ij = k_i . q_j / T with label i, loss, mean diagonal logit, dout = (p - I) / B as
    e2e_rows_kernel stores it, dk = dout q / T and dq = dout^T k / T, with their bounds."""
    B, d = q.shape
    q64, k64 = q.double(), k.double()
    l = (k64 @ q64.t()) / T
    lb = chain_bound(k, q, d + 2, T)
    # l as [B, 1 + (B - 1)] with the label first: softmax_rel is order-free, so permute column i to the front
    idx = torch.arange(B, device=l.device)
    order = torch.cat([idx[:, None], (idx[:, None] + 1 + torch.arange(B - 1, device=l.device)[None]) % B], 1)
    lo, lbo = l.gather(1, order), lb.gather(1, order)
    # normaliser: ceil(B / 256) exps per thread, 5 shuffle levels, 8 sequential adds; an exp and a division
    c_row = torch.full((B, 1), float(cdiv(B, 256) + 5 + 8 + 4 + 1), dtype=torch.float64, device=l.device)
    sm = softmax_rel(lo, lbo, c_row)
    loss, lossb = loss_bound(sm, lbo[:, 0], c_row)
    inv = torch.empty_like(order)
    inv.scatter_(1, order, torch.arange(B, device=l.device)[None].expand(B, B))
    p, rel = sm["p"].gather(1, inv), sm["rel"].gather(1, inv)
    eye = torch.eye(B, dtype=torch.float64, device=l.device)
    dout = (p - eye) / B
    # p - [j == i], times the fp32 1 / B (and its rounding)
    doutb = (rel * p + TINY + 3 * U * ((p - eye).abs() + rel * p)) / B
    dmag = (p - eye).abs() / B + doutb
    dk = dout @ q64 / T
    dkb = (doutb @ q64.abs() + (B + 2) * U * (dmag @ q64.abs())) / T
    dq = dout.t() @ k64 / T
    dqb = (doutb.t() @ k64.abs() + (B + 2) * U * (dmag.t() @ k64.abs())) / T
    return dict(loss=loss, lossb=lossb, ldiag=l.diagonal(), ldiagb=lb.diagonal(), dout=dout, doutb=doutb,
                dk=dk, dkb=dkb, dq=dq, dqb=dqb)


def e2e_grads_from_dout(q, k, dout, T):
    """e2e_grads_kernel teacher-forced on the stored dout: chains of B fmaf, times the fp32 1 / T."""
    B = q.shape[0]
    d64, q64, k64 = dout.double(), q.double(), k.double()
    return (d64 @ q64 / T, (B + 2) * U * (d64.abs() @ q64.abs()) / T,
            d64.t() @ k64 / T, (B + 2) * U * (d64.abs().t() @ k64.abs()) / T)
