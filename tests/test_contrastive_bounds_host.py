"""Host check of the contrastive head's error bounds (contrastive_bounds.py, derived in test_gpu_contrastive_head.py)
without an H100: an fp32 numpy restatement of the SIMT InfoNCE kernels' summation order (infonce_partial_tiled_kernel
and infonce_merge_kernel) stays within every bound, and perturbations the size of real bugs break them.  The same
shapes also run through the kernels themselves under the CPU emulator."""
import numpy as np
import pytest
import torch

import contrastive_bounds as cb
from emu_util import lib, ptr

f32 = np.float32


def _fma(a, b, c):
    # fp32 fma through float64: the product is exact there, the sum rounds twice (at most one fp32 ulp apart from
    # a true fma, in half-way cases only)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _warp_sum(v):
    """warp_sum over the last axis (32 lanes): xor butterfly, lane 0's value."""
    v = v.copy()
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(f32)
    return v[..., 0]


def simt_restated(q, k, mem, T, mutation=None):
    """The SIMT fused head in fp32, in the kernels' order.  Returns stats[2], dq, and the records [nch, B, d + 2].
    mutation: "last_chunk" (the merge skips the last chunk), "pos_term" (dq without (p_pos - 1) k), "mask_le" (a
    zero-padded key enters every ragged chunk), "split_shift" (every chunk after the first starts one key late)."""
    B, d = q.shape
    K = mem.shape[0]
    ck, kpt = cb.nce_ck(d), cb.nce_kpt(d)
    nch = cb.cdiv(K, ck)
    invT = f32(1.0 / T)
    rec = np.zeros((nch, B, d + 2), f32)
    for ch in range(nch):
        j0 = ch * ck + (1 if mutation == "split_shift" and ch > 0 else 0)
        nk = min(ck, K - j0)
        keys = np.zeros((ck, d), f32)
        keys[:nk] = mem[j0:j0 + nk]
        lg = np.zeros((B, ck), f32)
        for c in range(d):
            lg = _fma(q[:, c:c + 1], keys[None, :, c], lg)
        valid = np.arange(ck) < (nk + 1 if mutation == "mask_le" and nk < ck else nk)
        lg = np.where(valid, (lg * invT).astype(f32), f32(-3.0e38))
        mx = lg.max(1)
        p = np.where(valid, np.exp((lg - mx[:, None]).astype(f32)), f32(0))
        lane = p.reshape(B, kpt, 32)                       # lane owns keys lane + 32 t
        s = np.zeros((B, 32), f32)
        for t in range(kpt):
            s = (s + lane[:, t]).astype(f32)
        acc = np.zeros((B, d), f32)
        for j in range(ck):
            if valid[j]:
                acc = _fma(p[:, j:j + 1], keys[None, j], acc)
        rec[ch, :, 0], rec[ch, :, 1], rec[ch, :, 2:] = mx, _warp_sum(s), acc
    # merge: 128 threads over d, 4 warp partials added in order
    part = np.zeros((B, 128), f32)
    for c in range(d):
        part[:, c % 128] = _fma(q[:, c], k[:, c], part[:, c % 128])
    w = _warp_sum(part.reshape(B, 4, 32))
    lpos = ((((w[:, 0] + w[:, 1]).astype(f32) + w[:, 2]).astype(f32) + w[:, 3]).astype(f32) * invT).astype(f32)
    used = nch - 1 if mutation == "last_chunk" else nch
    M = lpos.copy()
    for ch in range(used):
        M = np.maximum(M, rec[ch, :, 0])
    S = np.exp((lpos - M).astype(f32))
    for ch in range(used):
        S = (S + (rec[ch, :, 1] * np.exp((rec[ch, :, 0] - M).astype(f32))).astype(f32)).astype(f32)
    stats = np.zeros(2, f32)
    for i in range(B):
        stats[0] = stats[0] + f32((np.log(S[i]) + M[i]).astype(f32) - lpos[i]) / f32(B)
        stats[1] = stats[1] + lpos[i] / f32(B)
    pp = (np.exp((lpos - M).astype(f32)) / S).astype(f32)
    a = ((pp - f32(1))[:, None] * k).astype(f32) if mutation != "pos_term" else np.zeros_like(k)
    for ch in range(used):
        wch = (np.exp((rec[ch, :, 0] - M).astype(f32)) / S).astype(f32)
        a = _fma(wch[:, None], rec[ch, :, 2:], a)
    dq = (a * f32(invT / f32(B))).astype(f32)
    return stats, dq, rec


def _inputs(B, K, d, regime, seed):
    rng = np.random.default_rng(seed)

    def unit(*s):
        x = rng.normal(size=s)
        return (x / np.linalg.norm(x, axis=-1, keepdims=True)).astype(f32)

    q = unit(B, d)
    k = unit(B, d) * f32(0.3) + q
    k = (k / np.linalg.norm(k, axis=1, keepdims=True)).astype(f32)
    mem = unit(K, d)
    if regime == "dom":                                    # q itself among the last keys: one negative dominates
        n = min(B, K - (cb.cdiv(K, cb.nce_ck(d)) - 1) * cb.nce_ck(d))
        mem[K - n:] = q[:n]
    return q, k, mem


def _worst(q, k, mem, T, stats, dq, rec):
    """Largest error / bound over every check of the fused SIMT head (end to end, records, merge)."""
    tq, tk, tm = (torch.from_numpy(a) for a in (q, k, mem))
    ex = cb.simt_expected(tq, tk, tm, T)
    out = {}
    loss, lossb = cb.mean_bound(ex["loss"], ex["lossb"])
    lpos, lposb = cb.mean_bound(ex["lpos"], ex["lposb"])
    checks = [("loss", stats[0], loss, lossb), ("lpos", stats[1], lpos, lposb), ("dq", dq, ex["dq"], ex["dqb"])]
    trec = torch.from_numpy(rec)
    checks += cb.simt_records_check(tq, tm, T, trec)
    mg = cb.simt_merge_expected(tq, tk, trec, T)
    checks += [("merge.dq", dq, mg["dq"], mg["dqb"])]
    for name, got, want, bound in checks:
        err = (torch.as_tensor(np.asarray(got, np.float64)) - want).abs()
        out[name] = float((err / bound).max())
    return out


_SHAPES = [(5, 1, 32, 0.07, "rand"), (33, 129, 32, 1.0, "dom"), (7, 200, 64, 0.2, "rand"), (4, 257, 128, 0.07, "dom"),
           (3, 130, 256, 1.0, "rand")]


@pytest.mark.parametrize("B,K,d,T,regime", _SHAPES)
def test_restated_simt_head_stays_within_bounds(B, K, d, T, regime):
    q, k, mem = _inputs(B, K, d, regime, B + K + d)
    stats, dq, rec = simt_restated(q, k, mem, T)
    worst = _worst(q, k, mem, T, stats, dq, rec)
    print("restated B=%d K=%d d=%d T=%g %s: %s" % (B, K, d, T, regime,
                                                     " ".join("%s %.3f" % kv for kv in worst.items())))
    assert max(worst.values()) <= 1.0, worst


# (mutation, shape, a check it must break): each shape is one where the mutation is visible
_MUTANTS = [("last_chunk", (33, 129, 32, 1.0, "dom"), "dq"),
            ("last_chunk", (4, 257, 128, 0.07, "dom"), "loss"),
            ("pos_term", (7, 200, 64, 0.2, "rand"), "dq"),
            ("mask_le", (33, 129, 32, 1.0, "dom"), "rec.s"),
            ("mask_le", (3, 130, 256, 1.0, "rand"), "loss"),
            ("split_shift", (7, 200, 64, 0.2, "rand"), "rec.acc")]


@pytest.mark.parametrize("mutation,shape,check", _MUTANTS, ids=["%s-%s" % (m[0], m[2]) for m in _MUTANTS])
def test_bug_sized_perturbations_break_the_bounds(mutation, shape, check):
    B, K, d, T, regime = shape
    q, k, mem = _inputs(B, K, d, regime, B + K + d)
    stats, dq, rec = simt_restated(q, k, mem, T, mutation=mutation)
    worst = _worst(q, k, mem, T, stats, dq, rec)
    print("%s: %s" % (mutation, " ".join("%s %.3g" % kv for kv in worst.items())))
    assert worst[check] > 1.0, worst


@pytest.mark.parametrize("B,K,d,T,regime", _SHAPES)
def test_emulated_simt_head_stays_within_bounds(B, K, d, T, regime):
    """gccb_infonce_fused itself (the SIMT path: the emulator has no tensor cores) under the same bounds, with the
    records read back from the workspace at (chunk, row) * (d + 2)."""
    Lb = lib()
    q, k, mem = _inputs(B, K, d, regime, B + K + d)
    nch = cb.cdiv(K, cb.nce_ck(d))
    stats = np.full(2, np.nan, f32)
    dq = np.full((B, d), np.nan, f32)
    nbytes = Lb.gccb_infonce_workspace(B, d, K)
    assert nbytes == nch * B * (d + 2) * 4
    ws = np.full(nbytes // 4, np.nan, f32)
    rc = Lb.gccb_infonce_fused(ptr(q), ptr(k), ptr(mem), B, d, K, T, ptr(stats), ptr(dq), ptr(ws), nbytes, None)
    assert rc == 0, Lb.gccb_last_error()
    worst = _worst(q, k, mem, T, stats, dq, ws.reshape(nch, B, d + 2))
    print("emulated B=%d K=%d d=%d T=%g %s: %s" % (B, K, d, T, regime,
                                                     " ".join("%s %.3f" % kv for kv in worst.items())))
    assert max(worst.values()) <= 1.0, worst


def test_e2e_bounds_hold_for_a_restated_row_pass():
    """The E2E bounds against an fp32 restatement of e2e_rows_kernel / e2e_grads_kernel (one thread's strided
    terms, a warp butterfly, 8 warp sums; chains of B fmaf), and a dropped diagonal term breaks them."""
    B, d, T = 40, 32, 0.2
    q, k, _ = _inputs(B, 1, d, "rand", 11)
    invT, invB = f32(1.0 / T), f32(1.0 / B)
    lg = np.zeros((B, B), f32)
    for c in range(d):
        lg = _fma(k[:, None, c], q[None, :, c], lg)
    lg = (lg * invT).astype(f32)
    mx = lg.max(1)
    e = np.exp((lg - mx[:, None]).astype(f32))
    thr = np.zeros((B, 256), f32)
    thr[:, :B] = e                                         # B <= 256: one term per thread
    w = _warp_sum(thr.reshape(B, 8, 32))
    S = np.zeros(B, f32)
    for i in range(8):
        S = (S + w[:, i]).astype(f32)
    eye = np.eye(B, dtype=f32)
    dout = (((e / S[:, None]).astype(f32) - eye).astype(f32) * invB).astype(f32)
    ex = cb.e2e_expected(torch.from_numpy(q), torch.from_numpy(k), T)
    for bad in (False, True):
        dd = dout.copy()
        if bad:
            dd[np.arange(B), np.arange(B)] += invB          # the -1 of the label left out
        dk = np.zeros((B, d), f32)
        for j in range(B):
            dk = _fma(dd[:, j:j + 1], q[None, j], dk)
        dk = (dk * invT).astype(f32)
        r_dout = float(((torch.from_numpy(dd).double() - ex["dout"]).abs() / ex["doutb"]).max())
        r_dk = float(((torch.from_numpy(dk).double() - ex["dk"]).abs() / ex["dkb"]).max())
        print("e2e restated%s: dout %.3g dk %.3g" % (" (no -1)" if bad else "", r_dout, r_dk))
        assert (r_dout > 1 and r_dk > 1) if bad else (r_dout <= 1 and r_dk <= 1)
