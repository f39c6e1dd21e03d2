"""CPU: the finetune kernels of csrc/finetune.cu under the fiber emulator -- the classification head against float64,
the clip-by-value optimiser steps against clip_grad_value_ + torch.optim, and the whole-graph feature gather against
indexing the cache directly.  Kernel LOGIC only; tests/test_gpu_finetune_engine.py runs them on an H100.

Head bounds (u = 2^-24, fp32 unit roundoff).  A logit is a fixed-order fma chain over H products plus the bias, so
|dlogit| <= (H + 1) u S with S = sum_h |x_h W_ch| + |bias_c|.  The loss of a row is lse - logit_y; exp and log add a
few ulps, so |dloss_row| <= 2 max_c |dlogit_c| + 8 u (|lse| + |logit_y|), and the mean keeps that bound.  A softmax
entry p_c moves by at most p_c (2 max |dlogit| + 8 u), so |d dlogits| <= (p_c (2 max |dlogit| + 8 u) + u) / b.
dfeat, dW and db are fixed-order sums of C, b and b such terms: each gets (K + 1) u sum |terms| for the sum itself
plus sum |W| (or |feat|) |d dlogits| from its inputs.  The tests use these bounds times 2."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from emu_util import NpBatch, lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets.graph_dataset import seed_first_union
from gcc_b200.datasets.labeled import _listed_csr, _simple_csr

U = 2.0 ** -24


# ---------------------------------------------------------------------------------------------- head
def _head_inputs(B, H, C, n_items, seed):
    rng = np.random.default_rng(seed)
    feat = rng.normal(size=(B, H)).astype(np.float32)
    W = (rng.normal(size=(C, H)) / np.sqrt(H)).astype(np.float32)
    bias = (rng.normal(size=C) * 0.1).astype(np.float32)
    labels = rng.integers(0, C, n_items).astype(np.int64)
    ids = rng.permutation(n_items)[:B].astype(np.int64)
    return feat, W, bias, labels, ids


def _run_head(feat, W, bias, ids, labels, b, eval_=False):
    B, H = feat.shape
    C = W.shape[0]
    L = lib()
    ws = np.zeros(L.gccb_ft_head_workspace(B, C) // 4 + 1, np.float32)
    dfeat = np.full((B, H), -7.0, np.float32)
    dW = np.full((C, H), -7.0, np.float32)
    db = np.full(C, -7.0, np.float32)
    stats = np.zeros(3, np.float32)
    rc = L.gccb_ft_head(ptr(feat), B, b, H, C, ptr(W), ptr(bias), ptr(ids), ptr(labels), len(labels),
                        1 if eval_ else 0, ptr(dfeat), ptr(dW), ptr(db), ptr(stats), ptr(ws), ws.nbytes, None)
    return rc, stats, dfeat, dW, db


def _head_ref(feat, W, bias, ids, labels, b, mutant=None):
    """float64 forward, loss, first-max correct count and gradients of rows 0..b-1.  mutant: 'wt' reads W as if it
    were stored [H][C], 'nob' drops the 1/b, 'last' counts the LAST maximum."""
    x, Wd, bd = feat[:b].astype(np.float64), W.astype(np.float64), bias.astype(np.float64)
    C, H = W.shape
    if mutant == "wt":
        Wd = W.reshape(-1).astype(np.float64).reshape(H, C).T
    y = labels[ids[:b]]
    z = x @ Wd.T + bd
    m = z.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(z - m).sum(1))
    loss = float(np.mean(lse - z[np.arange(b), y]))
    if mutant == "last":
        pred = C - 1 - np.argmax(z[:, ::-1], axis=1)
    else:
        pred = np.argmax(z, axis=1)
    correct = int((pred == y).sum())
    p = np.exp(z - lse[:, None])
    d = p.copy()
    d[np.arange(b), y] -= 1.0
    d = d if mutant == "nob" else d / b
    S = np.abs(x) @ np.abs(Wd).T + np.abs(bd)
    return dict(loss=loss, correct=correct, dfeat=d @ Wd, dW=d.T @ x, db=d.sum(0), z=z, p=p, d=d, S=S, lse=lse, y=y)


def _head_close(got, r, b, H, C, W, feat):
    """True when every output is inside the docstring's bounds (times 2)."""
    rc, stats, dfeat, dW, db = got
    dz = (H + 1) * U * r["S"]                                        # [b][C]
    dz_row = dz.max(1)
    loss_tol = np.mean(2 * dz_row + 8 * U * (np.abs(r["lse"]) + np.abs(r["z"][np.arange(b), r["y"]])))
    dd = (r["p"] * (2 * dz_row[:, None] + 8 * U) + U) / b           # bound on each dlogit
    Wa, xa = np.abs(W.astype(np.float64)), np.abs(feat[:b].astype(np.float64))
    dfeat_tol = (C + 1) * U * (np.abs(r["d"]) @ Wa) + dd @ Wa
    dW_tol = (b + 1) * U * (np.abs(r["d"]).T @ xa) + dd.T @ xa
    db_tol = (b + 1) * U * np.abs(r["d"]).sum(0) + dd.sum(0)
    return (abs(stats[0] - r["loss"]) <= 2 * loss_tol and int(stats[1]) == r["correct"] and int(stats[2]) == b
            and np.all(np.abs(dfeat[:b] - r["dfeat"]) <= 2 * dfeat_tol)
            and np.all(np.abs(dW - r["dW"]) <= 2 * dW_tol) and np.all(np.abs(db - r["db"]) <= 2 * db_tol))


HEAD_CASES = [(C, H, short) for C in (2, 5, 128) for H in (32, 64, 256) for short in (False, True)]


@pytest.mark.parametrize("C,H,short", HEAD_CASES, ids=["C%d-H%d-%s" % (c, h, "short" if s else "full")
                                                      for c, h, s in HEAD_CASES])
def test_head_matches_float64(C, H, short):
    B = 12
    b = 7 if short else B
    feat, W, bias, labels, ids = _head_inputs(B, H, C, 40, zlib.crc32(repr((C, H, short)).encode()))
    got = _run_head(feat, W, bias, ids, labels, b)
    assert got[0] == 0
    r = _head_ref(feat, W, bias, ids, labels, b)
    assert _head_close(got, r, b, H, C, W, feat)
    assert (got[1][:b] >= 0).all() and np.all(got[2][b:] == -7.0)  # rows beyond b are not written
    again = _run_head(feat, W, bias, ids, labels, b)
    for a, c in zip(got[1:], again[1:]):                            # bit-identical from run to run
        assert a.tobytes() == c.tobytes()
    ev = _run_head(feat, W, bias, ids, labels, b, eval_=True)      # forward only: same statistics, no gradients
    assert ev[0] == 0 and ev[1].tobytes() == got[1].tobytes() and np.all(ev[3] == -7.0)


def test_head_mutants_fail_a_case():
    """A kernel reading W transposed, dropping the 1/b or counting the last maximum would fail the comparison."""
    for mutant in ("wt", "nob", "last"):
        caught = False
        for C, H, short in HEAD_CASES + [("tie", 64, False)]:
            if C == "tie":
                feat, W, bias, labels, ids, b = _tie_inputs()
                C = W.shape[0]
            else:
                B = 12
                b = 7 if short else B
                feat, W, bias, labels, ids = _head_inputs(B, H, C, 40, zlib.crc32(repr((C, H, short)).encode()))
            got = _run_head(feat, W, bias, ids, labels, b)
            caught |= not _head_close(got, _head_ref(feat, W, bias, ids, labels, b, mutant), b, H, C, W, feat)
        assert caught, mutant


def _tie_inputs():
    """Classes 0 and 1 share their weights and bias and carry the largest logit of every row: exact ties."""
    feat, W, bias, labels, ids = _head_inputs(10, 64, 5, 10, 99)
    W[1] = W[0]
    bias[0] = bias[1] = 50.0
    labels[:] = np.arange(10) % 3 == 2                              # 7 rows labelled 0, 3 labelled 1
    ids = np.arange(10, dtype=np.int64)
    return feat, W, bias, labels, ids, 10


def test_head_ties_follow_the_first_maximum():
    feat, W, bias, labels, ids, b = _tie_inputs()
    rc, stats, *_ = _run_head(feat, W, bias, ids, labels, b)
    assert rc == 0 and int(stats[1]) == int((labels[ids] == 0).sum()) == 7


def test_head_refuses_unsupported_sizes():
    for C, H in ((129, 64), (5, 48)):
        feat, W, bias, labels, ids = _head_inputs(4, H, C, 8, 1)
        assert _run_head(feat, W, bias, ids, labels, 4)[0] == _capi.GCCB_ERR_BADARG
        assert b"gccb_ft_head" in lib().gccb_last_error()


# ---------------------------------------------------------------------------------------- clip by value
N = 1000
WD, EPS_ADAM, EPS_ADAGRAD = 0.05, 1e-8, 1e-10


def _grad(rng):
    g = (rng.normal(size=N) * 1.5).astype(np.float32)
    g[::11] = 1.0
    g[5::11] = -1.0                                                 # exactly at the bounds
    assert (np.abs(g) > 1).sum() > 100                               # and well beyond them
    return g


def _hyper(kind, lr, t, betas=(0.9, 0.999), lr_decay=0.0):
    if kind == "adam":
        return np.array([lr, 1 - betas[0] ** t, np.sqrt(1 - betas[1] ** t), 0], np.float32)
    if kind == "sgd":
        return np.array([lr, 0, 0, 0], np.float32)
    return np.array([lr / (1 + (t - 1) * lr_decay), 0, 0, 0], np.float32)


def _call_clip_value(kind, p, g, s0, s1, hyper, momentum=0.0, skip=None):
    L = lib()
    sw, mask = (ptr(skip), -1) if skip is not None else (None, 0)
    if kind == "adam":
        return L.gccb_clip_value_adam(ptr(p), ptr(g), ptr(s0), ptr(s1), N, ptr(hyper), 0.9, 0.999, EPS_ADAM, WD, 1.0,
                                      sw, mask, None)
    if kind == "sgd":
        return L.gccb_clip_value_sgd(ptr(p), ptr(g), ptr(s0), N, ptr(hyper), momentum, WD, 1.0, sw, mask, None)
    return L.gccb_clip_value_adagrad(ptr(p), ptr(g), ptr(s0), N, ptr(hyper), EPS_ADAGRAD, WD, 1.0, sw, mask, None)


def _ref64(kind, p, g, s0, s1, hyper, momentum, clamp_after_decay=False):
    """float64 restatement; clamp_after_decay is the wrong order (clamp(g + wd p) instead of clamp(g) + wd p)."""
    p, s0 = p.astype(np.float64), s0.astype(np.float64)
    s1 = s1.astype(np.float64)
    h = hyper.astype(np.float64)
    d = np.clip(g + WD * p, -1, 1) if clamp_after_decay else np.clip(g, -1, 1) + WD * p
    if kind == "adam":
        s0 = 0.9 * s0 + 0.1 * d
        s1 = 0.999 * s1 + 0.001 * d * d
        p = p - (h[0] / h[1]) * s0 / (np.sqrt(s1) / h[2] + EPS_ADAM)
    elif kind == "sgd":
        if momentum:
            s0 = momentum * s0 + d
            d = s0
        p = p - h[0] * d
    else:
        s0 = s0 + d * d
        p = p - h[0] * d / (np.sqrt(s0) + EPS_ADAGRAD)
    return p, s0, s1


CLIP_CASES = [("adam", 0.0, 0.0), ("sgd", 0.0, 0.0), ("sgd", 0.9, 0.0), ("adagrad", 0.0, 0.05)]


@pytest.mark.parametrize("kind,momentum,lr_decay", CLIP_CASES)
def test_clip_value_steps_match_torch(kind, momentum, lr_decay):
    """Five steps against clip_grad_value_(., 1) + torch.optim on float32 CPU tensors, the LR changed before every
    step as the warm-up schedule does; each step is also held to the float64 restatement, and the wrong order
    (clamping after the weight decay is added) is shown to fall outside the bar."""
    rng = np.random.default_rng(zlib.crc32(repr((kind, momentum, lr_decay)).encode()))
    p = rng.normal(size=N).astype(np.float32)
    s0, s1 = np.zeros(N, np.float32), np.zeros(N, np.float32)
    tp = torch.nn.Parameter(torch.from_numpy(p.copy()))
    if kind == "adam":
        opt = torch.optim.Adam([tp], lr=0.1, betas=(0.9, 0.999), weight_decay=WD)
    elif kind == "sgd":
        opt = torch.optim.SGD([tp], lr=0.1, momentum=momentum, weight_decay=WD)
    else:
        opt = torch.optim.Adagrad([tp], lr=0.1, lr_decay=lr_decay, weight_decay=WD)
    wrong_caught, lr_sum = False, 0.0
    for t in range(1, 6):
        lr = 0.02 * t
        g = _grad(rng)
        g0 = g.copy()
        tp.grad = torch.from_numpy(g.copy())
        torch.nn.utils.clip_grad_value_([tp], 1)
        for grp in opt.param_groups:
            grp["lr"] = lr
        opt.step()
        hyper = _hyper(kind, lr, t, lr_decay=lr_decay)
        want, ws0, ws1 = _ref64(kind, p, g, s0, s1, hyper, momentum)
        wrong, _, _ = _ref64(kind, p, g, s0, s1, hyper, momentum, clamp_after_decay=True)
        assert _call_clip_value(kind, p, g, s0, s1, hyper, momentum) == 0
        assert np.array_equal(g, g0)                                # the gradient is not written
        # Adam: the 1.3e-5 relative difference of exp_avg_sq (below) moves each update by at most ~1e-5 of lr
        lr_sum += lr
        atol = 1e-6 + (1e-5 * lr_sum if kind == "adam" else 0.0)
        assert np.allclose(p, tp.detach().numpy(), rtol=1e-5, atol=atol), t
        assert np.allclose(p, want, rtol=1e-5, atol=atol), t
        wrong_caught |= not np.allclose(p, wrong, rtol=1e-5, atol=atol)
        st = opt.state[tp]
        if kind == "adam":
            assert np.allclose(s0, st["exp_avg"].numpy(), rtol=1e-5, atol=1e-7)
            # the shared Adam rule weighs d*d by 1.0f - beta2 in fp32 (0.00099998713 for 0.999), torch by the fp32
            # rounding of the double 1 - beta2 (0.001): 1.3e-5 relative
            assert np.allclose(s1, st["exp_avg_sq"].numpy(), rtol=2e-5, atol=1e-9)
        elif kind == "adagrad":
            assert np.allclose(s0, st["sum"].numpy(), rtol=1e-5, atol=1e-9)
        elif momentum:
            assert np.allclose(s0, st["momentum_buffer"].numpy(), rtol=1e-5, atol=1e-7)
        else:
            assert not s0.any()
    assert wrong_caught


@pytest.mark.parametrize("kind", ["adam", "sgd", "adagrad"])
def test_clip_value_skip_word_is_a_no_op(kind):
    rng = np.random.default_rng(3)
    p, g = rng.normal(size=N).astype(np.float32), _grad(rng)
    s0, s1 = np.abs(rng.normal(size=N)).astype(np.float32), np.abs(rng.normal(size=N)).astype(np.float32)
    snap = [x.copy() for x in (p, g, s0, s1)]
    skip = np.array([_capi.FLAG_EDGE_OVERFLOW], np.int32)
    assert _call_clip_value(kind, p, g, s0, s1, _hyper(kind, 0.01, 1), 0.9, skip=skip) == 0
    assert all(a.tobytes() == b.tobytes() for a, b in zip(snap, (p, g, s0, s1)))
    skip[0] = 0
    assert _call_clip_value(kind, p, g, s0, s1, _hyper(kind, 0.01, 1), 0.9, skip=skip) == 0
    assert not np.array_equal(p, snap[0])


# ---------------------------------------------------------------------------------------- feature gather
class _Set:
    def __init__(self, graphs):
        self.seeds, self.items, ip, ix, no, eo = seed_first_union(graphs)
        self.indptr, self.indices = ip.astype(np.int64), ix.astype(np.int32)
        self.node_off, self.edge_off = no, eo
        self.c = _capi.GraphSet(ptr(self.indptr), ptr(self.indices), ptr(self.node_off), ptr(self.edge_off),
                                len(graphs))


def _feature_graphs():
    rng = np.random.RandomState(2)
    gs = [_simple_csr(np.array([0, 1]), np.array([1, 2]), 5, "iso"),          # vertices 3 and 4 isolated
          _listed_csr(np.zeros(0, np.int64), np.zeros(0, np.int64), 1, "one")]  # a one-node graph
    for i in range(4):
        n = int(rng.randint(3, 9))
        gs.append(_simple_csr(rng.randint(0, n, 2 * n), rng.randint(0, n, 2 * n), n, "r%d" % i))
    return gs


def _gather_features(s, ids, node_cap, edge_cap, cache, P):
    b = NpBatch(len(ids), node_cap, edge_cap)
    gids = np.asarray(ids, np.int64)
    assert lib().gccb_gather_graphs(C.byref(s.c), ptr(gids), C.byref(b.c), None) == 0
    pos = np.full((2, node_cap, P), -7.0, np.float32)
    assert lib().gccb_gather_features(C.byref(s.c), ptr(gids), C.byref(b.c), 0, ptr(cache), P, ptr(pos), None) == 0
    return b, pos


def test_gather_features_matches_cache_indexing():
    s = _Set(_feature_graphs())
    P = 8
    total = int(s.node_off[-1])
    cache = np.random.default_rng(4).normal(size=(total, P)).astype(np.float32)
    ids = [3, 1, 0, 5, 1, 2]                                        # out of order, the one-node graph twice
    N = int(sum(np.diff(s.node_off)[ids]))
    E = int(sum(np.diff(s.edge_off)[ids]))
    b, pos = _gather_features(s, ids, N + 2, E + 2, cache, P)
    want = np.concatenate([cache[s.node_off[i]:s.node_off[i + 1]] for i in ids])
    assert b.flags[0] == 0 and int(b.node_off[0, len(ids)]) == N
    assert pos[0, :N].tobytes() == want.tobytes()
    assert np.all(pos[0, N:] == -7.0) and np.all(pos[1] == -7.0)   # view 1 and rows beyond N untouched


def test_gather_features_leaves_an_empty_batch_alone():
    s = _Set(_feature_graphs())
    P = 4
    cache = np.ones((int(s.node_off[-1]), P), np.float32)
    ids = [0, 2, 3]
    N = int(sum(np.diff(s.node_off)[ids]))
    b, pos = _gather_features(s, ids, N - 1, 1000, cache, P)        # node overflow: published empty
    assert b.flags[0] == _capi.FLAG_NODE_OVERFLOW and b.node_off[0, len(ids)] == -1
    assert np.all(pos == -7.0)
