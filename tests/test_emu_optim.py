"""CPU: the SGD and Adagrad optimiser kernels (gccb_clip_sgd_ema, gccb_clip_adagrad_ema) under the fiber
emulator, against a float64 restatement on the fp32 inputs and against torch.optim.SGD / torch.optim.Adagrad.
Kernel LOGIC only; tests/test_gpu_optim.py runs them on an H100."""
import zlib

import numpy as np
import pytest
import torch

from emu_util import lib, ptr
from gcc_b200 import _capi

N_LIVE, N_ALL = 1000, 1300
ALPHA, WD, EPS = 0.999, 1e-5, 1e-10


def _clr(lr, t, lr_decay):
    return lr / (1 + (t - 1) * lr_decay)


def _call(kind, p, g, s, pe, hyper, *, momentum=0.9, wd=WD, clip=1.0, alpha=ALPHA, scale=1.0, skip=None):
    gn, ws = np.zeros(1, np.float32), np.zeros(1, np.float64)
    skip_word, mask = (ptr(skip), -1) if skip is not None else (None, 0)
    if kind == "sgd":
        rc = lib().gccb_clip_sgd_ema(ptr(p), ptr(g), ptr(s), ptr(pe), N_LIVE, len(p), ptr(hyper), momentum, wd, clip,
                                     alpha, scale, ptr(gn), ptr(ws), skip_word, mask, None)
    else:
        rc = lib().gccb_clip_adagrad_ema(ptr(p), ptr(g), ptr(s), ptr(pe), N_LIVE, len(p), ptr(hyper), EPS, wd, clip,
                                         alpha, scale, ptr(gn), ptr(ws), skip_word, mask, None)
    assert rc == 0
    return float(gn[0])


def _ref(kind, p, g, s, pe, step_lr, *, momentum=0.9, wd=WD, clip=1.0, alpha=ALPHA, scale=1.0):
    """float64: clip_grad_norm_ + torch.optim.{SGD,Adagrad}.step + moment_update on the live entries, EMA only
    on the tail.  step_lr is lr for SGD and clr for Adagrad."""
    p, pe = p.astype(np.float64), pe.astype(np.float64)
    s = None if s is None else s.astype(np.float64)
    gs = g.astype(np.float64) * scale
    total = float(np.sqrt((gs ** 2).sum()))
    coef = min(1.0, clip / (total + 1e-6)) if clip > 0 else 1.0
    d = coef * gs + wd * p[:N_LIVE]
    if kind == "sgd":
        if momentum != 0:
            s = momentum * s + d
            d = s
        p[:N_LIVE] -= step_lr * d
    else:
        s = s + d * d
        p[:N_LIVE] -= step_lr * d / (np.sqrt(s) + EPS)
    pe = alpha * pe + (1 - alpha) * p
    return p, s, pe, total, coef


def _inputs(rng, kind, momentum, g_scale):
    p = rng.normal(size=N_ALL).astype(np.float32)
    g = (rng.normal(size=N_LIVE) * g_scale).astype(np.float32)
    g[::17] = 0.0                                               # entries whose gradient is exactly zero
    pe = rng.normal(size=N_ALL).astype(np.float32)
    if kind == "sgd":
        s = (rng.normal(size=N_LIVE) * 0.1).astype(np.float32) if momentum != 0 else None
    else:
        s = np.abs(rng.normal(size=N_LIVE) * 0.01).astype(np.float32)
    return p, g, s, pe


CASES = [("sgd", dict(momentum=0.9)), ("sgd", dict(momentum=0.0)),
         ("adagrad", dict(lr_decay=0.0, t=1)), ("adagrad", dict(lr_decay=0.01, t=1)),
         ("adagrad", dict(lr_decay=0.0, t=7)), ("adagrad", dict(lr_decay=0.01, t=7))]


@pytest.mark.parametrize("kind,cfg", CASES, ids=lambda c: c if isinstance(c, str) else
                         "-".join("%s%s" % kv for kv in c.items()))
@pytest.mark.parametrize("g_scale,scale", [(1.0, 1.0), (1e-3, 1.0), (1.0, 0.25), (2e-3, 0.5)],
                         ids=["clip", "noclip", "clip-scaled", "noclip-scaled"])
def test_kernel_matches_float64(kind, cfg, g_scale, scale):
    rng = np.random.default_rng(zlib.crc32(repr((kind, cfg, g_scale, scale)).encode()))
    momentum = cfg.get("momentum", 0.9)
    p, g, s, pe = _inputs(rng, kind, momentum, g_scale)
    lr = 0.004
    step_lr = lr if kind == "sgd" else _clr(lr, cfg["t"], cfg["lr_decay"])
    p_o, s_o, pe_o, total, coef = _ref(kind, p, g, s, pe, step_lr, momentum=momentum, scale=scale)
    assert (coef < 1.0) == (g_scale == 1.0)                     # the clip is active exactly in the "clip" cases
    tail = p[N_LIVE:].copy()
    hyper = np.array([step_lr, 0, 0, 0], np.float32)
    gn = _call(kind, p, g, s, pe, hyper, momentum=momentum, scale=scale)
    assert np.isclose(gn, total, rtol=1e-5)
    assert np.allclose(p, p_o, rtol=1e-5, atol=1e-7)
    assert np.array_equal(p[N_LIVE:], tail)                     # the tail gets the EMA only
    assert np.allclose(pe, pe_o, rtol=1e-5, atol=1e-7)
    if s is not None:
        assert np.allclose(s, s_o, rtol=1e-5, atol=1e-7 if kind == "sgd" else 1e-12)
    zero = np.flatnonzero(g == 0)
    assert len(zero) > 50 and np.allclose(p[zero], p_o[zero], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_zero_gradient_without_weight_decay_moves_nothing(kind):
    rng = np.random.default_rng(5)
    p, g, s, pe = _inputs(rng, kind, 0.9, 1.0)
    g[:] = 0.0
    s[:] = 0.0
    p0 = p.copy()
    _call(kind, p, g, s, pe, np.array([0.01, 0, 0, 0], np.float32), wd=0.0)
    assert np.array_equal(p, p0) and not s.any()


@pytest.mark.parametrize("kind,momentum,lr_decay", [("sgd", 0.9, 0.0), ("sgd", 0.0, 0.0), ("adagrad", 0.0, 0.0),
                                                    ("adagrad", 0.0, 0.01)])
def test_five_steps_match_torch_optim(kind, momentum, lr_decay):
    """Five steps against torch.optim on float32 CPU tensors fed the same clipped gradients, with the LR changed
    before every step as the warm-up schedule does (train.py:411-417)."""
    rng = np.random.default_rng(17)
    p = rng.normal(size=N_ALL).astype(np.float32)
    pe = p.copy()
    s = np.zeros(N_LIVE, np.float32)
    tp = torch.nn.Parameter(torch.from_numpy(p[:N_LIVE].copy()))
    if kind == "sgd":
        opt = torch.optim.SGD([tp], lr=0.1, momentum=momentum, weight_decay=WD)
    else:
        opt = torch.optim.Adagrad([tp], lr=0.1, lr_decay=lr_decay, weight_decay=WD)
    for t in range(1, 6):
        lr = 0.05 * t
        g = rng.normal(size=N_LIVE).astype(np.float32)
        total = np.sqrt((g.astype(np.float64) ** 2).sum())
        g_clipped = (g * min(1.0, 1.0 / (total + 1e-6))).astype(np.float32)
        tp.grad = torch.from_numpy(g_clipped.copy())
        for grp in opt.param_groups:
            grp["lr"] = lr
        opt.step()
        hyper = np.array([lr if kind == "sgd" else _clr(lr, t, lr_decay), 0, 0, 0], np.float32)
        _call(kind, p, g_clipped, s, pe, hyper, momentum=momentum, clip=0.0)
        assert np.allclose(p[:N_LIVE], tp.detach().numpy(), rtol=1e-5, atol=1e-6), t
        st = opt.state[tp]
        if kind == "adagrad":
            assert float(st["step"]) == t
            assert np.allclose(s, st["sum"].numpy(), rtol=1e-5, atol=1e-9)
        elif momentum != 0:
            assert np.allclose(s, st["momentum_buffer"].numpy(), rtol=1e-5, atol=1e-7)
        else:
            assert "momentum_buffer" not in st and not s.any()


@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_skip_word_leaves_every_buffer_bit_identical(kind):
    rng = np.random.default_rng(9)
    p, g, s, pe = _inputs(rng, kind, 0.9, 1.0)
    snap = [x.copy() for x in (p, g, s, pe)]
    skip = np.array([_capi.FLAG_NODE_OVERFLOW], np.int32)
    _call(kind, p, g, s, pe, np.array([0.01, 0, 0, 0], np.float32), skip=skip)
    assert all(np.array_equal(a, b) for a, b in zip(snap, (p, g, s, pe)))
    skip[0] = 0                                                 # a clear skip word trains
    _call(kind, p, g, s, pe, np.array([0.01, 0, 0, 0], np.float32), skip=skip)
    assert not np.array_equal(p, snap[0]) and not np.array_equal(s, snap[2])


def test_bad_arguments_are_refused():
    p, g, pe = np.zeros(N_ALL, np.float32), np.zeros(N_LIVE, np.float32), np.zeros(N_ALL, np.float32)
    hyper, gn, ws = np.zeros(4, np.float32), np.zeros(1, np.float32), np.zeros(1, np.float64)
    L = lib()
    # momentum needs its buffer; without momentum it may be NULL
    assert L.gccb_clip_sgd_ema(ptr(p), ptr(g), None, ptr(pe), N_LIVE, N_ALL, ptr(hyper), 0.9, WD, 1.0, ALPHA, 1.0,
                               ptr(gn), ptr(ws), None, 0, None) == _capi.GCCB_ERR_BADARG
    assert L.gccb_clip_sgd_ema(ptr(p), ptr(g), None, ptr(pe), N_LIVE, N_ALL, ptr(hyper), 0.0, WD, 1.0, ALPHA, 1.0,
                               ptr(gn), ptr(ws), None, 0, None) == 0
    assert L.gccb_clip_adagrad_ema(ptr(p), ptr(g), None, ptr(pe), N_LIVE, N_ALL, ptr(hyper), EPS, WD, 1.0, ALPHA,
                                   1.0, ptr(gn), ptr(ws), None, 0, None) == _capi.GCCB_ERR_BADARG
    s = np.zeros(N_LIVE, np.float32)
    assert L.gccb_clip_adagrad_ema(ptr(p), ptr(g), ptr(s), ptr(pe), N_LIVE, N_LIVE - 1, ptr(hyper), EPS, WD, 1.0,
                                   ALPHA, 1.0, ptr(gn), ptr(ws), None, 0, None) == _capi.GCCB_ERR_BADARG
