"""CPU: the SIMT GIN training chain under the fiber emulator -- the last BatchNorm of a layer (BN_b) applied by the
kernels that read the layer's output, and BN_b's backward reduction inside the dh gather.  Pins the launch count of
one forward and one backward, every layer's stashed h in train and eval mode, and BN_b's running statistics after
one and two train-mode forwards, against the float64 oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from emu_util import lib, ptr
from gcc_b200 import _capi
from gcc_b200.models import layout as glayout
from oracle import model as om
from test_emu_gin import _batch, _oracle_view, _params

# launches per call at L = 5: forward = tables + x0 + 3 per GIN layer (agg+GEMM1, BN1+GEMM2, BN_a statistics)
# + pooling + heads; backward = heads + head weights + per layer (dh with BN_b's reduction, BN_a's reduction, GEMM2,
# GEMM1, two weight gradients with their reduces, three BatchNorm gradients) + dh0 + embedding
FWD_LAUNCHES_L5 = 16
BWD_LAUNCHES_L5 = 48


def _setup(L, H, B_=5, hops=12, seed=11):
    Lb = lib()
    b, views, pos = _batch(B_, hops)
    cfg = glayout.make_cfg(num_layers=L, hidden=H)
    flat, sd, _ = _params(cfg, np.random.default_rng(seed))
    rs, rtotal = glayout.running_slices(cfg)
    running = np.zeros(rtotal, np.float32)
    for key, (off, shape) in rs.items():
        running[off:off + shape[0]] = 1.0 if key.endswith("var") else 0.0
    acts = np.zeros(Lb.gccb_gin_acts_bytes(C.byref(cfg), b.B, b.node_cap), np.uint8)
    st = _capi.GinStash()
    assert Lb.gccb_gin_stash_layout(C.byref(cfg), b.B, b.node_cap, C.byref(st)) == 0, Lb.gccb_last_error()
    return Lb, b, views, pos, cfg, flat, sd, rs, running, acts, st


def _forward(Lb, cfg, b, view, pos, flat, running, nbt, bn_train, acts):
    feat = np.zeros((b.B, cfg.hidden), np.float32)
    rc = Lb.gccb_gin_forward(C.byref(cfg), C.byref(b.c), view, ptr(pos), ptr(flat), ptr(running), ptr(nbt), bn_train,
                             0, 0, -1, ptr(acts), acts.nbytes, ptr(feat), None, None)
    assert rc == 0, Lb.gccb_last_error()
    return feat


def _oracle_h(monkeypatch, sd, b, views, pos, view, L, bn_train):
    """Oracle forward of one view: every layer's h = relu(bn_b(y)) and the train-mode BatchNorm statistics."""
    seen = []
    bn = om._bn

    def record(x, *a, **k):
        y = bn(x, *a, **k)
        seen.append(y.detach())
        return y
    monkeypatch.setattr(om, "_bn", record)
    ov = _oracle_view(b, views, pos, view)
    _, _, stats = om.gin_encoder_forward(sd, ov["indptr"], ov["indices"], torch.from_numpy(ov["pos"]).double(),
                                         ov["seed"], ov["sub_deg"], ov["node_off"], num_layers=L, bn_train=bn_train)
    monkeypatch.setattr(om, "_bn", bn)
    return [torch.relu(seen[3 * l + 2]).numpy() for l in range(L - 1)], stats


def _check_h(acts, st, N, H, want):
    for l, w in enumerate(want):
        got = acts[st.h[l]:st.h[l] + N * H * 4].view(np.float32).reshape(N, H)
        assert np.allclose(got, w, rtol=1e-4, atol=1e-4 * float(np.abs(w).max())), (l, np.abs(got - w).max())


def test_launch_counts_per_call():
    L, H = 5, 64
    Lb, b, views, pos, cfg, flat, sd, rs, running, acts, st = _setup(L, H)
    nbt = np.zeros(3 * (L - 1), np.int64)
    n0 = Lb.gccb_launch_count()
    feat = _forward(Lb, cfg, b, 0, pos, flat, running, nbt, 1, acts)
    n1 = Lb.gccb_launch_count()
    assert n1 - n0 == FWD_LAUNCHES_L5
    w = np.random.default_rng(0).normal(size=feat.shape).astype(np.float32)
    grads = np.zeros_like(flat)
    ws = np.zeros(Lb.gccb_gin_backward_workspace(C.byref(cfg), b.B, b.node_cap), np.uint8)
    rc = Lb.gccb_gin_backward(C.byref(cfg), C.byref(b.c), 0, ptr(flat), ptr(acts), ptr(w), ptr(grads), 0, 0, -1,
                              ptr(ws), ws.nbytes, None)
    assert rc == 0, Lb.gccb_last_error()
    assert Lb.gccb_launch_count() - n1 == BWD_LAUNCHES_L5


@pytest.mark.parametrize("L,H", [(5, 64), (3, 128), (3, 32)])
def test_every_layer_h_and_running_statistics_vs_oracle(monkeypatch, L, H):
    """Two train-mode forwards (views 0, 1), then one eval-mode forward on the running statistics they left.
    After each: h of every layer, the last one (written by the pooling kernel) included; after each train-mode
    forward: the running mean / unbiased variance of all three BatchNorms of every layer (momentum 0.1, one update
    per forward) and num_batches_tracked."""
    Lb, b, views, pos, cfg, flat, sd, rs, running, acts, st = _setup(L, H)
    nbt = np.zeros(3 * (L - 1), np.int64)
    want_run = {k: running[off:off + s[0]].astype(np.float64) for k, (off, s) in rs.items()}
    for step, view in enumerate((0, 1)):
        _forward(Lb, cfg, b, view, pos, flat, running, nbt, 1, acts)
        h_o, stats = _oracle_h(monkeypatch, sd, b, views, pos, view, L, True)
        _check_h(acts, st, int(b.node_off[view, b.B]), H, h_o)
        for key in stats:
            mean, var = (t.numpy() for t in stats[key])
            want_run[key + "running_mean"] = 0.9 * want_run[key + "running_mean"] + 0.1 * mean
            want_run[key + "running_var"] = 0.9 * want_run[key + "running_var"] + 0.1 * var
        for key, (off, s) in rs.items():
            got, want = running[off:off + s[0]], want_run[key]
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * max(1.0, float(np.abs(want).max()))), \
                (step, key, np.abs(got - want).max())
        assert np.all(nbt == step + 1)
    # eval mode: both BatchNorms of the tail from the running statistics, which stay as they are
    run_before = running.copy()
    sd_eval = dict(sd)
    for key, (off, s) in rs.items():
        sd_eval[key] = torch.from_numpy(running[off:off + s[0]].astype(np.float64))
    _forward(Lb, cfg, b, 1, pos, flat, running, None, 0, acts)
    h_o, _ = _oracle_h(monkeypatch, sd_eval, b, views, pos, 1, L, False)
    _check_h(acts, st, int(b.node_off[1, b.B]), H, h_o)
    assert np.array_equal(running, run_before)
