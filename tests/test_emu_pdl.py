"""CPU: programmatic dependent launch in the hidden <= 64 training chain, under the fiber emulator.  Every kernel
launched with GCCB_LAUNCH_PDL must call pdl_wait() in every thread before it returns: otherwise its successor may
start before the predecessor's writes are visible, and the ordering stops being transitive.  One forward, InfoNCE,
backward, clip/update and enqueue at L = 5, hidden 64 and 32, with blocks that leave early: tiles past a short
batch's rows, a view published empty, a set skip word.  An emulator build with the wait removed from one kernel
fails the same check."""
import ctypes as C
import importlib.util
import os
import shutil

import numpy as np
import pytest

from emu_util import HERE, lib, ptr
from gcc_b200 import _capi
from test_emu_gin_chain import BWD_LAUNCHES_L5, FWD_LAUNCHES_L5, _setup

K_QUEUE = 300


def _pdl_log(Lb):
    f = Lb.gccb_emu_pdl_log
    f.restype, f.argtypes = C.c_char_p, [C.POINTER(C.c_ulonglong)]
    counts = (C.c_ulonglong * 2)()
    first = f(counts)
    return [int(x) for x in counts], first.decode()


def _run_chain(Lb, H, empty_view=False):
    """One step of the chain; returns {call: (launches, [pdl launches, unwaited], first offender)}."""
    L = 5
    _, b, views, pos, cfg, flat, sd, rs, running, acts, st = _setup(L, H, B_=5, hops=12)
    # a short batch: the stash and the grids are sized for twice the rows, so most tile-loop blocks exit at once
    b2 = _capi_batch_with_cap(b, 2 * b.node_cap + 130)
    pos2 = np.zeros((2, b2.node_cap, pos.shape[2]), np.float32)
    pos2[:, :b.node_cap] = pos
    if empty_view:
        b2.node_off[0, b2.B] = -1                  # published empty: heads and optimiser skip the step
    acts = np.zeros(Lb.gccb_gin_acts_bytes(C.byref(cfg), b2.B, b2.node_cap), np.uint8)
    nbt = np.zeros(3 * (L - 1), np.int64)
    B, d = b2.B, H
    out = {}

    def call(name, fn):
        _pdl_log(Lb)
        n0 = Lb.gccb_launch_count()
        assert fn() == 0, Lb.gccb_last_error()
        counts, first = _pdl_log(Lb)
        out[name] = (Lb.gccb_launch_count() - n0, counts, first)

    q = np.zeros((B, d), np.float32)
    call("forward", lambda: Lb.gccb_gin_forward(C.byref(cfg), C.byref(b2.c), 0, ptr(pos2), ptr(flat), ptr(running),
                                                ptr(nbt), 1, 5, 0, 0, ptr(acts), acts.nbytes, ptr(q), None, None))
    rng = np.random.default_rng(H)
    k = rng.normal(size=(B, d)).astype(np.float32)
    mem = rng.normal(size=(K_QUEUE, d)).astype(np.float32)
    stats = np.full(2, 7.0, np.float32)            # stale values: the partial pass zeroes them
    dq = np.zeros_like(q)
    ws = np.zeros(Lb.gccb_infonce_workspace(B, d, K_QUEUE), np.uint8)
    call("infonce", lambda: Lb.gccb_infonce_fused(ptr(q), ptr(k), ptr(mem), B, d, K_QUEUE, 0.07, ptr(stats), ptr(dq),
                                                  ptr(ws), ws.nbytes, None))
    grads = np.zeros_like(flat)
    bws = np.full(Lb.gccb_gin_backward_workspace(C.byref(cfg), B, b2.node_cap), 0xAB, np.uint8)   # stale reductions
    call("backward", lambda: Lb.gccb_gin_backward(C.byref(cfg), C.byref(b2.c), 0, ptr(flat), ptr(acts), ptr(dq),
                                                  ptr(grads), 5, 0, 0, ptr(bws), bws.nbytes, None))
    n = flat.size
    m, v, pe = np.zeros(n, np.float32), np.zeros(n, np.float32), flat.copy()
    hyper = np.array([1e-3, 0.1, 0.03, 0], np.float32)
    gn, wsd = np.zeros(1, np.float32), np.zeros(1, np.float64)
    flags = b2.flags
    flags[0] = 2 if empty_view else 0
    call("clip_update", lambda: Lb.gccb_clip_adam_ema(ptr(flat), ptr(grads), ptr(m), ptr(v), ptr(pe), n, n,
                                                      ptr(hyper), 0.9, 0.999, 1e-8, 1e-5, 1.0, 0.999, 1.0, ptr(gn),
                                                      ptr(wsd), ptr(flags), 3, None))
    idx = np.array([K_QUEUE - 2], np.int64)
    call("enqueue", lambda: Lb.gccb_moco_enqueue(ptr(mem), ptr(k), B, d, K_QUEUE, ptr(idx), 1, 0, ptr(flags), 3, None))
    return out, stats, grads


def _capi_batch_with_cap(b, node_cap):
    """b's two views in a batch with a larger node capacity (more tiles than rows)."""
    from emu_util import NpBatch
    nb = NpBatch(b.B, node_cap, b.edge_cap)
    nb.node_off[:] = b.node_off
    nb.edge_off[:] = b.edge_off
    nb.indptr[:, :b.node_cap + 1] = b.indptr
    nb.indptr[:, b.node_cap + 1:] = b.indptr[:, -1:]
    nb.indices[:] = b.indices
    for a in ("sub_deg", "graph_id", "orig_id"):
        getattr(nb, a)[:, :b.node_cap] = getattr(b, a)
    nb.counters[:] = b.counters
    return nb


EXPECTED = {"forward": FWD_LAUNCHES_L5, "infonce": 2, "backward": BWD_LAUNCHES_L5, "clip_update": 2, "enqueue": 2}


@pytest.mark.parametrize("H", [64, 32])
@pytest.mark.parametrize("empty_view", [False, True])
def test_every_programmatic_launch_waits_first(H, empty_view):
    Lb = lib()
    out, stats, grads = _run_chain(Lb, H, empty_view)
    for name, (launches, (pdl, unwaited), first) in out.items():
        assert launches == EXPECTED[name], (name, launches)
        assert pdl == launches, (name, pdl, launches)   # every launch of these calls is a programmatic dependent
        assert unwaited == 0, (name, unwaited, first)
    # the zeroing that replaced the memsets happened: InfoNCE statistics and BatchNorm-backward reductions
    if not empty_view:
        assert np.isfinite(stats).all() and abs(stats[0]) < 100 and np.isfinite(grads).all()
        assert np.abs(grads).max() < 1e6


def _sabotaged_lib(tmp_path):
    """The emulator library built from a copy of the sources with pdl_wait() removed from infonce_merge_kernel."""
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    root = str(tmp_path)
    shutil.copytree(os.path.join(mod.ROOT, "include"), os.path.join(root, "include"))
    csrc = os.path.join(root, "gcc_b200", "csrc")
    shutil.copytree(mod.CSRC, csrc)
    path = os.path.join(csrc, "moco.cu")
    src = open(path).read()
    at = src.index("infonce_merge_kernel(")
    wait = src.index("  pdl_wait();\n", at)
    assert wait < src.index("\n}\n", at)
    open(path, "w").write(src[:wait] + src[wait + len("  pdl_wait();\n"):])
    # this module instance of the emulator build compiles the edited copy into a directory of its own
    mod.ROOT, mod.CSRC = root, csrc
    mod.OUT = os.path.join(os.path.dirname(mod.LIB), "pdl_wait_removed")
    mod.LIB = os.path.join(mod.OUT, "libgccb200_emu.so")
    so = mod.build()
    return _capi.bind(C.CDLL(so), require_all=False)


def test_a_removed_wait_is_caught(tmp_path):
    Lb = _sabotaged_lib(tmp_path)
    out, _, _ = _run_chain(Lb, 64)
    launches, (pdl, unwaited), first = out["infonce"]
    assert unwaited == 1 and first == "infonce_merge_kernel", out["infonce"]
    assert all(out[n][1][1] == 0 for n in out if n != "infonce")
