"""The linear probe of csrc/probe.cu under the CPU emulator, against the numpy float64 restatement
(tests/probe_oracle.py): gradient, Hessian, Newton step and objective at widths 1 .. 256, row counts that are not a
multiple of the tile, 1, 2 and 47 classes, multi-label rows, a constant predictor, tied decision values, the
non-finite flag, refused widths, and a Hessian that is bit-identical however many problems share a launch."""
import numpy as np
import pytest

import probe_oracle as oracle
from emu_util import lib, ptr
from gcc_b200 import _capi


def data(n, d, c, seed, multi=False, folds=3):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    if multi:
        Y = (rng.random((n, c)) < 0.4).astype(np.uint8)
        Y[np.arange(n), rng.integers(0, c, n)] = 1
    else:
        lab = (X[:, 0] > 0).astype(int) * (c > 1) + rng.integers(0, c, n)
        Y = np.zeros((n, c), np.uint8)
        Y[np.arange(n), lab % c] = 1
    fo = (np.arange(n) % folds).astype(np.int32)
    return X, Y, fo


def ws_for(n, d, c, folds, batch):
    size = lib().gccb_probe_workspace(n, d, c, folds, batch)
    assert size > 0
    ws = np.zeros(size + 32, np.uint8)
    return ws[(-ws.ctypes.data) % 16:][:size]


def emu_system(X, Y, fo, W, C, folds, batch=0):
    L = lib()
    n, d = X.shape
    c = Y.shape[1]
    P = folds * c
    g = np.zeros((P, d + 1))
    H = np.zeros((P, d + 1, d + 1))
    st = np.zeros((P, d + 1))
    f = np.zeros(P)
    status = np.zeros(P, np.int32)
    ws = ws_for(n, d, c, folds, batch)
    X, Y, fo, W = (np.ascontiguousarray(a) for a in (X, Y, fo, W))
    rc = L.gccb_probe_system(ptr(X), n, d, ptr(Y), c, ptr(fo), folds, C, batch, ptr(W), ptr(g), ptr(H), ptr(st),
                             ptr(f), ptr(status), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return g, H, st, f, status


def emu_fit(X, Y, fo, C, folds, batch=0, max_iter=100):
    L = lib()
    n, d = X.shape
    c = Y.shape[1]
    P = folds * c
    w = np.zeros((P, d + 1))
    z = np.zeros((n, c))
    counts = np.zeros((folds, 3), np.int64)
    status = np.zeros(P, np.int32)
    gnorm = np.zeros(P)
    iters = np.zeros(P, np.int32)
    flags = np.zeros(1, np.int32)
    ws = ws_for(n, d, c, folds, batch)
    X, Y, fo = (np.ascontiguousarray(a) for a in (X, Y, fo))
    rc = L.gccb_probe_fit(ptr(X), n, d, ptr(Y), c, ptr(fo), folds, C, max_iter, batch, ptr(w), ptr(z), ptr(counts),
                          ptr(status), ptr(gnorm), ptr(iters), ptr(flags), ptr(ws), ws.nbytes, None)
    assert rc == 0, L.gccb_last_error()
    return dict(w=w, z=z, counts=counts, status=status, gnorm=gnorm, iters=iters, flags=int(flags[0]))


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("d", [1, 7, 63, 64, 65, 129, 256])
def test_gradient_hessian_and_step_match_the_oracle(d):
    n, c, folds = 45 if d > 64 else 77, 2, 2               # n not a multiple of the 32-row tile
    X, Y, fo = data(n, d, c, d, folds=folds)
    rng = np.random.default_rng(d + 1)
    W = rng.standard_normal((folds * c, d + 1)) * 0.1
    g, H, st, f, status = emu_system(X, Y, fo, W, 10.0, folds)
    for p, (go, Ho, so, fo_) in enumerate(oracle.systems(X, Y, fo, W, 10.0, folds)):
        assert rel(g[p], go) < 1e-12 and rel(H[p], Ho) < 1e-12
        assert abs(f[p] - fo_) <= 1e-12 * abs(fo_)
        if status[p] == 0:
            assert rel(st[p], so) < 1e-8
        assert np.array_equal(H[p], H[p].T)


@pytest.mark.parametrize("c", [1, 2, 47])
def test_fit_reaches_the_optimum_and_scores_its_topk(c):
    n, d, folds = 150, 5, 3
    X, Y, fo = data(n, d, c, 100 + c, folds=folds)
    r = emu_fit(X, Y, fo, 1.0, folds)
    assert r["flags"] == 0
    tp = fp = fn = 0
    for f in range(folds):
        for j in range(c):
            p = f * c + j
            tr = fo != f
            npos = int(Y[tr, j].sum())
            if npos == 0 or npos == tr.sum():
                assert r["status"][p] == (2 if npos else 3) and not r["w"][p].any()
                continue
            assert r["status"][p] == 1
            A, t = oracle._problem(X, Y, fo, f, j)
            assert rel(r["w"][p], oracle.newton(A, t, 1.0)) < 1e-8
        te = fo == f
        Z = np.stack([X[te].astype(np.float64) @ r["w"][f * c + j, :d] + r["w"][f * c + j, d] for j in range(c)], 1)
        for j in range(c):
            st = r["status"][f * c + j]
            if st in (2, 3):
                Z[:, j] = np.inf if st == 2 else -np.inf
        np.testing.assert_allclose(r["z"][te], Z, rtol=1e-12, atol=1e-12)
        ctp, cfp, cfn = oracle.topk_counts(r["z"][te], Y[te])
        assert tuple(r["counts"][f]) == (ctp, cfp, cfn)
        tp, fp, fn = tp + ctp, fp + cfp, fn + cfn
    if c == 1:
        assert (r["status"] == 2).all() and tp == n            # one class: every row predicts it


def test_multilabel_rows_and_a_class_absent_from_one_fold():
    n, d, c, folds = 120, 4, 5, 3
    X, Y, fo = data(n, d, c, 7, multi=True, folds=folds)
    Y[:, 4] = 0
    Y[fo == 0, 4] = 1                                         # class 4 only in fold 0's test rows
    r = emu_fit(X, Y, fo, 1.0, folds)
    assert r["flags"] == 0
    assert r["status"][0 * c + 4] == 3                         # fold 0 trains on no positive of class 4: -inf
    assert np.all(r["z"][fo == 0, 4] == -np.inf)
    for f in range(folds):
        assert tuple(r["counts"][f]) == oracle.topk_counts(r["z"][fo == f], Y[fo == f])


def test_tied_decision_values_break_to_the_lower_class():
    n, d, c, folds = 60, 3, 4, 2
    X, Y, fo = data(n, d, c, 9, folds=folds)
    Y[:] = 0
    Y[fo == 1, 0] = 1
    Y[fo == 1, 1] = 1                                        # fold 0 trains classes 0 and 1 on all-positive rows
    Y[fo == 0, 1] = 1                                        # fold 0's test rows: one label, class 1
    r = emu_fit(X, Y, fo, 1.0, folds)
    assert list(r["status"][:c]) == [2, 2, 3, 3]             # fold 0: +inf, +inf, -inf, -inf
    assert list(r["status"][c:]) == [3, 2, 3, 3]             # fold 1: only class 1 is positive in its training rows
    n0 = int((fo == 0).sum())
    assert tuple(r["counts"][0]) == (0, n0, n0)              # +inf tie between 0 and 1: class 0 is predicted
    assert tuple(r["counts"][1]) == (2 * (n - n0), 0, 0)     # class 1 (+inf), then class 0 of the -inf tie
    for f in range(folds):
        assert tuple(r["counts"][f]) == oracle.topk_counts(r["z"][fo == f], Y[fo == f])


def test_hessian_is_bit_identical_however_problems_share_a_launch():
    n, d, c, folds = 70, 9, 3, 3
    X, Y, fo = data(n, d, c, 11, folds=folds)
    W = np.random.default_rng(12).standard_normal((folds * c, d + 1)) * 0.2
    ref = emu_system(X, Y, fo, W, 1000.0, folds, batch=0)
    for batch in (1, 2, 5):
        got = emu_system(X, Y, fo, W, 1000.0, folds, batch=batch)
        for a, b in zip(ref[:4], got[:4]):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    r0 = emu_fit(X, Y, fo, 1000.0, folds)
    r1 = emu_fit(X, Y, fo, 1000.0, folds, batch=2)
    assert np.array_equal(r0["w"].view(np.uint64), r1["w"].view(np.uint64))
    assert np.array_equal(r0["z"].view(np.uint64), r1["z"].view(np.uint64))


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_nonfinite_row_raises_the_flag(bad):
    X, Y, fo = data(40, 3, 2, 13, folds=2)
    X[17, 1] = bad
    assert emu_fit(X, Y, fo, 1.0, 2)["flags"] & _capi.FLAG_NONFINITE


def test_iteration_limit_raises_the_flag():
    X, Y, fo = data(60, 3, 2, 14, folds=2)
    r = emu_fit(X, Y, fo, 1000.0, 2, max_iter=1)
    assert r["flags"] & _capi.FLAG_PROBE_NOCONV
    assert (r["status"] == 4).any() and r["gnorm"][r["status"] == 4].min() > 0


def test_refused_widths_and_workspace():
    L = lib()
    assert L.gccb_probe_workspace(10, 257, 2, 10, 0) == 0
    assert L.gccb_probe_workspace(10, 0, 2, 10, 0) == 0
    assert L.gccb_probe_workspace(10, 4, 1025, 10, 0) == 0
    assert L.gccb_probe_workspace(10, 4, 2, 65, 0) == 0
    X, Y, fo = data(20, 257, 2, 15, folds=2)
    z = np.zeros(64)
    ws = np.zeros(4096, np.uint8)
    rc = L.gccb_probe_fit(ptr(X), 20, 257, ptr(Y), 2, ptr(fo), 2, 1.0, 10, 0, ptr(z), ptr(z), ptr(z), ptr(z), ptr(z),
                          ptr(z), ptr(z), ptr(ws), ws.nbytes, None)
    assert rc == _capi.GCCB_ERR_BADARG and b"d <= 256" in L.gccb_last_error()
    X, Y, fo = data(20, 4, 2, 15, folds=2)
    rc = L.gccb_probe_fit(ptr(X), 20, 4, ptr(Y), 2, ptr(fo), 2, 1.0, 10, 0, ptr(z), ptr(z), ptr(z), ptr(z), ptr(z),
                          ptr(z), ptr(z), ptr(ws[(-ws.ctypes.data) % 16:]), 64, None)
    assert rc == _capi.GCCB_ERR_CAPACITY


def test_line_search_continues_along_the_same_step_past_four_lengths():
    # heavy-tailed rows: problems 2 and 3 (fold 1) meet a Newton step that needs more than four halvings, so the line
    # search runs a second window of step lengths in a further pass before the next Newton system
    rng = np.random.default_rng(1)
    X = np.clip(rng.standard_cauchy((40, 3)), -1e3, 1e3).astype(np.float32)
    lab = ((X[:, 0] + rng.standard_normal(40) * 0.5) > 0).astype(int)
    Y = np.zeros((40, 2), np.uint8)
    Y[np.arange(40), lab] = 1
    fo = (np.arange(40) % 2).astype(np.int32)
    r = emu_fit(X, Y, fo, 1000.0, 2)
    assert r["flags"] == 0 and (r["status"] == 1).all()
    for p in range(4):
        A, t = oracle._problem(X, Y, fo, p // 2, p % 2)
        assert rel(r["w"][p], oracle.newton(A, t, 1000.0)) < 1e-8
    for p in (2, 3):
        # one pass per accepted step and one to see convergence is not enough: a pass went to the second window
        short = emu_fit(X, Y, fo, 1000.0, 2, max_iter=int(r["iters"][p]) + 1)
        assert short["status"][p] == 4 and short["flags"] & _capi.FLAG_PROBE_NOCONV
