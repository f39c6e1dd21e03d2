"""A numpy float64 restatement of the linear probe of csrc/probe.cu (include/gccb200.h, DESIGN.md 4g): the
gradient, Hessian and Newton step of each (fold, class) problem, an independent Newton solve to the optimum, and the
top-k prediction with its micro-F1 counts."""
import numpy as np


def _problem(X, Y, folds, f, j):
    tr = folds != f
    return np.hstack([X[tr].astype(np.float64), np.ones((tr.sum(), 1))]), Y[tr, j].astype(np.float64)


def _reg(d):
    r = np.ones(d + 1)
    r[d] = 0.0
    return r


def objective(A, t, w, C):
    z = A @ w
    m = np.where(t > 0, z, -z)
    loss = np.where(m > 0, np.log1p(np.exp(-np.abs(m))), -m + np.log1p(np.exp(-np.abs(m))))
    return 0.5 * np.dot(w[:-1], w[:-1]) + C * loss.sum()


def system(A, t, w, C):
    """(gradient, Hessian, Newton step, objective) of one problem at w (intercept last)."""
    d = A.shape[1] - 1
    z = A @ w
    p = 1.0 / (1.0 + np.exp(-z))
    g = _reg(d) * w + C * (A.T @ (p - t))
    s = p * (1.0 - p)
    H = C * (A.T * s) @ A + np.diag(_reg(d))
    return g, H, -np.linalg.solve(H, g), objective(A, t, w, C)


def systems(X, Y, folds, W, C, n_folds):
    """system() of every problem p = f c + j at W [P, d + 1]."""
    c = Y.shape[1]
    out = []
    for f in range(n_folds):
        for j in range(c):
            A, t = _problem(X, Y, folds, f, j)
            out.append(system(A, t, W[f * c + j], C))
    return out


def newton(A, t, C, tol=1e-12, max_iter=200):
    """The optimum of one problem by plain damped Newton in float64 (numpy's solver, halving line search)."""
    w = np.zeros(A.shape[1])
    g0 = None
    for _ in range(max_iter):
        g, H, step, f = system(A, t, w, C)
        gn = np.abs(g).max()
        g0 = gn if g0 is None else g0
        if gn <= tol * max(1.0, g0):
            return w
        a = 1.0
        while a > 1e-8 and objective(A, t, w + a * step, C) > f + 1e-4 * a * g.dot(step) + 1e-12 * abs(f):
            a *= 0.5
        w = w + a * step
    return w


def topk_counts(Z, Y):
    """(tp, fp, fn) of the rows of decision values Z [n, c]: a row with k labels predicts the k classes of largest
    value, ties to the lower class."""
    tp = fp = fn = 0
    for z, y in zip(Z, Y):
        k = int(y.sum())
        order = sorted(range(len(z)), key=lambda j: (-z[j], j))[:k]
        hit = int(sum(y[j] for j in order))
        tp += hit
        fp += k - hit
        fn += k - hit
    return tp, fp, fn
