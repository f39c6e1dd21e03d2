"""Exact numpy restatement of the cosine top-k of csrc/knn.cu (include/gccb200.h, DESIGN.md 4f).

fp32 fma without math.fma: the product of two fp32 values is exact in float64 (48 significant bits), so
fma(a, b, c) = fp32(a*b + c) rounded once.  The float64 sum s = RN64(a*b + c) is rounded again to fp32; that double
rounding differs from a single rounding only when s lies exactly on an fp32 half-way point while the float64 addition
was inexact (a half-way point is a float64, so no other one can lie between the exact sum and s).  There the TwoSum
error term tells on which side the exact sum lies, and the result is the fp32 neighbour on that side.
"""
import numpy as np


def _halfway(s):
    """Mask of float64 values that lie exactly half-way between two adjacent fp32 values."""
    r = s.astype(np.float32)
    rd = r.astype(np.float64)
    other = np.nextafter(r, np.where(rd < s, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    with np.errstate(invalid="ignore", over="ignore"):
        mid = (rd + other.astype(np.float64)) * 0.5
    return (rd != s) & (mid == s)


def fma32(a, b, c):
    """Correctly rounded fp32 a*b + c, elementwise (broadcasting); a, b, c are fp32 arrays or scalars."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float32) for x in (a, b, c)))
    shape = a.shape
    a, b, c = (np.atleast_1d(x).ravel() for x in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)            # exact
    s = p + c.astype(np.float64)
    r = s.astype(np.float32)
    # cheap filter: a normal-range half-way point has its low 29 float64 mantissa bits equal to 1 << 28; values in
    # the fp32 subnormal range go through the exact test too
    cand = ((np.abs(s).view(np.int64) & 0x1FFFFFFF) == 0x10000000) | (np.abs(s) < 2.0 ** -125)
    if cand.any():
        i = np.nonzero(cand)[0]
        ss, pp, cc = s[i], p[i], c[i].astype(np.float64)
        bb = ss - pp
        err = (pp - (ss - bb)) + (cc - bb)                       # TwoSum: the exact sum is ss + err
        fix = _halfway(ss) & (err != 0)
        if fix.any():
            # the exact sum lies on err's side of the half-way point: take the fp32 neighbour on that side
            up = err[fix] > 0
            r0 = ss[fix].astype(np.float32)
            on_side = (r0.astype(np.float64) > ss[fix]) == up
            toward = np.where(up, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
            r[i[fix]] = np.where(on_side, r0, np.nextafter(r0, toward))
    return r.reshape(shape)


def normalize(x):
    """Rows of x [n, d] (fp32) -> normalised rows [n, d4] and a mask of rows holding a NaN or an Inf."""
    x = np.asarray(x, np.float32)
    n, d = x.shape
    d4 = (d + 3) & ~3
    xp = np.zeros((n, d4), np.float32)
    xp[:, :d] = x
    s = np.zeros(n, np.float32)
    for j in range(d4):
        s = fma32(xp[:, j], xp[:, j], s)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        den = np.sqrt(s)
        out = xp / den[:, None]
    out[s == 0] = 0.0
    return out.astype(np.float32), ~np.isfinite(x).all(axis=1)


def scores(qn, cn):
    """score[i, j] = sequential fp32 fma chain of qn[i, :] * cn[j, :] from +0 (normalised rows)."""
    acc = np.zeros((qn.shape[0], cn.shape[0]), np.float32)
    for j in range(qn.shape[1]):
        acc = fma32(qn[:, j, None], cn[None, :, j], acc)
    return acc


def topk(queries, cands, k, exclude=None):
    """(ids int64 [nq, k], scores fp32 [nq, k]): the first k candidates under (score descending, index ascending),
    -0 == +0 (reported as +0), exclude[i] (or -1) left out."""
    qn, _ = normalize(queries)
    cn, _ = normalize(cands)
    s = scores(qn, cn) + np.float32(0.0)                        # -0 -> +0
    nq, nc = s.shape
    ids = np.empty((nq, k), np.int64)
    out = np.empty((nq, k), np.float32)
    cand = np.arange(nc)
    for i in range(nq):
        keep = np.ones(nc, bool)
        if exclude is not None and 0 <= exclude[i] < nc:
            keep[exclude[i]] = False
        c = cand[keep]
        order = np.argsort(-s[i, keep].astype(np.float64), kind="stable")[:k]   # stable: ties by index
        ids[i] = c[order]
        out[i] = s[i, c[order]]
    return ids, out
