"""float64 checks of one graph's eigensolver output (gccb_posenc), shared by the emulator and the H100 tests of the
structure set (tests/eig_structures.py).  numpy / scipy only.

Notation: k = min(n - 2, pos_dim); U the k returned columns in descending order of their eigenvalues theta; R = L U -
U diag(theta) in float64 on the float32 output; lambda_1 >= lambda_2 >= ... the exact spectrum."""
import numpy as np
import scipy.sparse.linalg as sla

from oracle import posenc as opos

# per-column residual / orthonormality bars of each class (tests/test_gpu_parity2.py): the dense solver is a direct
# method; ChFSI up to 160 vertices converges to 1e-4; above, the documented stagnation bar (GCCB_CF_STAG = 2e-3 +
# 25 % for the float64 re-evaluation) -- a near-degenerate cluster wider than the 48-column block converges only
# to the cluster's own spread
RES_DENSE, RES_SMALL, RES_HUB, ORTHO = 2e-5, 1e-4, 2.5e-3, 1e-4
LAM_DENSE = 2e-6
EIGH_MAX = 3600            # dense float64 eigh up to here, eigsh (k + 16 vectors) above
KMAX = 32
NSTORE = KMAX + 16         # exact eigenpairs kept per graph


def bars(n, dense):
    """(residual bar, orthonormality bar) of the class an n-vertex graph goes to."""
    if dense:
        return RES_DENSE, RES_DENSE
    return (RES_SMALL, ORTHO) if n <= 160 else (RES_HUB, ORTHO)


def reference(g):
    """Exact top eigenpairs of L = D^-1/2 A D^-1/2 (D = column sums, duplicates summed, clipped to 1): dict(lap =
    the sparse matrix, w = the top min(n, NSTORE + 1) eigenvalues descending, V = their vectors)."""
    n = g["n"]
    lap = opos.normalized_adjacency(g["indptr"], g["indices"], n)
    if n <= EIGH_MAX:
        w, v = np.linalg.eigh(lap.toarray())
        w, v = w[::-1][:NSTORE + 1], v[:, ::-1][:, :NSTORE + 1]
    else:
        w, v = sla.eigsh(lap, k=NSTORE + 1, which="LA", tol=1e-13, ncv=4 * NSTORE, v0=np.ones(n))
        o = np.argsort(w)[::-1]
        w, v = w[o], v[:, o]
    return dict(lap=lap, w=w, V=v)


def _sin(U, V):
    """sin of the largest principal angle between span(U) (orthonormalised) and the orthonormal columns V."""
    Q, _ = np.linalg.qr(U)
    return float(np.linalg.norm(Q - V @ (V.T @ Q), 2))


def check(g, ref, u_all, lam_all, pos_dim, dense, kernel_res, worst):
    """Checks 1-4 on one graph's normalize = 0 output: u_all [n, pos_dim] float32 rows, lam_all [pos_dim] float32.
    Updates worst[check] with the largest error / bound ratio; raises AssertionError naming the graph."""
    n, name = g["n"], g["name"]
    k = min(n - 2, pos_dim)
    assert np.all(np.isfinite(u_all)) and np.all(np.isfinite(lam_all)), name
    if k <= 0:
        assert np.all(u_all == 0) and np.all(lam_all == 0), name
        return
    # 4. layout: columns / eigenvalues k.. exactly zero
    assert np.all(u_all[:, k:] == 0) and np.all(lam_all[k:] == 0), name
    lap = ref["lap"]
    U = u_all[:, :k][:, ::-1].astype(np.float64)                 # descending
    theta = lam_all[:k][::-1].astype(np.float64)
    LU = lap @ U
    R = LU - U * theta
    rq = (U * LU).sum(0) / (U * U).sum(0)
    col_res = np.linalg.norm(LU - U * rq, axis=0)
    ortho = float(np.abs(U.T @ U - np.eye(k)).max())
    res_bar, ortho_bar = bars(n, dense)
    # 1. residuals and orthonormality, and the kernel's own report
    _ratio(worst, "residual", col_res.max() / res_bar, name)
    _ratio(worst, "ortho", ortho / ortho_bar, name)
    _ratio(worst, "vs kernel residual", col_res.max() / (1.25 * kernel_res + 2e-5), name)
    # 4. eigenvalues ascending.  ChFSI orders its columns by the Ritz values of the last Rayleigh-Ritz step and reports
    # the Rayleigh quotients of the float32 columns X = Q W after it: inside a multiplet the two differ by the rounding
    # of X = Q W (measured 6e-7), so neighbours of a multiplet may be inverted by that much -- never by more than the
    # residual plus the rounding
    # residual plus the rounding.  The kernel's float32 Rayleigh quotient of a unit column is a sum of n products, each
    # at most 1 in size: it is within n * 2^-24 of the exact one (Higham's gamma_n bound).
    fp32_rq = n * 2.0 ** -24
    _ratio(worst, "ascending", max(0.0, -np.diff(lam_all[:k].astype(np.float64)).min(initial=0.0)) /
           (col_res.max() + 2 * fp32_rq), name)
    # 4. eigenvalue c belongs to column c: its Rayleigh quotient within the column's residual (plus that rounding)
    _ratio(worst, "column order", np.abs(rq - theta).max() / (col_res.max() + fp32_rq), name)
    # 4. sign: the largest-|.| component of every column (lowest row on ties) is positive
    big = np.argmax(np.abs(u_all[:, :k]), axis=0)
    assert np.all(u_all[big, np.arange(k)] > 0), (name, "sign")
    # 2. the top k: theta_j within ||R||_2 (+ the orthonormality defect) of the exact j-th largest eigenvalue
    w = ref["w"]
    rn = float(np.linalg.norm(R, 2))
    _ratio(worst, "top-k eigenvalues", np.abs(theta - w[:k]).max() / (rn + ortho + 1e-7), name)
    if dense:
        _ratio(worst, "dense eigenvalues", np.abs(theta - w[:k]).max() / LAM_DENSE, name)
    # 3. subspaces: Davis-Kahan wherever lambda_j - lambda_{j+1} > 10 ||R||_2 ...
    V = ref["V"]
    eps = rn + ortho
    for j in range(1, k + 1):
        if j >= len(w):
            break
        gap = w[j - 1] - w[j]
        if gap > 10 * rn and gap > 2 * eps:
            _ratio(worst, "subspace", _sin(U[:, :j], V[:, :j]) / (eps / (gap - eps) + 1e-7), name)
    # ... and where the cut lies inside a multiplet, the columns lie in the exact space up to its end
    if k < len(w) - 1 and not (w[k - 1] - w[k] > 10 * rn):
        for b in range(k + 1, len(w)):
            gap = w[b - 1] - w[b]
            if gap > 10 * rn and gap > 2 * eps:
                _ratio(worst, "multiplet membership", _sin(U, V[:, :b]) / (eps / (gap - eps) + 1e-7), name)
                break


def check_normalized(g, raw, nrm, worst):
    """5. normalize = 1 equals the row-normalised normalize = 0 output within 4 fp32 ulps; zero rows stay zero."""
    name = g["name"]
    r64 = raw.astype(np.float64)
    norm = np.sqrt((r64 * r64).sum(1, keepdims=True))
    zero = norm[:, 0] == 0
    assert np.all(nrm[zero] == 0), (name, "zero rows")
    want = r64[~zero] / norm[~zero]
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(nrm[~zero].astype(np.float64) - want) / ulp
    if err.size:
        _ratio(worst, "normalize ulps", float(err.max()) / 4.0, name)


def _ratio(worst, what, r, name):
    r = float(r)
    if r > worst.get(what, (0.0, ""))[0]:
        worst[what] = (r, name)
    assert r <= 1.0, (name, what, r)


def report(title, worst_by_class):
    """One line per class: the worst error / bound ratio of every check and the graph it came from."""
    print(title)
    for cls, worst in worst_by_class.items():
        print("  %-12s %s" % (cls, ", ".join("%s %.3f (%s)" % (w, r, g) for w, (r, g) in sorted(worst.items()))))
