"""GPU (H100): a linear-probe problem that fails is never scored as converged -- a constant column that duplicates
the unpenalised intercept makes the float64 Hessian singular, and fit_probe raises GccbError naming the fold, the
class and the non-positive pivot instead of returning weights."""
import numpy as np
import pytest

from gcc_b200 import _lib
from gcc_b200.tasks import linear_probe as lp

pytestmark = pytest.mark.gpu


def test_non_positive_pivot_is_reported():
    rng = np.random.default_rng(0)
    n = 2000
    X = np.stack([rng.standard_normal(n), np.full(n, 1e8)], 1).astype(np.float32)
    lab = (X[:, 0] + 0.5 * rng.standard_normal(n) > 0).astype(int)
    Y = lp.label_matrix(lab)
    with pytest.raises(_lib.GccbError, match=r"fold \d+, class \d+ did not converge \(non-positive Cholesky pivot\)"):
        lp.fit_probe(X, Y, lp.fold_ids(Y, 0))
    X[:, 1] = 1.0                                           # a benign constant column converges
    res = lp.fit_probe(X, Y, lp.fold_ids(Y, 0))
    assert (res.status == 1).all()
