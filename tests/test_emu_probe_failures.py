"""Failure paths of the linear probe (csrc/probe.cu) under the CPU emulator: a problem whose Hessian meets a
non-positive Cholesky pivot ends with status GCCB_PROBE_NOT_PD and raises GCCB_FLAG_PROBE_NOCONV, so that no caller
can score it as if it had converged; a problem that converges never raises the flag."""
import numpy as np
import pytest

from gcc_b200 import _capi
from test_emu_probe import emu_fit


def constant_column(K, n=60, seed=0):
    """Rows [N(0, 1), K]: the constant column duplicates the unpenalised intercept, so for large K the Hessian is
    singular in float64."""
    rng = np.random.default_rng(seed)
    X = np.stack([rng.standard_normal(n), np.full(n, K)], 1).astype(np.float32)
    lab = (X[:, 0] + 0.5 * rng.standard_normal(n) > 0).astype(int)
    Y = np.zeros((n, 2), np.uint8)
    Y[np.arange(n), lab] = 1
    return X, Y, (np.arange(n) % 2).astype(np.int32)


@pytest.mark.parametrize("K", [1e6, 1e8, 1e12])
def test_non_positive_pivot_raises_the_flag(K):
    X, Y, fo = constant_column(K)
    r = emu_fit(X, Y, fo, 1000.0, 2)
    assert (r["status"] == _capi.GCCB_PROBE_NOT_PD).any()
    assert r["flags"] & _capi.FLAG_PROBE_NOCONV
    assert set(r["status"]) <= {_capi.GCCB_PROBE_CONVERGED, _capi.GCCB_PROBE_NOT_PD}


def test_a_moderate_constant_column_converges_without_the_flag():
    X, Y, fo = constant_column(1e3)
    r = emu_fit(X, Y, fo, 1000.0, 2)
    assert (r["status"] == _capi.GCCB_PROBE_CONVERGED).all() and r["flags"] == 0
