"""CPU: the eigensolver kernels (gcc_b200/csrc/posenc.cu) under the fiber emulator on the structure set
(tests/eig_structures.py) up to 384 vertices -- the dense classes and the single-CTA ChFSI classes -- with the float64
checks of tests/eig_checks.py (residuals, the top k, subspaces, layout, feature widths, normalisation), under the
shipped dispatch and under GCCB200_DENSE_MAX=228.  tests/test_gpu_eigensolver.py runs the same checks on the H100
over the whole set; a failure there that passes here is a hardware-only one."""
import ctypes as C

import numpy as np
import pytest

import eig_checks as ec
import eig_structures as es
from emu_util import NpBatch, lib, ptr

NMAX = 384
# every feature width under the shipped dispatch, two under the dense one (the emulator is slow: ~40 s a call)
CASES = [("default", 32), ("default", 2), ("default", 5), ("default", 16), ("default", 31), ("dense", 32),
         ("dense", 5)]


@pytest.fixture(scope="module")
def structs():
    graphs = [g for g in es.structures() if g["n"] <= NMAX]
    return graphs, [ec.reference(g) for g in graphs]


def _posenc(b, pos_dim, normalize):
    L = lib()
    pos = np.full((2, b.node_cap, pos_dim), np.nan, np.float32)
    eig = np.full((2 * b.B, pos_dim), np.nan, np.float32)
    ws = np.zeros(L.gccb_posenc_workspace(b.B, b.node_cap), np.uint8)
    b.flags[:] = 0
    assert L.gccb_posenc(C.byref(b.c), pos_dim, normalize, ptr(pos), ptr(eig), ptr(ws), ws.nbytes, None) == 0, \
        L.gccb_last_error()
    n = 2 * b.B
    return pos, eig, ws[68 * n:72 * n].view(np.float32).copy()


@pytest.mark.parametrize("solver,pos_dim", CASES)
def test_structures_match_float64(structs, monkeypatch, solver, pos_dim):
    if solver == "dense":
        monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    else:
        monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
    graphs, refs = structs
    half = (len(graphs) + 1) // 2
    views = [graphs[:half], graphs[half:] + graphs[:1] * (2 * half - len(graphs))]
    b = NpBatch.from_subgraphs(views)
    raw, eig, kres = _posenc(b, pos_dim, 0)
    assert b.flags[0] == 0
    nrm, eig1, _ = _posenc(b, pos_dim, 1)
    assert b.flags[0] == 0 and np.array_equal(eig, eig1)
    worst = {}
    for v in (0, 1):
        end = b.node_off[v, b.B]
        assert np.all(np.isfinite(raw[v, :end])) and np.all(np.isnan(raw[v, end:])), v    # rows of the batch only
        for gi, g in enumerate(views[v]):
            i = gi if v == 0 else half + gi
            a, z = b.node_off[v, gi], b.node_off[v, gi + 1]
            cls = es.eig_class(g["n"], solver)
            w = worst.setdefault(cls, {})
            ec.check(g, refs[i % len(graphs)], raw[v, a:z], eig[v * b.B + gi], pos_dim, cls.startswith("dense"),
                     float(kres[v * b.B + gi]), w)
            ec.check_normalized(g, raw[v, a:z], nrm[v, a:z], w)
    ec.report("emulated eigensolver [%s], pos_dim %d: worst error / bound per class" % (solver, pos_dim),
              {c: worst[c] for c in es.CLASS_ORDER if c in worst})
