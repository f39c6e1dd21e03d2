"""GPU (H100): the linear probe of csrc/probe.cu (gcc_b200.tasks.linear_probe) -- weights at the float64 optimum of an
independent Newton solve at widths 64, 128 and 256, predictions equal to a converged sklearn fit row for row, micro-F1
within 0.01 of the reference evaluator, bit-identical weights across runs and launch batching, generate.py rows
through the command lines (a labelled .npz graph and an x2dgl corpus of whole graphs), and the error paths."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import probe_oracle as oracle
from gcc_b200 import _lib
from gcc_b200.tasks import linear_probe as lp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _data(n, d, c, seed, noise=1.0, multi=False):
    """Rows with a linear signal per class plus label noise: no class is separable, so every optimum is finite."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    U = rng.standard_normal((d, c)) / np.sqrt(d)
    S = X.astype(np.float64) @ U * 3.0 + noise * rng.standard_normal((n, c))
    if multi:
        Y = (S > 0.8).astype(np.uint8)
        Y[np.arange(n), S.argmax(1)] = 1
    else:
        Y = np.zeros((n, c), np.uint8)
        Y[np.arange(n), S.argmax(1)] = 1
    return X, Y


@pytest.mark.parametrize("d", [64, 128, 256])
def test_weights_reach_the_float64_optimum(d):
    n, c = 20000, 2
    X, Y = _data(n, d, c, d)
    folds = lp.fold_ids(Y, 0)
    res = lp.fit_probe(X, Y, folds)
    assert (res.status == 1).all()
    worst = 0.0
    for f in (0, 7):
        for j in range(c):
            A, t = oracle._problem(X, Y, folds, f, j)
            want = oracle.newton(A, t, 1000.0)
            worst = max(worst, np.abs(res.weights[f, j] - want).max() / np.abs(want).max())
    print("d=%d: worst relative weight error against float64 Newton %.3e, iterations %d..%d"
          % (d, worst, res.iters.min(), res.iters.max()))
    assert worst < 1e-8


def test_predictions_equal_converged_sklearn():
    from sklearn.linear_model import LogisticRegression
    from sklearn.multiclass import OneVsRestClassifier
    n, d, c = 3000, 16, 4
    X, Y = _data(n, d, c, 5)
    folds = lp.fold_ids(Y, 0)
    res = lp.fit_probe(X, Y, folds)
    tp = 0
    for f in range(10):
        tr, te = folds != f, folds == f
        clf = OneVsRestClassifier(LogisticRegression(C=1000, tol=1e-12, max_iter=100000))
        clf.fit(X[tr].astype(np.float64), Y[tr])
        want = np.asarray(clf.predict_proba(X[te].astype(np.float64))).argmax(1)
        z = res.decision[te]
        top2 = np.sort(z, 1)[:, -2:]
        assert (top2[:, 1] - top2[:, 0] > 1e-9).all()             # no near-tie decides a row
        got = z.argmax(1)
        assert np.array_equal(got, want), "fold %d: %d rows differ" % (f, (got != want).sum())
        tp += int(Y[te][np.arange(te.sum()), got].sum())
        assert abs(res.f1[f] - Y[te][np.arange(te.sum()), got].mean()) < 1e-12
    print("micro-F1 %.6f over %d rows, equal to converged sklearn" % (res.f1.mean(), n))


@pytest.mark.parametrize("multi", [False, True])
def test_micro_f1_near_the_reference_evaluator(multi):
    from gcc_b200.tasks.node_classification import NodeClassification
    if multi:
        X, Y = _data(1500, 64, 6, 9, noise=1.5, multi=True)
    else:
        X, Y = _data(1190, 64, 4, 8, noise=1.5)                    # usa_airport: 1190 nodes, 4 classes
    ref = object.__new__(NodeClassification)
    ref.seed = 0
    want = ref._evaluate(X.astype(np.float64), Y.astype(np.float32), 10)["Micro-F1"]
    got = float(lp.fit_probe(X, Y, lp.fold_ids(Y, 0)).f1.mean())
    print("%s: micro-F1 %.4f (GPU probe) vs %.4f (reference evaluator), gap %.4f"
          % ("multi-label" if multi else "usa_airport-shaped", got, want, got - want))
    assert abs(got - want) < 0.01


def test_weights_are_bit_identical_across_runs_and_batching():
    X, Y = _data(20000, 64, 3, 11)
    folds = lp.fold_ids(Y, 0)
    a = lp.fit_probe(X, Y, folds)
    b = lp.fit_probe(X, Y, folds)
    per_fold = lp.fit_probe(X, Y, folds, batch=3)                # one fold's problems per launch
    one = lp.fit_probe(X, Y, folds, batch=1)
    for r in (b, per_fold, one):
        assert np.array_equal(a.weights.view(np.uint64), r.weights.view(np.uint64))
        assert np.array_equal(a.decision.view(np.uint64), r.decision.view(np.uint64))
        assert np.array_equal(a.f1, r.f1)


def _run(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-s", "-m"] + args, cwd=str(cwd), env=env, capture_output=True, text=True)


def test_generate_rows_of_a_labelled_npz_end_to_end(tmp_path):
    from gcc_b200.datasets import synthetic
    from test_gpu_generate import _ckpt, _main
    g = synthetic.erdos_renyi(600, 3000, seed=4)
    deg = np.diff(g.indptr)
    y = (deg > np.median(deg)).astype(np.int64) + (deg > np.percentile(deg, 80))
    path = str(tmp_path / "mine.npz")
    np.savez(path, indptr=g.indptr, indices=g.indices, y=y)
    _main(_ckpt(tmp_path, "gin64"), path, 0)
    emb = str(tmp_path / "mine.npy")
    assert np.load(emb).shape == (600, 64)
    out = _run(["gcc_b200.tasks.linear_probe", "--emb-path", emb, "--dataset", path], tmp_path)
    assert out.returncode == 0, out.stderr
    print("linear_probe:", out.stdout.strip())
    assert out.stdout.startswith('{"Micro-F1": ')
    out = _run(["gcc_b200.tasks.node_classification", "--dataset", path, "--model", "from_numpy", "--hidden-size",
                "64", "--emb-path", emb], tmp_path)
    assert out.returncode == 0, out.stderr
    print("node_classification:", out.stdout.strip())
    assert out.stdout.startswith("{'Micro-F1': ")


def test_whole_graph_corpus_end_to_end(tmp_path):
    from gcc_b200.datasets import x2dgl
    from test_gpu_whole_graph_embed import _main
    from test_gpu_generate import _ckpt
    rng = np.random.RandomState(3)
    d = tmp_path / "edges"
    d.mkdir()
    files = []
    for i in range(40):
        n = int(rng.randint(20, 60))
        e = [(j, (j + 1) % n) for j in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(n * (1 + i % 2))]
        e = [(u, v) for u, v in e if u != v]
        p = d / ("g%02d.txt" % i)
        p.write_text("".join("%d %d\n" % uv for uv in e))
        files.append(str(p))
    corpus = str(tmp_path / "mine.bin")
    x2dgl.main(["--graph-dir", str(d), "--save-file", corpus, "--graph-files"] + files)
    rows = _main(_ckpt(tmp_path, "gin64"), corpus, B=8, whole_graphs=True).numpy()
    assert rows.shape == (40, 64)
    np.savez(str(tmp_path / "labels.npz"), graph_labels=np.arange(40) % 2)
    out = _run(["gcc_b200.tasks.linear_probe", "--emb-path", str(tmp_path / "mine.graphs.npy"), "--dataset",
                str(tmp_path / "labels.npz")], tmp_path)
    assert out.returncode == 0, out.stderr
    print("linear_probe (whole graphs):", out.stdout.strip())
    assert out.stdout.startswith('{"Micro-F1": ')


def test_nan_row_is_named_and_nonconvergence_is_reported():
    X, Y = _data(500, 8, 2, 13)
    folds = lp.fold_ids(Y, 0)
    Xb = X.copy()
    Xb[123, 4] = np.nan
    with pytest.raises(_lib.GccbError, match="row 123 holds a NaN"):
        lp.fit_probe(Xb, Y, folds)
    with pytest.raises(_lib.GccbError, match=r"fold \d+, class \d+ did not converge .* gradient norm"):
        lp.fit_probe(X, Y, folds, max_iter=1)
    with pytest.raises(ValueError, match="257"):
        lp.fit_probe(np.zeros((10, 257), np.float32), Y[:10], folds[:10])
    torch.cuda.synchronize()
