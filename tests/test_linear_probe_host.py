"""Host side of the linear probe (gcc_b200.tasks.linear_probe): label matrices, fold ids equal to the reference
evaluators' folds, the dataset readers, the finetune .npz path of tasks.node_classification, and the refusals of a
row count that differs from the label count and of a set that does not fit in device memory."""
import numpy as np
import pytest

from gcc_b200 import _lib
from gcc_b200.tasks import linear_probe as lp
from gcc_b200.tasks import node_classification as nc


def test_label_matrix_one_hot_and_multilabel():
    Y = lp.label_matrix(np.array([2, 0, 1, 2]))
    assert Y.dtype == np.uint8 and Y.shape == (4, 3)
    assert np.array_equal(Y.argmax(1), [2, 0, 1, 2]) and (Y.sum(1) == 1).all()
    M = np.array([[1, 0, 1], [0, 0, 1]], np.float32)
    assert np.array_equal(lp.label_matrix(M), M.astype(np.uint8))
    with pytest.raises(ValueError):
        lp.label_matrix(np.array([1, -1]))


@pytest.mark.parametrize("seed", [0, 3])
def test_fold_ids_are_the_reference_folds(seed):
    from sklearn.model_selection import StratifiedKFold
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 5, 300)
    Y = lp.label_matrix(y).astype(np.float32)
    fo = lp.fold_ids(Y, seed)
    # node evaluator: skf.split(np.zeros(n), argmax labels); graph evaluator: kf.split(x, y)
    node = StratifiedKFold(n_splits=10, shuffle=True, random_state=seed).split(np.zeros(300), Y.argmax(1).tolist())
    graph = StratifiedKFold(n_splits=10, shuffle=True, random_state=seed).split(rng.random((300, 4)), y)
    for f, ((_, a), (_, b)) in enumerate(zip(node, graph)):
        assert np.array_equal(np.nonzero(fo == f)[0], a) and np.array_equal(a, b)
    assert (fo >= 0).all()


def _npz(tmp_path, y, n=None):
    n = len(y) if n is None else n
    indptr = np.arange(n + 1, dtype=np.int64)
    indices = (np.arange(n, dtype=np.int32) + 1) % n
    path = str(tmp_path / "g.npz")
    np.savez(path, indptr=indptr, indices=indices, y=y)
    return path


def test_load_task_reads_the_finetune_npz_and_graph_labels(tmp_path):
    rng = np.random.default_rng(1)
    emb = rng.standard_normal((50, 8)).astype(np.float32)
    np.save(str(tmp_path / "e.npy"), emb)
    X, Y = lp.load_task(_npz(tmp_path, rng.integers(0, 3, 50)), str(tmp_path / "e.npy"))
    assert np.array_equal(X, emb) and Y.shape == (50, 3)
    multi = (rng.random((50, 4)) < 0.5).astype(np.int64)
    X, Y = lp.load_task(_npz(tmp_path, multi), str(tmp_path / "e.npy"))
    assert np.array_equal(Y, multi)
    np.savez(str(tmp_path / "gl.npz"), graph_labels=np.arange(50) % 2)
    X, Y = lp.load_task(str(tmp_path / "gl.npz"), str(tmp_path / "e.npy"))
    assert Y.shape == (50, 2) and np.array_equal(Y.argmax(1), np.arange(50) % 2)


def test_row_count_mismatch_names_both_counts(tmp_path):
    np.save(str(tmp_path / "e.npy"), np.zeros((49, 8), np.float32))
    with pytest.raises(ValueError, match="49 embedding rows for 50 label rows"):
        lp.load_task(_npz(tmp_path, np.arange(50) % 3), str(tmp_path / "e.npy"))
    np.savez(str(tmp_path / "gl.npz"), graph_labels=np.arange(48) % 2)
    with pytest.raises(ValueError, match="49 embedding rows for 48 graph labels"):
        lp.load_task(str(tmp_path / "gl.npz"), str(tmp_path / "e.npy"))
    with pytest.raises(ValueError, match="49 embedding rows for 50 label rows"):
        lp._check_shapes(49, 8, 3, 50, 49)
    with pytest.raises(ValueError, match="width 300"):
        lp._check_shapes(5, 300, 3, 5, 5)


def test_node_classification_reads_the_finetune_npz(tmp_path, capsys):
    rng = np.random.default_rng(2)
    y = rng.integers(0, 3, 200)
    emb = (np.eye(3)[y] * 2 + 0.3 * rng.standard_normal((200, 3))).astype(np.float32)
    np.save(str(tmp_path / "e.npy"), emb)
    path = _npz(tmp_path, y)
    ret = nc.main(["--dataset", path, "--model", "from_numpy", "--hidden-size", "3", "--emb-path",
                   str(tmp_path / "e.npy")])
    assert ret["Micro-F1"] > 0.9
    assert "Micro-F1" in capsys.readouterr().out
    multi = np.zeros((200, 3), np.int64)
    multi[np.arange(200), y] = 1
    multi[::4, (y[::4] + 1) % 3] = 1
    ret2 = nc.main(["--dataset", _npz(tmp_path, multi), "--model", "from_numpy", "--hidden-size", "3", "--emb-path",
                    str(tmp_path / "e.npy")])
    assert 0 < ret2["Micro-F1"] <= 1
    np.save(str(tmp_path / "short.npy"), emb[:150])
    with pytest.raises(ValueError, match="150 embedding rows for 200 label rows"):
        nc.main(["--dataset", path, "--model", "from_numpy", "--hidden-size", "3", "--emb-path",
                 str(tmp_path / "short.npy")])


def test_memory_refusal_names_the_sizes(monkeypatch):
    import torch
    lib = _lib.get()
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 30, 80 << 30))
    monkeypatch.setattr(torch.cuda, "memory_reserved", lambda *a: 0)
    monkeypatch.setattr(torch.cuda, "memory_allocated", lambda *a: 0)

    class Dev:
        def __init__(self, *a):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False
    monkeypatch.setattr(torch.cuda, "device", Dev)
    need = lp.probe_bytes(2_000_000, 64, 47)
    assert need > lib.gccb_probe_workspace(2_000_000, 64, 47, 10, 0) > 0
    with pytest.raises(_lib.GccbError, match=r"2000000 rows of width 64 with 47 classes x 10 folds need [\d.]+ GB"):
        lp.check_memory(2_000_000, 64, 47, dev=0)
    lp.check_memory(1000, 64, 4, dev=0)                          # a small set fits
