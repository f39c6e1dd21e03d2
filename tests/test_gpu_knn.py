"""GPU (H100): the cosine top-k of csrc/knn.cu (gcc_b200.tasks.knn) -- bit for bit against the numpy restatement
(tests/knn_oracle.py) on random, clustered and duplicate-heavy sets up to 5k x 50k at widths 32 .. 256 and on a
sampled 200k x 200k search; the same bits across candidate splits, query chunks and `--gpu 0 0`; scores within the
fp32 error bound of the float64 top-k; generate.py rows through the command line; Recall@20/40 against the
reference evaluator; error paths."""
import os
import types

import numpy as np
import pytest
import torch

import knn_oracle as oracle
from gcc_b200 import _lib
from gcc_b200.tasks import knn

pytestmark = pytest.mark.gpu


def _rows(kind, n, d, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.standard_normal((n, d)).astype(np.float32)
    if kind == "clustered":                                   # 50 tight clusters: many near-equal scores
        centres = rng.standard_normal((50, d))
        return (centres[rng.integers(0, 50, n)] + 1e-3 * rng.standard_normal((n, d))).astype(np.float32)
    base = rng.standard_normal((200, d)).astype(np.float32)  # duplicate-heavy: 200 distinct rows, exact ties
    return base[rng.integers(0, 200, n)]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _check_sampled(Q, C, ids, scores, k, sample, exclude=None):
    """Rows `sample` of the GPU result against the oracle, bit for bit."""
    ex = None if exclude is None else exclude[sample]
    want_ids, want_sc = oracle.topk(Q[sample], C, k, ex)
    np.testing.assert_array_equal(ids[sample], want_ids)
    assert np.array_equal(scores[sample].view(np.uint32), want_sc.view(np.uint32))


@pytest.mark.parametrize("kind,nq,nc,d,k", [("random", 5000, 50000, 32, 20), ("clustered", 4000, 30000, 64, 40),
                                            ("duplicates", 3000, 40000, 128, 128), ("random", 5000, 50000, 256, 20),
                                            ("duplicates", 700, 900, 130, 7)])
def test_matches_the_oracle_bit_for_bit(kind, nq, nc, d, k):
    Q = _rows(kind, nq, d, 1)
    C = _rows(kind, nc, d, 2)
    ids, sc = (t.cpu().numpy() for t in knn.topk_cosine(_dev(Q), _dev(C), k))
    rng = np.random.default_rng(0)
    sample = np.sort(rng.choice(nq, 32, replace=False))
    sample[-1] = nq - 1                                        # the last, partial query tile
    _check_sampled(Q, C, ids, sc, k, sample)


def test_bits_do_not_depend_on_splits_or_query_chunks():
    Q = _rows("duplicates", 3000, 64, 3)
    C = _rows("duplicates", 30000, 64, 4)
    q, c = _dev(Q), _dev(C)
    ex = torch.arange(3000, dtype=torch.int64, device="cuda")
    ref_ids, ref_sc = knn.topk_cosine(q, c, 40, exclude=ex)
    for kw in (dict(splits=1), dict(splits=3), dict(splits=17), dict(splits=128),
               dict(chunk_bytes=1 << 20), dict(chunk_bytes=1, splits=5)):
        ids, sc = knn.topk_cosine(q, c, 40, exclude=ex, **kw)
        assert torch.equal(ids, ref_ids), kw
        assert torch.equal(sc.view(torch.int32), ref_sc.view(torch.int32)), kw
    ids, sc = (t.cpu().numpy() for t in (ref_ids, ref_sc))
    _check_sampled(Q, C, ids, sc, 40, np.arange(0, 3000, 97), exclude=np.arange(3000))


def test_scores_lie_within_the_fp32_bound_of_the_float64_top_k():
    d, k = 64, 40
    Q = _rows("random", 2000, d, 5)
    C = _rows("random", 20000, d, 6)
    ids, sc = (t.cpu().numpy() for t in knn.topk_cosine(_dev(Q), _dev(C), k))
    q64 = Q / np.linalg.norm(Q.astype(np.float64), axis=1, keepdims=True)
    c64 = C / np.linalg.norm(C.astype(np.float64), axis=1, keepdims=True)
    tol = 4 * (d + 4) * 2.0 ** -24                           # normalisation of both rows plus a d-term fma chain
    for i in range(0, 2000, 50):
        cos = c64 @ q64[i]
        assert np.all(np.abs(sc[i] - cos[ids[i]]) <= tol)
        best = np.sort(cos)[::-1][:k]
        assert np.all(np.abs(np.sort(cos[ids[i]])[::-1] - best) <= 2 * tol)


def test_large_search_is_exact_on_sampled_queries():
    n, d, k = 200_000, 64, 20
    X = _rows("random", n, d, 7)
    x = _dev(X)
    ex = torch.arange(n, dtype=torch.int64, device="cuda")
    ids, sc = (t.cpu().numpy() for t in knn.topk_cosine(x, x, k, exclude=ex))
    sample = np.random.default_rng(1).choice(n, 12, replace=False)
    _check_sampled(X, X, ids, sc, k, sample, exclude=np.arange(n))


def test_recall_matches_the_reference_evaluator():
    from gcc_b200.tasks.similarity_search import SimilaritySearch
    rng = np.random.default_rng(9)
    n, d = 600, 32
    emb_1 = rng.standard_normal((n, d))
    perm = rng.permutation(n)
    emb_2 = emb_1[perm] + 2.0 * rng.standard_normal((n, d))   # row perm[j] of emb_1 is row j of emb_2
    inv = np.argsort(perm)
    # no near-ties: keep the names whose match scores at least 1e-4 away from every other candidate (leaving names
    # out only removes competitors), so that fp32 and float64 rank every match alike
    a = emb_1 / np.linalg.norm(emb_1, axis=1, keepdims=True)
    b = emb_2 / np.linalg.norm(emb_2, axis=1, keepdims=True)
    S = a @ b.T
    gap = np.abs(S - S[np.arange(n), inv][:, None])
    gap[np.arange(n), inv] = 1.0
    names = [i for i in range(n) if gap[i].min() > 1e-4]
    assert len(names) > n // 2
    dict_1 = {"v%d" % i: i for i in names}
    dict_2 = {"v%d" % i: int(inv[i]) for i in names}
    n = len(names)
    want = SimilaritySearch._evaluate(object.__new__(SimilaritySearch), emb_1.copy(), emb_2.copy(), dict_1, dict_2)
    keys = sorted(dict_1)
    reindex = [dict_2[key] for key in keys]
    q = _dev(emb_1[[dict_1[key] for key in keys]].astype(np.float32))
    c = _dev(emb_2[reindex].astype(np.float32))
    ids = knn.topk_cosine(q, c, 40)[0].cpu().numpy()
    truth = np.arange(n)[:, None]                            # key i's match is row i of the reindexed emb_2
    got = {"Recall @ %d" % k: float(np.mean((ids[:, :k] == truth).any(1))) for k in (20, 40)}
    assert 0.05 < got["Recall @ 20"] < 0.95                  # a search that is neither trivial nor hopeless
    assert got == pytest.approx(want, abs=0)


def _cli(tmp_path, emb, name, gpu, extra=()):
    argv = ["--emb-path", emb, "--k", "20", "--output", str(tmp_path / name)] + list(extra)
    if gpu is not None:
        argv += ["--gpu"] + [str(g) for g in gpu]
    knn.main(argv)
    return (np.load(str(tmp_path / name) + ".ids.npy"), np.load(str(tmp_path / name) + ".scores.npy"))


def test_generate_rows_through_the_command_line(tmp_path):
    import argparse
    import generate
    from gcc_b200.models import GraphEncoder
    opt = argparse.Namespace(positional_embedding_size=32, max_node_freq=8, max_edge_freq=8, max_degree=512,
                             freq_embedding_size=16, degree_embedding_size=16, hidden_size=64, num_layer=5,
                             set2set_iter=6, set2set_lstm_layer=3, model="gin", norm=True, rw_hops=64,
                             subgraph_size=128, restart_prob=0.8, seed=5, model_folder=str(tmp_path))
    torch.manual_seed(1)
    model = GraphEncoder(degree_input=True, **{kw: getattr(opt, a) for kw, a in generate.ENCODER_KWARGS.items()})
    ckpt = str(tmp_path / "ckpt.pth")
    torch.save({"opt": opt, "model": model.state_dict(), "epoch": 1}, ckpt)
    generate.main(types.SimpleNamespace(load_path=ckpt, dataset="synthetic-er", graph_nodes=3000, graph_edges=15000,
                                        batch_size=256, gpu=None))
    emb = str(tmp_path / "synthetic-er.npy")
    X = np.load(emb)
    ids, sc = _cli(tmp_path, emb, "one", None)
    x = _dev(X)
    want_ids, want_sc = knn.topk_cosine(x, x, 20, exclude=torch.arange(len(X), device="cuda"))
    np.testing.assert_array_equal(ids, want_ids.cpu().numpy())
    assert np.array_equal(sc.view(np.uint32), want_sc.cpu().numpy().view(np.uint32))
    assert not (ids == np.arange(len(X))[:, None]).any()     # the query's own row is left out
    ids2, sc2 = _cli(tmp_path, emb, "two", [0, 0])
    assert open(str(tmp_path / "one.ids.npy"), "rb").read() == open(str(tmp_path / "two.ids.npy"), "rb").read()
    assert open(str(tmp_path / "one.scores.npy"), "rb").read() == open(str(tmp_path / "two.scores.npy"), "rb").read()
    # --nodes and --candidates: subset queries against another file
    np.save(tmp_path / "ids.npy", np.array([5, 2999, 5, 17]))
    np.save(tmp_path / "cands.npy", X[::3])
    ids3, sc3 = _cli(tmp_path, emb, "three", [0, 0], ["--nodes", str(tmp_path / "ids.npy"), "--candidates",
                                                        str(tmp_path / "cands.npy")])
    w_ids, w_sc = knn.topk_cosine(x[[5, 2999, 5, 17]], _dev(X[::3]), 20)
    np.testing.assert_array_equal(ids3, w_ids.cpu().numpy())
    assert np.array_equal(sc3, w_sc.cpu().numpy())


def test_error_paths(tmp_path):
    x = _dev(_rows("random", 100, 16, 11))
    bad = x.clone()
    bad[37, 3] = float("nan")
    with pytest.raises(_lib.GccbError, match="candidates row 37"):
        knn.topk_cosine(x, bad, 5)
    bad[37, 3] = float("inf")
    with pytest.raises(_lib.GccbError, match="queries row 37"):
        knn.topk_cosine(bad, x, 5)
    with pytest.raises(ValueError, match="admissible"):
        knn.topk_cosine(x, x, 100, exclude=torch.arange(100, device="cuda"))
    with pytest.raises(ValueError):
        knn.topk_cosine(x, x, 129)
    with pytest.raises(ValueError):
        knn.topk_cosine(x, x[:, :8].contiguous(), 5)
    with pytest.raises(_lib.GccbError):
        knn.topk_cosine(x.cpu(), x, 5)
    # a failing shard: the other is terminated and no partial files stay
    X = _rows("random", 100, 16, 11)
    X[90, 0] = np.nan
    np.save(tmp_path / "a.npy", X)
    with pytest.raises(RuntimeError, match="NaN"):
        _cli(tmp_path, str(tmp_path / "a.npy"), "bad", [0, 0])
    assert not os.path.exists(str(tmp_path / "bad.ids.npy")) and not os.path.exists(str(tmp_path / "bad.scores.npy"))
