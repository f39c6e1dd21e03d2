"""Host-only pieces of the similarity search: the oracle's fp32 fma against exact rational arithmetic (including
half-way cases that a float64 sum rounds the wrong way), and the command line's parsing, query rows, shard split and
output layout."""
from fractions import Fraction

import numpy as np
import pytest

import knn_oracle as oracle
from gcc_b200.tasks import knn

F32 = np.float32


def exact_fma(a, b, c):
    """fp32(a*b + c) rounded once to nearest even, from exact rationals."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(x))                                   # float64 of x may itself be rounded: fix below
    lo = r if Fraction(float(r)) <= x else np.nextafter(r, F32(-np.inf))
    hi = np.nextafter(lo, F32(np.inf))
    dl, dh = x - Fraction(float(lo)), Fraction(float(hi)) - x
    if dl < dh:
        return lo
    if dh < dl:
        return hi
    return lo if (lo.view(np.uint32) & 1) == 0 else hi


def test_fma_half_way_cases_round_once():
    # a*b = 2^-24 (1 + 2^-30): exact sum 1 + 2^-24 + 2^-54 lies just above the half-way point 1 + 2^-24; the float64
    # sum drops the 2^-54 and lands on it, and ties-to-even would give 1.0
    a, b, c = F32(2.0 ** -24 * (1 + 2.0 ** -10)), F32(1 - 2.0 ** -10 + 2.0 ** -20), F32(1.0)
    assert oracle.fma32(a, b, c) == F32(1 + 2.0 ** -23) == exact_fma(a, b, c)
    assert F32(np.float64(a) * np.float64(b) + np.float64(c)) == F32(1.0)       # the naive double rounding
    # a*b = 2^-24 (1 - 2^-30) below the half-way point 1 + 3 * 2^-24 of an odd c: ties-to-even would round up
    a, b, c = F32(2.0 ** -24 * (1 + 2.0 ** -15)), F32(1 - 2.0 ** -15), F32(1 + 2.0 ** -23)
    assert oracle.fma32(a, b, c) == c == exact_fma(a, b, c)
    assert F32(np.float64(a) * np.float64(b) + np.float64(c)) != c
    # negative mirror images
    assert oracle.fma32(-a, b, -c) == -c


def test_fma_matches_exact_rounding_on_random_and_signed_zero_cases():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(3000) * np.exp2(rng.integers(-30, 30, 3000))).astype(F32)
    b = (rng.standard_normal(3000) * np.exp2(rng.integers(-30, 30, 3000))).astype(F32)
    c = (rng.standard_normal(3000) * np.exp2(rng.integers(-60, 30, 3000))).astype(F32)
    c[::5] = -(a[::5].astype(np.float64) * b[::5]).astype(F32)                  # near-cancellation
    got = oracle.fma32(a, b, c)
    want = np.array([exact_fma(x, y, z) for x, y, z in zip(a, b, c)], F32)
    assert np.array_equal(got, want)
    # signs of zero: +0 + (-0 product) = +0; a tiny negative sum rounds to -0
    assert not np.signbit(oracle.fma32(F32(-1.0), F32(0.0), F32(0.0)))
    tiny = oracle.fma32(F32(-2.0 ** -80), F32(2.0 ** -80), F32(0.0))
    assert tiny == 0 and np.signbit(tiny)


def test_oracle_order_is_score_descending_then_index():
    Q = np.array([[1.0, 0.0]], F32)
    Cd = np.array([[0.0, 1.0], [1.0, 0.0], [2.0, 0.0], [-1.0, 0.0], [0.0, 0.0], [3.0, 0.0]], F32)
    ids, sc = oracle.topk(Q, Cd, 6)
    assert ids.tolist() == [[1, 2, 5, 0, 4, 3]]
    assert sc.tolist() == [[1.0, 1.0, 1.0, 0.0, 0.0, -1.0]]
    ids, _ = oracle.topk(Q, Cd, 3, exclude=np.array([2]))
    assert ids.tolist() == [[1, 5, 0]]


def test_command_line_parsing_and_query_rows(tmp_path):
    A = np.zeros((50, 8), F32)
    np.save(tmp_path / "a.npy", A)
    np.save(tmp_path / "b.npy", np.zeros((30, 8), F32))
    np.save(tmp_path / "c.npy", np.zeros((30, 7), F32))
    (tmp_path / "ids.txt").write_text("4 9\n4\n")
    base = ["--emb-path", str(tmp_path / "a.npy"), "--output", str(tmp_path / "out")]
    args = knn.parse_args(base)
    assert args.k == 20 and args.gpu is None and args.candidates is None and args.nodes is None
    ids, nc, d = knn.query_rows(args)
    assert np.array_equal(ids, np.arange(50)) and nc == 50 and d == 8
    args = knn.parse_args(base + ["--candidates", str(tmp_path / "b.npy"), "--nodes", str(tmp_path / "ids.txt"),
                                  "--k", "30", "--gpu", "0", "0"])
    ids, nc, d = knn.query_rows(args)
    assert ids.tolist() == [4, 9, 4] and nc == 30 and args.gpu == [0, 0]
    with pytest.raises(SystemExit):                           # within A, 49 admissible candidates
        knn.query_rows(knn.parse_args(base + ["--k", "50"]))
    with pytest.raises(SystemExit):
        knn.query_rows(knn.parse_args(base + ["--k", "129", "--candidates", str(tmp_path / "b.npy")]))
    with pytest.raises(SystemExit):                           # widths differ
        knn.query_rows(knn.parse_args(base + ["--candidates", str(tmp_path / "c.npy")]))
    (tmp_path / "bad.txt").write_text("50\n")
    with pytest.raises(SystemExit):
        knn.query_rows(knn.parse_args(base + ["--nodes", str(tmp_path / "bad.txt")]))


@pytest.mark.parametrize("n,workers", [(1, 1), (10, 3), (7, 7), (3, 5)])
def test_query_shards_are_contiguous_and_cover_every_query_once(n, workers):
    import generate
    shards = generate.split_shards(n, 1, workers)
    covered = np.concatenate([np.arange(lo, hi) for lo, hi in shards])
    assert np.array_equal(covered, np.arange(n))
    sizes = [hi - lo for lo, hi in shards]
    assert max(sizes) - min(sizes) <= 1


def test_output_layout(tmp_path, monkeypatch):
    """main() writes PREFIX.ids.npy (int64) and PREFIX.scores.npy (float32), [queries, k], row i = query i; a failing
    search leaves no files behind."""
    np.save(tmp_path / "a.npy", np.zeros((12, 4), F32))
    (tmp_path / "ids.txt").write_text("3 1 3\n")

    def fake_search(emb_path, cand_path, query_ids, k, gpu, ids_out, scores_out):
        ids_out[:] = np.asarray(query_ids)[:, None] * 100 + np.arange(k)
        scores_out[:] = np.arange(k, dtype=F32)[None, :]

    monkeypatch.setattr(knn, "search_rows", fake_search)
    prefix = str(tmp_path / "out")
    paths = knn.main(["--emb-path", str(tmp_path / "a.npy"), "--nodes", str(tmp_path / "ids.txt"), "--k", "5",
                      "--output", prefix])
    assert paths == [prefix + ".ids.npy", prefix + ".scores.npy"]
    ids, sc = np.load(paths[0]), np.load(paths[1])
    assert ids.dtype == np.int64 and sc.dtype == np.float32 and ids.shape == sc.shape == (3, 5)
    assert ids[:, 0].tolist() == [300, 100, 300]

    def failing(*a):
        raise RuntimeError("boom")

    monkeypatch.setattr(knn, "search_rows", failing)
    prefix2 = str(tmp_path / "fail")
    with pytest.raises(RuntimeError):
        knn.main(["--emb-path", str(tmp_path / "a.npy"), "--k", "5", "--output", prefix2])
    assert not (tmp_path / "fail.ids.npy").exists() and not (tmp_path / "fail.scores.npy").exists()
