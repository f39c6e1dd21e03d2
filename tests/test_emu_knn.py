"""The cosine top-k of csrc/knn.cu under the CPU emulator, bit for bit against the numpy restatement
(tests/knn_oracle.py): widths 1 .. 130, k from 1 to every candidate, several candidate splits, ties, zero rows, ±0
scores, exclusion, the non-finite flag, refused arguments and queues that overflow several times in one tile."""
import numpy as np
import pytest

import knn_oracle as oracle
from emu_util import lib, ptr
from gcc_b200 import _capi


def emu_knn(Q, Cd, k, exclude=None, splits=0, reuse_from=None):
    """gccb_knn on host buffers -> (status, ids, scores, flags, workspace).  reuse_from: the workspace of an earlier
    call, which holds the normalised candidates (the call passes cands = NULL)."""
    L = lib()
    Q = np.ascontiguousarray(Q, np.float32)
    Cd = np.ascontiguousarray(Cd, np.float32)
    nq, d = Q.shape
    nc = Cd.shape[0]
    ws = reuse_from
    if ws is None:
        ws = np.zeros(L.gccb_knn_workspace(nq, nc, d, k, splits) + 32, np.uint8)
    wsv = ws[(-ws.ctypes.data) % 16:]                       # 16-byte aligned, at the same place for a reused buffer
    ids = np.full((nq, k), -7, np.int64)
    sc = np.full((nq, k), np.nan, np.float32)
    flags = np.zeros(1, np.int32)
    ex = None if exclude is None else np.ascontiguousarray(exclude, np.int64)
    rc = L.gccb_knn(ptr(Q), nq, None if reuse_from is not None else ptr(Cd), nc, d, k, ptr(ex), splits, ptr(ids),
                    ptr(sc), ptr(flags), ptr(wsv), wsv.nbytes, None)
    return rc, ids, sc, int(flags[0]), ws


def check(Q, Cd, k, exclude=None, splits=0):
    rc, ids, sc, flags, _ = emu_knn(Q, Cd, k, exclude, splits)
    assert rc == 0, lib().gccb_last_error()
    assert flags == 0
    want_ids, want_sc = oracle.topk(Q, Cd, k, exclude)
    np.testing.assert_array_equal(ids, want_ids)
    assert np.array_equal(sc.view(np.uint32), want_sc.view(np.uint32))
    return ids, sc


@pytest.mark.parametrize("d", [1, 3, 4, 64, 130])
@pytest.mark.parametrize("splits", [1, 2, 7])
def test_random_rows_match_the_oracle_bit_for_bit(d, splits):
    rng = np.random.default_rng(d * 10 + splits)
    Q = rng.standard_normal((70, d)).astype(np.float32)
    Cd = rng.standard_normal((300, d)).astype(np.float32)
    check(Q, Cd, 40, splits=splits)


@pytest.mark.parametrize("k", [1, 40, 128, 300])
def test_every_k_up_to_all_candidates(k):
    rng = np.random.default_rng(k)
    Q = rng.standard_normal((9, 16)).astype(np.float32)
    Cd = rng.standard_normal((300, 16)).astype(np.float32)
    if k > 128:
        rc, *_ = emu_knn(Q, Cd, k)
        assert rc == _capi.GCCB_ERR_BADARG                   # k is at most 128
        Cd = Cd[:100]
        k = 100                                               # k = nc: every candidate, in order
    for s in (1, 2, 7):
        check(Q, Cd, k, splits=s)


def test_all_equal_rows_rank_by_index():
    Q = np.ones((5, 8), np.float32)
    Cd = np.tile(np.arange(1, 9, dtype=np.float32), (260, 1))
    for s in (1, 2, 7):
        ids, _ = check(Q, Cd, 40, splits=s)
        assert np.array_equal(ids, np.tile(np.arange(40), (5, 1)))


def test_duplicated_rows_zero_rows_and_signed_zero_scores():
    rng = np.random.default_rng(3)
    base = rng.standard_normal((20, 12)).astype(np.float32)
    Cd = base[rng.integers(0, 20, 400)]                      # every row repeated ~20 times
    Cd[::7] = 0.0                                            # zero rows score +0 against everything
    Q = np.concatenate([base[:6], np.zeros((2, 12), np.float32)])
    Q[6, :] = 0.0
    # rows orthogonal to a query: products of opposite sign that cancel to ±0
    Q[7, :2] = (1.0, 1.0)
    Cd[3, :] = 0.0
    Cd[3, :2] = (1.0, -1.0)
    Cd[5, :] = 0.0
    Cd[5, :2] = (-1.0, 1.0)
    for s in (1, 2, 7):
        ids, sc = check(Q, Cd, 128, splits=s)
    assert np.all(sc[6] == 0) and not np.signbit(sc[6]).any()        # zero query: every score +0
    assert np.array_equal(ids[6], np.arange(128))


def test_exclusion_leaves_the_given_id_out():
    rng = np.random.default_rng(5)
    X = rng.standard_normal((150, 6)).astype(np.float32)
    ex = np.arange(40, dtype=np.int64)
    ex[3] = -1                                               # no exclusion for this query
    ex[4] = 10_000                                           # outside the candidates: nothing excluded
    for s in (1, 2, 7):
        ids, _ = check(X[:40], X, 20, exclude=ex, splits=s)
    assert ids[0, 0] != 0 and ids[3, 0] == 3 and ids[4, 0] == 4
    for i in range(40):
        if i not in (3, 4):
            assert i not in ids[i]
    rc, *_ = emu_knn(X[:40], X[:100], 100, exclude=ex)
    assert rc == _capi.GCCB_ERR_BADARG                       # k > nc - 1 admissible candidates
    assert b"admissible" in lib().gccb_last_error()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_rows_raise_the_flag(bad):
    rng = np.random.default_rng(6)
    Q = rng.standard_normal((4, 5)).astype(np.float32)
    Cd = rng.standard_normal((50, 5)).astype(np.float32)
    Cd[17, 2] = bad
    assert emu_knn(Q, Cd, 3)[3] & _capi.FLAG_NONFINITE
    Cd[17, 2] = 0
    Q[1, 4] = bad
    assert emu_knn(Q, Cd, 3)[3] & _capi.FLAG_NONFINITE
    Q[1, 4] = 0
    assert emu_knn(Q, Cd, 3)[3] == 0
    Q[1, 4] = bad
    assert np.array_equal(oracle.normalize(Q)[1], np.arange(4) == 1)


def test_refused_arguments():
    L = lib()
    Q = np.ones((2, 4), np.float32)
    assert emu_knn(Q, Q, 3)[0] == _capi.GCCB_ERR_BADARG                   # k > nc
    assert emu_knn(np.ones((2, 513), np.float32), np.ones((3, 513), np.float32), 1)[0] == _capi.GCCB_ERR_BADARG
    assert L.gccb_knn_workspace(2, 2, 0, 1, 0) == 0
    assert L.gccb_knn_workspace(2, 2, 4, 129, 0) == 0
    assert L.gccb_knn_workspace(2, 2, 4, 1, 129) == 0
    ids = np.zeros(2, np.int64)
    sc = np.zeros(2, np.float32)
    fl = np.zeros(1, np.int32)
    ws = np.zeros(64, np.uint8)                                              # too small
    rc = L.gccb_knn(ptr(Q), 2, ptr(Q), 2, 4, 1, None, 0, ptr(ids), ptr(sc), ptr(fl), ptr(ws[(-ws.ctypes.data) % 16:]),
                    16, None)
    assert rc == _capi.GCCB_ERR_CAPACITY


def test_queue_overflows_several_times_in_one_tile():
    # candidates in ascending score order: every one beats the current k-th, so a 128-candidate tile pushes 128 keys
    # per query through a 32-key queue (k = 1: four merges in the tile), and through a 64-key queue at k = 40
    d = 4
    t = np.linspace(0.0, 1.2, 1000, dtype=np.float32)
    Cd = np.stack([np.cos(t), np.sin(t), np.zeros_like(t), np.zeros_like(t)], 1).astype(np.float32)
    # scores against (0, 1) are sin(t): they ascend with the index, so every tile overflows its queues again
    Q = np.tile(np.array([[0.0, 1.0, 0.0, 0.0]], np.float32), (3, 1))
    for k in (1, 40):
        for s in (1, 2):
            check(Q, Cd, k, splits=s)


def test_reused_candidates_and_query_chunks_give_the_same_bits():
    rng = np.random.default_rng(8)
    Q = rng.standard_normal((150, 20)).astype(np.float32)
    Cd = rng.standard_normal((200, 20)).astype(np.float32)
    rc, ids, sc, _, ws = emu_knn(Q, Cd, 10, splits=2)
    assert rc == 0
    # the second chunk reads the candidates the first call normalised into the workspace (cands = NULL)
    rc, ids2, sc2, _, _ = emu_knn(Q[70:], Cd, 10, splits=3, reuse_from=ws)
    assert rc == 0
    np.testing.assert_array_equal(ids2, ids[70:])
    assert np.array_equal(sc2.view(np.uint32), sc[70:].view(np.uint32))
