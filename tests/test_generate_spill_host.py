"""Host-only planning of the re-run of an overflowed batch (gcc_b200.embed.spill_groups) and generate.py's line about
it: groups are consecutive, cover every ego-net pair once and fit both views' capacities; a pair too large for the
default capacity is alone, on buffers of its size; lower-bound counts are measured again, never used as sizes."""
import numpy as np
import pytest

import generate
from gcc_b200.embed import spill_groups

NODE_CAP, EDGE_CAP = 1000, 16000


def _check_cover(groups, sizes, node_cap, edge_cap):
    lo = 0
    for g_lo, g_hi, n_cap, e_cap in groups:
        assert g_lo == lo and g_hi > g_lo                      # consecutive, in order, none empty
        lo = g_hi
        part = sizes[g_lo:g_hi]
        if g_hi - g_lo == 1 and ((part[0, [0, 2]] > node_cap).any() or (part[0, [1, 3]] > edge_cap).any()):
            assert n_cap >= part[0, [0, 2]].max() and e_cap >= part[0, [1, 3]].max()
            continue
        assert (n_cap, e_cap) == (node_cap, edge_cap)
        tot = part.sum(axis=0)
        assert tot[0] <= n_cap and tot[2] <= n_cap               # the q and k views: separate limits
        assert tot[1] <= e_cap and tot[3] <= e_cap
    assert lo == len(sizes)


def _random_sizes(rng, b, big=0.0):
    n = rng.randint(2, 400, size=(b, 2))
    m = n * rng.randint(1, 30, size=(b, 2))
    sizes = np.stack([n[:, 0], m[:, 0], n[:, 1], m[:, 1]], axis=1).astype(np.int64)
    huge = rng.rand(b) < big
    sizes[huge, 0] *= 4
    sizes[huge, 3] *= 40
    return sizes


@pytest.mark.parametrize("seed,b,big", [(0, 64, 0.0), (1, 256, 0.0), (2, 256, 0.05), (3, 17, 0.3), (4, 1, 1.0)])
def test_groups_are_consecutive_cover_every_pair_once_and_fit_both_views(seed, b, big):
    sizes = _random_sizes(np.random.RandomState(seed), b, big)
    groups, remeasure = spill_groups(sizes, np.ones(b, bool), NODE_CAP, EDGE_CAP)
    assert remeasure == []
    _check_cover(groups, sizes, NODE_CAP, EDGE_CAP)


def test_groups_are_greedy_and_views_have_separate_limits():
    # q views fill node_cap after two pairs; k views fill edge_cap after three
    sizes = np.array([[500, 10, 1, 6000]] * 2 + [[1, 10, 1, 6000]] * 3, dtype=np.int64)
    groups, _ = spill_groups(sizes, np.ones(5, bool), NODE_CAP, EDGE_CAP)
    assert groups == [(0, 2, NODE_CAP, EDGE_CAP), (2, 4, NODE_CAP, EDGE_CAP), (4, 5, NODE_CAP, EDGE_CAP)]
    # a pair exactly at the capacity fits on its own buffers of the default size
    groups, _ = spill_groups(np.array([[NODE_CAP, EDGE_CAP, NODE_CAP, EDGE_CAP]]), [True], NODE_CAP, EDGE_CAP)
    assert groups == [(0, 1, NODE_CAP, EDGE_CAP)]


def test_a_pair_above_the_capacity_is_alone_on_buffers_of_its_size():
    sizes = np.array([[10, 20, 10, 20],
                      [3000, 40000, 2900, 41000],       # both vertices and edges above the default
                      [10, 20, 10, 20],
                      [20, 100, 30, 90000],             # edges of the k view alone
                      [1001, 5, 4, 5]], dtype=np.int64)  # vertices of the q view alone
    groups, remeasure = spill_groups(sizes, np.ones(5, bool), NODE_CAP, EDGE_CAP)
    assert remeasure == []
    assert groups == [(0, 1, NODE_CAP, EDGE_CAP), (1, 2, 3000, 41000), (2, 3, NODE_CAP, EDGE_CAP),
                      (3, 4, 30, 90000), (4, 5, 1001, 5)]
    _check_cover(groups, sizes, NODE_CAP, EDGE_CAP)


def test_lower_bound_counts_are_measured_again_not_used_as_sizes():
    sizes = np.array([[10, 20, 10, 20], [40000, 39999, 40000, 39999], [10, 20, 10, 20], [5, 4, 5, 8]], np.int64)
    exact = np.array([True, False, True, False])
    groups, remeasure = spill_groups(sizes, exact, NODE_CAP, EDGE_CAP)
    assert groups is None and remeasure == [1, 3]
    # once measured, the exact counts size the pair
    sizes[1] = [40000, 2_000_000, 39000, 1_900_000]
    sizes[3] = [5, 12, 5, 8]
    groups, remeasure = spill_groups(sizes, np.ones(4, bool), NODE_CAP, EDGE_CAP)
    assert remeasure == [] and groups == [(0, 1, NODE_CAP, EDGE_CAP), (1, 2, 40000, 2_000_000),
                                          (2, 4, NODE_CAP, EDGE_CAP)]


def test_generate_states_the_batches_it_replanned():
    assert generate.replan_line([(0, (0, 0))], 12) == "re-planned 0 of 12 batches: every batch fit the default capacity"
    line = generate.replan_line([(2, (3000, 41000)), (0, (0, 0)), (1, (5000, 20000))], 30)
    assert line.startswith("re-planned 3 of 30 batches")
    assert line.endswith("largest ego-net met: 5000 vertices, 20000 edges")
