"""CPU: the eigensolver structure set (tests/eig_structures.py) is what it claims to be."""
import numpy as np
import pytest

import eig_structures as es
from oracle import posenc as opos


@pytest.fixture(scope="module")
def graphs():
    return es.structures()


def test_every_graph_is_a_symmetric_csr(graphs):
    for g in graphs:
        n, ip, ix = g["n"], g["indptr"], g["indices"]
        assert ip.dtype == np.int32 and ix.dtype == np.int32 and len(ip) == n + 1 and ip[0] == 0, g["name"]
        assert ip[-1] == len(ix) == g["m"] and np.all(np.diff(ip) >= 0), g["name"]
        assert len(ix) == 0 or (ix.min() >= 0 and ix.max() < n), g["name"]
        rows = np.repeat(np.arange(n), np.diff(ip))
        fwd = np.sort(rows.astype(np.int64) * n + ix)
        bwd = np.sort(ix.astype(np.int64) * n + rows)
        assert np.array_equal(fwd, bwd), g["name"]                      # symmetric as a multiset of entries
        for r in range(0, n, max(1, n // 16)):
            assert np.all(np.diff(ix[ip[r]:ip[r + 1]]) >= 0), g["name"]
        if g["family"] != "multi":
            assert len(np.unique(fwd)) == len(fwd) and not np.any(rows == ix), g["name"]


def test_multigraphs_have_parallel_edges_and_self_loops(graphs):
    for g in (g for g in graphs if g["family"] == "multi"):
        rows = np.repeat(np.arange(g["n"]), np.diff(g["indptr"]))
        key = rows.astype(np.int64) * g["n"] + g["indices"]
        assert len(np.unique(key)) < len(key) and np.any(rows == g["indices"]), g["name"]
        loops = key[rows == g["indices"]]
        _, cnt = np.unique(loops, return_counts=True)
        assert np.all(cnt % 2 == 0), g["name"]                         # a self loop enters its row twice


def test_sizes_reach_every_class(graphs):
    """eig_class restated: every size class under both dispatches, the class edges, k = -1 .. 3."""
    sizes = {g["n"] for g in graphs}
    for n in (1, 2, 3, 4, 5, 96, 97, 144, 145, 160, 161, 228, 229, 384, 385, 1536, 1537, 3584, 3585):
        assert n in sizes, n
    assert es.eig_class(96) == "dense<=96" and es.eig_class(97) == "chfsi<=160"
    assert es.eig_class(160) == "chfsi<=160" and es.eig_class(161) == "chfsi<=384"
    assert es.eig_class(384) == "chfsi<=384" and es.eig_class(385) == "chfsi<=1536"
    assert es.eig_class(1536) == "chfsi<=1536" and es.eig_class(1537) == "chfsi<=3584"
    assert es.eig_class(3584) == "chfsi<=3584" and es.eig_class(3585) == "chfsi<=L2"
    assert es.eig_class(144, "dense") == "dense<=144" and es.eig_class(145, "dense") == "dense<=228"
    assert es.eig_class(228, "dense") == "dense<=228" and es.eig_class(229, "dense") == "chfsi<=384"
    for solver in ("default", "dense"):
        got = {es.eig_class(g["n"], solver) for g in graphs}
        want = set(es.CLASS_ORDER) - ({"dense<=144", "dense<=228"} if solver == "default" else {"chfsi<=160"})
        assert got == want, (solver, got)
    fam = {}
    for g in graphs:
        fam.setdefault(g["family"], set()).add(es.eig_class(g["n"]))
    for f, cls in fam.items():
        if f not in ("hub_heavy", "er_sparse", "hub_mix"):
            assert "dense<=96" in cls and any(c.startswith("chfsi") for c in cls), (f, cls)
    for c in ("chfsi<=1536", "chfsi<=3584", "chfsi<=L2"):
        assert len({g["family"] for g in graphs if es.eig_class(g["n"]) == c}) >= 3, c
    assert sum(g["n"] > 1536 for g in graphs) <= 8                    # the float64 reference of these dominates


def test_ring_cut_falls_inside_a_double_eigenvalue(graphs):
    for g in (g for g in graphs if g["family"] == "ring" and g["n"] > 34):
        w = np.linalg.eigvalsh(opos.normalized_adjacency(g["indptr"], g["indices"], g["n"]).toarray())[::-1]
        assert abs(w[31] - w[32]) < 1e-12 and w[30] - w[31] > 1e-6, g["name"]        # lambda_32 = lambda_33


def test_whole_graph_structures(graphs):
    """Components with isolated vertices, more than 48 components (eigenvalue 1 more degenerate than the block) and
    an all-isolated graph above 96 vertices."""
    by = {g["name"]: g for g in graphs}
    for g in graphs:
        deg = np.diff(g["indptr"])
        if g["family"] == "components":
            assert np.any(deg == 0), g["name"]
        if g["family"] == "isolated":
            assert g["m"] == 0
    assert any(g["family"] == "isolated" and g["n"] > 96 for g in graphs)
    g = by["many_components_190_60"]
    w = np.linalg.eigvalsh(opos.normalized_adjacency(g["indptr"], g["indices"], g["n"]).toarray())
    assert np.sum(np.abs(w - 1) < 1e-9) == 60 > 48


def test_hub_heavy_slabs(graphs):
    """More than GCCB_CL_MAXHEAVY rows of degree > GCCB_CL_HEAVY in one slab of the 192-row and of the 448-row
    cluster class, so the kernel's hub-row list overflows there."""
    heavy = {es.eig_class(g["n"]): max(es.heavy_rows_per_slab(g)) for g in graphs if g["family"] == "hub_heavy"}
    assert heavy.get("chfsi<=1536", 0) > es.CL_MAXHEAVY and heavy.get("chfsi<=3584", 0) > es.CL_MAXHEAVY, heavy
    g = next(g for g in graphs if g["name"] == "hub_heavy_1536")
    assert es.slab_rows(g["n"]) == 192                                  # a full 192-row slab
