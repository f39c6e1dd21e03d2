#!/usr/bin/env python
"""Generate tests/golden/baselines_golden.npz by executing the REAL reference embedders from a checkout of THUDM/GCC
(read-only): gcc/models/emb/prone.py (ProNE) and gcc/models/emb/_graphwave (GraphWave).

Stand-ins, everything else that runs is the reference's own code on the current scipy / networkx / sklearn:
  - matplotlib, matplotlib.pyplot, seaborn: empty modules (only plotting helpers use them);
  - scipy.sum: `sum` over the list of sparse terms (the alias left scipy);
  - `.A` on scipy sparse matrices: `.toarray()` (removed in scipy 1.14);
  - gcc.models.emb: a bare package, as in make_golden_tasks.py, so that its __init__ (which loads every embedder
    and from_numpy) is not executed.

Graphs, each built the way the reference task builds it (nx.Graph for node classification, nx.MultiGraph for
similarity search), with its vertices added in ascending id order first so that row r is the r-th smallest id:
  - usa / hindex (nx.Graph) and kdd / icdm (nx.MultiGraph): the edge lists of tasks_golden.npz;
  - hub (nx.Graph, 181 vertices): a hub with a self loop and 30 pendant paths of 6, some paths cross-linked;
  - split (nx.MultiGraph, 160 vertices): two random components of 100 and 60 vertices, every 5th pair repeated.

Stored per graph g: g_edge_index, g_multi, g_n, g_dim (ProNE's dimension: 16 on the tiny graphs, 64 otherwise),
g_taus and g_cheb (GraphWave's scales and Chebyshev coefficients), g_chi (GraphWave(64), float32), g_F_row /
g_F_col / g_F_val (ProNE's F), g_a (the tSVD features _chebyshev_gaussian receives, randomized_svd with
random_state=0, rounded to float32 before the propagation runs on them), g_mm (the matrix it hands to the dense SVD)
and g_emb (its output).  Also bessel = iv(0..4, 0.5).

Run:  GCC_REFERENCE=<checkout of THUDM/GCC> python tests/golden/make_golden_baselines.py [output.npz]
"""
import os
import sys
import types

import networkx as nx
import numpy as np
import scipy
import scipy.sparse as sp
from scipy.special import iv

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("GCC_REFERENCE")
if not REF or not os.path.isdir(REF):
    raise SystemExit("set GCC_REFERENCE to a checkout of THUDM/GCC")

mpl = types.ModuleType("matplotlib")
mpl.pyplot = types.ModuleType("matplotlib.pyplot")
sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": mpl.pyplot, "seaborn": types.ModuleType("seaborn")})
scipy.sum = lambda xs: sum(xs[1:], xs[0])
for cls in (sp.csr_matrix, sp.csc_matrix, sp.coo_matrix, sp.csr_array, sp.csc_array, sp.coo_array):
    cls.A = property(lambda s: s.toarray())
for name, path in (("gcc", "gcc"), ("gcc.models", "gcc/models"), ("gcc.models.emb", "gcc/models/emb")):
    m = types.ModuleType(name)
    m.__path__ = [os.path.join(REF, path)]
    sys.modules[name] = m

import gcc.models.emb.prone as ref_prone  # noqa: E402
from gcc.models.emb._graphwave.graphwave import compute_cheb_coeff_basis, graphwave_alg  # noqa: E402

_randomized_svd = ref_prone.randomized_svd
# prone.py passes random_state=None explicitly, so the seed has to replace that keyword, not default it
ref_prone.randomized_svd = lambda *args, **kwargs: _randomized_svd(*args, **dict(kwargs, random_state=0))


def _hub(rng):
    pairs = [(0, 0)]
    for p in range(30):
        base = 1 + 6 * p
        pairs.append((0, base))
        pairs += [(base + i, base + i + 1) for i in range(5)]
        if p % 4 == 0:
            pairs.append((base + 5, 1 + 6 * ((p + 7) % 30) + 2))
    return np.array(pairs, np.int64).T


def _split(rng):
    pairs = []
    for lo, n in ((0, 100), (100, 60)):
        pairs += [(lo + i, lo + (i + 1) % n) for i in range(n)]
        for _ in range(2 * n):
            a, b = rng.randint(0, n, 2)
            if a != b:
                pairs.append((lo + a, lo + b))
    pairs += pairs[::5]
    return np.array(pairs, np.int64).T


def _nx_graph(edge_index, multi):
    G = nx.MultiGraph() if multi else nx.Graph()
    G.add_nodes_from(np.unique(edge_index).tolist())
    G.add_edges_from(edge_index.T.tolist())
    return G


def main():
    rng = np.random.RandomState(20240601)
    t = np.load(os.path.join(HERE, "tasks_golden.npz"))
    graphs = [("usa", t["usa_edge_index"], False, 16), ("hindex", t["hindex_edge_index"], False, 16),
              ("kdd", t["ss0_edge_index"], True, 16), ("icdm", t["ss1_edge_index"], True, 16),
              ("hub", _hub(rng), False, 64), ("split", _split(rng), True, 64)]
    out = {"names": np.array([g[0] for g in graphs]), "bessel": np.array([iv(i, 0.5) for i in range(5)])}
    for name, ei, multi, dim in graphs:
        G = _nx_graph(ei, multi)
        n = G.number_of_nodes()
        out[name + "_edge_index"], out[name + "_multi"], out[name + "_n"] = ei, np.bool_(multi), np.int64(n)
        # GraphWave(64).train(G) is graphwave_alg(G, linspace(0, 100, 64 // 4)); called directly for its scales too
        chi, _, taus = graphwave_alg(G, np.linspace(0, 100, 16))
        out[name + "_taus"] = np.asarray(taus)
        out[name + "_cheb"] = np.array([compute_cheb_coeff_basis(tau, 30) for tau in taus])
        out[name + "_chi"] = np.asarray(chi, np.float32)

        model = ref_prone.ProNE(dim)
        model.num_node = n
        model.matrix0 = sp.csr_matrix(nx.adjacency_matrix(G))
        captured = {}
        rand = model._get_embedding_rand

        def get_rand(F):
            captured["F"] = sp.coo_matrix(F)
            return rand(F)

        model._get_embedding_rand = get_rand
        a = model._pre_factorization(model.matrix0, model.matrix0)
        a = a.astype(np.float32).astype(np.float64)
        dense = model._get_embedding_dense

        def get_dense(mm, d):
            captured["mm"] = np.array(mm, copy=True)
            return dense(mm, d)

        model._get_embedding_dense = get_dense
        emb = model._chebyshev_gaussian(model.matrix0, a, model.step, model.mu, model.theta)
        F = captured["F"]
        out.update({name + "_dim": np.int64(dim), name + "_F_row": F.row.astype(np.int32),
                    name + "_F_col": F.col.astype(np.int32), name + "_F_val": F.data,
                    name + "_a": a.astype(np.float32), name + "_mm": captured["mm"], name + "_emb": emb})
        print(name, "n", n, "chi", out[name + "_chi"].shape, "emb", emb.shape)
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "baselines_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d bytes" % os.path.getsize(path))


if __name__ == "__main__":
    main()
