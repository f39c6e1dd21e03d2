"""Seeded, numpy-only generator of local-id CSR graphs for the eigensolver tests (gcc_b200/csrc/posenc.cu).

Every graph is a dict(name, family, n, m, indptr, indices, subv) with int32 arrays, rows sorted, every edge stored in
both directions; multigraphs keep their parallel edges and enter a self loop twice into its row, the way
downstream.multigraph_from_edge_index stores them.  `structures()` is the whole set: every family reaches the dense
solver and at least one Chebyshev-filtered subspace (ChFSI) class, every size class of the solver is reached, at its
edges too, and the cluster and L2 classes hold at least three structurally different graphs each.

Long paths, rings and grids stay at n <= 384: their top spectrum is a gap-less quadratic run towards 1, which no
fixed-degree Chebyshev filter separates at larger n; ego-nets and the whole graphs of the graph datasets have a
small diameter."""
import numpy as np

DN_A, DN_B, DN_C = 96, 144, 228                  # dense solver classes (the last two only under GCCB200_DENSE_MAX)
CF_NSM, CF_NSM_C, CF_D1, CF_D = 160, 384, 1536, 3584
CLUSTER = 8                                      # CTAs of the cluster kernel: slabs of ceil(n / 8) rows
CL_HEAVY, CL_MAXHEAVY = 192, 16                  # cluster kernel: hub-row degree and hub-row list length
DENSE_MAX = {"default": DN_A, "dense": DN_C}


def eig_class(n, solver="default"):
    """The size class posenc.cu sends an n-vertex graph to (eig_class)."""
    if n <= DENSE_MAX[solver]:
        return "dense<=%d" % next(c for c in (DN_A, DN_B, DN_C) if n <= c)
    return "chfsi<=%s" % next((c for c in (CF_NSM, CF_NSM_C, CF_D1, CF_D) if n <= c), "L2")


CLASS_ORDER = ["dense<=96", "dense<=144", "dense<=228", "chfsi<=160", "chfsi<=384", "chfsi<=1536", "chfsi<=3584",
               "chfsi<=L2"]


def slab_rows(n):
    return -(-n // CLUSTER)


def csr(n, src, dst, multi=False):
    """Symmetric CSR of the undirected edges (src, dst).  Simple graphs drop self loops and duplicates."""
    src, dst = np.asarray(src, np.int64).ravel(), np.asarray(dst, np.int64).ravel()
    if not multi:
        keep = src != dst
        src, dst = src[keep], dst[keep]
    r, c = np.concatenate([src, dst]), np.concatenate([dst, src])
    key = r * n + c
    key = np.sort(key) if multi else np.unique(key)
    r, c = key // n, key % n
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, r + 1, 1)
    return np.cumsum(indptr).astype(np.int32), c.astype(np.int32)


def _graph(name, family, n, src, dst, multi=False):
    indptr, indices = csr(n, src, dst, multi)
    return dict(name=name, family=family, n=n, m=len(indices), indptr=indptr, indices=indices,
                subv=np.arange(n, dtype=np.int32))


def _empty():
    return np.zeros(0, np.int64), np.zeros(0, np.int64)


def _tree(rng, n):
    if n < 2:
        return _empty()
    return np.arange(1, n), np.array([rng.integers(0, i) for i in range(1, n)])


def _tree_plus(rng, n, extra):
    s, d = _tree(rng, n)
    e = rng.integers(0, n, (extra, 2))
    return np.concatenate([s, e[:, 0]]), np.concatenate([d, e[:, 1]])


def _hub_paths(rng, n, hubs=1):
    """`hubs` centres (a path among them) with pendant paths of one and two edges: eigenvalues 1/sqrt 2 and
    sqrt(2/3) of high multiplicity."""
    src, dst = list(range(1, hubs)), list(range(hubs - 1))
    v = hubs
    while v < n:
        h = int(rng.integers(0, hubs))
        if v + 1 < n and rng.random() < 0.5:
            src += [h, v]
            dst += [v, v + 1]
            v += 2
        else:
            src.append(h)
            dst.append(v)
            v += 1
    return np.array(src), np.array(dst)


def _star(n):
    return np.zeros(n - 1, np.int64), np.arange(1, n)


def _ring(n):
    return np.arange(n), (np.arange(n) + 1) % n


def _path(n):
    return np.arange(n - 1), np.arange(1, n)


def _grid(r, c):
    idx = np.arange(r * c).reshape(r, c)
    src = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    dst = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    return src, dst


def _bipartite(a, b):
    s, d = np.meshgrid(np.arange(a), a + np.arange(b), indexing="ij")
    return s.ravel(), d.ravel()


def _er(rng, n, p):
    iu = np.triu_indices(n, 1)
    keep = rng.random(len(iu[0])) < p
    return iu[0][keep], iu[1][keep]


def _er_sparse(rng, n, avg_deg):
    e = rng.integers(0, n, (n * avg_deg // 2, 2))
    return e[:, 0], e[:, 1]


def _union(parts):
    """parts: [(n_i, src_i, dst_i)] -> one graph, offsets in order (an isolated vertex is (1, [], []))."""
    src, dst, off = [], [], 0
    for n, s, d in parts:
        src.append(np.asarray(s, np.int64) + off)
        dst.append(np.asarray(d, np.int64) + off)
        off += n
    return off, np.concatenate(src), np.concatenate(dst)


def _cliques(sizes):
    parts = []
    for m in sizes:
        iu = np.triu_indices(m, 1)
        parts.append((m, iu[0], iu[1]))
    return _union(parts)


def _components(rng, n, big):
    """Components: ER pieces, trees, stars and dense near-cliques of the given sizes, then isolated vertices up to
    n (the whole graphs of COLLAB / IMDB / REDDIT)."""
    parts = []
    for i, m in enumerate(big):
        kind = i % 4
        if kind == 0:
            parts.append((m,) + _er(rng, m, 0.8))
        elif kind == 1:
            parts.append((m,) + _tree(rng, m))
        elif kind == 2:
            parts.append((m,) + _star(m))
        else:
            parts.append((m,) + _er(rng, m, 0.3))
    used = sum(big)
    parts += [(1,) + _empty()] * (n - used)
    order = rng.permutation(len(parts))                 # isolated vertices between the components
    return _union([parts[i] for i in order])


def _many_components(n, ncomp):
    """ncomp triangles and edges (eigenvalue 1 of multiplicity ncomp), isolated vertices after them."""
    parts, used = [], 0
    ntri = (n - 2 * ncomp) // 2
    for i in range(ncomp):
        m = 3 if i < ntri else 2
        iu = np.triu_indices(m, 1)
        parts.append((m, iu[0], iu[1]))
        used += m
    assert used <= n
    parts += [(1,) + _empty()] * (n - used)
    return _union(parts)


def _multi(rng, n, avg_deg, loops):
    """A multigraph: a random tree plus random extra edges, every edge repeated 1..5 times, `loops` self loops."""
    s, d = _tree_plus(rng, n, n * avg_deg // 2)
    t = rng.integers(1, 6, len(s))
    s, d = np.repeat(s, t), np.repeat(d, t)
    lv = rng.integers(0, n, loops)
    return np.concatenate([s, lv]), np.concatenate([d, lv])


def _hub_mix(rng, n, hubs, hub_deg, avg_deg):
    """Sparse random background plus `hubs` vertices with hub_deg random neighbours each."""
    s, d = _tree_plus(rng, n, n * avg_deg // 2)
    hs = np.repeat(np.arange(hubs), hub_deg)
    hd = rng.integers(0, n, hubs * hub_deg)
    return np.concatenate([s, hs]), np.concatenate([d, hd])


def structures(seed=0):
    """The whole structure set, in a fixed order."""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, family, n, sd, multi=False):
        out.append(_graph(name, family, n, sd[0], sd[1], multi))

    # ego-net-like: random trees, trees with a few extra edges, hubs with pendant paths
    for n in (1, 3, 60, 97, 161, 229, 700, 1537):
        add("tree_%d" % n, "tree", n, _tree(rng, n))
    for n in (2, 4, 90, 145, 300, 1100, 3585):
        add("tree_plus_%d" % n, "tree_plus", n, _tree_plus(rng, n, max(1, n // 20)))
    for n, h in ((5, 1), (95, 1), (144, 1), (160, 2), (228, 1), (385, 3), (1536, 4), (3584, 6)):
        add("hub_paths_%d" % n, "hub_paths", n, _hub_paths(rng, n, h))
    # stars: eigenvalue 0 of multiplicity n - 2
    for n in (33, 145, 384, 801):
        add("star_%d" % n, "star", n, _star(n))
    # rings (every eigenvalue but +-1 double: the k = 32 cut falls inside a pair) and paths (already tridiagonal)
    for n in (64, 96, 161, 384):
        add("ring_%d" % n, "ring", n, _ring(n))
    for n in (3, 96, 229, 300):
        add("path_%d" % n, "path", n, _path(n))
    # 2-D grids and complete bipartite graphs: eigenvalue -1, large multiplicities
    for r, c in ((8, 12), (12, 12), (10, 16), (16, 24)):
        add("grid_%dx%d" % (r, c), "grid", r * c, _grid(r, c))
    for a, b in ((30, 66), (40, 120), (100, 300), (20, 1517)):
        add("bipartite_%dx%d" % (a, b), "bipartite", a + b, _bipartite(a, b))
    # dense: Erdos-Renyi with p 0.3-0.6 (a dense bulk spectrum) and unions of cliques
    for n, p in ((80, 0.5), (144, 0.4), (229, 0.3), (385, 0.5)):
        add("er_dense_%d" % n, "er_dense", n, _er(rng, n, p))
    for sizes in ((20, 20, 30, 26), (40, 40, 40, 40, 25), (60, 60, 60, 60, 60, 40)):
        n, s, d = _cliques(sizes)
        add("cliques_%d" % n, "cliques", n, (s, d))
    # whole graphs: components plus isolated vertices, more than 48 components, all isolated
    for n, big in ((90, (30, 20, 10)), (228, (60, 40, 30, 20)), (490, (180, 120, 60, 30, 20))):
        n, s, d = _components(rng, n, big)
        add("components_%d" % n, "components", n, (s, d))
    for n, nc in ((96, 40), (190, 60), (480, 150)):
        n, s, d = _many_components(n, nc)
        add("many_components_%d_%d" % (n, nc), "many_components", n, (s, d))
    for n in (50, 97, 400):
        add("isolated_%d" % n, "isolated", n, _empty())
    # multigraphs: parallel edges and self loops
    for n in (40, 150, 384, 900):
        add("multi_%d" % n, "multi", n, _multi(rng, n, 3, max(2, n // 10)), multi=True)
    # hub-heavy dense graphs: more than 16 rows of degree > 192 in one cluster slab (192- and 448-row slabs)
    add("hub_heavy_400", "hub_heavy", 400, _er(rng, 400, 0.6))
    add("hub_heavy_1536", "hub_heavy", 1536, _er(rng, 1536, 0.2))
    add("hub_heavy_1600", "hub_heavy", 1600, _er(rng, 1600, 0.2))
    # the L2 class (n > 3584): sparse random and hub mixtures (simple top spectra: the float64 reference is eigsh)
    add("er_sparse_4000", "er_sparse", 4000, _er_sparse(rng, 4000, 8))
    add("hub_mix_5000", "hub_mix", 5000, _hub_mix(rng, 5000, 12, 600, 4))
    return out


def representatives(graphs, solver="default"):
    """One graph per size class for the placement-invariance checks (the first of each class in set order), and
    every hub-heavy graph."""
    seen, reps = set(), []
    for g in graphs:
        c = eig_class(g["n"], solver)
        if g["n"] >= 3 and (c not in seen or g["family"] == "hub_heavy"):
            seen.add(c)
            reps.append(g)
    return reps


def heavy_rows_per_slab(g):
    """Rows of degree > CL_HEAVY in each cluster slab of ceil(n / 8) rows."""
    deg = np.diff(g["indptr"])
    R = slab_rows(g["n"])
    return [int((deg[q * R:(q + 1) * R] > CL_HEAVY).sum()) for q in range(CLUSTER)]
