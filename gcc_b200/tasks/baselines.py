"""The reference's embedding baselines, GraphWave and ProNE (gcc/models/emb), on the GPU in float64, and a command
line that saves their rows for the frozen-embedding evaluators:

    python -m gcc_b200.tasks.baselines --task node_classification --dataset usa_airport --model prone \\
        --hidden-size 64 --output-dir <dir>        # then node_classification --model from_numpy --emb-path <dir>/usa_airport.npy
    python -m gcc_b200.tasks.baselines --task similarity_search --dataset kdd_icdm --model graphwave \\
        --hidden-size 64 --output-dir <dir>        # then similarity_search --model from_numpy_align (kdd.npy, icdm.npy)

The sparse arithmetic is csrc/baselines.cu (gccb_graphwave, gccb_prone_factor, gccb_prone_propagate,
gccb_spmm_f64).  ProNE's tall-skinny QR and its small SVDs are torch.linalg on the device (DESIGN.md).

Each task hands the embedder the graph the reference's task builds from the edge list:
  node classification  nx.Graph:      a listed pair (either direction) is one edge of weight 1, a self loop too;
  similarity search    nx.MultiGraph: A[u,v] counts the listed pairs (u,v) and (v,u); a listed (x,x) adds 1.
The vertex set is the vertices that appear in an edge, relabelled 0..n-1 in ascending order.
"""
import argparse
import math
import os
from collections import namedtuple

import numpy as np

from .. import _lib

WGraph = namedtuple("WGraph", "indptr indices vals nodes")   # symmetric CSR with float64 weights, nodes: original ids

ORDER = 30                    # _graphwave/graphwave.py:21
ETA_MAX, ETA_MIN = 0.95, 0.80
GRAPHWAVE_WORKSPACE = 2 << 30  # bytes of heat blocks: one block up to ~8k vertices, several beyond


def _csr(nodes, u, v, w):
    """Symmetric CSR of the (local u, local v, weight) triples, duplicates summed, rows ascending."""
    n = len(nodes)
    key = u * n + v
    order = np.argsort(key, kind="stable")
    key, w = key[order], w[order]
    uniq, start = np.unique(key, return_index=True)
    vals = np.add.reduceat(w, start) if len(w) else w
    rows = uniq // n
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, rows + 1, 1)
    return WGraph(np.cumsum(indptr), (uniq % n).astype(np.int32), vals.astype(np.float64), nodes)


def _local(edge_index):
    src, dst = (np.asarray(a, dtype=np.int64).reshape(-1) for a in edge_index)
    nodes = np.unique(np.concatenate([src, dst]))
    return nodes, np.searchsorted(nodes, src), np.searchsorted(nodes, dst)


def graph_from_pairs(edge_index):
    """nx.Graph(edge_index) as node classification builds it: de-duplicated pairs of weight 1, self loops kept
    with weight 1 (networkx puts w on the diagonal)."""
    nodes, s, d = _local(edge_index)
    n = len(nodes)
    a, b = np.minimum(s, d), np.maximum(s, d)
    pairs = np.unique(a * n + b)
    a, b = pairs // n, pairs % n
    off = a != b
    u = np.concatenate([a, b[off]])
    v = np.concatenate([b, a[off]])
    return _csr(nodes, u, v, np.ones(len(u)))


def multigraph_from_pairs(edge_index):
    """nx.MultiGraph(edge_index) as similarity search builds it: every listed pair is an edge; A[u,v] counts the
    pairs listed as (u,v) or (v,u), and a listed self loop adds 1 to A[x,x]."""
    nodes, s, d = _local(edge_index)
    off = s != d
    u = np.concatenate([s, d[off]])
    v = np.concatenate([d, s[off]])
    return _csr(nodes, u, v, np.ones(len(u)))


def graphwave_scales(n):
    """The two heat scales of GraphWave's automatic mode, the smallest nonzero Laplacian eigenvalue approximated by
    1/n: s = -ln(eta) sqrt(n / 2) for eta = ETA_MAX, ETA_MIN."""
    root = math.sqrt(n / 2.0)
    return np.array([-math.log(ETA_MAX) * root, -math.log(ETA_MIN) * root])


def cheb_coeffs(scale, order=ORDER):
    """Chebyshev interpolation coefficients of exp(-scale (x + 1)) on [-1, 1] at the `order` Chebyshev nodes
    theta_j = (2j - 1) pi / (2 order):  c_k = (2 / order) sum_j exp(-scale (cos theta_j + 1)) cos(k theta_j),
    k = 0 .. order, with c_0 halved."""
    theta = (2.0 * np.arange(1, order + 1) - 1.0) * math.pi / (2.0 * order)
    samples = np.exp(-scale * (np.cos(theta) + 1.0))
    coeffs = np.cos(np.outer(np.arange(order + 1), theta)) @ samples * (2.0 / order)
    coeffs[0] *= 0.5
    return coeffs


def bessel_i(order, x):
    """Modified Bessel function of the first kind I_order(x) (scipy.special.iv) by its power series."""
    term = (x / 2.0) ** order / math.factorial(order)
    total, m = 0.0, 0
    while term > 1e-300 and (m == 0 or term > 1e-18 * total):
        total += term
        m += 1
        term *= (x / 2.0) ** 2 / (m * (m + order))
    return total


def _device_graph(g):
    import torch
    _lib.require_device()
    dev = torch.device("cuda")
    return (torch.from_numpy(g.indptr).to(dev), torch.from_numpy(g.indices).to(dev),
            torch.from_numpy(g.vals).to(dev))


def _as_wgraph(graph):
    if isinstance(graph, WGraph):
        return graph
    indptr, indices, vals = graph
    return WGraph(np.asarray(indptr, np.int64), np.asarray(indices, np.int32), np.asarray(vals, np.float64),
                  np.arange(len(indptr) - 1))


class GraphWave:
    """GraphWave(dimension, scale=100).train(graph) -> chi [n, 4 (dimension // 4)] (gcc/models/emb/graphwave.py).
    graph: a WGraph or (indptr, indices, vals) of a symmetric weighted CSR.  block_cols: identity columns per heat
    block (default: as many as `workspace_bytes` holds); the result does not depend on it."""

    def __init__(self, dimension, scale=100, workspace_bytes=GRAPHWAVE_WORKSPACE, block_cols=None, **kwargs):
        self.dimension = dimension
        self.scale = scale
        self.workspace_bytes = workspace_bytes
        self.block_cols = block_cols

    def train(self, graph):
        import torch
        g = _as_wgraph(graph)
        n = len(g.indptr) - 1
        n_times = self.dimension // 4
        if n_times < 1 or n_times > 64:
            raise ValueError("GraphWave needs 4 <= dimension < 260, got %d" % self.dimension)
        lib = _lib.get()
        per_col = lib.gccb_graphwave_workspace(n, 2) // 2
        bc = self.block_cols or max(1, min(n, self.workspace_bytes // per_col))
        bc = min(bc, n)
        cheb = np.ascontiguousarray(np.concatenate([cheb_coeffs(t, ORDER) for t in graphwave_scales(n)]))
        times = np.ascontiguousarray(np.linspace(0, self.scale, n_times), np.float64)
        indptr, indices, vals = _device_graph(g)
        ws = torch.empty(lib.gccb_graphwave_workspace(n, bc), dtype=torch.uint8, device="cuda")
        chi = torch.empty((n, 4 * n_times), dtype=torch.float64, device="cuda")
        _lib.check(lib.gccb_graphwave(_lib.dptr(indptr), _lib.dptr(indices), _lib.dptr(vals), n,
                                      cheb.ctypes.data, ORDER, times.ctypes.data, n_times, bc, _lib.dptr(ws),
                                      ws.numel(), _lib.dptr(chi), _lib.stream_ptr()), "gccb_graphwave")
        return chi.cpu().numpy()


def _spmm(lib, dg, X):
    """dg X on the device, dg = (indptr, indices, values)."""
    import torch
    indptr, indices, vals = dg
    n = indptr.numel() - 1
    _check_rows(X, n, "block")
    X = X.contiguous()
    Y = torch.empty_like(X)
    _lib.check(lib.gccb_spmm_f64(_lib.dptr(indptr), _lib.dptr(indices), _lib.dptr(vals), n, X.shape[1],
                                 X.shape[1], 1.0, 0.0, None, None, 0.0, _lib.dptr(X), 0.0, None, _lib.dptr(Y),
                                 _lib.stream_ptr()), "gccb_spmm_f64")
    return Y


def _check_rows(X, n, what):
    """The kernels read an n-row block of the graph's size: anything else is refused before it reaches them."""
    if X.dim() != 2 or X.shape[0] != n or X.shape[1] < 1:
        raise ValueError("%s of shape %s: expected %d rows (the graph's vertices) and at least one column"
                         % (what, tuple(X.shape), n))


def _flip_scale_normalize(U, s, d):
    """sklearn's svd_flip (each column's largest-magnitude entry positive), then U[:, :d] sqrt(s), rows
    l2-normalised (sklearn.preprocessing.normalize: zero rows stay zero)."""
    import torch
    idx = U.abs().argmax(dim=0)
    signs = torch.sign(U[idx, torch.arange(U.shape[1], device=U.device)])
    signs[signs == 0] = 1
    U = (U * signs)[:, :d] * torch.sqrt(s[:d])
    norm = U.norm(dim=1, keepdim=True)
    return U / torch.where(norm == 0, torch.ones_like(norm), norm)


class ProNE:
    """ProNE(dimension, step=5, mu=0.2, theta=0.5).train(graph) -> [n, dimension] (gcc/models/emb/prone.py).
    The randomized SVD's start block comes from the Philox stream keyed by `seed`, or from train(omega=...)."""

    def __init__(self, dimension, step=5, mu=0.2, theta=0.5, seed=0, **kwargs):
        self.dimension = dimension
        self.step = step
        self.mu = mu
        self.theta = theta
        self.seed = seed

    def _check(self, n):
        if n < self.dimension:
            raise ValueError("ProNE of dimension %d needs at least as many vertices; the graph has %d"
                             % (self.dimension, n))

    def factorize(self, graph):
        """(F, F^T) values on the graph's pattern, as device tensors."""
        import torch
        g = _as_wgraph(graph)
        n = len(g.indptr) - 1
        lib = _lib.get()
        dg = _device_graph(g)
        F = torch.empty_like(dg[2])
        FT = torch.empty_like(dg[2])
        ws = torch.empty(lib.gccb_prone_factor_workspace(n), dtype=torch.uint8, device="cuda")
        _lib.check(lib.gccb_prone_factor(*(_lib.dptr(t) for t in dg), n, _lib.dptr(ws), ws.numel(), _lib.dptr(F),
                                         _lib.dptr(FT), _lib.stream_ptr()), "gccb_prone_factor")
        return dg, F, FT

    def omega(self, n):
        import torch
        cols = min(self.dimension + 10, n)
        out = torch.empty((n, cols), dtype=torch.float64, device="cuda")
        _lib.check(_lib.get().gccb_gaussian_f64(_lib.dptr(out), n, cols, self.seed, _lib.stream_ptr()),
                   "gccb_gaussian_f64")
        return out

    def tsvd(self, graph, omega=None, n_iter=5):
        """randomized_svd(F, dimension, n_oversamples=10, n_iter=5) with QR as the power-iteration normaliser;
        returns (singular values, features U sqrt(s) row-normalised), both device tensors."""
        import torch
        g = _as_wgraph(graph)
        n = len(g.indptr) - 1
        self._check(n)
        lib = _lib.get()
        dg, F, FT = self.factorize(g)
        f, ft = (dg[0], dg[1], F), (dg[0], dg[1], FT)
        if omega is None:
            Q = self.omega(n)
        else:
            Q = torch.as_tensor(omega, dtype=torch.float64, device="cuda")
            _check_rows(Q, n, "omega")
            if Q.shape[1] > n:
                raise ValueError("omega has %d columns, more than the graph's %d vertices" % (Q.shape[1], n))
        for _ in range(n_iter):
            Q = torch.linalg.qr(_spmm(lib, f, Q)).Q
            Q = torch.linalg.qr(_spmm(lib, ft, Q)).Q
        Q = torch.linalg.qr(_spmm(lib, f, Q)).Q.contiguous()
        B = _spmm(lib, ft, Q).T                                  # Q^T F
        Uh, s, _ = torch.linalg.svd(B, full_matrices=False)
        return s[:self.dimension], _flip_scale_normalize(Q @ Uh, s, self.dimension)

    def propagate(self, graph, a):
        """_chebyshev_gaussian(A, a, step, mu, theta): (mm, embedding) as device tensors."""
        import torch
        g = _as_wgraph(graph)
        n = len(g.indptr) - 1
        a = torch.as_tensor(a, dtype=torch.float64, device="cuda").contiguous()
        _check_rows(a, n, "a")
        if self.step == 1:
            return a, a
        lib = _lib.get()
        dg = _device_graph(g)
        k = a.shape[1]
        bessel = np.ascontiguousarray([bessel_i(i, self.theta) for i in range(self.step)], np.float64)
        ws = torch.empty(lib.gccb_prone_propagate_workspace(n, k), dtype=torch.uint8, device="cuda")
        mm = torch.empty_like(a)
        _lib.check(lib.gccb_prone_propagate(*(_lib.dptr(t) for t in dg), n, _lib.dptr(a), k, self.mu,
                                            bessel.ctypes.data, self.step, _lib.dptr(ws), ws.numel(), _lib.dptr(mm),
                                            _lib.stream_ptr()), "gccb_prone_propagate")
        U, s, _ = torch.linalg.svd(mm, full_matrices=False)
        return mm, _flip_scale_normalize(U, s, self.dimension)

    def train(self, graph, omega=None):
        g = _as_wgraph(graph)
        _, a = self.tsvd(g, omega)
        return self.propagate(g, a)[1].cpu().numpy()


MODELS = {"prone": ProNE, "graphwave": GraphWave}


def embed_edge_index(model, edge_index, multigraph):
    """(nodes, rows): the baseline's rows for the vertices that appear in edge_index."""
    g = (multigraph_from_pairs if multigraph else graph_from_pairs)(edge_index)
    return g.nodes, model.train(g)


def main(argv=None):
    from ..datasets.downstream import SSDataset, create_node_classification_dataset, node_dataset_graph
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--task", choices=["node_classification", "similarity_search"], required=True)
    ap.add_argument("--dataset", type=str, required=True)
    ap.add_argument("--model", choices=sorted(MODELS), required=True)
    ap.add_argument("--hidden-size", type=int, required=True)
    ap.add_argument("--output-dir", type=str, required=True)
    ap.add_argument("--seed", type=int, default=0, help="Philox key of ProNE's randomized SVD")
    ap.add_argument("--root", type=str, default="data", help="directory of the downstream datasets")
    args = ap.parse_args(argv)
    if args.model == "graphwave" and args.hidden_size % 4:
        ap.error("graphwave writes 4 * (hidden_size // 4) columns: --hidden-size must be a multiple of 4")
    model = MODELS[args.model](args.hidden_size, seed=args.seed)
    os.makedirs(args.output_dir, exist_ok=True)
    if args.task == "node_classification":
        data = create_node_classification_dataset(args.dataset, args.root).data
        edge_index = data.edge_index.numpy()
        rows = np.zeros((node_dataset_graph(args.dataset, args.root).num_nodes, args.hidden_size))
        nodes, emb = embed_edge_index(model, edge_index, multigraph=False)
        rows[nodes] = emb
        outs = {args.dataset: rows}
    else:
        name_1, name_2 = args.dataset.split("_")[:2]
        ss = SSDataset(os.path.join(args.root, "panther"), name_1, name_2)
        outs = {}
        for name, d in zip((name_1, name_2), ss.data):
            # Panther ids with edges are numbered 0.. in order of appearance: row v is vertex v
            outs[name] = embed_edge_index(model, d.edge_index.numpy(), multigraph=True)[1]
    for name, rows in outs.items():
        path = os.path.join(args.output_dir, name + ".npy")
        np.save(path, rows)
        print("saved %s embeddings %s to %s" % (args.model, rows.shape, path))
    return outs


if __name__ == "__main__":
    main()
