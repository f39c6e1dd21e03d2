"""A minimal stand-in for DGL 0.4.3, used ONLY by tests/golden/make_golden.py to
execute the REAL reference modules (gcc/**, train.py of a reference checkout)
without DGL, which was not installable there (SURVEY.md section 8c).

Everything here encodes the [M] (recalled, unverifiable) DGL semantics the
oracle documents; everything *outside* this file that runs during golden
generation is the reference's own code.  Test infrastructure, not product.
"""
import sys
import types

import numpy as np
import scipy.sparse as sparse
import torch
import torch.nn as nn


class StubGraph:
    """Just enough of DGLGraph for the reference's hot path."""

    def __init__(self, n, src, dst, parent_nid=None, batch_num_nodes=None):
        self.n = int(n)
        self.src = np.asarray(src, dtype=np.int64)   # edge u -> v
        self.dst = np.asarray(dst, dtype=np.int64)
        self.ndata = {}
        self.edata = {}
        self.parent_nid = parent_nid
        self.batch_num_nodes = list(batch_num_nodes) if batch_num_nodes else [self.n]
        self.batch_size = len(self.batch_num_nodes)

    @classmethod
    def from_csr(cls, indptr, indices):
        indptr = np.asarray(indptr, dtype=np.int64)
        n = len(indptr) - 1
        row = np.repeat(np.arange(n), np.diff(indptr))
        # CSR row v lists v's neighbours u; symmetric graphs -> store edges u -> v
        return cls(n, np.asarray(indices, dtype=np.int64), row)

    def number_of_nodes(self):
        return self.n

    def number_of_edges(self):
        return len(self.src)

    def nodes(self):
        return torch.arange(self.n)

    def in_degrees(self):
        return torch.from_numpy(np.bincount(self.dst, minlength=self.n)).long()

    def in_degree(self, v):
        return int((self.dst == int(v)).sum())

    def to(self, device):
        return self

    def readonly(self, flag=True):
        return self

    def subgraph(self, nodes):
        """[M] new ids follow `nodes` order; all parent edges with both ends inside,
        multiplicity kept; per-destination order = parent adjacency order."""
        nodes = [int(v) for v in (nodes.tolist() if hasattr(nodes, "tolist") else nodes)]
        pos = {v: i for i, v in enumerate(nodes)}
        order = np.lexsort((self.src, self.dst))     # group by dst, src ascending
        s2, d2 = [], []
        by_dst = {}
        for e in order:
            by_dst.setdefault(int(self.dst[e]), []).append(int(self.src[e]))
        for v in nodes:
            for u in by_dst.get(v, []):
                if u in pos:
                    s2.append(pos[u])
                    d2.append(pos[v])
        return StubGraph(len(nodes), s2, d2, parent_nid=np.array(nodes))

    def adjacency_matrix_scipy(self, transpose=False, return_edge_ids=True):
        """[M] rows = dst, cols = src, data = 1 (transpose=False)."""
        r, c = (self.src, self.dst) if transpose else (self.dst, self.src)
        return sparse.coo_matrix((np.ones(len(r)), (r, c)), shape=(self.n, self.n)).tocsr()

    # helpers for our own oracle / tests
    def batched_csr(self):
        order = np.lexsort((np.arange(len(self.src)), self.dst))
        # keep insertion order inside each destination row
        order = np.argsort(self.dst, kind="stable")
        indptr = np.zeros(self.n + 1, dtype=np.int64)
        np.cumsum(np.bincount(self.dst, minlength=self.n), out=indptr[1:])
        return indptr, self.src[order].astype(np.int32)


def batch(graphs):
    """[M] dgl.batch: node/edge ids offset by cumulative counts, ndata concatenated."""
    off, src, dst, bnn = 0, [], [], []
    for g in graphs:
        src.append(g.src + off)
        dst.append(g.dst + off)
        off += g.n
        bnn.append(g.n)
    bg = StubGraph(off, np.concatenate(src) if src else [], np.concatenate(dst) if dst else [],
                   batch_num_nodes=bnn)
    for key in graphs[0].ndata:
        bg.ndata[key] = torch.cat([g.ndata[key] for g in graphs], dim=0)
    return bg


class GINConv(nn.Module):
    """[M] dgl.nn.pytorch.conv.GINConv(apply_func, 'sum', init_eps, learn_eps)."""

    def __init__(self, apply_func, aggregator_type, init_eps=0, learn_eps=False):
        super().__init__()
        assert aggregator_type == "sum"
        self.apply_func = apply_func
        if learn_eps:
            self.eps = nn.Parameter(torch.FloatTensor([init_eps]))
        else:
            self.register_buffer("eps", torch.FloatTensor([init_eps]))

    def forward(self, graph, feat):
        src = torch.from_numpy(graph.src)
        dst = torch.from_numpy(graph.dst)
        neigh = torch.zeros_like(feat).index_add_(0, dst, feat[src])
        rst = (1 + self.eps) * feat + neigh
        if self.apply_func is not None:
            rst = self.apply_func(rst)
        return rst


class SumPooling(nn.Module):
    def forward(self, graph, feat):
        gid = torch.repeat_interleave(torch.arange(graph.batch_size),
                                      torch.tensor(graph.batch_num_nodes))
        return torch.zeros(graph.batch_size, feat.shape[1], dtype=feat.dtype).index_add_(0, gid, feat)


class _Unused(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()


class Set2Set(nn.Module):
    """Only the parameter container (state_dict keys set2set.lstm.*); the gin
    branch never calls it (graph_encoder.py:189-190)."""

    def __init__(self, input_dim, n_iters, n_layers):
        super().__init__()
        self.lstm = nn.LSTM(2 * input_dim, input_dim, n_layers)


# random_walk_with_restart is bound by make_golden.py to the oracle's pure-Python walk
_rwr_impl = None


def random_walk_with_restart(g, seeds, restart_prob, max_nodes_per_seed):
    return _rwr_impl(g, seeds, restart_prob, max_nodes_per_seed)


def install():
    """Register fake `dgl` (and matplotlib) modules in sys.modules."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    dgl = mod("dgl", batch=batch, DGLGraph=StubGraph)
    dgl.random = mod("dgl.random", seed=lambda s: None)
    dgl.backend = mod("dgl.backend", asnumpy=lambda t: t.numpy())
    dgl.data = mod("dgl.data", AmazonCoBuy=None, Coauthor=None)
    dgl.data.utils = mod("dgl.data.utils")
    dgl.data.tu = mod("dgl.data.tu", TUDataset=None)
    dgl.nodeflow = mod("dgl.nodeflow", NodeFlow=None)
    dgl.contrib = mod("dgl.contrib")
    dgl.contrib.sampling = mod("dgl.contrib.sampling",
                               random_walk_with_restart=random_walk_with_restart)
    dgl.nn = mod("dgl.nn")
    dgl.nn.pytorch = mod("dgl.nn.pytorch", Set2Set=Set2Set, NNConv=_Unused)
    dgl.nn.pytorch.conv = mod("dgl.nn.pytorch.conv", GINConv=GINConv)
    dgl.nn.pytorch.glob = mod("dgl.nn.pytorch.glob", SumPooling=SumPooling,
                              AvgPooling=_Unused, MaxPooling=_Unused)
    dgl.model_zoo = mod("dgl.model_zoo")
    dgl.model_zoo.chem = mod("dgl.model_zoo.chem")
    dgl.model_zoo.chem.gnn = mod("dgl.model_zoo.chem.gnn", GATLayer=_Unused)
    if "matplotlib" not in sys.modules:
        try:
            import matplotlib  # noqa: F401
        except ImportError:
            mpl = mod("matplotlib")
            mpl.pyplot = mod("matplotlib.pyplot")
    # the reference hard-codes .cuda(); make it a no-op on this CPU-only box
    torch.Tensor.cuda = lambda self, *a, **k: self
    nn.Module.cuda = lambda self, *a, **k: self
    torch.cuda.synchronize = lambda *a, **k: None
    return dgl
