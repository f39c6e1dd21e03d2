"""Device-resident ego-net dataset: the GPU replacement of the reference's CPU DataLoader.

Mirrors the surface of gcc/datasets/graph_dataset.py that train.py touches
(LoadBalanceGraphDataset ctor kwargs, .total, .jobs, .dgl_graphs_file, iteration
yielding (graph_q, graph_k)) -- SURVEY.md section 8b -- but sampling, induction,
positional features and batching all run as CUDA kernels over a CSR kept in HBM:

  reference (CPU worker processes)                      here (device kernels)
  __iter__: np.random.choice(p ~ deg^.75)   :85-92   -> gccb_draw_seeds
  __getitem__: budget + dgl RWR             :113-130 -> gccb_sample_batch (walk)
  _rwr_trace_to_dgl_graph                   data_util.py:218-239 -> gccb_sample_batch (induce)
  _add_undirected_graph_positional_embedding data_util.py:266-281 -> gccb_posenc
  batcher()/dgl.batch, pickling, H2D        data_util.py:26-32, train.py:382-383 -> (nothing: already batched on device)

Randomness is the counter-based "RWR-Philox v1" stream (DESIGN.md), so a batch is a
pure function of (run seed, sample ids) -- independent of worker count or world size.
"""
import ctypes as C
import math
import operator

import numpy as np
import torch

from .. import _capi, _lib
from . import synthetic
from .data_util import BatchedSubgraphs

HOPCAP = 64


def load_graphs(spec):
    """CSRGraph | list[CSRGraph] | path to .npz(indptr, indices[, graph_sizes]) | path to a DGL save_graphs
    .bin -> (union CSR, sizes)."""
    if isinstance(spec, synthetic.CSRGraph):
        return spec, [spec.num_nodes]
    if isinstance(spec, (list, tuple)):
        return synthetic.disjoint_union(spec), [g.num_nodes for g in spec]
    if isinstance(spec, str):
        if spec.endswith(".npz"):
            z = np.load(spec)
            g = synthetic.CSRGraph(z["indptr"].astype(np.int64), z["indices"].astype(np.int32),
                                   len(z["indptr"]) - 1, spec)
            sizes = z["graph_sizes"].tolist() if "graph_sizes" in z.files else [g.num_nodes]
            return g, sizes
        if spec.endswith(".bin"):
            # DGL 0.4.x save_graphs file (gcc/utils/x2dgl.py:129-131), read without DGL: graph_dataset.py:26-28
            # (load_graphs) and :58-60 (load_labels "graph_sizes").  Layout restated from memory: datasets/dgl_bin.py
            from . import dgl_bin
            graphs, labels = dgl_bin.read_dgl_bin(spec)
            sizes = labels["graph_sizes"].tolist() if "graph_sizes" in labels else [g.num_nodes for g in graphs]
            if sizes != [g.num_nodes for g in graphs]:
                raise ValueError("%s: label graph_sizes disagrees with the stored graphs" % spec)
            return (graphs[0] if len(graphs) == 1 else synthetic.disjoint_union(graphs)), sizes
        raise NotImplementedError("unknown graph file type %r (use DGL .bin or .npz)" % spec)
    raise TypeError("unsupported graph spec %r" % (spec,))


def budget_for_degree(deg, rw_hops, restart_prob, exponent=0.75):
    """max_nodes_per_seed: gcc/datasets/graph_dataset.py:113-124 (pretraining loader, deg^0.75) or
    :243-254 (GraphDataset family used by generate.py / finetuning, plain degree) -- same arithmetic."""
    d = (deg ** 0.75) if exponent == 0.75 else deg
    return max(rw_hops, int((d * math.e / (math.e - 1) / restart_prob) + 0.5))


class DeviceGraph:
    """Parent CSR + sampler tables in HBM (built once; the reference re-loads graphs per worker,
    graph_dataset.py:23-30)."""

    def __init__(self, graph, rw_hops, restart_prob, key, device, budget_exponent=0.75, budget_cap=None):
        as_t = lambda x, dt: (x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))).to(
            device=device, dtype=dt).contiguous()
        self.indptr = as_t(graph.indptr, torch.int64)
        self.indices = as_t(graph.indices, torch.int32)
        deg = self.indptr[1:] - self.indptr[:-1]
        if int(deg.min()) <= 0:
            raise ValueError("zero-degree vertices are not allowed (the reference removes them, "
                             "gcc/utils/x2dgl.py:61; DGL aborts on them)")
        self.num_nodes = self.indptr.numel() - 1
        self.max_degree = int(deg.max())
        # budget depends only on the seed's degree -> small host-built table (exact Python arithmetic)
        uniq = torch.unique(deg).cpu().numpy()
        table = np.zeros(self.max_degree + 1, dtype=np.int32)
        for d in uniq:
            table[d] = budget_for_degree(int(d), rw_hops, restart_prob, budget_exponent)
        table = np.maximum.accumulate(table)          # unused degrees: any value; keep monotone
        if budget_cap:                                 # capacity knob (sampler sweeps on graphs with huge hubs);
            table = np.minimum(table, int(budget_cap))  # deviates from the reference formula above the cap
        self.max_budget = int(table.max())
        p = deg.double() ** 0.75                       # graph_dataset.py:86-87
        p = p / p.sum()
        cdf = torch.cumsum(p, 0)
        self.cdf = (cdf / cdf[-1]).contiguous()
        self.restart_thresh = min(int(restart_prob * 4294967296.0), 0xFFFFFFFF)
        self.key = int(key)
        self.budget_table = torch.from_numpy(table).to(device)
        self.c = _capi.Graph(self.indptr.data_ptr(), self.indices.data_ptr(), self.num_nodes,
                             self.budget_table.data_ptr(), len(table), self.max_budget,
                             self.restart_thresh, 0, self.key)
        self.nbytes = self.indptr.numel() * 8 + self.indices.numel() * 4


class BatchBuffers:
    """Caller-owned device memory behind one gccb_batch_t (both views of B pairs)."""

    def __init__(self, B, node_cap, edge_cap, pos_dim, max_budget, device):
        lib = _lib.get()
        i32 = dict(dtype=torch.int32, device=device)
        self.B, self.node_cap, self.edge_cap, self.pos_dim = B, node_cap, edge_cap, pos_dim
        self.node_off = torch.zeros(2, B + 1, **i32)
        self.edge_off = torch.zeros(2, B + 1, **i32)
        self.indptr = torch.zeros(2, node_cap + 1, **i32)
        self.indices = torch.zeros(2, edge_cap, **i32)
        self.sub_deg = torch.zeros(2, node_cap, **i32)
        self.graph_id = torch.zeros(2, node_cap, **i32)
        self.orig_id = torch.zeros(2, node_cap, **i32)
        self.counters = torch.zeros(2 * B, 4, dtype=torch.int64, device=device)
        self.flags = torch.zeros(1, **i32)
        self.pos = torch.zeros(2, node_cap, pos_dim, dtype=torch.float32, device=device)
        self.eigvals = torch.zeros(2 * B, pos_dim, dtype=torch.float32, device=device)
        self.seeds = torch.zeros(B, dtype=torch.int64, device=device)
        self.sample_ids = torch.zeros(B, dtype=torch.int64, device=device)
        self.ws_sample = torch.zeros(max(lib.gccb_sample_batch_workspace(B, max_budget, edge_cap), 8),
                                     dtype=torch.uint8, device=device)
        self.ws_posenc = torch.zeros(max(lib.gccb_posenc_workspace(B, node_cap), 8),
                                     dtype=torch.uint8, device=device)
        self.c = _capi.Batch(B, node_cap, edge_cap, 0, self.node_off.data_ptr(),
                             self.edge_off.data_ptr(), self.indptr.data_ptr(),
                             self.indices.data_ptr(), self.sub_deg.data_ptr(),
                             self.graph_id.data_ptr(), self.orig_id.data_ptr(),
                             self.counters.data_ptr(), self.flags.data_ptr())

    def eig_debug(self):
        """(iterations, worst residual) per ego-net of the last gccb_posenc on these buffers, read
        from the debug area of its workspace (posenc.cu: worklist[7][2B] | counts[7] | iters[2B] |
        pad to 64 ints | res[2B]).  Direct-Jacobi ego-nets report minus their sweep count, ego-nets solved by
        the dense tridiagonal solver (a direct method) report 0 iterations and their measured residual."""
        B, NC = self.B, 7
        ints = self.ws_posenc.view(torch.int32)
        o = NC * 2 * B + NC
        ni = ((o + 2 * B + 63) // 64) * 64
        return ints[o:o + 2 * B].clone(), self.ws_posenc[ni * 4: ni * 4 + 2 * B * 4].view(torch.float32).clone()

    def check_flags(self):
        """Host sync: raise on any device-side failure flag.  Eigensolver non-convergence is not
        fatal (the reference itself falls back to zeros after 10 ARPACK retries,
        data_util.py:249-257): it is counted and reported once."""
        f = int(self.flags.item())
        if f:
            self.flags.zero_()
            if f & _capi.FLAG_EIG_NOCONV:
                self.eig_noconv_events = getattr(self, "eig_noconv_events", 0) + 1
                if self.eig_noconv_events == 1:
                    import warnings
                    warnings.warn("gcc_b200: an ego-net eigensolve hit its iteration limit "
                                  "(residual above 2.5e-4); features kept as is")
                f &= ~_capi.FLAG_EIG_NOCONV
            if f:
                raise _lib.GccbError("device flags: " + "; ".join(
                    n for b, n in _capi.FLAG_NAMES.items() if f & b))


class LoadBalanceGraphDataset(torch.utils.data.IterableDataset):
    """Same constructor as the reference (graph_dataset.py:34-47) plus `device`, `seed`,
    `batch_size` and capacity knobs.  `dgl_graphs_file` may be a CSRGraph, a list of
    CSRGraphs or an .npz path."""

    def __init__(self, rw_hops=64, restart_prob=0.8, positional_embedding_size=32,
                 step_dist=[1.0, 0.0, 0.0], num_workers=1, dgl_graphs_file="./data/small.bin",
                 num_samples=10000, num_copies=1, graph_transform=None, aug="rwr", num_neighbors=5,
                 device="cuda", seed=0, batch_size=32, node_cap=None, edge_cap=None, budget_cap=None):
        super(LoadBalanceGraphDataset).__init__()
        assert sum(step_dist) == 1.0
        assert positional_embedding_size > 1
        if list(step_dist) != [1.0, 0.0, 0.0]:
            raise NotImplementedError("only the default step_dist=[1,0,0] (q and k share the seed, "
                                      "graph_dataset.py:39,104-106) is on the accelerated path")
        if aug != "rwr":
            raise NotImplementedError("aug='ns' is not on the accelerated path (train.py never sets it)")
        if graph_transform is not None:
            raise NotImplementedError("graph_transform is unused by train.py and unsupported here")
        self.rw_hops, self.restart_prob = rw_hops, restart_prob
        self.positional_embedding_size = positional_embedding_size
        self.step_dist, self.num_samples, self.num_neighbors = step_dist, num_samples, num_neighbors
        self.dgl_graphs_file, self.aug, self.graph_transform = dgl_graphs_file, aug, graph_transform
        graph, graph_sizes = load_graphs(dgl_graphs_file)
        # the reference's greedy size-descending worker balance (graph_dataset.py:63-76); kept for
        # API parity (.jobs) -- on device every graph of the union is resident, nothing is sharded
        assert num_workers % num_copies == 0
        jobs = [list() for _ in range(num_workers // num_copies)]
        workloads = [0] * (num_workers // num_copies)
        for idx, size in sorted(enumerate(graph_sizes), key=operator.itemgetter(1), reverse=True):
            argmin = workloads.index(min(workloads))
            workloads[argmin] += size
            jobs[argmin].append(idx)
        self.jobs = jobs * num_copies
        self.total = self.num_samples * num_workers
        self.num_workers = num_workers
        self.length = graph.num_nodes
        self.device = torch.device(device)
        self.seed = int(seed)
        self.batch_size = int(batch_size)
        _lib.require_device()
        self.graph = DeviceGraph(graph, rw_hops, restart_prob, self.seed, self.device, budget_cap=budget_cap)
        B = self.batch_size
        mb = self.graph.max_budget
        self.node_cap = int(node_cap or (B * min(mb + HOPCAP, 320) + mb + HOPCAP))
        self.edge_cap = int(edge_cap or self.node_cap * 16)
        self.buffers = BatchBuffers(B, self.node_cap, self.edge_cap, positional_embedding_size, mb,
                                    self.device)
        self.next_sample = 0

    def __len__(self):
        return self.total

    # -- one batch, fully on device (no host sync) ---------------------------------------------
    def sample_batch(self, first_sample=None, seeds=None, buffers=None, posenc=True):
        """Draw (or take) B seeds, walk, induce, batch and compute positional features for both
        views.  Returns the BatchBuffers (device).  `seeds`: optional int64 tensor [B]."""
        lib = _lib.get()
        buf = buffers or self.buffers
        B = buf.B
        st = _lib.stream_ptr()
        if first_sample is None:
            first_sample = self.next_sample
            self.next_sample += B
        if seeds is None:
            _lib.check(lib.gccb_draw_seeds(_lib.dptr(self.graph.cdf), self.graph.num_nodes,
                                           self.graph.key, int(first_sample), B, _lib.dptr(buf.seeds),
                                           _lib.dptr(buf.sample_ids), st), "gccb_draw_seeds")
        else:
            buf.seeds.copy_(seeds, non_blocking=True)
            buf.sample_ids.copy_(torch.arange(first_sample, first_sample + B, device=self.device))
        _lib.check(lib.gccb_sample_batch(C.byref(self.graph.c), _lib.dptr(buf.seeds),
                                         _lib.dptr(buf.sample_ids), C.byref(buf.c),
                                         _lib.dptr(buf.ws_sample), buf.ws_sample.numel(), st),
                   "gccb_sample_batch")
        if posenc:
            self.posenc(buf)
        return buf

    def posenc(self, buffers=None):
        """Positional features of both views of a sampled batch (data_util.py:242-281)."""
        buf = buffers or self.buffers
        _lib.check(_lib.get().gccb_posenc(C.byref(buf.c), buf.pos_dim, 1, _lib.dptr(buf.pos),
                                          _lib.dptr(buf.eigvals), _lib.dptr(buf.ws_posenc),
                                          buf.ws_posenc.numel(), _lib.stream_ptr()), "gccb_posenc")

    def __iter__(self):
        """Yields batched (graph_q, graph_k) -- what DataLoader(collate_fn=batcher()) yields in the
        reference.  One epoch = total // batch_size batches (train.py:356)."""
        for _ in range(self.total // self.batch_size):
            buf = self.sample_batch()
            yield BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1)


class NodeClassificationDataset:
    """generate.py's dataset (graph_dataset.py:279-309 on top of GraphDataset :218-275): item idx is
    NODE idx of one graph, seeds are taken in order (no sampling), both views walk from the seed
    (step_dist [1,0,0]) with budget max(rw_hops, int(deg*e/(e-1)/restart + 0.5)) -- plain degree,
    unlike the pretraining loader.  `dataset` is a CSRGraph or an .npz path (the reference's
    downloaded datasets need the network / DGL).  Iterating yields batched (graph_q, graph_k, count)
    with `count` valid pairs (the last batch is padded with the last node)."""

    def __init__(self, dataset, rw_hops=64, subgraph_size=64, restart_prob=0.8,
                 positional_embedding_size=32, step_dist=[1.0, 0.0, 0.0], device="cuda", seed=0,
                 batch_size=256, node_cap=None, edge_cap=None):
        assert positional_embedding_size > 1
        if list(step_dist) != [1.0, 0.0, 0.0]:
            raise NotImplementedError("only step_dist=[1,0,0] (generate.py never sets another)")
        self.rw_hops, self.subgraph_size, self.restart_prob = rw_hops, subgraph_size, restart_prob
        self.positional_embedding_size, self.step_dist = positional_embedding_size, step_dist
        graph, _ = load_graphs(dataset)
        self.device = torch.device(device)
        _lib.require_device()
        self.graph = DeviceGraph(graph, rw_hops, restart_prob, int(seed), self.device, budget_exponent=1.0)
        self.length = self.total = self.graph.num_nodes
        self.batch_size = B = int(min(batch_size, self.length))
        mb = self.graph.max_budget
        self.node_cap = int(node_cap or (B * min(mb + HOPCAP, 320) + mb + HOPCAP))
        self.edge_cap = int(edge_cap or self.node_cap * 16)
        self.buffers = BatchBuffers(B, self.node_cap, self.edge_cap, positional_embedding_size, mb, self.device)
        self._sampler = LoadBalanceGraphDataset.sample_batch

    def __len__(self):
        return self.length

    def __iter__(self):
        B = self.batch_size
        for start in range(0, self.length, B):
            count = min(B, self.length - start)
            seeds = torch.arange(start, start + B, device=self.device).clamp_(max=self.length - 1)
            buf = self._sampler(self, first_sample=start, seeds=seeds)
            buf.check_flags()
            yield BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1), count

    posenc = LoadBalanceGraphDataset.posenc
