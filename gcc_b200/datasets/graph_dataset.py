"""Device-resident ego-net dataset: the GPU replacement of the reference's CPU DataLoader.

Mirrors the surface of gcc/datasets/graph_dataset.py that train.py touches
(LoadBalanceGraphDataset ctor kwargs, .total, .jobs, .dgl_graphs_file, iteration
yielding (graph_q, graph_k)) -- SURVEY.md section 8b -- but sampling, induction,
positional features and batching all run as CUDA kernels over a CSR kept in HBM:

  reference (CPU worker processes)                      here (device kernels)
  __iter__: np.random.choice(p ~ deg^.75)   :85-92   -> gccb_draw_seeds
  __getitem__: budget + dgl RWR             :113-130 -> gccb_sample_batch (walk)
    step_dist key seed, dgl random_walk     :104-110 -> gccb_pair_seeds, then gccb_sample_batch_pairs
    aug="ns" neighbour sampling             :131-162 -> gccb_ns_batch
  _rwr_trace_to_dgl_graph                   data_util.py:218-239 -> gccb_sample_batch (induce)
  _add_undirected_graph_positional_embedding data_util.py:266-281 -> gccb_posenc
  batcher()/dgl.batch, pickling, H2D        data_util.py:26-32, train.py:382-383 -> (nothing: already batched on device)

Randomness is the counter-based "RWR-Philox v1" stream (DESIGN.md), so a batch is a
pure function of (run seed, sample ids) -- independent of worker count or world size.
"""
import copy
import ctypes as C
import math
import operator

import numpy as np
import torch

from .. import _capi, _lib
from . import synthetic
from .data_util import BatchedSubgraphs

HOPCAP = 64
NS_NODE_CAP_MAX = (2 ** 31 - 1) // 256 - 1   # gccb_ns_batch: an ego-net over its cap counts node_cap + 1 vertices


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


def walk_capacity(B, max_budget, node_cap=None, edge_cap=None, clip=None):
    """(node_cap, edge_cap) for B walks of budget <= max_budget, unless given: B ego-nets of max_budget + HOPCAP
    vertices (on average at most `clip`, if given) plus one more, and 16 edge slots per vertex."""
    per = max_budget + HOPCAP
    node_cap = int(node_cap or B * (per if clip is None else min(per, clip)) + per)
    return node_cap, int(edge_cap or node_cap * 16)


class BatchBuffers:
    """Caller-owned device memory behind one gccb_batch_t (both views of B pairs).  max_budget sizes the
    sampler's workspace; None for buffers that only whole-graph batches fill (gccb_gather_graphs needs none)."""

    def __init__(self, B, node_cap, edge_cap, pos_dim, max_budget, device):
        lib = _lib.get()
        i32 = dict(dtype=torch.int32, device=device)
        self.B, self.node_cap, self.edge_cap, self.pos_dim = B, node_cap, edge_cap, pos_dim
        self.max_budget = max_budget
        self._narrowed = {}
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
        self.seeds_k = torch.zeros(B, dtype=torch.int64, device=device)      # key-view seeds of step_dist
        self.sample_ids = torch.zeros(B, dtype=torch.int64, device=device)
        ws = lib.gccb_sample_batch_workspace(B, max_budget, edge_cap) if max_budget is not None else 0
        self.ws_sample = torch.zeros(max(ws, 8), dtype=torch.uint8, device=device)
        self.ws_posenc = torch.zeros(max(lib.gccb_posenc_workspace(B, node_cap), 8),
                                     dtype=torch.uint8, device=device)
        self.c = self._batch_struct()

    def _batch_struct(self):
        return _capi.Batch(self.B, self.node_cap, self.edge_cap, 0, self.node_off.data_ptr(),
                           self.edge_off.data_ptr(), self.indptr.data_ptr(),
                           self.indices.data_ptr(), self.sub_deg.data_ptr(),
                           self.graph_id.data_ptr(), self.orig_id.data_ptr(),
                           self.counters.data_ptr(), self.flags.data_ptr())

    def narrow(self, b):
        """The same memory as a batch of b <= B pairs (the short last batch of an epoch): node_off / edge_off
        laid out [2][b+1] and counters [2b][4] at the front of the full arrays, every per-node array, the flag
        word and the workspaces shared.  Cached per b; narrow(B) is these buffers."""
        if b == self.B:
            return self
        if not 0 < b < self.B:
            raise ValueError("a batch of %d pairs does not fit buffers of %d" % (b, self.B))
        if b not in self._narrowed:
            s = copy.copy(self)
            s.B, s._narrowed = b, {}
            s.node_off = self.node_off.view(-1)[:2 * (b + 1)].view(2, b + 1)
            s.edge_off = self.edge_off.view(-1)[:2 * (b + 1)].view(2, b + 1)
            s.counters = self.counters[:2 * b]
            s.eigvals = self.eigvals[:2 * b]
            s.seeds, s.seeds_k, s.sample_ids = self.seeds[:b], self.seeds_k[:b], self.sample_ids[:b]
            s.c = s._batch_struct()
            self._narrowed[b] = s
        return self._narrowed[b]

    def posenc(self):
        """Positional features of both views of the batch these buffers hold (data_util.py:242-281), on the
        current stream."""
        _lib.check(_lib.get().gccb_posenc(C.byref(self.c), self.pos_dim, 1, _lib.dptr(self.pos),
                                          _lib.dptr(self.eigvals), _lib.dptr(self.ws_posenc),
                                          self.ws_posenc.numel(), _lib.stream_ptr()), "gccb_posenc")

    def mark_absent(self, view):
        """Mark view `view` absent for the eigensolver, which then solves the other view alone: zero offsets and
        counters, node_off[view, B] = -1 (posenc.cu classify kernel)."""
        self.node_off[view].zero_()
        self.edge_off[view].zero_()
        self.node_off[view, self.B] = -1
        self.counters[view * self.B:(view + 1) * self.B].zero_()

    def eig_debug(self):
        """(iterations, worst residual) per ego-net of the last gccb_posenc on these buffers, read
        from the debug area at the start of its workspace (posenc.cu: phase[2B][8] int64 | iters[2B] int32 |
        res[2B] float32).  Ego-nets solved by the dense tridiagonal solver (a direct method) report 0
        iterations and their measured residual."""
        n = 2 * self.B
        ws = self.ws_posenc
        return ws[64 * n:68 * n].view(torch.int32).clone(), ws[68 * n:72 * n].view(torch.float32).clone()

    def eig_phases(self):
        """[2B][8] int64 phase cycle counters per ego-net of the last gccb_posenc (thread 0 of each CTA, rank 0 of
        each cluster), from the same debug area; posenc.cu names the phases of each solver."""
        n = 2 * self.B
        return self.ws_posenc[:64 * n].view(torch.int64).view(n, 8).clone()

    def check_flags(self):
        """Host sync: raise on any device-side failure flag.  Eigensolver non-convergence is not
        fatal (the reference itself falls back to zeros after 10 ARPACK retries,
        data_util.py:249-257): it is counted and reported once."""
        f = int(self.flags.item())
        if f:
            self.flags.zero_()
            self.raise_flags(f)

    def raise_flags(self, f, where=""):
        """Interpret a flag word already read from these buffers: warn once on eigensolver non-convergence, raise
        GccbError (prefixed by `where`) on any other flag."""
        if f & _capi.FLAG_EIG_NOCONV:
            self.eig_noconv_events = getattr(self, "eig_noconv_events", 0) + 1
            if self.eig_noconv_events == 1:
                import warnings
                warnings.warn("gcc_b200: an ego-net eigensolve hit its iteration limit "
                              "with a residual above 2e-3; features kept as is")
            f &= ~_capi.FLAG_EIG_NOCONV
        if f:
            raise _lib.GccbError(where + "device flags: " + "; ".join(
                n for b, n in _capi.FLAG_NAMES.items() if f & b))


def step_cdf(step_dist):
    """float64 CDF of step_dist (the number of hops between the q and k seeds, graph_dataset.py:104-110), or None
    for the default [1, 0, 0] (both views share the seed).  Lengths 1 to 3, as the reference's random_walk allows."""
    p = [float(x) for x in step_dist]
    if not 1 <= len(p) <= 3 or min(p) < 0.0 or abs(sum(p) - 1.0) > 1e-9:
        raise ValueError("step_dist must hold 1 to 3 probabilities summing to 1, got %r" % (step_dist,))
    if p[0] == 1.0:
        return None
    cdf = np.cumsum(np.array(p, dtype=np.float64))
    return np.ascontiguousarray(cdf / cdf[-1])


def sample_pairs(ds, buf, first_sample, seeds=None, sample_ids=None):
    """Both views of buf's B pairs with sample ids first_sample.. (or `sample_ids`, device int64 [B], with given
    seeds), walked on ds.graph with no host sync.  Seeds: drawn
    (gccb_draw_seeds), or `seeds` (device int64 [B], or buf.seeds already written).  Views: by ds.step_cdf (None: the
    k view shares the seed; else gccb_pair_seeds draws buf.seeds_k) and ds.aug ("rwr": gccb_sample_batch, or
    gccb_sample_batch_pairs for separate seeds; "ns": gccb_ns_batch).  Returns buf."""
    lib, st, g = _lib.get(), _lib.stream_ptr(), ds.graph
    if seeds is None:
        _lib.check(lib.gccb_draw_seeds(_lib.dptr(g.cdf), g.num_nodes, g.key, int(first_sample), buf.B,
                                       _lib.dptr(buf.seeds), _lib.dptr(buf.sample_ids), st), "gccb_draw_seeds")
    else:
        if seeds is not buf.seeds:
            buf.seeds.copy_(seeds, non_blocking=True)
        if sample_ids is not None:
            buf.sample_ids.copy_(sample_ids, non_blocking=True)
        else:
            torch.arange(first_sample, first_sample + buf.B, device=buf.seeds.device, out=buf.sample_ids)
    cdf, aug = getattr(ds, "step_cdf", None), getattr(ds, "aug", "rwr")   # the labeled datasets: the defaults
    seeds_k = buf.seeds
    if cdf is not None:
        _lib.check(lib.gccb_pair_seeds(C.byref(g.c), cdf.ctypes.data, len(cdf), _lib.dptr(buf.seeds),
                                       _lib.dptr(buf.sample_ids), buf.B, _lib.dptr(buf.seeds_k), st),
                   "gccb_pair_seeds")
        seeds_k = buf.seeds_k
    ws = (_lib.dptr(buf.ws_sample), buf.ws_sample.numel(), st)
    if aug == "ns":
        _lib.check(lib.gccb_ns_batch(C.byref(g.c), _lib.dptr(buf.seeds), _lib.dptr(seeds_k), _lib.dptr(buf.sample_ids),
                                     ds.rw_hops, ds.num_neighbors, C.byref(buf.c), *ws), "gccb_ns_batch")
    elif seeds_k is buf.seeds:
        _lib.check(lib.gccb_sample_batch(C.byref(g.c), _lib.dptr(buf.seeds), _lib.dptr(buf.sample_ids),
                                         C.byref(buf.c), *ws), "gccb_sample_batch")
    else:
        _lib.check(lib.gccb_sample_batch_pairs(C.byref(g.c), _lib.dptr(buf.seeds), _lib.dptr(seeds_k),
                                               _lib.dptr(buf.sample_ids), C.byref(buf.c), *ws),
                   "gccb_sample_batch_pairs")
    return buf


class LoadBalanceGraphDataset(torch.utils.data.IterableDataset):
    """Same constructor as the reference (graph_dataset.py:34-47) plus `device`, `seed`,
    `batch_size` and capacity knobs.  `dgl_graphs_file` may be a CSRGraph, a list of
    CSRGraphs or an .npz path.

    step_dist = [p0, p1, p2]: the k view's seed is the end of a 0-, 1- or 2-hop uniform walk from the q seed, drawn
    per sample on the device; both views keep the q seed's walk budget (graph_dataset.py:104-130).  aug="ns" replaces
    RWR by neighbour sampling: rw_hops layers, each expanding the previous one by at most num_neighbors neighbours
    per vertex (:131-162).  With the reference's default rw_hops (train.py: 256) that reaches most of a component;
    an ego-net holds at most gccb_ns_ego_cap(num_neighbors) vertices (4096 at num_neighbors = 5) and a view at most
    node_cap, and a view that does not fit is skipped like any overflowing batch."""

    def __init__(self, rw_hops=64, restart_prob=0.8, positional_embedding_size=32,
                 step_dist=[1.0, 0.0, 0.0], num_workers=1, dgl_graphs_file="./data/small.bin",
                 num_samples=10000, num_copies=1, graph_transform=None, aug="rwr", num_neighbors=5,
                 device="cuda", seed=0, batch_size=32, node_cap=None, edge_cap=None, budget_cap=None):
        super(LoadBalanceGraphDataset).__init__()
        assert sum(step_dist) == 1.0
        assert positional_embedding_size > 1
        self.step_cdf = step_cdf(step_dist)
        if aug not in ("rwr", "ns"):
            raise NotImplementedError("aug=%r: the reference defines 'rwr' and 'ns'" % (aug,))
        if aug == "ns" and int(num_neighbors) < 1:
            raise ValueError("aug='ns' needs num_neighbors >= 1")
        if graph_transform is not None:
            raise NotImplementedError("graph_transform is an arbitrary callable on DGLGraphs: it cannot run on the "
                                      "device and is unsupported here")
        self.rw_hops, self.restart_prob = rw_hops, restart_prob
        self.positional_embedding_size = positional_embedding_size
        self.step_dist, self.num_samples, self.num_neighbors = step_dist, num_samples, int(num_neighbors)
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
        self.node_cap, self.edge_cap = walk_capacity(B, mb, node_cap, edge_cap, clip=320)
        if aug == "ns":
            # the ns workspace holds ego-nets of up to ego_cap vertices: sizing the buffers' sampler workspace as for
            # that walk budget gives every copy of them (PretrainEngine's run-ahead ring) room for it
            ego_cap = int(_lib.get().gccb_ns_ego_cap(self.num_neighbors))
            if ego_cap == 0:
                raise ValueError("num_neighbors=%d is too large for aug='ns'" % self.num_neighbors)
            if self.node_cap > NS_NODE_CAP_MAX:
                raise ValueError("aug='ns' takes node_cap <= %d, got %d" % (NS_NODE_CAP_MAX, self.node_cap))
            mb = max(mb, ego_cap)
        self.buffers = BatchBuffers(B, self.node_cap, self.edge_cap, positional_embedding_size, mb,
                                    self.device)
        self.next_sample = 0

    def __len__(self):
        return self.total

    # -- one batch, fully on device (no host sync) ---------------------------------------------
    def sample_batch(self, first_sample=None, seeds=None, buffers=None, posenc=True):
        """Draw (or take) B seeds, walk, induce, batch and compute positional features for both
        views.  Returns the BatchBuffers (device).  `seeds`: optional int64 tensor [B]."""
        buf = buffers or self.buffers
        if first_sample is None:
            first_sample = self.next_sample
            self.next_sample += buf.B
        sample_pairs(self, buf, first_sample, seeds)
        if posenc:
            buf.posenc()
        return buf

    def posenc(self, buffers=None):
        """Positional features of both views of a sampled batch (BatchBuffers.posenc)."""
        (buffers or self.buffers).posenc()

    def __iter__(self):
        """Yields batched (graph_q, graph_k) -- what DataLoader(collate_fn=batcher()) yields in the
        reference.  One epoch = total // batch_size batches (train.py:356)."""
        for _ in range(self.total // self.batch_size):
            buf = self.sample_batch()
            yield BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1)


class _EpochOrder:
    """Pretraining on a downstream dataset (train.py:547-586): the reference's map-style DataLoader with
    shuffle=False, drop_last=False.  An epoch is items 0..total-1 in order, in batches of B; the last one holds
    total mod B items when that is not 0.  PretrainEngine numbers its batches j = 0, 1, ... and asks for batch j
    with first_sample = j * B (parallel.first_sample_id on one GPU); j counts on across epochs.  The reference
    trains these datasets on one GPU only, so the engine refuses world_size > 1 for them."""

    epoch_ordered = True

    def __len__(self):
        return self.length

    def posenc(self, buffers=None):
        """Positional features of both views of a batch (BatchBuffers.posenc)."""
        (buffers or self.buffers).posenc()

    def steps_per_epoch(self):
        return -(-self.total // self.batch_size)

    def _locate(self, first_sample):
        """(epoch, first item, item count) of the engine's batch that starts at first_sample."""
        B = self.batch_size
        if first_sample is None:
            first_sample = self.next_batch * B
            self.next_batch += 1
        epoch, idx = divmod(int(first_sample) // B, self.steps_per_epoch())
        a = idx * B
        return epoch, a, min(B, self.total - a)


class NodeClassificationDataset(_EpochOrder):
    """generate.py's dataset (graph_dataset.py:279-309 on top of GraphDataset :218-275): item idx is
    NODE idx of one graph, seeds are taken in order (no sampling), both views walk from the seed
    (step_dist [1,0,0]; another step_dist walks the k view from a 1- or 2-hop neighbour, graph_dataset.py:227-275)
    with budget max(rw_hops, int(deg*e/(e-1)/restart + 0.5)) of the q seed -- plain degree, unlike the pretraining
    loader.  `dataset` is a CSRGraph or an .npz path (the reference's
    downloaded datasets need the network / DGL).  Iterating yields batched (graph_q, graph_k, count)
    with `count` valid pairs (the last batch is padded with the last node).  sample_batch() is the
    pretraining interface (see _EpochOrder)."""

    def __init__(self, dataset, rw_hops=64, subgraph_size=64, restart_prob=0.8,
                 positional_embedding_size=32, step_dist=[1.0, 0.0, 0.0], device="cuda", seed=0,
                 batch_size=256, node_cap=None, edge_cap=None):
        assert positional_embedding_size > 1
        self.step_cdf = step_cdf(step_dist)
        self.aug, self.num_neighbors = "rwr", 5
        self.rw_hops, self.subgraph_size, self.restart_prob = rw_hops, subgraph_size, restart_prob
        self.positional_embedding_size, self.step_dist = positional_embedding_size, step_dist
        graph, _ = load_graphs(dataset)
        self.device = torch.device(device)
        _lib.require_device()
        self.graph = DeviceGraph(graph, rw_hops, restart_prob, int(seed), self.device, budget_exponent=1.0)
        self.length = self.total = self.graph.num_nodes
        self.batch_size = B = int(min(batch_size, self.length))
        mb = self.graph.max_budget
        self.node_cap, self.edge_cap = walk_capacity(B, mb, node_cap, edge_cap, clip=320)
        # a given capacity is a memory limit; at the default one, EmbedEngine re-runs a batch that overflows it
        self.caps_given = node_cap is not None or edge_cap is not None
        self.buffers = BatchBuffers(B, self.node_cap, self.edge_cap, positional_embedding_size, mb, self.device)
        self.next_batch = 0

    def __iter__(self):
        B = self.batch_size
        for start in range(0, self.length, B):
            count = min(B, self.length - start)
            seeds = torch.arange(start, start + B, device=self.device).clamp_(max=self.length - 1)
            buf = sample_pairs(self, self.buffers, start, seeds)
            buf.posenc()
            buf.check_flags()
            yield BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1), count

    def sample_batch(self, first_sample=None, seeds=None, buffers=None, posenc=True):
        """Batch number first_sample // B of the epoch order, on the device with no host sync: seeds are the
        epoch's items a .. a+b-1, and Philox sample id epoch * total + item gives every item fresh walk randomness
        in every epoch (sample ids are never reused).  Returns the buffers narrowed to the b pairs."""
        if seeds is not None:
            raise ValueError("a node dataset trains on its nodes in order: the seeds are not the caller's")
        epoch, a, b = self._locate(first_sample)
        buf = (buffers or self.buffers).narrow(b)
        torch.arange(a, a + b, device=self.device, out=buf.seeds)
        sample_pairs(self, buf, epoch * self.total + a, buf.seeds)
        if posenc:
            buf.posenc()
        return buf


def seed_first_union(graphs):
    """Every graph relabelled seed first -- its first maximum out-degree vertex (graph_dataset.py:361) moved to
    row 0 by labeled.seed_first -- and the set as one union CSR (the gccb_graph_set_t layout).  Returns (seeds,
    items = [(indptr, indices)] per relabelled graph, indptr, indices as union ids, node_off, edge_off), int64."""
    from .labeled import seed_first
    seeds = np.array([int(np.argmax(np.diff(g.indptr))) for g in graphs], dtype=np.int64)
    items = [seed_first(g.indptr, g.indices, s)[:2] for g, s in zip(graphs, seeds)]
    node_off = np.concatenate([[0], np.cumsum([len(ip) - 1 for ip, _ in items])]).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum([len(ix) for _, ix in items])]).astype(np.int64)
    indptr = np.concatenate([ip[:-1] + e for (ip, _), e in zip(items, edge_off)] + [edge_off[-1:]])
    indices = np.concatenate([np.asarray(ix, dtype=np.int64) + a for (_, ix), a in zip(items, node_off)])
    return seeds, items, indptr.astype(np.int64), indices, node_off, edge_off


def first_bad_graph(indptr, indices, node_off):
    """The first graph of a union CSR (host arrays) holding a row that is not non-decreasing or that names a vertex
    outside the graph -- what gccb_seed_first_union reports as GCCB_FLAG_BAD_ROW -- or None."""
    indptr, node_off = np.asarray(indptr, np.int64), np.asarray(node_off, np.int64)
    indices = np.asarray(indices, np.int64)
    row = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    graph = np.searchsorted(node_off, row, side="right") - 1
    bad = (indices < node_off[graph]) | (indices >= node_off[graph + 1])
    bad[1:] |= (indices[1:] < indices[:-1]) & (row[1:] == row[:-1])
    i = np.flatnonzero(bad)
    return int(graph[i[0]]) if len(i) else None


def sorted_rows(graph):
    """graph with every row non-decreasing (a row's entries reordered, as seed_first orders them); graph itself when
    its rows already are."""
    indptr, indices = np.asarray(graph.indptr, np.int64), np.asarray(graph.indices)
    if len(indices) < 2:
        return graph
    start = np.zeros(len(indices), bool)
    start[indptr[:-1][np.diff(indptr) > 0]] = True
    if not ((indices[1:] < indices[:-1]) & ~start[1:]).any():
        return graph
    row = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    return synthetic.CSRGraph(indptr, indices[np.lexsort((indices, row))].astype(np.int32), graph.num_nodes,
                              graph.name)


def set_memory_error(n_nodes, n_edges, n_graphs, free):
    """The message refusing a whole-graph set whose union CSR and its relabelled copy (int64 offsets, int32 ids, int64
    graph offsets and seeds) do not fit in `free` bytes of device memory, or None when they fit."""
    csr = 8 * (n_nodes + 1) + 4 * n_edges
    need = 2 * csr + 8 * (3 * n_graphs + 2)
    if need <= free:
        return None
    return ("a set of %d graphs (%d vertices, %d edge entries) needs %.2f GB of device memory for its union CSR and "
            "its relabelled copy (%.2f GB each), %.2f GB are free; sets that do not fit are not supported"
            % (n_graphs, n_nodes, n_edges, need / 1e9, csr / 1e9, free / 1e9))


class DeviceGraphSet:
    """Whole graphs relabelled seed first on the device (gccb_seed_first_union: seeds, node offsets and sizes kept on
    the host), their union CSR on the device as a gccb_graph_set_t, and the positional-feature cache (rows per vertex,
    eigenvalues per graph).  Datasets and their fold views share one by reference.  DeviceGraphSet(graphs) takes a list
    of CSRGraphs; from_union takes the (union, sizes) load_graphs returns, and makes no per-graph host arrays.  The
    whole union is uploaded, then relabelled into a copy; the input is freed once the copy is made."""

    def __init__(self, graphs, device):
        graphs = list(graphs)
        # seed_first_union sorts each relabelled row; the device relabel keeps rows non-decreasing, so it is given
        # non-decreasing rows
        union = sorted_rows(synthetic.disjoint_union(graphs))
        self._build(union.indptr, union.indices, [g.num_nodes for g in graphs], device, "the graph list")

    @classmethod
    def from_union(cls, union, sizes, device, name="the union"):
        """The set of graphs `sizes` (vertex counts, in order) of the union CSRGraph `union`, whose rows must be
        non-decreasing and stay inside their graph (GccbError names the first graph that breaks this)."""
        self = cls.__new__(cls)
        self._build(union.indptr, union.indices, sizes, device, name)
        return self

    def _build(self, indptr, indices, sizes, device, name):
        self.device = dev = torch.device(device)
        sizes = np.asarray(sizes, dtype=np.int64).reshape(-1)
        node_off = np.zeros(len(sizes) + 1, dtype=np.int64)
        np.cumsum(sizes, out=node_off[1:])
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        G, V = len(sizes), int(node_off[-1])
        if G == 0 or sizes.min() < 0 or len(indptr) != V + 1:
            raise ValueError("%s: graph sizes (%d graphs, %d vertices) do not match a CSR of %d rows"
                             % (name, G, V, len(indptr) - 1))
        E = int(indptr[-1])
        if V > 2 ** 31:
            raise _lib.GccbError("%s: %d vertices; union vertex ids must fit int32" % (name, V))
        _lib.require_device()
        with torch.cuda.device(dev):
            free = torch.cuda.mem_get_info()[0] + torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
        msg = set_memory_error(V, E, G, free)
        if msg:
            raise _lib.GccbError("%s: %s" % (name, msg))
        edge_off = indptr[node_off]
        to = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt)
        src_ptr, src_idx = to(indptr, torch.int64), to(indices, torch.int32)
        self.node_off, self.edge_off = to(node_off, torch.int64), to(edge_off, torch.int64)
        src = _capi.GraphSet(src_ptr.data_ptr(), src_idx.data_ptr(), self.node_off.data_ptr(),
                             self.edge_off.data_ptr(), G)
        self.indptr = torch.empty(V + 1, dtype=torch.int64, device=dev)
        self.indices = torch.empty(E, dtype=torch.int32, device=dev)
        seeds = torch.empty(G, dtype=torch.int64, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.get().gccb_seed_first_union(C.byref(src), V, E, _lib.dptr(seeds), _lib.dptr(self.indptr),
                                                        _lib.dptr(self.indices), _lib.dptr(flags), _lib.stream_ptr()),
                       "gccb_seed_first_union")
        if int(flags.item()):
            g = first_bad_graph(indptr, np.asarray(indices), node_off)
            raise _lib.GccbError("%s: graph %d has a row that is not non-decreasing or names a vertex outside the "
                                 "graph" % (name, g))
        del src_ptr, src_idx
        self.seeds = seeds.cpu().numpy()
        self.node_off_host = node_off
        self.sizes, self.nnz = sizes, np.diff(edge_off)
        self.c = _capi.GraphSet(self.indptr.data_ptr(), self.indices.data_ptr(), self.node_off.data_ptr(),
                                self.edge_off.data_ptr(), G)
        self.features = self.eigvals = None
        self._items = None

    def __len__(self):
        return len(self.sizes)

    @property
    def items(self):
        """[(indptr int64, indices int32)] per relabelled graph in local ids, as seed_first_union lists them: copied
        from the device union on first use."""
        if self._items is None:
            ip, ix, no = self.indptr.cpu().numpy(), self.indices.cpu().numpy(), self.node_off_host
            self._items = [(ip[a:b + 1] - ip[a], (ix[ip[a]:ip[b]] - a).astype(np.int32))
                           for a, b in zip(no[:-1], no[1:])]
        return self._items

    def buffers(self, B, pos_dim):
        """BatchBuffers that hold any B graphs of the set: the capacity of the B largest, plus 8, and no sampler
        workspace (gccb_gather_graphs needs none)."""
        top = lambda counts: int(np.sort(counts)[::-1][:B].sum()) + 8
        return BatchBuffers(B, top(self.sizes), top(self.nnz), pos_dim, None, self.device)

    def gather(self, ids, buf):
        """Both views of buf's batch are the graphs `ids` (device int64 [buf.B]): gccb_gather_graphs, no host sync."""
        _lib.check(_lib.get().gccb_gather_graphs(C.byref(self.c), _lib.dptr(ids), C.byref(buf.c), _lib.stream_ptr()),
                   "gccb_gather_graphs")

    def feature_cache(self, pos_dim, B):
        """Positional features of every vertex of the union [vertices][pos_dim] (and self.eigvals [graphs][pos_dim]),
        computed on first use, in batches of B consecutive ids, whose rows are the union's rows in order.  The
        eigensolver is deterministic, so these are what gccb_posenc computes for a graph in any batch."""
        if self.features is None:
            no, n = self.node_off_host, len(self.sizes)
            cache = torch.empty(int(no[-1]), pos_dim, dtype=torch.float32, device=self.device)
            eigvals = torch.empty(n, pos_dim, dtype=torch.float32, device=self.device)
            full = self.buffers(B, pos_dim)
            ids = torch.arange(n, dtype=torch.int64, device=self.device)
            for a in range(0, n, B):
                b = min(B, n - a)
                buf = full.narrow(b)
                self.gather(ids[a:a + b], buf)
                buf.mark_absent(1)
                buf.posenc()
                cache[no[a]:no[a + b]].copy_(buf.pos[0, :no[a + b] - no[a]])
                eigvals[a:a + b].copy_(buf.eigvals[:b])
            full.check_flags()
            self.features, self.eigvals = cache, eigvals
        return self.features

    def gather_features(self, ids, buf):
        """View 0's positional rows (gccb_gather_features) and eigenvalues of the graphs `ids` (device int64 [buf.B])
        from the feature cache, which feature_cache() has built.  No host sync."""
        _lib.check(_lib.get().gccb_gather_features(C.byref(self.c), _lib.dptr(ids), C.byref(buf.c), 0,
                                                   _lib.dptr(self.features), buf.pos_dim, _lib.dptr(buf.pos),
                                                   _lib.stream_ptr()), "gccb_gather_features")
        torch.index_select(self.eigvals, 0, ids, out=buf.eigvals[:buf.B])


INT32_MAX = 2 ** 31 - 1     # the batch layout's offsets are int32


def whole_graph_plan(sizes, nnz, ids, B):
    """(node_cap, edge_cap) of buffers that hold every batch of whole graphs `ids` (graph ids, in order; batches are
    every B of them): the largest batch's vertex and edge-entry totals, plus 8.  GccbError names a batch that does not
    fit the int32 batch layout, and its largest graph."""
    ids = np.asarray(ids, dtype=np.int64)
    if not len(ids):
        return 8, 8
    starts = np.arange(0, len(ids), B)
    n = np.add.reduceat(np.asarray(sizes, np.int64)[ids], starts)
    m = np.add.reduceat(np.asarray(nnz, np.int64)[ids], starts)
    node_cap, edge_cap = int(n.max()) + 8, int(m.max()) + 8
    if max(node_cap, edge_cap) > INT32_MAX:
        t = int(np.argmax(np.maximum(n, m)))
        chunk = ids[t * B:(t + 1) * B]
        big = int(chunk[np.argmax(np.asarray(nnz, np.int64)[chunk])])
        raise _lib.GccbError("batch of rows %d..%d (graph ids %d..%d): %d vertices and %d edge entries exceed the "
                             "int32 batch layout; its largest graph, %d, has %d vertices and %d edge entries"
                             % (t * B, t * B + len(chunk) - 1, chunk[0], chunk[-1], n[t], m[t], big, sizes[big],
                                nnz[big]))
    return node_cap, edge_cap


class WholeGraphDataset:
    """generate.py's whole-graph rows (graph_dataset.py:311-340 with entire_graph=True): item i is graph i of a
    corpus, relabelled seed first on the device (DeviceGraphSet), and its row is the encoding of the whole graph.
    `dataset` is a list of CSRGraphs, or the (union CSRGraph, sizes) pair load_graphs returns for a .bin or .npz
    corpus.  EmbedEngine takes it as its dataset: its ring buffers are sized exactly from the batches it runs (plan),
    and a batch's data path (prepare) is the gather of its graphs, view 1 marked absent, and the positional features
    of view 0."""

    whole_graphs = True

    def __init__(self, dataset, positional_embedding_size=32, device="cuda", batch_size=256, name="the corpus"):
        assert positional_embedding_size > 1
        self.device = torch.device(device)
        if isinstance(dataset, tuple) and len(dataset) == 2 and isinstance(dataset[0], synthetic.CSRGraph):
            self.graph_set = DeviceGraphSet.from_union(dataset[0], dataset[1], self.device, name)
        else:
            self.graph_set = DeviceGraphSet(dataset, self.device)
        self.positional_embedding_size = positional_embedding_size
        self.length = self.total = len(self.graph_set)
        self.batch_size = int(min(batch_size, self.total))

    def plan(self, ids):
        """(node_cap, edge_cap) for the batches of the graph ids `ids` (whole_graph_plan)."""
        gs = self.graph_set
        return whole_graph_plan(gs.sizes, gs.nnz, ids, self.batch_size)

    def buffers(self, node_cap, edge_cap):
        return BatchBuffers(self.batch_size, node_cap, edge_cap, self.positional_embedding_size, None, self.device)

    def prepare(self, buf, ids):
        """View 0 of buf = the whole graphs `ids` (device int64 [buf.B]) with their positional features; view 1 marked
        absent, so the eigensolver solves view 0 alone.  No host sync."""
        self.graph_set.gather(ids, buf)
        buf.mark_absent(1)
        buf.posenc()
        return buf


class GraphClassificationDataset(_EpochOrder):
    """graph_dataset.py:311-340 (entire_graph=True) for pretraining: item idx is GRAPH idx, and q and k are
    both the whole graph with its seed on the first maximum out-degree vertex.  The reference also walks an
    RWR trace per view and then discards it; nothing is walked here.  Each graph is relabelled seed first
    once, on the device (DeviceGraphSet), and the set lives there as one union CSR; a batch is
    gccb_gather_graphs of the epoch's next graph ids.  Positional features come from a deterministic
    eigensolver, so the two views' features are identical (the reference starts ARPACK from a random vector
    per view).  `dataset` is a name of downstream.GRAPH_DSETS (TU files under ./data), a list of CSRGraphs or
    a (graphs, labels) pair; the graphs keep their listed multi-edges (downstream.graph_dataset_graphs)."""

    def __init__(self, dataset, rw_hops=64, subgraph_size=64, restart_prob=0.8, positional_embedding_size=32,
                 step_dist=[1.0, 0.0, 0.0], device="cuda", seed=0, batch_size=32):
        from . import downstream
        assert positional_embedding_size > 1
        if step_cdf(step_dist) is not None:
            raise NotImplementedError("step_dist other than [1,0,0] on whole graphs would need the k view relabelled "
                                      "seed first around another vertex, per view and batch; unsupported")
        self.rw_hops, self.subgraph_size, self.restart_prob = rw_hops, subgraph_size, restart_prob
        self.positional_embedding_size, self.step_dist = positional_embedding_size, step_dist
        self.entire_graph = True
        if isinstance(dataset, str):
            graphs, _ = downstream.graph_dataset_graphs(dataset)
        elif isinstance(dataset, tuple) and len(dataset) == 2:
            graphs = list(dataset[0])
        else:
            graphs = list(dataset)
        self.length = self.total = len(graphs)
        self.device = torch.device(device)
        _lib.require_device()
        self.graph_set = DeviceGraphSet(graphs, self.device)
        self.seeds = self.graph_set.seeds                                    # each item's seed
        self.batch_size = B = int(min(batch_size, self.total))
        self.buffers = self.graph_set.buffers(B, positional_embedding_size)
        self.node_cap, self.edge_cap = self.buffers.node_cap, self.buffers.edge_cap
        self.next_batch = 0

    @property
    def items(self):
        """Each item's relabelled graph (DeviceGraphSet.items)."""
        return self.graph_set.items

    def sample_batch(self, first_sample=None, seeds=None, buffers=None, posenc=True):
        """Batch number first_sample // B of the epoch order: graphs a .. a+b-1 in both views, on the device with
        no host sync.  Returns the buffers narrowed to the b pairs."""
        if seeds is not None:
            raise ValueError("a graph dataset trains on its graphs in order: the seeds are not the caller's")
        _, a, b = self._locate(first_sample)
        buf = (buffers or self.buffers).narrow(b)
        torch.arange(a, a + b, device=self.device, out=buf.seeds)
        self.graph_set.gather(buf.seeds, buf)
        if posenc:
            buf.posenc()
        return buf
