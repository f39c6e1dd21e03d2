"""Labeled datasets of the finetune loop (reference: gcc/datasets/graph_dataset.py:342-433,
gcc/datasets/data_util.py:35-113,227-236, train.py:516-545).

  reference                                              here
  NodeClassificationDatasetLabeled.__getitem__ :398-424  ego-net of node idx, budget = rw_hops (NOT the degree
      (one RWR trace of max_nodes_per_seed=rw_hops,        formula: :412), sampled / induced / encoded by the same
      _rwr_trace_to_dgl_graph, label = y[idx].argmax())    device kernels as pretraining; only view 0 is used
  GraphClassificationDatasetLabeled.getitem :359-378     entire_graph=True: the subgraph is the WHOLE graph
      (entire_graph=True, seed = argmax out-degree,        (data_util.py:227-236), the seed one-hot sits on the
      cached in self.dict at construction :355)            max-degree node.  The device batch layout marks row 0 of
                                                           each graph as the seed, so each graph is relabelled once
                                                           (seed first, on the device); GIN, sum pooling and the
                                                           eigenvector features are permutation-equivariant.
  labeled_batcher() data_util.py:35-41                   batches(): (BatchedSubgraphs, LongTensor labels)
  Edgelist data_util.py:61-113                           Edgelist (same file formats, own parser)
  TUDataset (dgl.data, downloads)                        read_tu_dataset (the public TU text layout) or an .npz bundle

The reference downloads its datasets; there is no network here, so `dataset` may also be an in-memory
object -- (CSRGraph, labels) / (list[CSRGraph], labels) -- or a path.
"""
import copy
import os
from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from . import synthetic
from .data_util import BatchedSubgraphs
from .graph_dataset import BatchBuffers, DeviceGraph, DeviceGraphSet, sample_pairs, walk_capacity

Data = namedtuple("Data", ["x", "edge_index", "y"])          # data_util.py:44

GRAPH_CLASSIFICATION_DSETS = ["collab", "imdb-binary", "imdb-multi", "rdt-b", "rdt-5k"]   # train.py:37
_TU_NAMES = {"imdb-binary": "IMDB-BINARY", "imdb-multi": "IMDB-MULTI", "rdt-b": "REDDIT-BINARY",
             "rdt-5k": "REDDIT-MULTI-5K", "collab": "COLLAB"}                                # data_util.py:48-54
_EDGELIST_NAMES = {                                                                         # data_util.py:193-211
    "usa_airport": ("data/struc2vec/", "usa-airports"), "brazil_airport": ("data/struc2vec/", "brazil-airports"),
    "europe_airport": ("data/struc2vec/", "europe-airports"),
    "h-index-rand-1": ("data/hindex/", "aminer_hindex_rand1_5000"),
    "h-index-top-1": ("data/hindex/", "aminer_hindex_top1_5000"),
    "h-index": ("data/hindex/", "aminer_hindex_rand20intop200_5000")}


class Edgelist:
    """`<root>/<name>.edgelist` ("u v" per line) + `<name>.nodelabel` ("u label" per line): nodes are
    numbered in order of first appearance, every edge is stored in both directions, labels are numbered in
    order of first appearance -- except the h-index sets, whose label is (value > median)
    (data_util.py:61-113).  .data.y is one-hot [num_nodes, num_labels]."""

    def __init__(self, root, name):
        self.name = name
        node2id, pairs = {}, []
        with open(os.path.join(root, name + ".edgelist")) as f:
            for line in f:
                if not line.strip():
                    continue
                u, v = (int(t) for t in line.split()[:2])
                for w in (u, v):
                    if w not in node2id:
                        node2id[w] = len(node2id)
                pairs.append((node2id[u], node2id[v]))
        n = len(node2id)
        nodes, raw = [], []
        with open(os.path.join(root, name + ".nodelabel")) as f:
            for line in f:
                if not line.strip():
                    continue
                u, lab = (int(t) for t in line.split()[:2])
                nodes.append(node2id[u])
                raw.append(lab)
        if "hindex" in name:
            med = np.median(raw)
            labels, n_labels = [int(v > med) for v in raw], len(set(raw))
        else:
            label2id = {}
            for lab in raw:
                if lab not in label2id:
                    label2id[lab] = len(label2id)
            labels, n_labels = [label2id[v] for v in raw], len(label2id)
        assert n == len(set(nodes)), "every node needs exactly one label line"
        y = torch.zeros(n, n_labels)
        y[nodes, labels] = 1
        e = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
        both = np.stack([e, e[:, ::-1]], axis=1).reshape(-1, 2)       # (u, v), (v, u), ... like the reference
        self.node2id = node2id
        self.data = Data(x=None, edge_index=torch.from_numpy(both.T.copy()), y=y)
        self.transform = None

    def get(self, idx):
        assert idx == 0
        return self.data


def graph_from_edge_index(edge_index, num_nodes=None):
    """NodeClassificationDataset._create_dgl_graph (graph_dataset.py:300-308): num_nodes = max id + 1, every
    listed edge added in both directions.  The device sampler needs a simple graph: duplicates and self loops
    are dropped like x2dgl.py does for the pretraining corpus (a multi-edge only changes walk probabilities)."""
    src, dst = (np.asarray(a, dtype=np.int64) for a in edge_index)
    n = int(max(src.max(), dst.max())) + 1 if num_nodes is None else int(num_nodes)
    return _simple_csr(src, dst, n, "edge_index")


def read_tu_dataset(root, name, multigraph=False):
    """The public TU layout: <name>_A.txt ("u, v" 1-based, both directions listed), <name>_graph_indicator.txt
    (graph id of node i, 1-based), <name>_graph_labels.txt.  Returns (list[CSRGraph], int64 labels numbered from 0
    in order of sorted distinct values, like dgl.data.TUDataset).  multigraph=True keeps every listed entry once,
    repeated pairs and self loops included, as dgl.data.TUDataset's graphs do; the default makes simple graphs."""
    base = os.path.join(root, name, name)
    ind = np.loadtxt(base + "_graph_indicator.txt", dtype=np.int64).reshape(-1) - 1
    a = np.loadtxt(base + "_A.txt", dtype=np.int64, delimiter=",").reshape(-1, 2) - 1
    raw = np.loadtxt(base + "_graph_labels.txt", dtype=np.int64).reshape(-1)
    values = np.unique(raw)
    labels = np.searchsorted(values, raw)
    n_graphs = int(ind.max()) + 1
    assert len(raw) == n_graphs
    first = np.searchsorted(ind, np.arange(n_graphs))                # node ids are grouped by graph
    sizes = np.bincount(ind, minlength=n_graphs)
    gid = ind[a[:, 0]]
    assert np.all(gid == ind[a[:, 1]]), "edge across graphs"
    graphs = []
    order = np.argsort(gid, kind="stable")
    a, gid = a[order], gid[order]
    bounds = np.searchsorted(gid, np.arange(n_graphs + 1))
    for g in range(n_graphs):
        e = a[bounds[g]:bounds[g + 1]] - first[g]
        make = _listed_csr if multigraph else _simple_csr
        graphs.append(make(e[:, 0], e[:, 1], int(sizes[g]), "%s_%d" % (name, g)))
    return graphs, labels


def _listed_csr(src, dst, n, name):
    """CSR of the directed entries src -> dst exactly as listed (rows non-decreasing), isolated vertices kept."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    order = np.lexsort((dst, src))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=indptr[1:])
    return synthetic.CSRGraph(indptr, dst[order].astype(np.int32), n, name)


def _simple_csr(src, dst, n, name):
    """Symmetric simple CSR that KEEPS isolated vertices (a whole TU graph is the subgraph; dropping nodes
    would change the sum pooling)."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    keep = src != dst
    key = np.unique(np.concatenate([src[keep] * n + dst[keep], dst[keep] * n + src[keep]]))
    s, d = key // n, key % n
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(s, minlength=n), out=indptr[1:])
    return synthetic.CSRGraph(indptr, d.astype(np.int32), n, name)


def seed_first(indptr, indices, seed):
    """Relabel one graph so that `seed` becomes node 0 and the others keep their relative order (the order
    _rwr_trace_to_dgl_graph gives an ego-net: subv = [seed] + rest, data_util.py:221-226).  Returns
    (indptr, indices, perm) with perm[new] = old; neighbour lists stay ascending in the new ids."""
    indptr = np.asarray(indptr, dtype=np.int64)
    n = len(indptr) - 1
    perm = np.concatenate([[seed], np.arange(seed), np.arange(seed + 1, n)]).astype(np.int64)
    inv = np.empty(n, dtype=np.int64)
    inv[perm] = np.arange(n)
    deg = np.diff(indptr)[perm]
    new_ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=new_ptr[1:])
    new_idx = np.empty(len(indices), dtype=np.int32)
    for new, old in enumerate(perm):
        nb = inv[np.asarray(indices[indptr[old]:indptr[old + 1]], dtype=np.int64)]
        nb.sort()
        new_idx[new_ptr[new]:new_ptr[new + 1]] = nb
    return new_ptr, new_idx, perm


def fill_whole_graphs(buf, graphs, view=0):
    """Write whole (already relabelled) graphs into view `view` of a BatchBuffers as one batch; the other view
    is marked absent for the eigensolver (node_off[.., B] = -1, posenc.cu classify kernel).  Host-side
    assembly, the reference the tests hold gccb_gather_graphs (DeviceGraphSet.gather) to."""
    B = buf.B
    assert len(graphs) == B
    sizes = np.array([len(g[0]) - 1 for g in graphs], dtype=np.int64)
    nnz = np.array([len(g[1]) for g in graphs], dtype=np.int64)
    node_off = np.zeros(B + 1, dtype=np.int64)
    edge_off = np.zeros(B + 1, dtype=np.int64)
    np.cumsum(sizes, out=node_off[1:])
    np.cumsum(nnz, out=edge_off[1:])
    N, E = int(node_off[-1]), int(edge_off[-1])
    if N > buf.node_cap or E > buf.edge_cap:
        raise _lib.GccbError("whole-graph batch (%d nodes, %d edges) exceeds the buffers (%d, %d)"
                             % (N, E, buf.node_cap, buf.edge_cap))
    indptr = np.empty(N + 1, dtype=np.int32)
    indices = np.empty(E, dtype=np.int32)
    gid = np.repeat(np.arange(B, dtype=np.int32), sizes)
    for g, (ip, ix) in enumerate(graphs):
        a, e = node_off[g], edge_off[g]
        indptr[a:a + sizes[g]] = e + np.asarray(ip[:-1], dtype=np.int64)
        indices[e:e + nnz[g]] = a + np.asarray(ix, dtype=np.int64)
    indptr[N] = E
    deg = np.diff(indptr).astype(np.int32)
    dev = buf.pos.device
    put = lambda dst, arr: dst.copy_(torch.from_numpy(arr).to(dev, non_blocking=True))
    put(buf.node_off[view], node_off.astype(np.int32))
    put(buf.edge_off[view], edge_off.astype(np.int32))
    put(buf.indptr[view, :N + 1], indptr)
    put(buf.indices[view, :E], indices)
    put(buf.sub_deg[view, :N], deg)
    put(buf.graph_id[view, :N], gid)
    put(buf.orig_id[view, :N], np.arange(N, dtype=np.int32))
    cnt = np.zeros((B, 4), dtype=np.int64)
    cnt[:, 0], cnt[:, 1] = sizes, nnz
    put(buf.counters[view * B:(view + 1) * B], cnt)
    BatchBuffers.mark_absent(buf, 1 - view)        # buf: BatchBuffers, or any object with its arrays
    return buf


class _LabeledBase:
    """Index-addressed dataset + the batch iterator that replaces DataLoader(Subset(dataset, idx),
    collate_fn=labeled_batcher()) (train.py:543-545,576-592)."""

    def __len__(self):
        return self.length

    def _buffers(self, B):
        if B not in self._bufs:
            self._bufs[B] = self._new_buffers(B)
        return self._bufs[B]

    def batches(self, indices=None, batch_size=None, shuffle=False, rng=None):
        """Yields (graph_q, y): graph_q a BatchedSubgraphs of len(chunk) graphs, y int64 labels on the device.
        The last batch may be smaller (DataLoader's drop_last=False)."""
        idx = np.arange(self.length) if indices is None else np.asarray(indices, dtype=np.int64)
        if shuffle:
            idx = (rng or np.random).permutation(idx)
        bs = int(batch_size or self.batch_size)
        for a in range(0, len(idx), bs):
            chunk = idx[a:a + bs]
            yield self._make_batch(chunk), torch.from_numpy(self.labels[chunk]).to(self.device)

    def _make_batch(self, chunk):
        """device_batch of the host item ids `chunk`, then a host sync that raises on a device flag."""
        buf = self.device_batch(torch.from_numpy(np.ascontiguousarray(chunk)).to(self.device))
        buf.check_flags()
        return BatchedSubgraphs(buf, 0)

    def num_batches(self, n_items, batch_size=None):
        bs = int(batch_size or self.batch_size)
        return (n_items + bs - 1) // bs

    def fold_view(self):
        """This dataset for one more cross-validation fold on the same device: the read-only device state (graph or
        graph set with its feature cache, device labels) is shared, while the BatchBuffers (and with them the
        flag word) and the sampler's next_sample counter are the fold's own and start as a freshly built dataset's
        do, so the fold draws the batches a fresh dataset would give it.  Folds on separate streams may use their
        views concurrently once the stream that built this dataset has been waited on."""
        if hasattr(self, "feature_cache"):
            self.feature_cache()                       # built now, on the stream the folds' streams wait on
        view = copy.copy(self)
        view._bufs = {}
        if hasattr(self, "next_sample"):
            view.next_sample = 0
        return view


class NodeClassificationDatasetLabeled(_LabeledBase):
    """graph_dataset.py:381-424.  `dataset`: a name of data_util.create_node_classification_dataset's Edgelist
    family (files under ./data), an Edgelist, a (CSRGraph, y) pair or an .npz with indptr / indices / y
    (y one-hot [n, C] or int labels [n])."""

    def __init__(self, dataset, rw_hops=64, subgraph_size=64, restart_prob=0.8, positional_embedding_size=32,
                 step_dist=[1.0, 0.0, 0.0], cat_prone=False, device="cuda", seed=0, batch_size=32,
                 node_cap=None, edge_cap=None):
        assert positional_embedding_size > 1
        self.rw_hops, self.subgraph_size, self.restart_prob = rw_hops, subgraph_size, restart_prob
        self.positional_embedding_size, self.step_dist = positional_embedding_size, step_dist
        graph, y = self._load(dataset)
        y = np.asarray(y)
        self.data = Data(x=None, edge_index=None, y=torch.from_numpy(y) if y.ndim == 2 else None)
        self.labels = (y.argmax(axis=1) if y.ndim == 2 else y).astype(np.int64)      # :424 / train.py:534
        self.num_classes = int(y.shape[1]) if y.ndim == 2 else int(self.labels.max()) + 1
        self.device = torch.device(device)
        _lib.require_device()
        self.labels_dev = torch.from_numpy(self.labels).to(self.device)      # FinetuneEngine's label table
        # max_nodes_per_seed = rw_hops for every seed (:412): the degree formula capped at rw_hops
        self.graph = DeviceGraph(graph, rw_hops, restart_prob, int(seed), self.device, budget_exponent=1.0,
                                 budget_cap=rw_hops)
        self.length = self.total = self.graph.num_nodes
        assert len(self.labels) == self.length
        self.batch_size = int(min(batch_size, self.length))
        self._caps = (node_cap, edge_cap)
        self._bufs = {}
        self.next_sample = 0

    @staticmethod
    def _load(dataset):
        if isinstance(dataset, Edgelist):
            return graph_from_edge_index(dataset.data.edge_index.numpy()), dataset.data.y.numpy()
        if isinstance(dataset, (tuple, list)) and len(dataset) == 2:
            return dataset[0], dataset[1]
        if isinstance(dataset, str) and dataset.endswith(".npz"):
            z = np.load(dataset)
            g = synthetic.CSRGraph(z["indptr"].astype(np.int64), z["indices"].astype(np.int32),
                                   len(z["indptr"]) - 1, dataset)
            return g, z["y"]
        if isinstance(dataset, str) and dataset in _EDGELIST_NAMES:
            e = Edgelist(*_EDGELIST_NAMES[dataset])
            return graph_from_edge_index(e.data.edge_index.numpy()), e.data.y.numpy()
        raise NotImplementedError("node classification dataset %r: pass an Edgelist, (CSRGraph, y), an .npz or one of %s"
                                  % (dataset, sorted(_EDGELIST_NAMES)))

    def _new_buffers(self, B):
        mb = self.graph.max_budget
        return BatchBuffers(B, *walk_capacity(B, mb, *self._caps), self.positional_embedding_size, mb, self.device)

    def device_batch(self, ids):
        """Ego-nets of the items `ids` (device int64 [b]) and their features, with no host sync.  A batch over its
        capacity is published empty with the buffers' flag raised; the caller reads the flag."""
        buf = self._buffers(ids.numel())
        first = self.next_sample                       # fresh walk randomness for every item drawn, like the reference
        self.next_sample += buf.B
        sample_pairs(self, buf, first, ids)
        buf.posenc()
        return buf


class GraphClassificationDatasetLabeled(_LabeledBase):
    """graph_dataset.py:342-378.  `dataset`: one of GRAPH_CLASSIFICATION_DSETS (TU files under ./data/<NAME>/),
    a (list[CSRGraph], labels) pair or an .npz with indptr / indices / graph_sizes / graph_labels of the
    disjoint union."""

    def __init__(self, dataset, rw_hops=64, subgraph_size=64, restart_prob=0.8, positional_embedding_size=32,
                 step_dist=[1.0, 0.0, 0.0], device="cuda", seed=0, batch_size=32):
        assert positional_embedding_size > 1
        self.rw_hops, self.subgraph_size, self.restart_prob = rw_hops, subgraph_size, restart_prob
        self.positional_embedding_size, self.step_dist = positional_embedding_size, step_dist
        self.entire_graph = True
        graphs, labels = self._load(dataset)
        self.labels = np.asarray(labels, dtype=np.int64).reshape(-1)
        self.num_classes = int(self.labels.max()) + 1                   # dataset.num_labels
        self.length = self.total = len(graphs)
        assert len(self.labels) == self.length
        self.device = torch.device(device)
        _lib.require_device()
        # the reference's self.dict (:355): every item is prepared once.  seed = argmax degree (:361, first
        # maximum), moved to row 0; the relabelled items form one union CSR on the device
        self.graph_set = DeviceGraphSet(graphs, self.device)
        self.seeds = self.graph_set.seeds                                    # each item's seed
        self.batch_size = int(min(batch_size, self.length))
        self._bufs = {}
        self.labels_dev = torch.from_numpy(self.labels).to(self.device)      # FinetuneEngine's label table

    @staticmethod
    def _load(dataset):
        if isinstance(dataset, (tuple, list)) and len(dataset) == 2:
            return list(dataset[0]), dataset[1]
        if isinstance(dataset, str) and dataset.endswith(".npz"):
            z = np.load(dataset)
            indptr, indices, sizes = z["indptr"].astype(np.int64), z["indices"].astype(np.int64), z["graph_sizes"]
            graphs, a = [], 0
            for i, n in enumerate(sizes):
                ip = indptr[a:a + n + 1]
                graphs.append(synthetic.CSRGraph(ip - ip[0], (indices[ip[0]:ip[-1]] - a).astype(np.int32), int(n),
                                                 "%s_%d" % (dataset, i)))
                a += int(n)
            return graphs, z["graph_labels"]
        if isinstance(dataset, str) and dataset in _TU_NAMES:
            return read_tu_dataset("data", _TU_NAMES[dataset])
        raise NotImplementedError("graph classification dataset %r: pass (graphs, labels), an .npz or one of %s"
                                  % (dataset, GRAPH_CLASSIFICATION_DSETS))

    @property
    def items(self):
        """Each item's relabelled graph (DeviceGraphSet.items)."""
        return self.graph_set.items

    def _new_buffers(self, B):
        return self.graph_set.buffers(B, self.positional_embedding_size)

    def feature_cache(self):
        """The graph set's feature cache (DeviceGraphSet.feature_cache), built in batches of batch_size graphs."""
        return self.graph_set.feature_cache(self.positional_embedding_size, self.batch_size)

    def device_batch(self, ids):
        """The whole graphs `ids` (device int64 [b]) with no host sync: the union gather and, in view 0, the cached
        features.  The buffers hold the b largest graphs, so a batch never overflows."""
        buf = self._buffers(ids.numel())
        self.feature_cache()
        self.graph_set.gather(ids, buf)
        self.graph_set.gather_features(ids, buf)
        return buf


def labeled_batcher():
    """API parity with data_util.py:35-41: batches() already yields (graph_q, labels)."""
    def batcher_dev(batch):
        return batch[0] if isinstance(batch, list) and len(batch) == 1 else batch
    return batcher_dev
