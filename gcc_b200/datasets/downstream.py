"""Downstream datasets of the reference's "freeze" evaluation (generate.py + gcc/tasks), as multigraphs.

  reference                                                  here
  NodeClassificationDataset._create_dgl_graph                multigraph_from_edge_index: num_nodes = max id + 1,
      (graph_dataset.py:301-309)                                 every listed pair added in both directions,
                                                                 parallel edges and self loops kept (DGL keeps them)
  SSSingleDataset / SSDataset (data_util.py:111-191)         SSSingleDataset / SSDataset: Panther .graph / .dict
  create_node_classification_dataset (data_util.py:193-215)  create_node_classification_dataset
  TUDataset graph_lists (dgl.data.tu)                        labeled.read_tu_dataset(..., multigraph=True)

The Edgelist files (airports, h-index) and the Panther files already list every edge in both directions, so the
builder's second direction doubles each of them, and a Panther edge of weight t appears 2t times: that is what the
reference's DGL graph holds, so walks, induced degrees, GIN sums and positional features all see those
multiplicities.  The finetune loader (labeled.NodeClassificationDatasetLabeled) still de-duplicates; see DESIGN.md.
"""
import os

import numpy as np
import torch

from .labeled import _EDGELIST_NAMES, _TU_NAMES, Data, Edgelist, _listed_csr, read_tu_dataset

SS_DSETS = ["kdd", "icdm", "sigir", "cikm", "sigmod", "icde"]                    # data_util.py:212
NODE_DSETS = list(_EDGELIST_NAMES) + SS_DSETS
GRAPH_DSETS = list(_TU_NAMES)


def multigraph_from_edge_index(edge_index, name="edge_index"):
    """_create_dgl_graph (graph_dataset.py:301-309) as a CSR: row v lists the heads of v's out-edges,
    non-decreasing, a neighbour repeated once per parallel edge (the gccb_graph_t contract)."""
    src, dst = (np.asarray(a, dtype=np.int64).reshape(-1) for a in edge_index)
    n = int(max(src.max(), dst.max())) + 1
    return _listed_csr(np.concatenate([src, dst]), np.concatenate([dst, src]), n, name)


def _read_panther_graph(path, node2id):
    """Header line skipped, then "x y t" rows: t times (x, y) and (y, x), ids numbered in order of first
    appearance (data_util.py:121-143)."""
    pairs = []
    with open(path) as f:
        f.readline()
        for line in f:
            x, y, t = (int(v) for v in line.split())
            for w in (x, y):
                if w not in node2id:
                    node2id[w] = len(node2id)
            pairs.extend([(node2id[x], node2id[y]), (node2id[y], node2id[x])] * t)
    e = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    return torch.from_numpy(e.T.copy())


class SSSingleDataset:
    """One Panther graph `<root>/<name>.graph` (data_util.py:111-143)."""

    def __init__(self, root, name):
        self.data = Data(x=None, edge_index=_read_panther_graph(os.path.join(root, name + ".graph"), {}), y=None)
        self.transform = None

    def get(self, idx):
        assert idx == 0
        return self.data


class SSDataset:
    """Two Panther graphs and their `.dict` files ("name<TAB>id" per line; an id that no edge names is
    appended to the numbering): .data = [Data(edge_index, y=name -> node id)] x 2 (data_util.py:145-191)."""

    def __init__(self, root, name1, name2):
        self.data, self.node2id = [], []
        for name in (name1, name2):
            node2id = {}
            edge_index = _read_panther_graph(os.path.join(root, name + ".graph"), node2id)
            name_dict = {}
            with open(os.path.join(root, name + ".dict")) as f:
                for line in f:
                    key, str_x = line.split("\t")
                    x = int(str_x)
                    if x not in node2id:
                        node2id[x] = len(node2id)
                    name_dict[key] = node2id[x]
            self.data.append(Data(x=None, edge_index=edge_index, y=name_dict))
            self.node2id.append(node2id)
        self.node2id_1, self.node2id_2 = self.node2id
        self.transform = None

    def get(self, idx):
        assert idx == 0
        return self.data


def create_node_classification_dataset(name, root="data"):
    """data_util.py:193-215: airports and h-index (Edgelist), Panther graphs (SSSingleDataset)."""
    if name in _EDGELIST_NAMES:
        sub, stem = _EDGELIST_NAMES[name]
        return Edgelist(os.path.join(root, os.path.basename(sub.rstrip("/"))), stem)
    if name in SS_DSETS:
        return SSSingleDataset(os.path.join(root, "panther"), name)
    raise NotImplementedError("node dataset %r: one of %s" % (name, NODE_DSETS))


def node_dataset_graph(name, root="data"):
    """The multigraph generate.py embeds for a named node dataset."""
    return multigraph_from_edge_index(create_node_classification_dataset(name, root).data.edge_index.numpy(), name)


def graph_dataset_graphs(name, root="data"):
    """(list of multigraph CSRs, labels) of a TU set, the graphs generate.py embeds whole."""
    if name not in _TU_NAMES:
        raise NotImplementedError("graph dataset %r: one of %s" % (name, GRAPH_DSETS))
    return read_tu_dataset(root, _TU_NAMES[name], multigraph=True)
