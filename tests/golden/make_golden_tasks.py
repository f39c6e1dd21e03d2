#!/usr/bin/env python
"""Generate tests/golden/tasks_golden.npz by executing the REAL reference readers and evaluators from a checkout of
THUDM/GCC (read-only):

  - gcc.datasets.data_util: Edgelist (airports and h-index layouts), SSSingleDataset, SSDataset;
  - gcc.datasets.graph_dataset: NodeClassificationDataset._create_dgl_graph (edge lists as the DGL graph holds them);
  - gcc.tasks: NodeClassification._evaluate, GraphClassification.svc_classify, SimilaritySearch._evaluate.

The input files are small ones written here (parallel edges, Panther weights t up to 5, self loops, .dict names
without edges); their text is stored in the fixture so the tests read the very same files.  Evaluator inputs are
seeded embeddings and labels.

Stand-ins, everything else that runs is the reference's own code:
  - dgl: dgl_stub.py, as for make_golden.py; its graph gains add_nodes / add_edges here (the builder API
    _create_dgl_graph calls), keeping every added edge: DGL keeps parallel edges and self loops.
  - gcc.models.emb: its package imports the GraphWave baseline, which needs seaborn and pandas.  The stand-in package
    loads the reference's own gcc/models/emb/from_numpy.py; ProNE and GraphWave are not used.

Run:  GCC_REFERENCE=<checkout of THUDM/GCC> python tests/golden/make_golden_tasks.py
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("GCC_REFERENCE")
if not REF or not os.path.isdir(REF):
    raise SystemExit("set GCC_REFERENCE to a checkout of THUDM/GCC")
sys.path.insert(0, HERE)

import dgl_stub  # noqa: E402

dgl = dgl_stub.install()


class BuilderGraph(dgl_stub.StubGraph):
    def __init__(self):
        super().__init__(0, [], [])

    def add_nodes(self, n):
        self.n += int(n)

    def add_edges(self, src, dst):
        self.src = np.concatenate([self.src, np.asarray(src, dtype=np.int64)])
        self.dst = np.concatenate([self.dst, np.asarray(dst, dtype=np.int64)])


dgl.DGLGraph = BuilderGraph
sys.path.insert(0, REF)
emb = types.ModuleType("gcc.models.emb")
spec = importlib.util.spec_from_file_location("gcc.models.emb.from_numpy",
                                              os.path.join(REF, "gcc", "models", "emb", "from_numpy.py"))
from_numpy = importlib.util.module_from_spec(spec)
spec.loader.exec_module(from_numpy)
for k in ("Zero", "FromNumpy", "FromNumpyGraph", "FromNumpyAlign"):
    setattr(emb, k, getattr(from_numpy, k))
emb.ProNE = emb.GraphWave = None
sys.modules["gcc.models.emb"] = emb

import gcc.datasets.data_util as ref_du  # noqa: E402
import gcc.datasets.graph_dataset as ref_gd  # noqa: E402
from gcc.tasks.graph_classification import GraphClassification  # noqa: E402
from gcc.tasks.node_classification import NodeClassification  # noqa: E402
from gcc.tasks.similarity_search import SimilaritySearch  # noqa: E402


def _edgelist_text(rng, n, m, labels_of):
    """Raw ids are shuffled so that first-appearance numbering differs from them; every 7th line is repeated
    (a parallel edge), one line is a self loop."""
    raw = rng.permutation(np.arange(100, 100 + 3 * n, 3))
    lines = ["%d %d" % (raw[i], raw[(i + 1) % n]) for i in range(n)]            # a ring: every node has an edge
    for _ in range(m):
        a, b = rng.randint(0, n, 2)
        if a != b:
            lines.append("%d %d" % (raw[a], raw[b]))
    lines += lines[::7]
    lines.append("%d %d" % (raw[3], raw[3]))
    lab = ["%d %d" % (raw[i], labels_of(i)) for i in rng.permutation(n)]
    return "\n".join(lines) + "\n", "\n".join(lab) + "\n"


def _panther_text(rng, n, m, names, extra):
    raw = rng.permutation(np.arange(7, 7 + 5 * n, 5))
    rows = ["%d %d %d" % (raw[i], raw[(i + 1) % n], rng.randint(1, 6)) for i in range(n)]
    for _ in range(m):
        a, b = rng.randint(0, n, 2)
        rows.append("%d %d %d" % (raw[a], raw[b], rng.randint(1, 6)))
    rows.append("%d %d 2" % (raw[1], raw[1]))                                     # a self loop of weight 2
    graph = "%d %d\n" % (n, len(rows)) + "\n".join(rows) + "\n"
    ids = list(raw[:len(names) - extra]) + [int(raw.max()) + 11 * (i + 1) for i in range(extra)]   # ids without edges
    d = "".join("%s\t%d\n" % (nm, x) for nm, x in zip(names, ids))
    return graph, d


def _dict_arrays(prefix, d):
    keys = sorted(d)
    return {prefix + "_keys": np.array(keys), prefix + "_ids": np.array([d[k] for k in keys], np.int64)}


def main():
    rng = np.random.RandomState(20191213)
    files = {}
    files["struc2vec/usa-airports.edgelist"], files["struc2vec/usa-airports.nodelabel"] = \
        _edgelist_text(rng, 40, 90, lambda i: [11, 3, 7, 3][i % 4])
    files["hindex/aminer_hindex_rand1_5000.edgelist"], files["hindex/aminer_hindex_rand1_5000.nodelabel"] = \
        _edgelist_text(rng, 30, 60, lambda i: int(rng.randint(0, 40)))
    names = ["author%03d" % i for i in range(60)]
    files["panther/kdd.graph"], files["panther/kdd.dict"] = _panther_text(rng, 35, 50, names[:30], 3)
    files["panther/icdm.graph"], files["panther/icdm.dict"] = _panther_text(rng, 28, 40, names[10:40], 2)
    out = {"files/" + k: np.array(v) for k, v in files.items()}

    with tempfile.TemporaryDirectory() as tmp:
        for k, v in files.items():
            os.makedirs(os.path.dirname(os.path.join(tmp, k)), exist_ok=True)
            with open(os.path.join(tmp, k), "w") as f:
                f.write(v)
        for tag, sub, stem in (("usa", "struc2vec", "usa-airports"), ("hindex", "hindex", "aminer_hindex_rand1_5000")):
            e = ref_du.Edgelist(os.path.join(tmp, sub), stem)
            out[tag + "_edge_index"] = e.data.edge_index.numpy()
            out[tag + "_y"] = e.data.y.numpy()
            g = ref_gd.NodeClassificationDataset._create_dgl_graph(None, e.data)
            out[tag + "_graph_src"], out[tag + "_graph_dst"], out[tag + "_graph_n"] = g.src, g.dst, np.int64(g.n)
        s = ref_du.SSSingleDataset(os.path.join(tmp, "panther"), "kdd")
        out["kdd_edge_index"] = s.data.edge_index.numpy()
        g = ref_gd.NodeClassificationDataset._create_dgl_graph(None, s.data)
        out["kdd_graph_src"], out["kdd_graph_dst"], out["kdd_graph_n"] = g.src, g.dst, np.int64(g.n)
        ss = ref_du.SSDataset(os.path.join(tmp, "panther"), "kdd", "icdm")
        for i, d in enumerate(ss.data):
            out["ss%d_edge_index" % i] = d.edge_index.numpy()
            out.update(_dict_arrays("ss%d_dict" % i, d.y))

    # evaluators on seeded embeddings
    n, h, c = 200, 16, 4
    lab = rng.randint(0, c, n)
    y = np.zeros((n, c), np.float32)
    y[np.arange(n), lab] = 1
    multi = rng.choice(n, 30, replace=False)                     # rows with two labels: top-k with k = 2
    y[multi, (lab[multi] + 1) % c] = 1
    x = rng.randn(n, h) + 0.8 * np.eye(c, h)[lab]
    nc = NodeClassification.__new__(NodeClassification)
    nc.seed = 3
    out["nc_x"], out["nc_y"], out["nc_seed"] = x, y, np.int64(nc.seed)
    out["nc_result"] = np.float64(nc._evaluate(x, torch.Tensor(y), 10)["Micro-F1"])

    gx = rng.randn(120, h)
    gy = (gx[:, 0] + 0.5 * gx[:, 1] + 0.3 * rng.randn(120) > 0).astype(np.int64) + (gx[:, 2] > 1.2)
    gc = GraphClassification.__new__(GraphClassification)
    gc.seed = 5
    out["gc_x"], out["gc_y"], out["gc_seed"] = gx, gy, np.int64(gc.seed)
    out["gc_result"] = np.float64(gc.svc_classify(gx, gy, False)["Micro-F1"])

    e1 = rng.randn(50, h)
    perm = rng.permutation(45)
    e2 = np.concatenate([e1[perm] + 3.0 * rng.randn(45, h), rng.randn(5, h)])
    d1 = {"n%02d" % i: i for i in range(50)}
    d1["far1"] = 60                                              # beyond emb_1: filtered out
    d2 = {"n%02d" % perm[i]: i for i in range(45)}
    d2["far1"], d2["x"] = 3, 70
    out["ss_e1"], out["ss_e2"] = e1, e2
    out.update(_dict_arrays("ss_d1", d1))
    out.update(_dict_arrays("ss_d2", d2))
    res = SimilaritySearch._evaluate(None, e1.copy(), e2.copy(), d1, d2)
    out["ss_recall20"], out["ss_recall40"] = np.float64(res["Recall @ 20"]), np.float64(res["Recall @ 40"])
    print({k: float(v) for k, v in out.items() if k.endswith(("result", "recall20", "recall40"))})

    path = os.path.join(HERE, "tasks_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "(%d arrays)" % len(out))


if __name__ == "__main__":
    main()
