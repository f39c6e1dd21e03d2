"""Generate tests/golden/x2dgl_golden.npz by running the REAL reference converter, gcc/utils/x2dgl.py of a reference
checkout, under tests/golden/dgl_stub.py -- its yuxiao_kdd17_graph_to_dgl and its __main__ flow (directory scan of
the `todo` names, sort by vertex count, save_graphs with "graph_sizes").

Run:  GCC_REFERENCE=<checkout of THUDM/GCC> python tests/golden/make_golden_x2dgl.py

The fixtures are small seeded .lscc files named after `todo` entries, with self loops, duplicates in both
orientations, isolated vertices and ids at n - 1.  The stub's graph class gains what x2dgl.py calls; the DGL 0.4.3
semantics it restates are [M] (recalled, not checked against DGL):
  [M] DGLGraph().from_scipy_sparse_matrix(A): one edge row -> col per stored entry of A, in CSR order;
  [M] remove_nodes(vids): the listed vertices and their edges go, the others are relabelled 0.. in increasing
      old-id order, edge order kept;
  [M] save_graphs(filename, g_list, labels): captured here instead of written.
Test infrastructure, not product.
"""
import os
import runpy
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import dgl_stub  # noqa: E402

FIXTURES = [  # (todo name, n, m, seed)
    ("ca-DBLP-NetRep.txt.lpm.lscc", 40, 70, 1),
    ("ca-IMDB-NetRep.txt.lpm.lscc", 25, 40, 2),
    ("soc-Academia-NetRep.txt.lpm.lscc", 60, 140, 3),
]


class X2dglGraph(dgl_stub.StubGraph):
    def __init__(self):
        super().__init__(0, [], [])

    def from_scipy_sparse_matrix(self, A):
        A = A.tocsr()
        row = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
        self.n, self.src, self.dst = A.shape[0], row.astype(np.int64), A.indices.astype(np.int64)

    def remove_nodes(self, vids):
        gone = np.zeros(self.n, bool)
        gone[np.atleast_1d(np.asarray(vids, dtype=np.int64))] = True
        new_id = np.cumsum(~gone) - 1
        keep = ~gone[self.src] & ~gone[self.dst]
        self.src, self.dst = new_id[self.src[keep]], new_id[self.dst[keep]]
        self.n = int((~gone).sum())

    def __repr__(self):
        return "DGLGraph(num_nodes=%d, num_edges=%d)" % (self.n, len(self.src))


saved = {}


def save_graphs(filename, g_list, labels=None):
    saved.update(filename=filename, graphs=list(g_list), labels=labels)


def make_lscc(n, m, seed):
    rng = np.random.default_rng(seed)
    hi = n - n // 5                                  # the top fifth of the ids are isolated ...
    u = rng.integers(0, hi, m)
    v = rng.integers(0, hi, m)
    v[: m // 10] = u[: m // 10]                      # self loops
    u[m // 10: m // 10 + 5], v[m // 10: m // 10 + 5] = v[:5] + 1, u[:5]
    u[-4:], v[-4:] = v[-8:-4], u[-8:-4]              # duplicates in the other orientation
    u[-5], v[-5] = n - 1, 0                          # ... except n - 1
    lines = ["n %d" % n] + ["%d %d" % (i, 1000 + i) for i in range(n)] + ["m %d" % m]
    lines += ["%d %d %d" % (a, b, rng.integers(1, 5)) for a, b in zip(u, v)]
    return ("\n".join(lines) + "\n").encode()


def main(ref_root):
    script = os.path.join(ref_root, "gcc", "utils", "x2dgl.py")
    dgl = dgl_stub.install()
    dgl.DGLGraph = X2dglGraph
    dgl.data.utils.save_graphs = save_graphs
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, n, m, seed in FIXTURES:
            text = make_lscc(n, m, seed)
            with open(os.path.join(d, name), "wb") as f:
                f.write(text)
            out["text_" + name] = np.frombuffer(text, np.uint8)
        # the written graphs carry no file name: map them back through each file's vertex count
        convert = runpy.run_path(script, run_name="x2dgl_ref")["yuxiao_kdd17_graph_to_dgl"]
        name_of = {convert(os.path.join(d, name)).number_of_nodes(): name for name, *_ in FIXTURES}
        assert len(name_of) == len(FIXTURES), "fixture vertex counts must be distinct"
        argv = sys.argv
        sys.argv = ["x2dgl.py", "--graph-dir", d, "--save-file", os.path.join(d, "small.bin"), "--embed-dim", "64"]
        try:
            runpy.run_path(script, run_name="__main__")
        finally:
            sys.argv = argv
    graphs = saved["graphs"]
    sizes = saved["labels"]["graph_sizes"]
    assert isinstance(sizes, torch.Tensor)
    for i, g in enumerate(graphs):
        order = np.lexsort((g.src, g.dst))           # in-CSR: row = destination, neighbours ascending
        indptr = np.zeros(g.n + 1, np.int64)
        np.cumsum(np.bincount(g.dst, minlength=g.n), out=indptr[1:])
        out["file%d" % i] = np.array(name_of[g.n])
        out["indptr%d" % i] = indptr
        out["indices%d" % i] = g.src[order].astype(np.int32)
    out["graph_sizes"] = sizes.numpy().astype(np.int64)
    out["count"] = np.array(len(graphs))
    np.savez_compressed(os.path.join(HERE, "x2dgl_golden.npz"), **out)
    return graphs


if __name__ == "__main__":
    REF = os.environ.get("GCC_REFERENCE")
    if not REF:
        raise SystemExit("set GCC_REFERENCE to a checkout of THUDM/GCC")
    main(REF)
