"""Host-only logic of whole-graph embedding: the ring's buffer plan (the largest batch that runs, not the B largest
graphs), shard boundaries over graph ids, output naming of --whole-graphs, the graph-classification labels of a TU
directory and of an .npz, the device-memory refusal, and the row contract's host helpers."""
import numpy as np
import pytest

import generate
from gcc_b200 import _lib
from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import (first_bad_graph, seed_first_union, set_memory_error, sorted_rows,
                                             whole_graph_plan)
from gcc_b200.tasks.graph_classification import graph_labels


def test_plan_is_the_largest_batch_not_the_largest_graphs():
    sizes = np.array([100, 1, 1, 1, 90, 1, 1, 1], np.int64)
    nnz = np.array([400, 0, 2, 0, 500, 2, 0, 0], np.int64)
    # batches of 4 in order: (103, 402) and (93, 502); the two largest graphs together would be (190, 900)
    assert whole_graph_plan(sizes, nnz, np.arange(8), 4) == (103 + 8, 502 + 8)
    # an id list: batches [4, 0] and [1, 1] -- the order given, repeats allowed
    assert whole_graph_plan(sizes, nnz, [4, 0, 1, 1], 2) == (190 + 8, 900 + 8)
    assert whole_graph_plan(sizes, nnz, [1, 2, 3], 2) == (2 + 8, 2 + 8)
    assert whole_graph_plan(sizes, nnz, [], 2) == (8, 8)


def test_plan_refuses_a_batch_beyond_int32():
    sizes = np.array([5, 2 ** 30, 2 ** 30, 7], np.int64)
    nnz = np.array([4, 2 ** 30, 2 ** 30 + 1, 0], np.int64)
    assert whole_graph_plan(sizes, nnz, [0, 1, 3], 1)[0] == 2 ** 30 + 8
    with pytest.raises(_lib.GccbError, match=r"rows 0\.\.1 \(graph ids 1\.\.2\).*largest graph, 2"):
        whole_graph_plan(sizes, nnz, [1, 2, 0, 3], 2)


def test_graph_id_shards_are_whole_batches():
    # 1,000 graphs in batches of 64: 16 batches over 3 shards -> 6, 5, 5
    shards = generate.split_shards(1000, 64, 3)
    assert shards == [(0, 384), (384, 704), (704, 1000)]
    assert all(lo % 64 == 0 for lo, _ in shards)


def test_whole_graph_output_names(tmp_path):
    assert generate.output_stem("corpus.bin", True) == "corpus.graphs"
    assert generate.output_stem("/a/b/corpus.npz", True) == "corpus.graphs"
    assert generate.output_stem("/a/b/corpus.bin", False) == "corpus"
    assert generate.output_stem("imdb-binary", True) == "imdb-binary"
    d = tmp_path / "MYSET"
    d.mkdir()
    assert generate.whole_graph_source(str(d)) is None                 # no MYSET_A.txt: not a TU directory
    (d / "MYSET_A.txt").write_text("1, 2\n2, 1\n")
    assert generate.whole_graph_source(str(d) + "/") == "tu-dir"
    assert generate.output_stem(str(d) + "/", True) == "MYSET"
    assert generate.whole_graph_source("imdb-binary") == "tu-name"
    assert generate.whole_graph_source("corpus.bin") is None
    base = ["--load-path", "x.pth", "--dataset", "c.bin"]
    assert generate.parse_args(base).whole_graphs is False
    assert generate.parse_args(base + ["--whole-graphs"]).whole_graphs is True


def test_graph_classification_labels(tmp_path):
    d = tmp_path / "MYSET"
    d.mkdir()
    (d / "MYSET_graph_labels.txt").write_text("7\n-1\n7\n3\n")
    assert graph_labels(str(d)).tolist() == [2, 0, 2, 1]             # numbered by sorted distinct value
    np.savez(tmp_path / "c.npz", indptr=np.zeros(1), indices=np.zeros(0), graph_labels=np.array([1, 0, 1]))
    assert graph_labels(str(tmp_path / "c.npz")).tolist() == [1, 0, 1]
    np.savez(tmp_path / "nolabels.npz", indptr=np.zeros(1))
    with pytest.raises(ValueError, match="graph_labels"):
        graph_labels(str(tmp_path / "nolabels.npz"))


def test_graph_classification_checks_the_row_count(tmp_path):
    from gcc_b200.tasks import graph_classification
    np.savez(tmp_path / "c.npz", graph_labels=np.array([1, 0, 1, 0]))
    np.save(tmp_path / "rows.npy", np.zeros((3, 4), np.float32))
    with pytest.raises(ValueError, match="3 embedding rows for 4 graph labels"):
        graph_classification.main(["--dataset", str(tmp_path / "c.npz"), "--model", "from_numpy_graph",
                                   "--hidden-size", "4", "--emb-path", str(tmp_path / "rows.npy")])


def test_memory_refusal_gives_the_sizes():
    assert set_memory_error(1000, 5000, 10, 10 ** 9) is None
    msg = set_memory_error(10 ** 9, 2 * 10 ** 10, 10 ** 6, 80 * 10 ** 9)
    assert msg is not None
    assert "1000000 graphs (1000000000 vertices, 20000000000 edge entries)" in msg
    assert "176.02 GB" in msg and "88.00 GB each" in msg and "80.00 GB are free" in msg


def test_sorted_rows_and_first_bad_graph():
    rng = np.random.RandomState(0)
    graphs = []
    for i in range(5):
        n = 6
        indptr = np.arange(0, 3 * n + 1, 3, dtype=np.int64)
        graphs.append(synthetic.CSRGraph(indptr, rng.randint(0, n, 3 * n).astype(np.int32), n, "g%d" % i))
    union = synthetic.disjoint_union(graphs)
    node_off = np.arange(0, 31, 6)
    fixed = sorted_rows(union)
    assert first_bad_graph(fixed.indptr, fixed.indices, node_off) is None
    assert sorted_rows(fixed) is fixed
    # the relabel of the sorted union is the relabel of the graphs as given: seed_first sorts each row
    _, _, ip, ix, _, _ = seed_first_union(graphs)
    want_bad = first_bad_graph(union.indptr, union.indices, node_off)
    assert want_bad is not None
    back = [synthetic.CSRGraph(g.indptr, fixed.indices[6 * 3 * i:6 * 3 * (i + 1)] - 6 * i, 6, g.name)
            for i, g in enumerate(graphs)]
    _, _, ip2, ix2, _, _ = seed_first_union(back)
    assert np.array_equal(ip, ip2) and np.array_equal(ix, ix2)
