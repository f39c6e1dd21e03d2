"""Frozen-embedding evaluators of the reference (gcc/tasks): node classification, graph classification and
similarity search on the `.npy` rows generate.py writes.  They are scikit-learn fits on the host, as in the
reference, and stay there: at the named datasets' sizes (a few thousand rows of 64) a host fit takes seconds.  For
the millions of rows generate.py writes for a large graph or corpus, the GPU has tools with an exact definition:
`gcc_b200.tasks.knn`, a cosine top-k for similarity search, and `gcc_b200.tasks.linear_probe`, the node evaluator's
one-vs-rest logistic regression (C = 1000) solved to a stated tolerance in float64, for node and graph labels.

    python -m gcc_b200.tasks.node_classification  --dataset usa_airport --model from_numpy --hidden-size 64 --emb-path <npy>
    python -m gcc_b200.tasks.graph_classification --dataset imdb-binary --model from_numpy_graph --hidden-size 64 --emb-path <npy>
    python -m gcc_b200.tasks.similarity_search    --dataset kdd_icdm --model from_numpy_align --hidden-size 64 \\
        --emb-path-1 <kdd.npy> --emb-path-2 <icdm.npy>
    python -m gcc_b200.tasks.linear_probe         --dataset <name | y.npz | graph labels> --emb-path <npy>
"""
import numpy as np


class Zero:
    """All-zero embeddings (gcc/models/emb/from_numpy.py: Zero)."""

    def __init__(self, hidden_size, **kwargs):
        self.hidden_size = hidden_size

    def train(self, nodes):
        return np.zeros((len(nodes), self.hidden_size))


class FromNumpy:
    """Rows of a saved `.npy` (FromNumpy): train(nodes) returns the rows of `nodes`, the vertices that appear in
    the edge list.  The reference walks networkx's node order and writes each row back to its own node id, so
    row v of the task's feature matrix is row v of the file, and a vertex without edges keeps a zero row."""

    def __init__(self, hidden_size, emb_path, **kwargs):
        self.hidden_size = hidden_size
        self.emb = np.load(emb_path)

    def train(self, nodes):
        return self.emb[nodes]


class FromNumpyGraph(FromNumpy):
    """One row per graph (FromNumpyGraph): the file as it is."""

    def train(self, nodes):
        assert nodes is None
        return self.emb


class FromNumpyAlign:
    """Two `.npy` files, one per graph of a similarity-search pair (FromNumpyAlign): each graph takes the first
    unused file whose row count equals its vertex count."""

    def __init__(self, hidden_size, emb_path_1, emb_path_2, **kwargs):
        self.hidden_size = hidden_size
        self.emb = [np.load(emb_path_1), np.load(emb_path_2)]
        self.used = [False, False]

    def train(self, nodes):
        for i in (0, 1):
            if len(nodes) == self.emb[i].shape[0] and not self.used[i]:
                self.used[i] = True
                return self.emb[i][nodes]
        raise NotImplementedError("no unused embedding file has %d rows" % len(nodes))


def _baseline(name):
    def make(*args, **kwargs):
        raise NotImplementedError("the %s baseline is not a build_model model; save its rows with `python -m "
                                  "gcc_b200.tasks.baselines --model %s ...` (or embeddings saved by generate.py) and "
                                  "evaluate them with --model from_numpy / from_numpy_graph / from_numpy_align"
                                  % (name, name.lower()))
    return make


def build_model(name, hidden_size, **model_args):
    """gcc/tasks/__init__.py: build_model."""
    return {
        "zero": Zero,
        "from_numpy": FromNumpy,
        "from_numpy_align": FromNumpyAlign,
        "from_numpy_graph": FromNumpyGraph,
        "prone": _baseline("ProNE"),
        "graphwave": _baseline("GraphWave"),
    }[name](hidden_size, **model_args)


def edge_nodes(edge_index):
    """Vertices that appear in an edge list, ascending: the rows the reference's networkx graph holds."""
    return np.unique(np.asarray(edge_index).reshape(-1))
