"""Graph classification on frozen embeddings (gcc/tasks/graph_classification.py): an RBF SVC (C = 100000) under a
shuffled stratified 10-fold split; the mean accuracy is reported under the reference's key, "Micro-F1".

`--dataset` is one of the five TU names (labels from data/<NAME>), the path of any TU directory NAME (labels from
its NAME_graph_labels.txt, numbered as read_tu_dataset numbers them: by sorted distinct value), or an .npz holding
`graph_labels`, one per graph -- the rows generate.py writes for a TU directory or, with --whole-graphs, for a
corpus file."""
import argparse
import os
import warnings

import numpy as np
from sklearn.metrics import accuracy_score
from sklearn.model_selection import StratifiedKFold
from sklearn.svm import SVC

from ..datasets.downstream import graph_dataset_graphs
from . import build_model

warnings.filterwarnings("ignore")


def graph_labels(dataset, root="data"):
    """int64 labels of `dataset`: a TU name (read under root), a TU directory path or an .npz with graph_labels."""
    if dataset.endswith(".npz"):
        with np.load(dataset) as z:
            if "graph_labels" not in z.files:
                raise ValueError("%s holds no graph_labels" % dataset)
            return np.asarray(z["graph_labels"], dtype=np.int64).reshape(-1)
    name = os.path.basename(os.path.normpath(dataset))
    path = os.path.join(os.path.normpath(dataset), name + "_graph_labels.txt")
    if os.path.isfile(path):
        raw = np.loadtxt(path, dtype=np.int64).reshape(-1)
        return np.searchsorted(np.unique(raw), raw)                   # as read_tu_dataset numbers them
    return graph_dataset_graphs(dataset, root)[1]


class GraphClassification:
    def __init__(self, dataset, model, hidden_size, num_shuffle, seed, root="data", **model_args):
        assert model == "from_numpy_graph"
        self.labels = graph_labels(dataset, root)
        self.model = build_model(model, hidden_size, **model_args)
        self.hidden_size = hidden_size
        self.num_shuffle = num_shuffle
        self.seed = seed

    def train(self):
        x = self.model.train(None)
        if len(x) != len(self.labels):
            raise ValueError("%d embedding rows for %d graph labels: the rows must be one per graph, in order"
                             % (len(x), len(self.labels)))
        return self.svc_classify(x, self.labels)

    def svc_classify(self, x, y):
        """svc_classify(search=False); the grid search of search=True is not reached by any reference command."""
        kf = StratifiedKFold(n_splits=10, shuffle=True, random_state=self.seed)
        accuracies = []
        for train_index, test_index in kf.split(x, y):
            classifier = SVC(C=100000)
            classifier.fit(x[train_index], y[train_index])
            accuracies.append(accuracy_score(y[test_index], classifier.predict(x[test_index])))
        return {"Micro-F1": np.mean(accuracies)}


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--dataset", type=str, required=True)
    parser.add_argument("--model", type=str, required=True)
    parser.add_argument("--hidden-size", type=int, required=True)
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--num-shuffle", type=int, default=10)
    parser.add_argument("--emb-path", type=str, default="")
    args = parser.parse_args(argv)
    task = GraphClassification(args.dataset, args.model, args.hidden_size, args.num_shuffle, args.seed,
                               emb_path=args.emb_path)
    ret = task.train()
    print(ret)
    return ret


if __name__ == "__main__":
    main()
