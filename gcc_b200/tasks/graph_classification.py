"""Graph classification on frozen embeddings (gcc/tasks/graph_classification.py): an RBF SVC (C = 100000) under a
shuffled stratified 10-fold split; the mean accuracy is reported under the reference's key, "Micro-F1"."""
import argparse
import warnings

import numpy as np
from sklearn.metrics import accuracy_score
from sklearn.model_selection import StratifiedKFold
from sklearn.svm import SVC

from ..datasets.downstream import graph_dataset_graphs
from . import build_model

warnings.filterwarnings("ignore")


class GraphClassification:
    def __init__(self, dataset, model, hidden_size, num_shuffle, seed, root="data", **model_args):
        assert model == "from_numpy_graph"
        _, self.labels = graph_dataset_graphs(dataset, root)
        self.model = build_model(model, hidden_size, **model_args)
        self.hidden_size = hidden_size
        self.num_shuffle = num_shuffle
        self.seed = seed

    def train(self):
        return self.svc_classify(self.model.train(None), self.labels)

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
