"""Node classification on frozen embeddings (gcc/tasks/node_classification.py): one-vs-rest logistic regression
(C = 1000) that predicts each test node's top-k labels, k = its label count, under a shuffled stratified 10-fold
split of the argmax labels; the mean micro-F1 over the folds is reported as {"Micro-F1": ...}.

`--dataset` is one of the five named node datasets (labels from data/, rows of the vertices that have edges, zeros
elsewhere) or an .npz holding `y`, the finetune format (one label per row, or a 2-D 0/1 label matrix): its rows are
the embedding file's rows as they are.  The same fit on the GPU, solved to a stated tolerance and at any size, is
`gcc_b200.tasks.linear_probe`."""
import argparse
import warnings
from collections import defaultdict

import numpy as np
import scipy.sparse as sp
from sklearn.linear_model import LogisticRegression
from sklearn.metrics import f1_score
from sklearn.model_selection import StratifiedKFold
from sklearn.multiclass import OneVsRestClassifier

from ..datasets.downstream import create_node_classification_dataset
from . import build_model, edge_nodes
from .linear_probe import label_matrix

warnings.filterwarnings("ignore")


class NodeClassification:
    def __init__(self, dataset, model, hidden_size, num_shuffle, seed, root="data", **model_args):
        if dataset.endswith(".npz"):
            self.data = None
            with np.load(dataset) as z:
                if "y" not in z.files:
                    raise ValueError("%s holds no y" % dataset)
                self.label_matrix = label_matrix(z["y"])
        else:
            self.data = create_node_classification_dataset(dataset, root).data
            self.label_matrix = self.data.y.numpy()
        self.num_nodes, self.num_classes = self.label_matrix.shape
        self.model = build_model(model, hidden_size, **model_args)
        self.hidden_size = hidden_size
        self.num_shuffle = num_shuffle
        self.seed = seed

    def train(self):
        if self.data is None:                                       # an .npz: the file's rows as they are
            emb = getattr(self.model, "emb", None)
            if emb is not None and len(emb) != self.num_nodes:
                raise ValueError("%d embedding rows for %d label rows: the rows must be one per node, in order"
                                 % (len(emb), self.num_nodes))
            nodes = np.arange(self.num_nodes)
            return self._evaluate(np.asarray(self.model.train(nodes), np.float64), self.label_matrix,
                                  self.num_shuffle)
        nodes = edge_nodes(self.data.edge_index.numpy())
        features_matrix = np.zeros((self.num_nodes, self.hidden_size))
        features_matrix[nodes] = self.model.train(nodes)
        return self._evaluate(features_matrix, self.label_matrix, self.num_shuffle)

    def _evaluate(self, features_matrix, label_matrix, num_shuffle):
        label_matrix = np.asarray(label_matrix, dtype=np.float32)
        skf = StratifiedKFold(n_splits=10, shuffle=True, random_state=self.seed)
        labels = label_matrix.argmax(axis=1).tolist()
        results = defaultdict(list)
        for train_idx, test_idx in skf.split(np.zeros(len(labels)), labels):
            clf = TopKRanker(LogisticRegression(C=1000))
            clf.fit(features_matrix[train_idx], label_matrix[train_idx])
            y_test = label_matrix[test_idx]
            preds = clf.predict(features_matrix[test_idx], y_test.sum(axis=1).astype(np.int64).tolist())
            results[""].append(f1_score(y_test, preds, average="micro"))
        return {"Micro-F1" + k: sum(v) / len(v) for k, v in sorted(results.items())}


class TopKRanker(OneVsRestClassifier):
    def predict(self, X, top_k_list):
        assert X.shape[0] == len(top_k_list)
        probs = np.asarray(super().predict_proba(X))
        all_labels = sp.lil_matrix(probs.shape)
        for i, k in enumerate(top_k_list):
            for label in self.classes_[probs[i, :].argsort()[-k:]].tolist():
                all_labels[i, label] = 1
        return all_labels


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--dataset", type=str, required=True)
    parser.add_argument("--model", type=str, required=True)
    parser.add_argument("--hidden-size", type=int, required=True)
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--num-shuffle", type=int, default=10)
    parser.add_argument("--emb-path", type=str, default="")
    args = parser.parse_args(argv)
    task = NodeClassification(args.dataset, args.model, args.hidden_size, args.num_shuffle, args.seed,
                              emb_path=args.emb_path)
    ret = task.train()
    print(ret)
    return ret


if __name__ == "__main__":
    main()
