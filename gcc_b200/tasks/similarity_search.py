"""Similarity search on frozen embeddings (gcc/tasks/similarity_search.py): for every name the two Panther graphs
share, rank the second graph's shared vertices by cosine similarity to the name's vertex in the first graph and
report how often the true match is among the top 20 / 40, as {"Recall @ 20": ..., "Recall @ 40": ...}.
`--dataset a_b` names the pair (e.g. kdd_icdm)."""
import argparse
from collections import defaultdict

import numpy as np

from ..datasets.downstream import SSDataset
from . import build_model, edge_nodes


class SimilaritySearch:
    def __init__(self, dataset_1, dataset_2, model, hidden_size, root="data", **model_args):
        self.data = SSDataset(root + "/panther", dataset_1, dataset_2).data
        self.model = build_model(model, hidden_size, **model_args)
        self.hidden_size = hidden_size

    def _train_wrap(self, data):
        nodes = edge_nodes(data.edge_index.numpy())
        features_matrix = np.zeros((len(nodes), self.hidden_size))
        features_matrix[nodes] = self.model.train(nodes)
        return features_matrix

    def train(self):
        emb_1 = self._train_wrap(self.data[0])
        emb_2 = self._train_wrap(self.data[1])
        return self._evaluate(emb_1, emb_2, self.data[0].y, self.data[1].y)

    def _evaluate(self, emb_1, emb_2, dict_1, dict_2):
        # sorted: the reference iterates a set of strings, whose order (and so the winner of an exact score tie)
        # changes with the interpreter's hash seed
        shared_keys = [k for k in sorted(set(dict_1.keys()) & set(dict_2.keys()))
                       if dict_1[k] < emb_1.shape[0] and dict_2[k] < emb_2.shape[0]]
        emb_1 = emb_1 / np.linalg.norm(emb_1, axis=1).reshape(-1, 1)
        emb_2 = emb_2 / np.linalg.norm(emb_2, axis=1).reshape(-1, 1)
        reindex = [dict_2[key] for key in shared_keys]
        reindex_dict = {x: i for i, x in enumerate(reindex)}
        emb_2 = emb_2[reindex]
        k_list = [20, 40]
        results = defaultdict(list)
        for key in shared_keys:
            idxs = emb_2.dot(emb_1[dict_1[key]]).argsort()[::-1]
            for k in k_list:
                results[k].append(int(reindex_dict[dict_2[key]] in idxs[:k]))
        return {"Recall @ %d" % k: sum(results[k]) / len(results[k]) for k in k_list}


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--dataset", type=str, required=True)
    parser.add_argument("--model", type=str, required=True)
    parser.add_argument("--hidden-size", type=int, required=True)
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--emb-path-1", type=str, default="")
    parser.add_argument("--emb-path-2", type=str, default="")
    args = parser.parse_args(argv)
    name_1, name_2 = args.dataset.split("_")[:2]
    task = SimilaritySearch(name_1, name_2, args.model, args.hidden_size,
                            emb_path_1=args.emb_path_1, emb_path_2=args.emb_path_2)
    ret = task.train()
    print(ret)
    return ret


if __name__ == "__main__":
    main()
