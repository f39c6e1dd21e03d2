#!/usr/bin/env python
"""generate.py -- the reference's inference export (generate.py:33-134) on the H100 kernels.

Loads a pretraining checkpoint (`--load-path`, written by this repo's train.py or by the reference:
same `model` state_dict keys), walks two ego-nets from EVERY node of the target graph in order
(NodeClassificationDataset, graph_dataset.py:279-309), encodes both with the model in eval mode
(BatchNorm running statistics, no dropout) and saves (f(q) + f(k)) / 2 as `<model_folder>/<name>.npy`
(generate.py:48-53,133-134).  The reference batches the whole dataset into ONE batch (:90); here
the nodes go through in `--batch-size` chunks -- eval-mode encoding is per-graph, so the result is
the same.  `--dataset` is an .npz CSR (indptr, indices) or `synthetic-<kind>`: the reference's named
datasets need the network / DGL (SURVEY.md 8f N2, N3).
"""
import argparse
import os

import numpy as np
import torch

from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
from gcc_b200.models import GraphEncoder

# checkpoint["opt"] attribute -> GraphEncoder keyword (train.py:601-620 builds the model from these)
ENCODER_KWARGS = {
    "positional_embedding_size": "positional_embedding_size", "max_node_freq": "max_node_freq",
    "max_edge_freq": "max_edge_freq", "max_degree": "max_degree",
    "freq_embedding_size": "freq_embedding_size", "degree_embedding_size": "degree_embedding_size",
    "output_dim": "hidden_size", "node_hidden_dim": "hidden_size", "edge_hidden_dim": "hidden_size",
    "num_layers": "num_layer", "num_step_set2set": "set2set_iter",
    "num_layer_set2set": "set2set_lstm_layer", "gnn_model": "model", "norm": "norm",
}


def test_moco(train_loader, model, opt):
    """Embedding of every item: mean of the two views' eval-mode features (generate.py:33-53)."""
    model.eval()
    chunks = []
    with torch.no_grad():
        for view_q, view_k, valid in train_loader:
            pair = torch.stack([model(view_q), model(view_k)])
            if pair.shape[1:] != (view_q.batch_size, opt.hidden_size):
                raise RuntimeError("encoder returned %s" % (tuple(pair.shape),))
            chunks.append(pair.mean(0)[:valid].cpu())        # the last chunk is padded: keep the valid pairs
    return torch.cat(chunks)


def resolve_graph(name, nodes, edges):
    """`--dataset`: an .npz path is passed through; synthetic-chunglu / synthetic-er are generated."""
    if name.endswith(".npz"):
        return name
    if name.endswith("chunglu"):
        return synthetic.chung_lu(nodes, edges, 0.5, seed=0)
    return synthetic.erdos_renyi(nodes, edges, seed=0)


def main(args_test):
    path = args_test.load_path
    if not os.path.isfile(path):
        raise SystemExit("=> no checkpoint found at '{}'".format(path))
    if not torch.cuda.is_available():
        raise SystemExit("generate.py needs a CUDA device (sm_90a); there is no CPU path")
    print("=> loading checkpoint '{}'".format(path))
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    print("=> loaded successfully '{}' (epoch {})".format(path, ckpt["epoch"]))
    opt = ckpt["opt"]
    gpu = args_test.gpu or 0
    torch.cuda.set_device(gpu)
    opt.device = torch.device("cuda", gpu)

    encoder = GraphEncoder(degree_input=True, **{kw: getattr(opt, attr) for kw, attr in ENCODER_KWARGS.items()})
    encoder.load_state_dict(ckpt["model"])
    encoder = encoder.to(opt.device)
    del ckpt

    nodes = NodeClassificationDataset(
        dataset=resolve_graph(args_test.dataset, args_test.graph_nodes, args_test.graph_edges),
        rw_hops=opt.rw_hops, subgraph_size=opt.subgraph_size, restart_prob=opt.restart_prob,
        positional_embedding_size=opt.positional_embedding_size, device=opt.device,
        seed=getattr(opt, "seed", 0), batch_size=args_test.batch_size)
    emb = test_moco(nodes, encoder, opt)

    stem = os.path.basename(args_test.dataset)
    stem = stem[:-4] if stem.endswith(".npz") else stem
    out = os.path.join(getattr(opt, "model_folder", "."), stem)
    np.save(out, emb.numpy())
    print("saved {} embeddings of dim {} to {}.npy".format(emb.shape[0], emb.shape[1], out))
    return emb


if __name__ == "__main__":
    ap = argparse.ArgumentParser("inference export: node embeddings from a pretraining checkpoint")
    ap.add_argument("--load-path", type=str, required=True, help="path to load model")
    ap.add_argument("--dataset", type=str, default="synthetic-er",
                    help=".npz CSR file (indptr, indices) or synthetic-er / synthetic-chunglu")
    ap.add_argument("--graph-nodes", type=int, default=2000, help="size of a synthetic target graph")
    ap.add_argument("--graph-edges", type=int, default=10000)
    ap.add_argument("--batch-size", type=int, default=256, help="nodes encoded per launch group")
    ap.add_argument("--gpu", default=None, type=int, help="GPU id to use.")
    main(ap.parse_args())
