#!/usr/bin/env python
"""generate.py -- the reference's inference export (generate.py:33-134) on the H100 kernels.

Loads a pretraining checkpoint (`--load-path`, written by this repo's train.py or by the reference:
same `model` state_dict keys), walks two ego-nets from EVERY node of the target graph in order
(NodeClassificationDataset, graph_dataset.py:279-309), encodes both with the model in eval mode
(BatchNorm running statistics, no dropout) and saves (f(q) + f(k)) / 2 as `<model_folder>/<name>.npy`
(generate.py:48-53,133-134).  The reference batches the whole dataset into ONE batch (:90); here
the nodes go through in `--batch-size` chunks -- eval-mode encoding is per-graph, so the result is
the same.

`--dataset` is one of the reference's downstream datasets, read from ./data as the reference reads them
(datasets/downstream.py), an .npz CSR (indptr, indices), a DGL .bin corpus or `synthetic-<kind>`:
  - node datasets (airports and h-index from data/struc2vec, data/hindex; kdd ... icde from data/panther): the
    multigraph of the reference's _create_dgl_graph, parallel edges kept, one row per node;
  - .bin corpora (datasets/dgl_bin.py, as train.py and x2dgl read and write them): one row per vertex of the union
    of the file's graphs, in file order (the ids load_graphs assigns);
  - graph datasets (the five TU sets from data/<NAME>, or a path to any TU directory NAME holding NAME_A.txt,
    NAME_graph_indicator.txt, ...): q and k are both the whole graph with the seed on its first maximum-degree vertex
    (entire_graph=True), so the row of a graph is the encoding of that whole graph; one row per graph, in the file's
    order.  A TU directory's rows go to `<model_folder>/<NAME>.npy`;
  - `--whole-graphs` on a .bin or .npz corpus with graph_sizes: one whole-graph row per graph of the file, in file
    order, saved as `<model_folder>/<stem>.graphs.npy` beside the vertex rows `<stem>.npy`.

Node and whole-graph rows go through gcc_b200.embed.EmbedEngine (the data path of `--prefetch` batches runs ahead of the encoder;
`--prefetch 0` is the serial loop) straight into the .npy file through a memmap, so host memory does not grow with
the graph.  `--nodes FILE` writes only the rows of the listed ids (node ids, or graph ids for whole graphs), in the file's
order.  `--gpu 0 1 ...` splits the
rows into one contiguous, batch-aligned shard per entry, each embedded by its own process on that device and written
at its offsets in the shared file; the same id may repeat.  A row depends only on (run seed, node id), so the shards
exchange nothing.  A batch whose ego-nets overflow the default capacity (a run of hubs of a power-law graph) is re-run
on buffers sized from its measured ego-nets; one line after the rows are saved says how many were, and the largest
ego-net met.  Whole graphs are relabelled seed first on the device (gccb_seed_first_union), and the ring's buffers are
sized from the largest batch that runs, so no whole-graph batch overflows; each process uploads the whole union.
"""
import argparse
import multiprocessing
import multiprocessing.connection
import os
import traceback

import numpy as np
import torch

from gcc_b200.datasets import downstream, synthetic
from gcc_b200.datasets.graph_dataset import NodeClassificationDataset, WholeGraphDataset, load_graphs
from gcc_b200.datasets.labeled import read_tu_dataset
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
WORKER_ERROR_CHARS = 16384                     # a worker's traceback, cut to fit the pipe without blocking


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


def is_tu_dir(path):
    """A TU directory NAME holding NAME_A.txt (and NAME_graph_indicator.txt, ...)."""
    name = os.path.basename(os.path.normpath(path))
    return os.path.isdir(path) and os.path.isfile(os.path.join(path, name + "_A.txt"))


def whole_graph_source(dataset):
    """A TU name, a TU directory, or None when `dataset` names no graph set (a .bin / .npz corpus embeds whole
    graphs only with --whole-graphs)."""
    if dataset in downstream.GRAPH_DSETS:
        return "tu-name"
    if is_tu_dir(dataset):
        return "tu-dir"
    return None


def resolve_whole_graphs(dataset):
    """The graphs `dataset` embeds whole: a list of CSRGraphs (TU sets, read as multigraphs, as the named sets are)
    or the (union, sizes) load_graphs returns for a .bin / .npz corpus."""
    kind = whole_graph_source(dataset)
    if kind == "tu-name":
        return downstream.graph_dataset_graphs(dataset)[0]
    if kind == "tu-dir":
        path = os.path.normpath(dataset)
        return read_tu_dataset(os.path.dirname(path), os.path.basename(path), multigraph=True)[0]
    return load_graphs(dataset)


def output_stem(dataset, whole_graphs):
    """The output file's name without .npy: the dataset name, a TU directory's NAME, or a corpus file's stem (with
    .graphs for its whole-graph rows, so they never overwrite its vertex rows)."""
    stem = os.path.basename(os.path.normpath(dataset))
    if stem.endswith(".npz") or stem.endswith(".bin"):
        stem = stem[:-4] + (".graphs" if whole_graphs else "")
    return stem


def resolve_graph(name, nodes, edges):
    """`--dataset`: a named node dataset is read from ./data as a multigraph; an .npz or .bin path is passed
    through; synthetic-chunglu / synthetic-er are generated."""
    if name in downstream.NODE_DSETS:
        return downstream.node_dataset_graph(name)
    if name.endswith(".npz") or name.endswith(".bin"):
        return name
    if name.endswith("chunglu"):
        return synthetic.chung_lu(nodes, edges, 0.5, seed=0)
    return synthetic.erdos_renyi(nodes, edges, seed=0)


def parse_gpus(gpu):
    """`--gpu`: None (device 0), one id, or a list of ids (one shard each; repeats allowed) -> list of ints."""
    if gpu is None:
        return [0]
    ids = [int(g) for g in gpu] if isinstance(gpu, (list, tuple)) else [int(gpu)]
    if not ids or min(ids) < 0:
        raise ValueError("--gpu takes one or more device ids >= 0, got %r" % (gpu,))
    return ids


def read_nodes(path):
    """`--nodes`: a .npy array or a text file of integer node ids (whitespace or newline separated) -> int64 [n]."""
    if path.endswith(".npy"):
        ids = np.load(path)
        if ids.ndim != 1 or not np.issubdtype(ids.dtype, np.integer):
            raise ValueError("%s: expected a 1-D integer array, got %s %s" % (path, ids.dtype, ids.shape))
    else:
        with open(path) as f:
            tokens = f.read().split()
        try:
            ids = np.array([int(t) for t in tokens], dtype=np.int64)
        except ValueError as e:
            raise ValueError("%s: node ids must be integers (%s)" % (path, e)) from None
    if ids.size == 0:
        raise ValueError("%s lists no node ids" % path)
    return ids.astype(np.int64)


def replan_line(stats, n_batches):
    """The line generate.py prints after the rows: batches re-planned of n_batches, from the shards' (count,
    (vertices, edges) of the largest ego-net) results, and the largest ego-net met."""
    count = sum(c for c, _ in stats)
    if not count:
        return "re-planned 0 of %d batches: every batch fit the default capacity" % n_batches
    n, m = max(big for _, big in stats)
    return ("re-planned %d of %d batches that overflowed the default capacity on buffers sized from their ego-nets; "
            "largest ego-net met: %d vertices, %d edges" % (count, n_batches, n, m))


def split_shards(n, batch_size, workers):
    """Rows 0..n-1 in batches of batch_size, split into `workers` contiguous runs of whole batches (the first
    n_batches mod workers runs get one batch more) -> one (lo, hi) per worker; workers beyond the batch count get
    empty runs (lo == hi)."""
    n_b = -(-n // batch_size)
    q, r = divmod(n_b, workers)
    out, b0 = [], 0
    for w in range(workers):
        b1 = b0 + q + (w < r)
        out.append((min(n, b0 * batch_size), min(n, b1 * batch_size)))
        b0 = b1
    return out


def _node_rows(load_path, graph, batch_size, prefetch, gpu, rows, out, whole=False):
    """Embed `rows` (a range of node ids or an int64 array of them) of `graph` on device `gpu` into `out`.  Returns
    (batches re-planned, (vertices, edges) of the largest ego-net they held).  whole: `graph` is what
    resolve_whole_graphs returns, `rows` are graph ids, and the result is (0, (node_cap, edge_cap) of the ring)."""
    from gcc_b200.embed import EmbedEngine
    torch.cuda.set_device(gpu)
    dev = torch.device("cuda", gpu)
    ckpt = torch.load(load_path, map_location="cpu", weights_only=False)
    opt = ckpt["opt"]
    encoder = GraphEncoder(degree_input=True, **{kw: getattr(opt, attr) for kw, attr in ENCODER_KWARGS.items()})
    encoder.load_state_dict(ckpt["model"])
    encoder = encoder.to(dev).eval()
    del ckpt
    if whole:
        items = WholeGraphDataset(graph, positional_embedding_size=opt.positional_embedding_size, device=dev,
                                  batch_size=batch_size)
    else:
        items = NodeClassificationDataset(
            dataset=graph, rw_hops=opt.rw_hops, subgraph_size=opt.subgraph_size, restart_prob=opt.restart_prob,
            positional_embedding_size=opt.positional_embedding_size, device=dev, seed=getattr(opt, "seed", 0),
            batch_size=batch_size)
    eng = EmbedEngine(items, encoder, prefetch=prefetch)
    eng.run(rows, out)
    torch.cuda.synchronize(dev)
    if whole:
        return 0, (eng.node_cap, eng.edge_cap)
    return eng.replanned, eng.largest_egonet


def _worker(load_path, dataset, graph_nodes, graph_edges, batch_size, prefetch, gpu, rows, out_file, lo, hi, conn,
            whole=False):
    """One shard in its own process: rows lo..hi-1 of the output file.  Sends _node_rows' result through conn, or
    the traceback if it fails."""
    try:
        graph = resolve_whole_graphs(dataset) if whole else resolve_graph(dataset, graph_nodes, graph_edges)
        out = np.lib.format.open_memmap(out_file, mode="r+")
        stats = _node_rows(load_path, graph, batch_size, prefetch, gpu, rows, out[lo:hi], whole)
        out.flush()
    except BaseException:
        conn.send(traceback.format_exc()[-WORKER_ERROR_CHARS:])
        raise SystemExit(1)
    conn.send(stats)


def _run_shards(args_test, gpus, shards, rows_of, out_file, prefetch, whole=False):
    """One process per non-empty shard; all of them joined.  If one fails, the others are terminated and its error
    is raised.  Returns the shards' _node_rows results."""
    ctx = multiprocessing.get_context("spawn")
    procs, stats = [], []
    try:
        for i, (gpu, (lo, hi)) in enumerate(zip(gpus, shards)):
            if lo == hi:
                continue
            recv, send = ctx.Pipe(duplex=False)
            p = ctx.Process(target=_worker, name="generate-shard-%d" % i,
                            args=(args_test.load_path, args_test.dataset, args_test.graph_nodes, args_test.graph_edges,
                                  args_test.batch_size, prefetch, gpu, rows_of(lo, hi), out_file, lo, hi, send,
                                  whole))
            p.start()
            send.close()
            procs.append((i, gpu, lo, hi, p, recv))
        pending = [p for *_, p, _ in procs]
        while pending:
            multiprocessing.connection.wait([p.sentinel for p in pending])
            for i, gpu, lo, hi, p, recv in procs:
                if p in pending and p.exitcode is not None:
                    pending.remove(p)
                    if p.exitcode != 0:
                        msg = recv.recv() if recv.poll() else "exit code %d" % p.exitcode
                        raise RuntimeError("generate.py: shard %d (gpu %d, rows %d..%d) failed:\n%s"
                                           % (i, gpu, lo, hi - 1, msg))
                    stats.append(recv.recv())
    finally:
        for *_, p, recv in procs:
            if p.is_alive():
                p.terminate()
        for *_, p, recv in procs:
            p.join()
            recv.close()
    return stats


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
    gpus = parse_gpus(getattr(args_test, "gpu", None))
    prefetch = getattr(args_test, "prefetch", 4)
    nodes_file = getattr(args_test, "nodes", None)
    whole = whole_graph_source(args_test.dataset) is not None
    if getattr(args_test, "whole_graphs", False):
        if not (args_test.dataset.endswith(".bin") or args_test.dataset.endswith(".npz")):
            raise SystemExit("--whole-graphs embeds the graphs of a .bin or .npz corpus; %r is not one"
                             % args_test.dataset)
        whole = True
    out = os.path.join(getattr(opt, "model_folder", "."), output_stem(args_test.dataset, whole))
    del ckpt

    if whole:
        graphs = resolve_whole_graphs(args_test.dataset)
        n_items = len(graphs[1]) if isinstance(graphs, tuple) else len(graphs)
        what = "graph"
    else:
        graph = resolve_graph(args_test.dataset, args_test.graph_nodes, args_test.graph_edges)
        n_items = load_graphs(graph)[0].num_nodes
        what = "node"
    ids = None
    if nodes_file:
        ids = read_nodes(nodes_file)
        if ids.min() < 0 or ids.max() >= n_items:
            raise SystemExit("%s: %s ids must lie in 0..%d" % (nodes_file, what, n_items - 1))
    n = n_items if ids is None else len(ids)
    rows_of = (lambda lo, hi: range(lo, hi)) if ids is None else (lambda lo, hi: ids[lo:hi])
    out_file = out + ".npy"
    emb = np.lib.format.open_memmap(out_file, mode="w+", dtype=np.float32, shape=(n, opt.hidden_size))
    B = min(args_test.batch_size, n_items)
    try:
        if len(gpus) == 1:
            stats = [_node_rows(path, graphs if whole else graph, args_test.batch_size, prefetch, gpus[0],
                                rows_of(0, n), emb, whole)]
        else:
            # shards aligned to the batches a one-GPU run makes, so every batch holds the same items
            stats = _run_shards(args_test, gpus, split_shards(n, B, len(gpus)), rows_of, out_file, prefetch, whole)
        emb.flush()
    except BaseException:
        del emb
        os.remove(out_file)
        raise
    print("saved {} embeddings of dim {} to {}".format(n, opt.hidden_size, out_file))
    if whole:
        print("whole graphs: batch buffers sized from the largest batch, up to %d vertices and %d edge entries"
              % max(big for _, big in stats))
    else:
        print(replan_line(stats, -(-n // B)))
    return torch.from_numpy(np.asarray(emb))


def parse_args(argv=None):
    ap = argparse.ArgumentParser("inference export: node embeddings from a pretraining checkpoint")
    ap.add_argument("--load-path", type=str, required=True, help="path to load model")
    ap.add_argument("--dataset", type=str, default="synthetic-er",
                    help="a downstream dataset (%s; files under ./data), a TU directory, an .npz CSR file (indptr, "
                         "indices), a DGL .bin corpus or synthetic-er / synthetic-chunglu"
                         % ", ".join(downstream.NODE_DSETS + downstream.GRAPH_DSETS))
    ap.add_argument("--graph-nodes", type=int, default=2000, help="size of a synthetic target graph")
    ap.add_argument("--graph-edges", type=int, default=10000)
    ap.add_argument("--batch-size", type=int, default=256, help="nodes (or whole graphs) encoded per launch group")
    ap.add_argument("--gpu", default=None, type=int, nargs="+",
                    help="GPU id(s): one shard of the rows per entry, each in its own process (repeats allowed)")
    ap.add_argument("--prefetch", type=int, default=4,
                    help="batches whose sampling and positional features run ahead of the encoder; 0 = serial")
    ap.add_argument("--nodes", type=str, default=None,
                    help="a .npy or text file of node ids (graph ids for whole graphs): write only their rows, in "
                         "the file's order")
    ap.add_argument("--whole-graphs", action="store_true",
                    help="a .bin or .npz corpus: one row per graph (the whole graph, seed on its first maximum-degree "
                         "vertex), saved as <stem>.graphs.npy")
    return ap.parse_args(argv)


if __name__ == "__main__":
    main(parse_args())
