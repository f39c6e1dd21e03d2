"""One finetune epoch with the torch-ops loop (train.train_finetune) and with FinetuneEngine, alternating, in one call
(DESIGN.md, finetuning).

    python profiles/finetune_time.py [--reps 3]

Two synthetic workloads a user of `train.py --finetune` runs:
  nodes   a Chung-Lu graph the size of usa_airport (about 1.2k vertices, 13.6k directed edges, 4 classes by degree),
          rw_hops 256, batch 32;
  graphs  2,000 sparse graphs averaging about 430 vertices, the size of REDDIT-BINARY, 2 classes, batch 32.
Encoder: GIN, 5 layers, hidden 64 (the reference's defaults); fold 0 of the 10-fold split.  Each arm runs one
untimed epoch, then --reps timed epochs per arm, alternating; an epoch is timed by the host clock between device
synchronisations.  The engine's whole-graph feature cache is built once at construction and timed separately.
Prints one JSON line per workload with the card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def node_set(dev):
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.labeled import NodeClassificationDatasetLabeled
    g = synthetic.chung_lu(1190, 6950, 0.5, seed=11)
    deg = np.diff(g.indptr)
    y = np.digitize(deg, np.quantile(deg, [0.25, 0.5, 0.75]))
    return NodeClassificationDatasetLabeled((g, y), rw_hops=256, batch_size=32, device=dev)


def graph_set(dev):
    from gcc_b200.datasets.labeled import GraphClassificationDatasetLabeled, _simple_csr
    rng = np.random.RandomState(12)
    graphs, labels = [], []
    for i in range(2000):
        n = int(np.clip(rng.lognormal(np.log(320), 0.8), 20, 3000))
        m = int(1.16 * n)
        src, dst = rng.randint(0, n, m), rng.randint(0, n, m)
        if i % 2:                                      # a discussion thread's hub
            hub = int(rng.randint(0, n))
            k = n // 4
            src, dst = np.concatenate([src, np.full(k, hub)]), np.concatenate([dst, rng.randint(0, n, k)])
        graphs.append(_simple_csr(src, dst, n, "g%d" % i))
        labels.append(i % 2)
    return GraphClassificationDatasetLabeled((graphs, np.array(labels)), batch_size=32, device=dev)


def encoder(dev, seed):
    import torch
    import train
    args = train.parse_option(["--finetune"])
    torch.manual_seed(seed)
    return train._make_encoder(args).to(dev), args


def run(name, ds, reps):
    import torch
    import train
    from gcc_b200.finetune import FinetuneEngine
    from sklearn.model_selection import StratifiedKFold
    dev = torch.device("cuda", 0)
    train_idx, _ = list(StratifiedKFold(10, shuffle=True, random_state=0).split(np.zeros(len(ds)), ds.labels))[0]
    H, C = 64, ds.num_classes
    mt, args = encoder(dev, 0)
    me, _ = encoder(dev, 0)
    lt, le = torch.nn.Linear(H, C).to(dev), torch.nn.Linear(H, C).to(dev)
    opt = types.SimpleNamespace(hidden_size=H, learning_rate=0.005, epochs=100, print_freq=10, tb_freq=250)
    opt_m = train.make_optimizer(args, mt.parameters())
    opt_o = torch.optim.Adam(lt.parameters(), lr=0.005, betas=(0.9, 0.999), weight_decay=1e-5)
    loader = train.LabeledLoader(ds, train_idx, 32, shuffle=True, seed=0)
    torch.cuda.synchronize()
    t0 = time.time()
    eng = FinetuneEngine(ds, me, le, lr=0.005)
    torch.cuda.synchronize()
    setup = time.time() - t0
    rng = np.random.RandomState(0)
    times = {"torch": [], "engine": []}
    ce = torch.nn.CrossEntropyLoss()
    for rep in range(reps + 1):
        for arm in ("torch", "engine"):
            torch.cuda.synchronize()
            t0 = time.time()
            if arm == "torch":
                train.train_finetune(rep + 1, loader, mt, lt, ce, opt_m, opt_o, None, opt)
            else:
                eng.train_epoch(rep + 1, rng.permutation(train_idx), 100, print_freq=10, tb_freq=250)
            torch.cuda.synchronize()
            if rep:
                times[arm].append(time.time() - t0)
    return dict(workload=name, items=len(ds), train_items=len(train_idx), steps=-(-len(train_idx) // 32),
                torch_epoch_s=[round(t, 4) for t in times["torch"]], engine_epoch_s=[round(t, 4) for t in times["engine"]],
                speedup=round(float(np.median(times["torch"]) / np.median(times["engine"])), 2),
                engine_setup_s=round(setup, 3), card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import contextlib
    import io

    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    for name, make in (("nodes", node_set), ("graphs", graph_set)):
        ds = make(dev)
        extra = {}
        if name == "nodes":
            extra = dict(directed_edges=int(ds.graph.indices.numel()), nodes=ds.graph.num_nodes)
        else:
            extra = dict(mean_vertices=round(float(ds.graph_set.sizes.mean()), 1))
        with contextlib.redirect_stdout(io.StringIO()):              # the per-step training lines
            r = run(name, ds, a.reps)
        r.update(extra)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
