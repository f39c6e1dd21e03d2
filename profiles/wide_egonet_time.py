"""Sampling and positional-feature time of wide ego-nets (walk budget above the walk CTA's shared memory) against
their vertex count, for hubs of about 20k to 200k neighbours.

Graph: vertex 0 joined to vertices 1..hub, beside a Chung-Lu graph of 2 * hub vertices; NodeClassificationDataset
(plain-degree budget, rw_hops 256, restart 0.8) with batches of one item, so that both views of the batch are the
hub's ego-nets.  Each timed call is one batch (two wide ego-nets) on the current stream between CUDA events, after
warm-up calls of the same shape.  Prints one JSON line per hub size, each with the card's name, power limit and SM
clock read in the same run, and writes the list to --out if given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def with_hub(hub, seed):
    from gcc_b200.datasets import synthetic
    g = synthetic.chung_lu(2 * hub, 10 * hub, exponent=0.5, seed=seed)
    src = np.repeat(np.arange(g.num_nodes, dtype=np.int64), np.diff(g.indptr)) + 1
    dst = g.indices.astype(np.int64) + 1
    src = np.concatenate([src, np.zeros(hub, np.int64)])
    dst = np.concatenate([dst, np.arange(1, hub + 1, dtype=np.int64)])
    return synthetic.from_pairs(src, dst, max(g.num_nodes, hub) + 1, "hub%d" % hub)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hubs", default="20000,50000,100000,200000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="JSON file of the rows")
    args = ap.parse_args()
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset, sample_pairs
    rows = []
    for hub in (int(h) for h in args.hubs.split(",")):
        g = with_hub(hub, seed=hub % 97)
        ds = NodeClassificationDataset(dataset=g, rw_hops=256, restart_prob=0.8, positional_embedding_size=32,
                                       device="cuda", seed=1, batch_size=1)
        buf = ds.buffers
        seeds = torch.zeros(1, dtype=torch.int64, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t_s, t_p = [], []
        for r in range(args.reps + 2):                      # two warm-up calls
            ev[0].record()
            sample_pairs(ds, buf, r, seeds)
            ev[1].record()
            buf.posenc()
            ev[2].record()
            torch.cuda.synchronize()
            if r >= 2:
                t_s.append(ev[0].elapsed_time(ev[1]))
                t_p.append(ev[1].elapsed_time(ev[2]))
        c = buf.counters.cpu().numpy()
        flags = int(buf.flags.item())
        buf.flags.zero_()
        row = dict(hub_neighbours=hub, budget=int(ds.graph.budget_table[hub].item()),
                   n=[int(c[0, 0]), int(c[1, 0])], m=[int(c[0, 1]), int(c[1, 1])],
                   sample_ms_per_egonet=float(np.median(t_s)) / 2, posenc_ms_per_egonet=float(np.median(t_p)) / 2,
                   sample_ms_min=float(np.min(t_s)) / 2, posenc_ms_min=float(np.min(t_p)) / 2, flags=flags,
                   card=card())
        print(json.dumps(row), flush=True)
        rows.append(row)
        del ds, buf
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
