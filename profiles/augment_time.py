"""Throughput of the data path alone (sampling + positional features, no training; and the sampler alone) on the C2
graph for the
reference's views: RWR with step_dist [1,0,0] (the default path, the control), RWR with [0.5,0.3,0.2], and
aug="ns" with rw_hops 2 / 3 / 4 and num_neighbors 5.  The arms run alternately, `--rounds` times each, in one
process; each round times `--batches` batches of B = 256 with CUDA events after `--warmup` untimed ones.

    python profiles/augment_time.py [--rounds 3 --batches 20 --warmup 3]

Prints one line per arm and round (pairs/s = B * batches / elapsed, with and without the positional features) and a
JSON summary of the medians."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gcc_b200.datasets import synthetic  # noqa: E402
from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset  # noqa: E402

ARMS = {
    "rwr [1,0,0]": dict(rw_hops=256),
    "rwr [0.5,0.3,0.2]": dict(rw_hops=256, step_dist=[0.5, 0.3, 0.2]),
    "ns hops 2": dict(rw_hops=2, aug="ns", num_neighbors=5),
    "ns hops 3": dict(rw_hops=3, aug="ns", num_neighbors=5),
    "ns hops 4": dict(rw_hops=4, aug="ns", num_neighbors=5),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    B = 256
    g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
    # ns ego-nets at 4 layers average ~700 vertices: room for B of 1024 (the default node_cap assumes RWR sizes)
    sets = {name: LoadBalanceGraphDataset(restart_prob=0.8, positional_embedding_size=32, dgl_graphs_file=g,
                                          batch_size=B, seed=0, node_cap=B * 1024 if "aug" in kw else None, **kw)
            for name, kw in ARMS.items()}
    rates = {name: [] for name in ARMS}
    sampler = {name: [] for name in ARMS}
    nodes = {}
    for r in range(args.rounds):
        for name, ds in sets.items():
            for _ in range(args.warmup):
                ds.sample_batch()
            torch.cuda.synchronize()
            ds.buffers.check_flags()
            for posenc, out in ((True, rates), (False, sampler)):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.batches):
                    ds.sample_batch(posenc=posenc)
                t1.record()
                torch.cuda.synchronize()
                ds.buffers.check_flags()
                out[name].append(B * args.batches / (t0.elapsed_time(t1) / 1e3))
            nodes[name] = int(ds.buffers.node_off[0, B]) / B
            print("round %d  %-18s %9.0f pairs/s, sampler alone %9.0f  (%.0f vertices per q ego-net in the last "
                  "batch)" % (r, name, rates[name][-1], sampler[name][-1], nodes[name]), flush=True)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "batch": B,
                      "pairs_per_s_median": {k: float(np.median(v)) for k, v in rates.items()},
                      "sampler_pairs_per_s_median": {k: float(np.median(v)) for k, v in sampler.items()},
                      "pairs_per_s_all": rates, "sampler_pairs_per_s_all": sampler, "q_vertices_per_egonet": nodes}))


if __name__ == "__main__":
    main()
