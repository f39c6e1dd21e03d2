"""Throughput of generate.py's node export on the C2 graph (Chung-Lu, 1M nodes, 20M pairs), B = 256: the serial loop
(EmbedEngine prefetch 0, `generate.py --prefetch 0`) against the run-ahead ring (prefetch 4, the default), for GIN
hidden 64, GIN hidden 128 and GAT hidden 64 (4 heads).  Each round embeds the same `--nodes` ids (a fixed random
sample of the graph, so that hubs and leaves come in their natural proportion) with each arm; a round is
timed on the host from the first launch to the last row in host memory.  The models run one after another,
the two arms of a model alternately.  Prints one line per arm and round, the
GPU's name, power limit and SM clock read in the same process, and a JSON summary of the medians.

    python profiles/generate_time.py [--rounds 3 --nodes 131072 --out out/generate_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gcc_b200.datasets import synthetic  # noqa: E402
from gcc_b200.datasets.graph_dataset import NodeClassificationDataset  # noqa: E402
from gcc_b200.embed import EmbedEngine  # noqa: E402
from gcc_b200.models import GraphEncoder  # noqa: E402

MODELS = {"gin h64": ("gin", 64), "gin h128": ("gin", 128), "gat h64": ("gat", 64)}


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True)
    return dict(zip(q.split(","), (v.strip() for v in r.stdout.strip().split(","))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nodes", type=int, default=131072, help="ids embedded per arm and round")
    ap.add_argument("--out", type=str, default=None, help="also write the JSON summary here")
    args = ap.parse_args()
    B = 256
    g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
    # generate.py's plain-degree walk budget (not pretraining's deg^0.75) gives the hubs of C2 ego-nets of thousands
    # of vertices: a batch of 256 random nodes needs more room than the default 320 vertices per ego-net
    ds = NodeClassificationDataset(dataset=g, rw_hops=256, restart_prob=0.8, positional_embedding_size=32,
                                   device="cuda", seed=0, batch_size=B, node_cap=B * 2048)
    ids = np.sort(np.random.RandomState(0).choice(ds.graph.num_nodes, args.nodes, replace=False))
    rates = {}
    for name, (gnn, H) in MODELS.items():                      # one model at a time: two engines in memory
        torch.manual_seed(0)
        model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                             node_hidden_dim=H, num_layers=5, norm=True, gnn_model=gnn,
                             degree_input=True).cuda().eval()
        arms = {"%s prefetch %d" % (name, p): EmbedEngine(ds, model, prefetch=p) for p in (0, 4)}
        out = {arm: np.empty((len(ids), H), np.float32) for arm in arms}
        for arm, eng in arms.items():                          # warm-up: every kernel, shape class and stream
            eng.run(ids[:4 * B], out[arm][:4 * B])
        for r in range(args.rounds):
            for arm, eng in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.run(ids, out[arm])
                torch.cuda.synchronize()
                rates.setdefault(arm, []).append(len(ids) / (time.perf_counter() - t0))
                print("round %d  %-20s %9.0f nodes/s" % (r, arm, rates[arm][-1]), flush=True)
        a, b = out[name + " prefetch 0"], out[name + " prefetch 4"]
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name     # the two arms compute the same rows
        del arms, model
        torch.cuda.empty_cache()
    state = gpu_state()
    med = {k: float(np.median(v)) for k, v in rates.items()}
    summary = {"gpu": state, "graph": "chung_lu 1M nodes 20M pairs", "batch": B, "nodes_per_round": len(ids),
               "nodes_per_s_median": med,
               "speedup_run_ahead_over_serial": {m: med[m + " prefetch 4"] / med[m + " prefetch 0"] for m in MODELS},
               "multi_gpu": "not measured" if torch.cuda.device_count() < 2 else "not run by this script",
               "nodes_per_s_all": rates}
    print("gpu: %s, power limit %s, SM clock %s (max %s)" % (state["name"], state["power.limit"], state["clocks.sm"],
                                                             state["clocks.max.sm"]))
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
