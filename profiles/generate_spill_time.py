"""generate.py's node export at the default capacity on the C2 graph (Chung-Lu, 1M nodes, 20M pairs), where the batches
of consecutive hubs overflow it and are re-run on buffers sized from their ego-nets (DESIGN §5e).

1. Every node, in order, GIN hidden 64, B = 256, rw_hops 256, generate.py's plain-degree budget, run-ahead ring
   (prefetch 4): wall time from the first launch to the last row in host memory, nodes/s, the batches re-planned,
   the wall time spent re-running them and the largest ego-net met.
2. With --baseline-embed FILE (an embed.py of another revision): profiles/generate_time.py's arms (explicit node_cap
   B * 2048, so nothing overflows; GIN h64, GIN h128, GAT h64; prefetch 0 and 4) with this revision's EmbedEngine and
   the baseline's, alternately, `--rounds` rounds each.  Both must write the same bytes.

Prints the GPU's name, power limit and SM clock read in the same process, and a JSON summary.

    python profiles/generate_spill_time.py [--rounds 3 --baseline-embed FILE --out out/generate_spill_time.json]
"""
import argparse
import importlib.util
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gcc_b200 import embed  # noqa: E402
from gcc_b200.datasets import synthetic  # noqa: E402
from gcc_b200.datasets.graph_dataset import NodeClassificationDataset  # noqa: E402
from gcc_b200.models import GraphEncoder  # noqa: E402
from profiles.generate_time import MODELS, gpu_state  # noqa: E402

B = 256


def encoder(gnn, H):
    torch.manual_seed(0)
    return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                        node_hidden_dim=H, num_layers=5, norm=True, gnn_model=gnn, degree_input=True).cuda().eval()


def dataset(g, node_cap=None):
    return NodeClassificationDataset(dataset=g, rw_hops=256, restart_prob=0.8, positional_embedding_size=32,
                                     device="cuda", seed=0, batch_size=B, node_cap=node_cap)


def whole_graph(g):
    """Part 1: every node at the default capacity, with the re-planned batches timed on the host."""
    ds = dataset(g)
    eng = embed.EmbedEngine(ds, encoder("gin", 64), prefetch=4)
    spill = []
    replan = eng._replan

    def timed(t):                                  # the ring has drained: its work is done before the clock starts
        t0 = time.perf_counter()
        replan(t)                                  # ends with the group's rows in host memory
        spill.append(time.perf_counter() - t0)
    eng._replan = timed
    eng.run(range(4 * B), np.empty((4 * B, 64), np.float32))              # warm-up: the hub batches spill
    n = ds.graph.num_nodes
    out = np.empty((n, 64), np.float32)
    spill.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.run(range(n), out)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert np.isfinite(out).all()
    res = {"nodes": n, "batches": -(-n // B), "wall_s": wall, "nodes_per_s": n / wall,
           "replanned_batches": eng.replanned, "replan_s": sum(spill), "replan_share": sum(spill) / wall,
           "replan_s_per_batch": spill, "largest_egonet_vertices_edges": list(eng.largest_egonet),
           "default_node_cap": ds.node_cap, "default_edge_cap": ds.edge_cap}
    print("whole graph, default capacity: %d nodes in %.2f s (%.0f nodes/s); %d of %d batches re-planned, %.2f s "
          "(%.1f %% of the wall time); largest ego-net %d vertices, %d edges"
          % (n, wall, n / wall, eng.replanned, res["batches"], sum(spill), 100 * res["replan_share"],
             *eng.largest_egonet), flush=True)
    return res


def load_baseline(path):
    spec = importlib.util.spec_from_file_location("gcc_b200._baseline_embed", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def ab(g, base, rounds, n_ids):
    """Part 2: generate_time.py's arms, this revision against the baseline, alternately."""
    ds = dataset(g, node_cap=B * 2048)
    ids = np.sort(np.random.RandomState(0).choice(ds.graph.num_nodes, n_ids, replace=False))
    rates = {}
    for name, (gnn, H) in MODELS.items():
        model = encoder(gnn, H)
        arms = {}
        for p in (0, 4):
            for rev, mod in (("baseline", base), ("this", embed)):
                arms["%s prefetch %d %s" % (name, p, rev)] = mod.EmbedEngine(ds, model, prefetch=p)
        out = {arm: np.empty((len(ids), H), np.float32) for arm in arms}
        for arm, eng in arms.items():
            eng.run(ids[:4 * B], out[arm][:4 * B])
        for r in range(rounds):
            for arm, eng in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.run(ids, out[arm])
                torch.cuda.synchronize()
                rates.setdefault(arm, []).append(len(ids) / (time.perf_counter() - t0))
                print("round %d  %-32s %9.0f nodes/s" % (r, arm, rates[arm][-1]), flush=True)
        for p in (0, 4):
            a, b = out["%s prefetch %d baseline" % (name, p)], out["%s prefetch %d this" % (name, p)]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (name, p)
        del arms, model
        torch.cuda.empty_cache()
    return {"nodes_per_round": n_ids, "nodes_per_s_median": {k: float(np.median(v)) for k, v in rates.items()},
            "nodes_per_s_all": rates, "same_bytes": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ab-nodes", type=int, default=131072, help="ids embedded per arm and round in part 2")
    ap.add_argument("--baseline-embed", type=str, default=None, help="embed.py of another revision (part 2)")
    ap.add_argument("--out", type=str, default=None, help="also write the JSON summary here")
    args = ap.parse_args()
    g = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0, device="cuda")
    summary = {"graph": "chung_lu 1M nodes 20M pairs", "batch": B, "whole_graph_default_capacity": whole_graph(g)}
    torch.cuda.empty_cache()
    if args.baseline_embed:
        summary["ab_explicit_capacity"] = ab(g, load_baseline(args.baseline_embed), args.rounds, args.ab_nodes)
    state = summary["gpu"] = gpu_state()
    print("gpu: %s, power limit %s, SM clock %s (max %s)" % (state["name"], state["power.limit"], state["clocks.sm"],
                                                             state["clocks.max.sm"]))
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
