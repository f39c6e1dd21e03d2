"""Wall time of the embedding baselines on G(n, 4n) random graphs at hidden 64 (DESIGN.md section 4).

    python profiles/baselines_time.py --arm gpu [--sizes 2000 5000 20000]
    GCC_REFERENCE=<checkout of THUDM/GCC> python profiles/baselines_time.py --arm cpu [--graphwave-max-n 2000]

gpu: GraphWave(64).train and ProNE(64).train of gcc_b200.tasks.baselines, one warm-up call, then the median of
     `--repeats` calls; each call copies the graph in and the rows out, and ends in a device synchronise.  The
     card's name, power limit and SM clocks are printed with the numbers.
cpu: the reference's own modules (gcc/models/emb) under the stand-ins of tests/golden/make_golden_baselines.py,
     one call each; GraphWave only up to --graphwave-max-n vertices (its heat matrices are dense n x n).
One JSON line per (arm, model, n).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def edge_list(n, seed=0):
    """G(n, 4n): 4n distinct pairs without self loops."""
    rng = np.random.RandomState(seed)
    seen = set()
    while len(seen) < 4 * n:
        a, b = rng.randint(0, n, 2)
        if a != b:
            seen.add((min(a, b), max(a, b)))
    return np.array(sorted(seen), np.int64).T


def run_gpu(sizes, repeats):
    import torch
    from gcc_b200.tasks import baselines
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": q, "torch": torch.__version__}))
    for n in sizes:
        g = baselines.graph_from_pairs(edge_list(n))
        for name, model in (("graphwave", baselines.GraphWave(64)), ("prone", baselines.ProNE(64))):
            model.train(g)
            times = []
            for _ in range(repeats):
                torch.cuda.synchronize()
                t = time.perf_counter()
                model.train(g)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t)
            print(json.dumps({"arm": "gpu", "model": name, "n": len(g.nodes), "seconds": statistics.median(times),
                              "all": times}), flush=True)


def run_cpu(sizes, graphwave_max_n):
    ref = os.environ.get("GCC_REFERENCE")
    if not ref:
        raise SystemExit("set GCC_REFERENCE to a checkout of THUDM/GCC")
    os.environ["GCC_REFERENCE"] = ref
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    sys.argv = sys.argv[:1]
    import make_golden_baselines  # noqa: F401  (installs the stand-ins and imports the reference modules)
    import networkx as nx
    from gcc.models.emb.graphwave import GraphWave
    from gcc.models.emb.prone import ProNE
    for n in sizes:
        G = nx.Graph()
        G.add_edges_from(edge_list(n).T.tolist())
        for name, model in (("graphwave", GraphWave(64)), ("prone", ProNE(64))):
            if name == "graphwave" and n > graphwave_max_n:
                print(json.dumps({"arm": "cpu", "model": name, "n": n, "seconds": None, "note": "not measured"}))
                continue
            t = time.perf_counter()
            model.train(G)
            print(json.dumps({"arm": "cpu", "model": name, "n": G.number_of_nodes(),
                              "seconds": time.perf_counter() - t, "cpus": os.cpu_count()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", choices=["gpu", "cpu"], required=True)
    ap.add_argument("--sizes", type=int, nargs="+", default=[2000, 5000, 20000])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--graphwave-max-n", type=int, default=2000)
    args = ap.parse_args()
    if args.arm == "gpu":
        run_gpu(args.sizes, args.repeats)
    else:
        run_cpu(args.sizes, args.graphwave_max_n)


if __name__ == "__main__":
    main()
