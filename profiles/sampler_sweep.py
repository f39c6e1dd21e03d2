#!/usr/bin/env python
"""BASELINE config 5: sampler + induction kernels only, 65,536 ego-nets per launch on a 10M-node /
200M-pair RMAT graph, rw_hops in {64, 128, 256, 512}: achieved ALGORITHMIC GB/s (SURVEY 8d byte
formula, counters emitted by the kernels) against the measured HBM peak.  Writes one JSON object."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gcc_b200  # noqa: F401
import torch

from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
scale = int(sys.argv[1]) if len(sys.argv) > 1 else 24
pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 200_000_000
B = int(sys.argv[3]) if len(sys.argv) > 3 else 32768          # pairs per launch -> 2B ego-nets
BUDGET_CAP = int(sys.argv[4]) if len(sys.argv) > 4 else 2000   # walk budgets above it are clipped (0 = the reference formula unclipped)
HOPS = [int(x) for x in sys.argv[5].split(",")] if len(sys.argv) > 5 else [64, 128, 256, 512]
REPS = int(sys.argv[6]) if len(sys.argv) > 6 else 3            # 1 under ncu
dev = torch.device("cuda")
g = synthetic.rmat_device(scale, pairs, seed=0, device=dev)
torch.cuda.synchronize()
deg = g.indptr[1:] - g.indptr[:-1]
info = {"graph": g.name, "nodes": g.num_nodes, "nnz": int(g.indices.numel()), "max_degree": int(deg.max()),
        "csr_bytes": int(g.indptr.numel() * 8 + g.indices.numel() * 4), "egonets_per_launch": 2 * B}
try:
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs", 3350.0))
    info["peak_source"] = "MEASURED_PEAKS.json"
except Exception:
    peak, info["peak_source"] = 3350.0, "H100 SXM data sheet, 3350 GB/s"
rows = []
for hops in HOPS:
    ds = LoadBalanceGraphDataset(rw_hops=hops, restart_prob=0.8, dgl_graphs_file=g, batch_size=B, seed=0,
                                 device=dev, node_cap=B * 1024, edge_cap=B * 1024 * 48, budget_cap=BUDGET_CAP or None)
    try:
        for i in range(2):
            ds.sample_batch(posenc=False)
        torch.cuda.synchronize()
        ds.buffers.check_flags()
    except Exception as e:                      # capacity overflow on this graph: record it, keep sweeping
        rows.append({"rw_hops": hops, "error": str(e)})
        print(rows[-1], file=sys.stderr)
        del ds
        torch.cuda.empty_cache()
        continue
    reps = REPS
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    acc = torch.zeros(4, dtype=torch.float64, device=dev)
    ev[0].record()
    for i in range(reps):
        ds.sample_batch(posenc=False)
        acc += ds.buffers.counters.double().sum(0)
    ev[1].record()
    torch.cuda.synchronize()
    ds.buffers.check_flags()
    ms = ev[0].elapsed_time(ev[1]) / reps
    n_sum, m_sum, t_sum, deg_sum = [float(x) / reps for x in acc.tolist()]
    alg = t_sum * 12 + (8 * n_sum + 4 * deg_sum) + 4 * (2 * n_sum + 2 * B + m_sum)
    rows.append({"rw_hops": hops, "ms_per_launch_group": ms, "egonets_per_sec": 2 * B / (ms / 1e3),
                 "algorithmic_bytes": alg, "achieved_gbs": alg / (ms / 1e3) / 1e9, "frac_of_hbm_peak": alg / (ms / 1e3) / 1e9 / peak,
                 "avg_nodes": n_sum / (2 * B), "avg_induced_edges": m_sum / (2 * B), "avg_walk_steps": t_sum / (2 * B),
                 "avg_scanned_neighbours": deg_sum / (2 * B), "max_budget": ds.graph.max_budget,
                 "seeds_with_clipped_budget_frac": float((ds.graph.budget_table[deg[ds.buffers.seeds]] >= BUDGET_CAP).double().mean()) if BUDGET_CAP else 0.0})
    print(rows[-1], file=sys.stderr)
    del ds
    torch.cuda.empty_cache()
info.update({"hbm_peak_gbs": peak, "sweep": rows,
             "note": "walk budgets above %d are clipped (capacity knob of the sweep; 0 = unclipped); inputs resident in HBM; "
                     "timed with CUDA events over %d launch groups (walk+unique, offsets, fill); physical DRAM bytes: the ncu "
                     "capture next to this file" % (BUDGET_CAP, REPS)})
print(json.dumps(info))
