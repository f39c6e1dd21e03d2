"""C2 pretraining throughput with the GAT encoder next to GIN, in one call (DESIGN.md, GAT section).

    python profiles/gat_time.py [--steps 50] [--warmup 10]

The C2 workload of bench.py (MoCo K = 16384, 5 layers, hidden 64, batch 256, rw_hops 256, the 1M-vertex Chung-Lu
graph) is trained for --warmup steps, then --steps timed steps between CUDA events, once with --model gin and once
with --model gat (4 heads, Set2Set 6 iterations x 3 LSTM layers).  Prints one JSON line per model with subgraphs/s
(2 x batch x steps / seconds, bench.py's `value`) and the card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run(model_name, steps, warmup):
    import torch
    import bench
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    cfg = bench.CONFIGS["c2"]
    dev = torch.device("cuda", 0)
    B, L, H, K = cfg["batch"], cfg["layers"], cfg["hidden"], cfg["K"]
    torch.manual_seed(0)
    g = bench.make_graph_device(cfg, dev)
    ds = LoadBalanceGraphDataset(rw_hops=cfg["rw_hops"], restart_prob=0.8, positional_embedding_size=32,
                                 dgl_graphs_file=g, num_samples=2000, num_workers=12, num_copies=6, batch_size=B,
                                 seed=0, device=dev)

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                            node_hidden_dim=H, num_layers=L, num_heads=4, num_step_set2set=6, num_layer_set2set=3,
                            norm=True, gnn_model=model_name, degree_input=True)

    model, ema = mk(), mk()
    ema.load_state_dict(model.state_dict())
    model, ema = model.to(dev), ema.to(dev)
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).to(dev)
    eng = PretrainEngine(ds, model, ema, contrast, moco=True)
    for _ in range(warmup):
        eng.step(lr=0.005)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        eng.step(lr=0.005)
    eng.wait_data_streams()
    ev[1].record()
    torch.cuda.synchronize()
    s = eng.read_stats()
    sec = ev[0].elapsed_time(ev[1]) / 1000.0
    return dict(model=model_name, subgraphs_per_s=round(2 * B * steps / sec, 1), step_ms=round(1000 * sec / steps, 3),
                loss=round(s["loss"], 5), card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    for m in ("gin", "gat"):
        print(json.dumps(run(m, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
