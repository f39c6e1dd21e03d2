#!/usr/bin/env python
"""GPU diagnostic: CUPTI kernel timeline (torch.profiler) of a few pipelined engine steps.
Writes a chrome trace to argv[2] (default: timeline.json.gz in the temporary directory).  Diagnostic only -- never a bench value."""
import contextlib
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gcc_b200  # noqa: F401  (sets CUDA_DEVICE_MAX_CONNECTIONS before CUDA starts)
import torch
from torch.profiler import ProfilerActivity, profile

import bench  # noqa: E402
from gcc_b200.contrastive.memory_moco import MemoryMoCo  # noqa: E402
from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset  # noqa: E402
from gcc_b200.engine import PretrainEngine  # noqa: E402
from gcc_b200.models import GraphEncoder  # noqa: E402

cfg = bench.CONFIGS[sys.argv[3] if len(sys.argv) > 3 else "c2"]
dev = torch.device("cuda")
g = bench.make_graph_device(cfg, dev)
B, L, H, K = cfg["batch"], cfg["layers"], cfg["hidden"], cfg["K"]
ds = LoadBalanceGraphDataset(rw_hops=cfg["rw_hops"], restart_prob=0.8, dgl_graphs_file=g, batch_size=B, seed=0)


def mk():
    return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                        node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True)


model, ema = mk(), mk()
ema.load_state_dict(model.state_dict())
model, ema = model.to(dev), ema.to(dev)
with contextlib.redirect_stdout(sys.stderr):
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).to(dev)
eng = PretrainEngine(ds, model, ema, contrast, moco=True, prefetch=int(sys.argv[1]) if len(sys.argv) > 1 else 4)
for _ in range(12):
    eng.step(lr=0.005)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(6):
        eng.step(lr=0.005)
    torch.cuda.synchronize()
out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(tempfile.gettempdir(), "timeline.json.gz")
prof.export_chrome_trace(out)
print("wrote", out)
