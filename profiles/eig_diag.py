#!/usr/bin/env python
"""GPU diagnostic: eigensolver iterations / residuals per size class on one C2 batch."""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from gcc_b200 import _lib  # noqa: E402
from gcc_b200.datasets.graph_dataset import LoadBalanceGraphDataset  # noqa: E402

cfg = bench.CONFIGS[sys.argv[1] if len(sys.argv) > 1 else "c2"]
dev = torch.device("cuda")
g = bench.make_graph_device(cfg, dev)
B = cfg["batch"]
ds = LoadBalanceGraphDataset(rw_hops=cfg["rw_hops"], restart_prob=0.8, dgl_graphs_file=g, batch_size=B, seed=0)
buf = ds.sample_batch(posenc=False)
torch.cuda.synchronize()
lib = _lib.get()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for rep in range(3):
    ev[0].record()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 1, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                               _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    ev[1].record()
    torch.cuda.synchronize()
    print("posenc ms", ev[0].elapsed_time(ev[1]))
iters, res = (t.cpu().numpy() for t in buf.eig_debug())
n = buf.counters[:, 0].cpu().numpy()
print("flags", int(buf.flags.item()))
for lo, hi in ((0, 96), (96, 160), (160, 384), (384, 1536), (1536, 100000)):
    m = (n > lo) & (n <= hi)
    if m.sum():
        print("n in (%d,%d]: count %d  iters mean %.2f max %d  res mean %.2e max %.2e" % (
            lo, hi, m.sum(), iters[m].mean(), iters[m].max(), res[m].mean(), res[m].max()))
big = np.argsort(-n)[:8]
print("largest:", [(int(n[i]), int(iters[i]), float(res[i])) for i in big])

# several batches: size extremes and eigensolver time
for st in range(1, 9):
    buf = ds.sample_batch(posenc=False)
    ev[0].record()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 1, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                               _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    ev[1].record()
    torch.cuda.synchronize()
    n = buf.counters[:, 0].cpu().numpy()
    it, rs = (t.cpu().numpy() for t in buf.eig_debug())
    top = np.argsort(-n)[:3]
    print("batch %d: posenc %.2f ms; largest (n, iters, res): %s; max iters %d" % (
        st, ev[0].elapsed_time(ev[1]), [(int(n[i]), int(it[i]), float("%.1e" % rs[i])) for i in top], it.max()))

# phase cycle counters of the last batch's ChFSI ego-nets (thread 0 of each CTA / rank 0 of each cluster)
phase = buf.eig_phases().cpu().numpy()
names = ["filter", "gram-schmidt", "H=QtLQ", "ritz", "X=QW", "residual"]
n = buf.counters[:, 0].cpu().numpy()
for lo, hi in ((96, 160), (160, 384), (384, 100000)):
    m = (n > lo) & (n <= hi) & (it > 0)
    if m.sum():
        tot = phase[m][:, :6].sum(0).astype(float)
        print("n in (%d,%d]: cycles/ego-net %.0f k; split %s; Jacobi rounds/ego-net: %.0f working + %.0f idle" % (
            lo, hi, tot.sum() / m.sum() / 1e3,
            ", ".join("%s %.0f%%" % (nm, 100 * t / tot.sum()) for nm, t in zip(names, tot)),
            phase[m][:, 6].mean(), phase[m][:, 7].mean()))
