#!/usr/bin/env python
"""GPU diagnostic: the dense tridiagonal eigensolver up to 96 (the default) and up to 228 vertices on the same batches
(gccb_posenc reads GCCB200_DENSE_MAX on every call), with the dense solver's phase cycle counters."""
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
lib = _lib.get()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]


def posenc(buf, dense_max):
    if dense_max is None:
        os.environ.pop("GCCB200_DENSE_MAX", None)
    else:
        os.environ["GCCB200_DENSE_MAX"] = str(dense_max)
    ev[0].record()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 1, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                               _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1])


variants = [("dense<=228", 228), ("dense<=96", None)]
tot = {k: [] for k, _ in variants}
for st in range(int(sys.argv[2]) if len(sys.argv) > 2 else 8):
    buf = ds.sample_batch(posenc=False)
    torch.cuda.synchronize()
    for name, dm in variants:
        posenc(buf, dm)                                  # warm (first call sets the smem attributes)
        tot[name].append(min(posenc(buf, dm) for _ in range(2)))
    flags = int(buf.flags.item())
    buf.flags.zero_()
    n = buf.counters[:, 0].cpu().numpy()
    print("batch %d: largest n %s, flags %d, posenc ms %s" % (
        st, sorted(n.tolist())[-3:], flags, ", ".join("%s %.2f" % (k, tot[k][-1]) for k, _ in variants)))
print("mean posenc ms per batch: " + ", ".join("%s %.3f" % (k, np.mean(v)) for k, v in tot.items()))
posenc(buf, 228)
it, res = buf.eig_debug()
it, res = it.cpu().numpy(), res.cpu().numpy()
ph = buf.eig_phases().cpu().numpy()
n = buf.counters[:, 0].cpu().numpy()
names = ["setup", "tridiagonalisation", "multisection", "inverse iteration", "gram-schmidt", "back-transformation"]
for lo, hi in ((0, 96), (96, 144), (144, 228)):
    m = (n > lo) & (n <= hi) & (it == 0)
    if m.sum():
        t = ph[m][:, :6].sum(0).astype(float)
        print("dense n in (%d,%d]: %d ego-nets, cycles/ego-net %.0f k; split %s; kernel-side residual max %.1e" % (
            lo, hi, m.sum(), t.sum() / m.sum() / 1e3, ", ".join("%s %.0f%%" % (nm, 100 * x / t.sum()) for nm, x in zip(names, t)),
            res[m].max()))
