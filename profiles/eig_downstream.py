#!/usr/bin/env python
"""CPU experiment (kernel LOGIC under the emulator of tests/emu + the torch-CPU oracle model): what does the
eigensolver's inexactness do downstream?  VERDICT r01, missing #6.

For one sampled batch (C2-like ego-nets, hubs included) the encoder (5-layer GIN, hidden 64, random init, train-mode
BatchNorm, float64 oracle model) is run on positional features from
  ours      the device solvers (emulated): default mix (dense n <= 96, ChFSI above), dense up to 228;
  ours*     the SAME vectors projected onto the exact invariant subspace of the top-k eigenvalues (the whole multiple
            eigenvalue the cut falls into included) and re-orthonormalised (float64 eigh, polar factor): what the
            solver would return if it were exact, in the same basis -- so the difference
            ours - ours* isolates the inexactness from the arbitrariness of the basis;
  ref1/ref2 two runs of the reference's own call (scipy eigsh, float64, random v0, data_util.py:242-263): the basis
            inside a multiple eigenvalue and every sign are arbitrary there, so ref1 - ref2 is the reference's own
            run-to-run spread.
Reported per graph: || f(ours) - f(ours*) || and || f(ref1) - f(ref2) || for the unit-norm embeddings f."""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from emu_util import NpBatch, lib, ptr  # noqa: E402
from gcc_b200.datasets import synthetic  # noqa: E402
from gcc_b200.models import GraphEncoder  # noqa: E402
from oracle import model as om  # noqa: E402
from oracle import posenc as opos  # noqa: E402
from oracle import rwr as orwr  # noqa: E402


def solver_features(views, dense_max):
    os.environ["GCCB200_DENSE_MAX"] = str(dense_max)
    L = lib()
    b = NpBatch.from_subgraphs(views)
    pos = np.zeros((2, b.node_cap, 32), np.float32)
    ws = np.zeros(L.gccb_posenc_workspace(b.B, b.node_cap), np.uint8)
    assert L.gccb_posenc(C.byref(b.c), 32, 0, ptr(pos), None, ptr(ws), ws.nbytes, None) == 0
    return b, pos                                          # raw unit eigenvectors (normalize = 0)


def finish(u):
    nrm = np.sqrt((u * u).sum(axis=1, keepdims=True))
    nrm[nrm == 0.0] = 1.0
    return u / nrm                                         # sklearn normalize(norm="l2"), data_util.py:260


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 48
    g = synthetic.chung_lu(100000, 2000000, seed=0)
    seeds = orwr.draw_seeds(orwr.seed_cdf(g.indptr), 42, range(B))
    bt = orwr.budget_table(int(np.diff(g.indptr).max()), 256, 0.8)
    subs = orwr.rwr_batch(g.indptr, g.indices, 42, np.arange(B), seeds, bt, orwr.restart_threshold(0.8),
                          int(bt.max()) + 65, 1 << 20)
    views = [subs[0::2], subs[1::2]]
    lst = views[0]                                         # the query view is enough
    sizes = np.array([s["n"] for s in lst])
    laps = [opos.normalized_adjacency(s["indptr"], s["indices"], s["n"]).toarray() for s in lst]
    exact = [np.linalg.eigh(a) for a in laps]
    feats = {}
    for name, dm in (("default (dense <= 96)", 96), ("dense <= 228", 228)):
        b, pos = solver_features(views, dm)
        got, proj = [], []
        for gi, s in enumerate(lst):
            a, z = b.node_off[0, gi], b.node_off[0, gi + 1]
            n = s["n"]
            k = min(n - 2, 32)
            x = pos[0, a:z, :k].astype(np.float64)
            w, v = exact[gi]
            lo = int(np.searchsorted(w, w[n - k] - 1e-7))  # the whole multiple eigenvalue the top-k cut falls into
            vk = v[:, lo:]                                 # exact invariant subspace that contains every valid answer
            y = vk @ (vk.T @ x)
            uu, _, vt = np.linalg.svd(y, full_matrices=False)
            y = uu @ vt                                    # closest orthonormal basis (polar factor)
            pad = np.zeros((n, 32 - k))
            got.append(np.hstack([finish(x), pad]))
            proj.append(np.hstack([finish(y), pad]))
        feats[name] = (np.vstack(got), np.vstack(proj))
    rng1, rng2 = np.random.RandomState(1), np.random.RandomState(2)
    ref = [np.vstack([opos.posenc_reference_call(s["indptr"], s["indices"], s["n"], 32, rng=r).astype(np.float64) for s in lst])
           for r in (rng1, rng2)]
    # the encoder
    torch.manual_seed(0)
    model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=64,
                         node_hidden_dim=64, num_layers=5, norm=True, gnn_model="gin", degree_input=True)
    P = {k: v.detach().double() for k, v in model.state_dict().items()}
    noff = b.node_off[0].astype(np.int64)
    N, M = int(noff[-1]), int(b.edge_off[0, b.B])
    seed_flag = np.zeros(N, np.int64)
    seed_flag[noff[:-1]] = 1
    args = (b.indptr[0, :N + 1].astype(np.int64), b.indices[0, :M].astype(np.int64))

    def embed(p):
        with torch.no_grad():
            f, _, _ = om.gin_encoder_forward(P, args[0], args[1], torch.from_numpy(p), seed_flag, b.sub_deg[0, :N], noff,
                                             num_layers=5, bn_train=True)
        return f.numpy()

    f_ref = [embed(r) for r in ref]
    d_ref = np.linalg.norm(f_ref[0] - f_ref[1], axis=1)
    print("batch: %d ego-nets, sizes min/median/max %d/%d/%d, %d above 160 vertices" % (
        len(lst), sizes.min(), np.median(sizes), sizes.max(), (sizes > 160).sum()))
    print("reference run-to-run spread  || f(ref1) - f(ref2) ||: median %.2e, max %.2e (unit-norm embeddings)" % (
        np.median(d_ref), d_ref.max()))
    for name, (x, y) in feats.items():
        d = np.linalg.norm(embed(x) - embed(y), axis=1)
        hub = sizes > 160
        per_node = np.abs(x - y).max(axis=1)
        cls = np.repeat(sizes, sizes)                      # ego-net size of every node row

        def worst(m):
            return per_node[m].max() if m.any() else 0.0
        print("%-22s || f(ours) - f(ours*) ||: median %.2e, max %.2e; ego-nets above 160 vertices: max %.2e; feature "
              "difference max |x - x*|: n <= 96 %.1e, 96 < n <= 228 %.1e, n > 228 %.1e" % (
                  name, np.median(d), d.max(), d[hub].max() if hub.any() else 0.0, worst(cls <= 96),
                  worst((cls > 96) & (cls <= 228)), worst(cls > 228)))


if __name__ == "__main__":
    main()
