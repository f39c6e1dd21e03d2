"""Whole-graph embedding: (a) the seed-first relabel of a graph corpus on the host (seed_first_union, one graph at a
time) against the device build (gccb_seed_first_union), on ~10^6 small synthetic graphs and on the same corpus with
three 10^5-vertex graphs added; the kernel is timed alone with CUDA events (median of 5) and its achieved bytes/s is
the algorithmic volume 2 * (8 * (V + 1) + 4 * E) + 16 * G over that time, against the H100 SXM data-sheet 3.35 TB/s.
(b) Whole-graph rows in graphs/s through EmbedEngine, serial (prefetch 0) against run-ahead (prefetch 4), GIN hidden
64 and 128, on a REDDIT-BINARY-sized synthetic set (2,000 graphs, ~430 vertices and ~1,000 entries on average),
B = 256; the arms alternate in one process and must write identical bytes.  Prints the GPU's name, power limit and SM
clock read in the same run, and a JSON summary.

    python profiles/graph_embed_time.py [--rounds 3 --out out/graph_embed_time.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gcc_b200 import _capi, _lib  # noqa: E402
from gcc_b200.datasets import synthetic  # noqa: E402
from gcc_b200.datasets.graph_dataset import DeviceGraphSet, WholeGraphDataset, seed_first_union  # noqa: E402
from gcc_b200.embed import EmbedEngine  # noqa: E402
from gcc_b200.models import GraphEncoder  # noqa: E402

PEAK_BW = 3.35e12


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True)
    return dict(zip(q.split(","), (v.strip() for v in r.stdout.strip().split(","))))


def small_corpus(G, seed):
    """G graphs of 1..8 vertices with 0..2 random entries per vertex (rows sorted; parallel edges, self loops and
    isolated vertices occur), as one union CSR and its sizes."""
    rng = np.random.RandomState(seed)
    n = rng.randint(1, 9, G)
    m = rng.randint(0, 3, G) * n
    return n, m, rng


def union_of(parts):
    """[(n [G], m [G], rng)] -> (union CSRGraph, sizes); entries drawn inside each graph."""
    sizes = np.concatenate([p[0] for p in parts])
    m = np.concatenate([p[1] for p in parts])
    rng = parts[0][2]
    node_off = np.concatenate([[0], np.cumsum(sizes)])
    gid = np.repeat(np.arange(len(sizes)), m)
    src = node_off[gid] + (rng.random_sample(len(gid)) * sizes[gid]).astype(np.int64)
    dst = node_off[gid] + (rng.random_sample(len(gid)) * sizes[gid]).astype(np.int64)
    order = np.lexsort((dst, src))
    V = int(node_off[-1])
    indptr = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=V), out=indptr[1:])
    return synthetic.CSRGraph(indptr, dst[order].astype(np.int32), V, "corpus"), sizes


def split(union, sizes):
    no = np.concatenate([[0], np.cumsum(sizes)])
    ip, ix = union.indptr, union.indices
    return [synthetic.CSRGraph(ip[a:b + 1] - ip[a], (ix[ip[a]:ip[b]] - a).astype(np.int32), int(b - a), "g")
            for a, b in zip(no[:-1], no[1:])]


def relabel_arm(name, union, sizes):
    graphs = split(union, sizes)
    V, E, G = union.num_nodes, len(union.indices), len(sizes)
    t0 = time.perf_counter()
    seed_first_union(graphs)
    host_s = time.perf_counter() - t0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = DeviceGraphSet.from_union(union, sizes, "cuda")
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0                          # upload, relabel, seeds to the host
    dev = torch.device("cuda")
    src_ptr = torch.from_numpy(union.indptr).to(dev)
    src_idx = torch.from_numpy(union.indices).to(dev)
    src = _capi.GraphSet(src_ptr.data_ptr(), src_idx.data_ptr(), s.node_off.data_ptr(), s.edge_off.data_ptr(), G)
    out_ip, out_ix = torch.empty_like(s.indptr), torch.empty_like(s.indices)
    seeds, flags = torch.empty(G, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    times = []
    for _ in range(6):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(_lib.get().gccb_seed_first_union(C.byref(src), V, E, _lib.dptr(seeds), _lib.dptr(out_ip),
                                                    _lib.dptr(out_ix), _lib.dptr(flags), _lib.stream_ptr()), "relabel")
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    kernel_s = float(np.median(times[1:]))
    assert torch.equal(out_ip, s.indptr) and torch.equal(out_ix, s.indices) and int(flags.item()) == 0
    nbytes = 2 * (8 * (V + 1) + 4 * E) + 16 * G
    r = dict(corpus=name, graphs=G, vertices=V, entries=E, host_s=host_s, device_build_s=build_s,
             kernel_s=kernel_s, kernel_bytes=nbytes, kernel_bw=nbytes / kernel_s,
             kernel_bw_frac=nbytes / kernel_s / PEAK_BW, host_over_kernel=host_s / kernel_s,
             host_over_build=host_s / build_s)
    print("relabel %-24s G=%d V=%d E=%d  host %.2f s  device build %.3f s  kernel %.3f ms  %.0f GB/s (%.1f %% of "
          "3.35 TB/s)  host/kernel %.0fx  host/build %.1fx"
          % (name, G, V, E, host_s, build_s, kernel_s * 1e3, nbytes / kernel_s / 1e9,
             100 * nbytes / kernel_s / PEAK_BW, host_s / kernel_s, host_s / build_s))
    return r


def reddit_like(seed=0):
    """2,000 graphs: vertex counts log-normal around 430 (6..3,782), a random tree plus 16 % extra edges, both
    directions listed."""
    rng = np.random.RandomState(seed)
    graphs = []
    for i in range(2000):
        n = int(np.clip(rng.lognormal(np.log(300), 0.8), 6, 3782))
        parent = (rng.random_sample(n - 1) * np.arange(1, n)).astype(np.int64)
        extra = rng.randint(0, n, (int(0.16 * n), 2))
        u = np.concatenate([np.arange(1, n), extra[:, 0]])
        v = np.concatenate([parent, extra[:, 1]])
        keep = u != v
        src, dst = np.concatenate([u[keep], v[keep]]), np.concatenate([v[keep], u[keep]])
        order = np.lexsort((dst, src))
        indptr = np.zeros(n + 1, np.int64)
        np.cumsum(np.bincount(src, minlength=n), out=indptr[1:])
        graphs.append(synthetic.CSRGraph(indptr, dst[order].astype(np.int32), n, "r%d" % i))
    return graphs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    state = gpu_state()
    print("gpu:", state)
    out = dict(gpu=state, relabel=[], embed={})
    small = small_corpus(1_000_000, 1)
    out["relabel"].append(relabel_arm("1M small graphs", *union_of([small])))
    rng = np.random.RandomState(2)
    big = (np.full(3, 100_000), np.full(3, 300_000), rng)
    out["relabel"].append(relabel_arm("1M small + 3 x 1e5-vertex", *union_of([small, big])))

    graphs = reddit_like()
    ds = WholeGraphDataset(graphs, positional_embedding_size=32, batch_size=256)
    print("reddit-like: %d graphs, %d vertices, %d entries" % (len(graphs), int(ds.graph_set.sizes.sum()),
                                                               int(ds.graph_set.nnz.sum())))
    for H in (64, 128):
        torch.manual_seed(0)
        model = GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                             node_hidden_dim=H, num_layers=5, norm=True, gnn_model="gin",
                             degree_input=True).cuda().eval()
        engines = {S: EmbedEngine(ds, model, prefetch=S) for S in (0, 4)}
        res, rows = {0: [], 4: []}, {}
        for S in (0, 4):                                        # warm-up: allocations, first launches
            engines[S].run(range(len(graphs)))
        for r in range(args.rounds):
            for S in (0, 4):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rows[S] = engines[S].run(range(len(graphs)))
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                res[S].append(len(graphs) / dt)
                print("embed gin h%d prefetch %d round %d: %.3f s, %.0f graphs/s" % (H, S, r, dt, len(graphs) / dt))
        assert rows[0].tobytes() == rows[4].tobytes(), "prefetch 0 and 4 wrote different rows"
        med = {S: float(np.median(v)) for S, v in res.items()}
        print("embed gin h%d: serial %.0f graphs/s, run-ahead %.0f graphs/s (%.2fx), identical bytes"
              % (H, med[0], med[4], med[4] / med[0]))
        out["embed"]["gin h%d" % H] = dict(serial=med[0], run_ahead=med[4], speedup=med[4] / med[0],
                                           node_cap=engines[4].node_cap, edge_cap=engines[4].edge_cap)
        del engines
    out["gpu_after"] = gpu_state()
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
