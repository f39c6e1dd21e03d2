"""Corpus builder timings at LiveJournal size (~4.8M vertices, ~69M edge lines) on one GPU: a seeded Chung-Lu .lscc
file and the plain edge list of the same edges, then

  * the read of each file (a sequential read into a 32 MiB buffer; the files were just written, so this is a read
    from the page cache, not from the disk);
  * the GPU build end to end (datasets/x2dgl.build_graph, host clock around work that ends in a synchronise);
  * its parts with CUDA events: the host-to-device copy of the text, the parse kernels alone on device-resident
    text (GB/s of text against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet), the cleaning
    (synthetic.from_keys_device: unique, bincount, remap, cumsum);
  * the host path (numpy parse + synthetic.from_pairs), checked array for array against the GPU build;
  * the reference's per-line loop (x2dgl.py:30-47) plus coo -> csr, restated, on the first 1M edge lines.

    python profiles/x2dgl_time.py --out DIR [--nodes 4800000 --lines 69000000]

The text files go to a temporary directory that is removed at the end; the JSON summary goes to --out.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402

import x2dgl_oracle  # noqa: E402
from gcc_b200 import _capi, _lib  # noqa: E402
from gcc_b200.datasets import synthetic, x2dgl  # noqa: E402

HBM_TBS = 3.35


def ascii_rows(cols, width=8):
    """Rows of non-negative ints (< 10^width) as ASCII text: the columns separated by ' ', rows ended by '\\n'."""
    m = len(cols[0])
    W = len(cols) * (width + 1)
    mat = np.zeros((m, W), np.uint8)
    keep = np.zeros((m, W), bool)
    for c, v in enumerate(cols):
        v = np.asarray(v, np.int64)
        nd = np.maximum(1, np.floor(np.log10(np.maximum(v, 1))).astype(np.int64) + 1)
        for k in range(width):
            mat[:, c * (width + 1) + k] = 48 + (v // 10 ** (width - 1 - k)) % 10
            keep[:, c * (width + 1) + k] = k >= width - nd
        mat[:, c * (width + 1) + width] = 32 if c + 1 < len(cols) else 10
        keep[:, c * (width + 1) + width] = True
    return mat[keep].tobytes()


def write_files(d, n, m, seed=0, piece=8_000_000):
    rng = np.random.default_rng(seed)
    w = (np.arange(n) + 1.0) ** -0.5
    cdf = np.cumsum(w) / w.sum()
    lscc, plain = os.path.join(d, "lj_size.lscc"), os.path.join(d, "lj_size.txt")
    with open(lscc, "wb") as fl, open(plain, "wb") as fp:
        fl.write(b"n %d\n" % n)
        ids = np.arange(n)
        fl.write(ascii_rows([ids, ids]))
        fl.write(b"m %d\n" % m)
        for a in range(0, m, piece):
            c = min(piece, m - a)
            u = np.minimum(np.searchsorted(cdf, rng.random(c), side="right"), n - 1)
            v = np.minimum(np.searchsorted(cdf, rng.random(c), side="right"), n - 1)
            fl.write(ascii_rows([u, v, rng.integers(1, 10, c)]))
            fp.write(ascii_rows([u, v]))
    return lscc, plain


def read_time(path):
    buf = bytearray(32 << 20)
    t = time.perf_counter()
    with open(path, "rb", buffering=0) as f:
        while f.readinto(buf):
            pass
    return time.perf_counter() - t


def cut_points(data, chunk):
    cuts, pos = [], 0
    while pos < len(data):
        end = pos + chunk
        if end >= len(data):
            cuts.append((pos, len(data)))
            break
        c = data.rfind(b"\n", pos, end) + 1
        cuts.append((pos, c))
        pos = c
    return cuts


def parts(path, chunk=x2dgl.DEFAULT_CHUNK, reps=3):
    """H2D copy, parse kernels and cleaning of one file, each timed with CUDA events."""
    lib = _lib.get()
    fmt = x2dgl.file_format(path)
    data = open(path, "rb").read()
    cuts = cut_points(data, chunk)
    host = torch.frombuffer(bytearray(data), dtype=torch.uint8).pin_memory()
    text = torch.empty(len(data), dtype=torch.uint8, device="cuda")
    cap = len(data) // 2 + 2
    keys = torch.empty(cap, dtype=torch.int64, device="cuda")
    ws_bytes = lib.gccb_edgelist_workspace(chunk)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    sp_ = _lib.stream_ptr()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    h2d, parse = [], []
    for _ in range(reps):
        ev[0].record()
        text.copy_(host, non_blocking=True)
        ev[1].record()
        torch.cuda.synchronize()
        h2d.append(ev[0].elapsed_time(ev[1]) / 1e3)
        ev[0].record()
        _lib.check(lib.gccb_edgelist_begin(fmt, _lib.dptr(ws), ws_bytes, sp_))
        for a, b in cuts:
            _lib.check(lib.gccb_edgelist_parse(ctypes.c_void_p(text.data_ptr() + a), b - a, fmt, _lib.dptr(keys), cap,
                                               _lib.dptr(ws), ws_bytes, sp_))
        _lib.check(lib.gccb_edgelist_finish(fmt, _lib.dptr(keys), _lib.dptr(ws), ws_bytes, sp_))
        ev[1].record()
        torch.cuda.synchronize()
        parse.append(ev[0].elapsed_time(ev[1]) / 1e3)
    st = _capi.EdgelistState.from_buffer_copy(ws[:ctypes.sizeof(_capi.EdgelistState)].cpu().numpy().tobytes())
    assert st.first_error == (1 << 64) - 1
    del text, host, ws
    clean = []
    for _ in range(reps):
        k = keys[:st.keys].clone()
        ev[0].record()
        synthetic.from_keys_device([k], int(st.n))
        ev[1].record()
        torch.cuda.synchronize()
        clean.append(ev[0].elapsed_time(ev[1]) / 1e3)
    nb = len(data)
    return dict(bytes=nb, chunks=len(cuts), keys=int(st.keys), h2d_s=h2d, h2d_GBs=nb / min(h2d) / 1e9,
                parse_s=parse, parse_GBs=nb / min(parse) / 1e9,
                parse_text_rate_over_hbm=(nb / min(parse)) / (HBM_TBS * 1e12), clean_s=clean)


def reference_loop(lscc, lines=1_000_000):
    """x2dgl.py:30-47 and :50-53 restated (the loop and coo -> csr), over the first `lines` edge lines."""
    t0 = time.perf_counter()
    with open(lscc, "r") as f:
        n = int(f.readline().split()[1])
        for i in range(n):
            f.readline()
        m = min(int(f.readline().split()[1]), lines)
        t1 = time.perf_counter()
        m_true = 0
        row, col = [0] * (2 * m), [0] * (2 * m)
        for i in range(m):
            u, v, _ = list(map(int, f.readline().split()))
            if u == v:
                continue
            u, v = min(u, v), max(u, v)
            row[m_true], col[m_true] = u, v
            m_true += 1
            row[m_true], col[m_true] = v, u
            m_true += 1
    t2 = time.perf_counter()
    A = sp.coo_matrix(([1] * m_true, (row[:m_true], col[:m_true])), shape=(n, n)).tocsr()
    t3 = time.perf_counter()
    return dict(edge_lines=m, skip_header_s=t1 - t0, loop_s=t2 - t1, coo_tocsr_s=t3 - t2, nnz=int(A.nnz))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory of the JSON summary")
    ap.add_argument("--nodes", type=int, default=4_800_000)
    ap.add_argument("--lines", type=int, default=69_000_000)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    res = {}
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print("gpu:", res["gpu"], flush=True)
    _lib.require_device()
    d = tempfile.mkdtemp(prefix="x2dgl_time_")
    try:
        t = time.perf_counter()
        lscc, plain = write_files(d, args.nodes, args.lines)
        res["write_s"] = time.perf_counter() - t
        warm = os.path.join(d, "warm.txt")
        with open(warm, "wb") as f:
            f.write(b"0 1\n1 2\n")
        x2dgl.build_graph(warm)
        for label, path in (("lscc", lscc), ("plain", plain)):
            r = dict(bytes=os.path.getsize(path), read_s=[read_time(path) for _ in range(2)])
            builds = []
            for _ in range(2):
                torch.cuda.synchronize()
                t = time.perf_counter()
                g = x2dgl.build_graph(path)
                torch.cuda.synchronize()
                builds.append(time.perf_counter() - t)
            r["gpu_build_s"] = builds
            r["graph"] = dict(nodes=g.num_nodes, nnz=len(g.indices))
            r["parts"] = parts(path)
            t = time.perf_counter()
            h = x2dgl_oracle.host_build(path)
            r["host_build_s"] = time.perf_counter() - t
            r["host_equals_gpu"] = bool(np.array_equal(h.indptr, g.indptr.cpu().numpy()) and
                                        np.array_equal(h.indices, g.indices.cpu().numpy()))
            del g, h
            torch.cuda.empty_cache()
            res[label] = r
            print(label, json.dumps(r), flush=True)
        res["reference_loop_1M"] = reference_loop(lscc)
        print("reference loop", json.dumps(res["reference_loop_1M"]), flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    with open(os.path.join(args.out, "x2dgl_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
