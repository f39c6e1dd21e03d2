"""Structural similarity search on the GPU: exact, deterministic cosine top-k over embedding rows.

    python -m gcc_b200.tasks.knn --emb-path A.npy [--candidates B.npy] --k 20 [--nodes ids.txt] [--gpu 0 1 ...] \\
        --output PREFIX            # writes PREFIX.ids.npy (int64) and PREFIX.scores.npy (float32), [queries, k]

For each query row, the k candidate rows of largest cosine similarity, in (score descending, index ascending) order.
Without --candidates the search runs within A and leaves each query's own row out.  The kernel is csrc/knn.cu
(gccb_knn); its definition of the normalisation, the scores and the order is in include/gccb200.h and DESIGN.md 4f.
The output is a function of the rows alone: query chunking, candidate splits and the number of GPUs do not change a
bit of it.
"""
import argparse
import multiprocessing
import multiprocessing.connection
import os
import traceback

import numpy as np

from .. import _capi, _lib

MAX_DIM = 512
MAX_K = 128
CHUNK_BYTES = 1 << 30          # bound on the workspace of one query chunk (plus the normalised candidates)
COPY_ROWS = 1 << 16            # rows per host <-> device copy of the command line: bounds its host memory
WORKER_ERROR_CHARS = 16384


def _check_rows(x, what):
    import torch
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise _lib.GccbError("%s: expected a CUDA tensor (there is no CPU path)" % what)
    if x.dtype != torch.float32 or x.dim() != 2:
        raise ValueError("%s: expected a 2-D float32 tensor, got %s %s" % (what, x.dtype, tuple(x.shape)))
    if not 1 <= x.shape[1] <= MAX_DIM:
        raise ValueError("%s: row width %d outside 1..%d" % (what, x.shape[1], MAX_DIM))
    if x.shape[0] < 1:
        raise ValueError("%s: no rows" % what)
    return x.contiguous()


def _chunk_rows(lib, nq, nc, dim, k, splits, budget):
    """Queries per gccb_knn call: all of them if the workspace fits `budget` beside the normalised candidates, else
    the largest multiple of 64 that does (at least 64)."""
    cands = lib.gccb_knn_workspace(1, nc, dim, k, splits)          # the candidate block, and one query
    rows = nq
    while rows > 64 and lib.gccb_knn_workspace(rows, nc, dim, k, splits) - cands > budget:
        rows = max(64, (rows // 2) // 64 * 64)
    return rows


def _raise_nonfinite(queries, candidates):
    import torch
    for what, x in (("queries", queries), ("candidates", candidates)):
        bad = torch.nonzero(~torch.isfinite(x).all(dim=1))
        if bad.numel():
            raise _lib.GccbError("%s row %d holds a NaN or an Inf" % (what, int(bad[0, 0])))
    raise _lib.GccbError("gccb_knn reported a NaN or an Inf in its input")


def topk_cosine(queries, candidates, k, exclude=None, splits=None, chunk_bytes=CHUNK_BYTES):
    """Exact cosine top-k on the current device (include/gccb200.h, gccb_knn).

    queries [nq, d], candidates [nc, d]: float32 CUDA tensors, 1 <= d <= 512.  k: 1..128.  exclude: None or an int64
    tensor [nq] of candidate ids to leave out (-1: none).  splits: candidate partitions of the score kernel (None:
    chosen from the shapes; the result does not depend on it).  Returns (ids int64 [nq, k], scores float32 [nq, k]),
    in (score descending, candidate index ascending) order.  The candidates are normalised once; the queries go
    through in chunks whose workspace stays within chunk_bytes, with no host synchronisation between them.  Raises
    GccbError naming the first row that holds a NaN or an Inf."""
    import torch
    lib = _lib.get()
    _lib.require_device()
    queries = _check_rows(queries, "queries")
    candidates = _check_rows(candidates, "candidates")
    nq, d = queries.shape
    nc = candidates.shape[0]
    if candidates.shape[1] != d:
        raise ValueError("queries have %d columns, candidates %d" % (d, candidates.shape[1]))
    if queries.device != candidates.device:
        raise ValueError("queries on %s, candidates on %s" % (queries.device, candidates.device))
    admissible = nc - (exclude is not None)
    if not 1 <= k <= MAX_K or k > admissible:
        raise ValueError("k = %d: need 1 <= k <= %d and at most the %d admissible candidates"
                         % (k, MAX_K, admissible))
    S = 0 if splits is None else int(splits)
    if exclude is not None:
        exclude = torch.as_tensor(exclude, dtype=torch.int64, device=queries.device).contiguous()
        if exclude.shape != (nq,):
            raise ValueError("exclude of shape %s, expected (%d,)" % (tuple(exclude.shape), nq))
    dev = queries.device
    with torch.cuda.device(dev):
        rows = _chunk_rows(lib, nq, nc, d, k, S, chunk_bytes)
        last = nq - (nq - 1) // rows * rows
        ws_bytes = max(lib.gccb_knn_workspace(rows, nc, d, k, S), lib.gccb_knn_workspace(last, nc, d, k, S))
        if ws_bytes == 0:
            raise ValueError("gccb_knn refuses nq=%d nc=%d d=%d k=%d splits=%d" % (nq, nc, d, k, S))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
        scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        stream = _lib.stream_ptr()
        for lo in range(0, nq, rows):
            n = min(rows, nq - lo)
            _lib.check(lib.gccb_knn(_lib.dptr(queries[lo:lo + n]), n, _lib.dptr(candidates) if lo == 0 else None,
                                    nc, d, k, None if exclude is None else _lib.dptr(exclude[lo:lo + n]), S,
                                    _lib.dptr(ids[lo:lo + n]), _lib.dptr(scores[lo:lo + n]), _lib.dptr(flags),
                                    _lib.dptr(ws), ws_bytes, stream), "gccb_knn")
        if int(flags.item()) & _capi.FLAG_NONFINITE:
            _raise_nonfinite(queries, candidates)
    return ids, scores


# ---- command line ---------------------------------------------------------------------------------------------------

def _to_device(rows, ids, dev):
    """rows[ids] (ids None: every row) as a float32 tensor on dev, copied COPY_ROWS rows at a time."""
    import torch
    n = rows.shape[0] if ids is None else len(ids)
    out = torch.empty((n, rows.shape[1]), dtype=torch.float32, device=dev)
    for lo in range(0, n, COPY_ROWS):
        hi = min(n, lo + COPY_ROWS)
        block = rows[lo:hi] if ids is None else rows[ids[lo:hi]]
        out[lo:hi] = torch.from_numpy(np.array(block, dtype=np.float32))       # a writable copy of the memmap rows
    return out


def _check_memory(nq, nc, d, k, dev):
    import torch
    lib = _lib.get()
    rows = _chunk_rows(lib, nq, nc, d, k, 0, CHUNK_BYTES)
    ws = max(lib.gccb_knn_workspace(rows, nc, d, k, 0), lib.gccb_knn_workspace(nq - (nq - 1) // rows * rows, nc, d,
                                                                               k, 0))
    need = 4 * (nq + nc) * d + 12 * nq * k + ws
    with torch.cuda.device(dev):
        free = torch.cuda.mem_get_info()[0] + torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
    if need > free:
        raise _lib.GccbError("knn: %d queries x %d candidates of width %d need %.2f GB of device memory (%.2f GB of "
                             "rows, %.2f GB of results, %.2f GB of workspace), %.2f GB are free; sets that do not fit "
                             "are not supported" % (nq, nc, d, need / 1e9, 4 * (nq + nc) * d / 1e9, 12 * nq * k / 1e9,
                                                    ws / 1e9, free / 1e9))


def search_rows(emb_path, cand_path, query_ids, k, gpu, ids_out, scores_out):
    """The search of the queries query_ids (row ids of emb_path) on device `gpu`, written into the [len, k] arrays
    ids_out / scores_out (memmaps or arrays).  Without cand_path the candidates are emb_path's rows and each query's
    own row is excluded."""
    import torch
    torch.cuda.set_device(gpu)
    dev = torch.device("cuda", gpu)
    A = np.load(emb_path, mmap_mode="r")
    C = A if cand_path is None else np.load(cand_path, mmap_mode="r")
    _check_memory(len(query_ids), C.shape[0], A.shape[1], k, dev)
    q = _to_device(A, query_ids, dev)
    c = _to_device(C, None, dev)
    excl = torch.from_numpy(np.asarray(query_ids, np.int64)).to(dev) if cand_path is None else None
    ids, scores = topk_cosine(q, c, k, exclude=excl)
    del q, c
    for lo in range(0, ids.shape[0], COPY_ROWS):
        hi = min(ids.shape[0], lo + COPY_ROWS)
        ids_out[lo:hi] = ids[lo:hi].cpu().numpy()
        scores_out[lo:hi] = scores[lo:hi].cpu().numpy()


def _worker(emb_path, cand_path, query_ids, k, gpu, prefix, lo, hi, conn):
    """One shard in its own process: result rows lo..hi-1.  Sends None, or the traceback if it fails."""
    try:
        ids_out = np.lib.format.open_memmap(prefix + ".ids.npy", mode="r+")
        scores_out = np.lib.format.open_memmap(prefix + ".scores.npy", mode="r+")
        search_rows(emb_path, cand_path, query_ids, k, gpu, ids_out[lo:hi], scores_out[lo:hi])
        ids_out.flush()
        scores_out.flush()
    except BaseException:
        conn.send(traceback.format_exc()[-WORKER_ERROR_CHARS:])
        raise SystemExit(1)
    conn.send(None)


def _run_shards(args, gpus, shards, query_ids):
    """One process per non-empty shard; if one fails, the others are terminated and its error is raised."""
    ctx = multiprocessing.get_context("spawn")
    procs = []
    try:
        for i, (gpu, (lo, hi)) in enumerate(zip(gpus, shards)):
            if lo == hi:
                continue
            recv, send = ctx.Pipe(duplex=False)
            p = ctx.Process(target=_worker, name="knn-shard-%d" % i,
                            args=(args.emb_path, args.candidates, query_ids[lo:hi], args.k, gpu, args.output, lo, hi,
                                  send))
            p.start()
            send.close()
            procs.append((i, gpu, lo, hi, p, recv))
        pending = [p for *_, p, _ in procs]
        while pending:
            multiprocessing.connection.wait([p.sentinel for p in pending])
            for i, gpu, lo, hi, p, recv in procs:
                if p in pending and p.exitcode is not None:
                    pending.remove(p)
                    if p.exitcode != 0:
                        msg = recv.recv() if recv.poll() else "exit code %d" % p.exitcode
                        raise RuntimeError("knn: shard %d (gpu %d, queries %d..%d) failed:\n%s"
                                           % (i, gpu, lo, hi - 1, msg))
    finally:
        for *_, p, recv in procs:
            if p.is_alive():
                p.terminate()
        for *_, p, recv in procs:
            p.join()
            recv.close()


def query_rows(args):
    """(row ids of the queries in --emb-path, number of candidate rows, row width) from the command line."""
    from generate import read_nodes
    A = np.load(args.emb_path, mmap_mode="r")
    if A.ndim != 2:
        raise SystemExit("%s: expected a 2-D array of rows, got shape %s" % (args.emb_path, A.shape))
    nc, d = A.shape
    if args.candidates is not None:
        C = np.load(args.candidates, mmap_mode="r")
        if C.ndim != 2 or C.shape[1] != d:
            raise SystemExit("%s: expected rows of width %d, got shape %s" % (args.candidates, d, C.shape))
        nc = C.shape[0]
    ids = np.arange(A.shape[0], dtype=np.int64)
    if args.nodes:
        ids = read_nodes(args.nodes)
        if ids.min() < 0 or ids.max() >= A.shape[0]:
            raise SystemExit("%s: query ids must lie in 0..%d" % (args.nodes, A.shape[0] - 1))
    admissible = nc - (args.candidates is None)
    if not 1 <= args.k <= min(MAX_K, admissible):
        raise SystemExit("--k %d: need 1 <= k <= %d and at most the %d admissible candidates"
                         % (args.k, MAX_K, admissible))
    if not 1 <= d <= MAX_DIM:
        raise SystemExit("rows of width %d: 1..%d are supported" % (d, MAX_DIM))
    return ids, nc, d


def main(argv=None):
    from generate import parse_gpus, split_shards
    args = parse_args(argv)
    ids, _, _ = query_rows(args)
    gpus = parse_gpus(args.gpu)
    n = len(ids)
    paths = [args.output + ".ids.npy", args.output + ".scores.npy"]
    ids_out = np.lib.format.open_memmap(paths[0], mode="w+", dtype=np.int64, shape=(n, args.k))
    scores_out = np.lib.format.open_memmap(paths[1], mode="w+", dtype=np.float32, shape=(n, args.k))
    try:
        if len(gpus) == 1:
            search_rows(args.emb_path, args.candidates, ids, args.k, gpus[0], ids_out, scores_out)
            ids_out.flush()
            scores_out.flush()
        else:
            del ids_out, scores_out
            _run_shards(args, gpus, split_shards(n, 1, len(gpus)), ids)
    except BaseException:
        for p in paths:
            if os.path.exists(p):
                os.remove(p)
        raise
    print("saved the top %d of %d queries to %s and %s" % (args.k, n, paths[0], paths[1]))
    return paths


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--emb-path", type=str, required=True, help="query rows: a 2-D float .npy (e.g. generate.py's)")
    ap.add_argument("--candidates", type=str, default=None,
                    help="candidate rows (.npy of the same width); default: --emb-path, each query's own row excluded")
    ap.add_argument("--k", type=int, default=20, help="neighbours per query, 1..%d" % MAX_K)
    ap.add_argument("--nodes", type=str, default=None,
                    help="a .npy or text file of query row ids: search only those, in the file's order")
    ap.add_argument("--gpu", default=None, type=int, nargs="+",
                    help="GPU id(s): one contiguous shard of the queries per entry, each in its own process")
    ap.add_argument("--output", type=str, required=True, help="prefix of PREFIX.ids.npy and PREFIX.scores.npy")
    return ap.parse_args(argv)


if __name__ == "__main__":
    main()
