"""Linear-probe classification on the GPU: exact one-vs-rest logistic regression over embedding rows.

    python -m gcc_b200.tasks.linear_probe --emb-path rows.npy --dataset D [--seed S] [--gpu I]

The model of the reference's node evaluator (OneVsRestClassifier(LogisticRegression(C=1000)), each test row predicting
its k labels' worth of classes), fitted to a stated tolerance in float64 on the GPU under the same shuffled
stratified 10-fold split of the argmax labels; prints the mean micro-F1 over the folds as {"Micro-F1": ...}.  The
kernel is csrc/probe.cu (gccb_probe_fit); the definition of the problems, the solver, its stopping rule and the
prediction is in include/gccb200.h and DESIGN.md 4g.  The result is a function of the inputs: it does not depend on
how many problems share a launch, or on the device.

D is a named node dataset (the feature matrix NodeClassification.train builds: the rows of the vertices that have
edges, zeros elsewhere), an .npz with `y` (the finetune format: the file's rows as they are; a 1-D y is one label per
row, a 2-D y a 0/1 label matrix), or anything graph_classification.graph_labels accepts (one row per graph).
"""
import argparse
import collections
import json

import numpy as np

from .. import _capi, _lib

MAX_DIM = 256
MAX_CLASSES = 1024
FOLDS = 10
MAX_ITER = 100

ProbeResult = collections.namedtuple("ProbeResult", ["weights", "decision", "f1", "iters", "status"])


def label_matrix(y):
    """0/1 uint8 [n, c]: a 1-D integer label vector one-hot (c = max + 1), a 2-D label matrix as it is."""
    y = np.asarray(y)
    if y.ndim == 1:
        y = y.astype(np.int64)
        if y.size and y.min() < 0:
            raise ValueError("labels must be non-negative, got %d" % y.min())
        Y = np.zeros((len(y), int(y.max()) + 1 if y.size else 1), np.uint8)
        Y[np.arange(len(y)), y] = 1
        return Y
    if y.ndim != 2:
        raise ValueError("labels of shape %s: expected a vector or a matrix" % (y.shape,))
    return (np.asarray(y) != 0).astype(np.uint8)


def fold_ids(Y, seed, folds=FOLDS):
    """The test fold of each row: StratifiedKFold(n_splits=folds, shuffle=True, random_state=seed) over Y.argmax(1),
    the folds both reference evaluators use."""
    from sklearn.model_selection import StratifiedKFold
    labels = np.asarray(Y).argmax(axis=1)
    out = np.full(len(labels), -1, np.int32)
    skf = StratifiedKFold(n_splits=folds, shuffle=True, random_state=seed)
    for f, (_, test) in enumerate(skf.split(np.zeros(len(labels)), labels)):
        out[test] = f
    return out


def _device_inputs(rows, Y, folds, dev):
    import torch

    def put(a, dtype):
        if isinstance(a, torch.Tensor):
            return a.to(device=dev, dtype=dtype).contiguous()
        return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dtype).contiguous()
    return put(rows, torch.float32), put(Y, torch.uint8), put(folds, torch.int32)


def probe_bytes(n, d, c, folds=FOLDS, batch=0):
    """Device bytes of a fit: the rows, labels and fold ids, the outputs and the workspace."""
    lib = _lib.get()
    P = folds * c
    return (4 * n * d + n * c + 4 * n + 8 * n * c + 8 * P * (d + 1) + 24 * folds + 16 * P +
            lib.gccb_probe_workspace(n, d, c, folds, batch))


def _free_bytes(dev):
    import torch
    with torch.cuda.device(dev if dev is not None else torch.cuda.current_device()):
        return torch.cuda.mem_get_info()[0] + torch.cuda.memory_reserved() - torch.cuda.memory_allocated()


def check_memory(n, d, c, folds=FOLDS, batch=0, dev=None):
    """The problems per launch for a fit of this shape: `batch` if given, else the largest of P = folds c, P/2, P/4,
    ... (at least 1) whose fit fits in the free device memory.  The result does not depend on it.  Raises GccbError
    with the sizes if even that does not fit."""
    lib = _lib.get()
    free = _free_bytes(dev)
    b = batch if batch > 0 else folds * c
    while batch <= 0 and b > 1 and probe_bytes(n, d, c, folds, b) > free:
        b = (b + 1) // 2
    need = probe_bytes(n, d, c, folds, b)
    if need > free:
        ws = lib.gccb_probe_workspace(n, d, c, folds, b)
        raise _lib.GccbError("linear probe: %d rows of width %d with %d classes x %d folds need %.2f GB of device "
                             "memory at %d problem%s per launch (%.2f GB of rows and labels, %.2f GB of decision "
                             "values, %.2f GB of workspace), %.2f GB are free; sets that do not fit are not supported"
                             % (n, d, c, folds, need / 1e9, b, "" if b == 1 else "s", (4 * n * d + n * c + 4 * n) / 1e9,
                                8 * n * c / 1e9, ws / 1e9, free / 1e9))
    return b


def _check_shapes(n, d, c, nY, nf):
    if nY != n:
        raise ValueError("%d embedding rows for %d label rows: the rows must be one per labelled item, in order"
                         % (n, nY))
    if nf != n:
        raise ValueError("%d fold ids for %d rows" % (nf, n))
    if not 1 <= d <= MAX_DIM:
        raise ValueError("rows of width %d: 1..%d are supported (every encoder width: 64, 128, 256)" % (d, MAX_DIM))
    if not 1 <= c <= MAX_CLASSES:
        raise ValueError("%d classes: 1..%d are supported" % (c, MAX_CLASSES))


def fit_probe(rows, Y, folds, C=1000.0, n_folds=FOLDS, batch=0, max_iter=MAX_ITER):
    """The one-vs-rest logistic regression of every (fold, class) problem on the current device (gccb_probe_fit).

    rows [n, d] float32 (numpy or CUDA tensor), Y [n, c] 0/1, folds [n] test fold ids in 0..n_folds-1.  batch: the
    problems per launch (0: as many as fit in free device memory; the result does not depend on it).  Returns a ProbeResult of numpy arrays: weights
    [n_folds, c, d + 1] float64 (intercept last; zeros for a constant predictor), decision [n, c] float64 (the decision
    values of each row under its own fold's problems, +-inf for a constant predictor), f1 [n_folds] (micro-F1 of each
    fold's test rows), iters and status [n_folds, c].  Raises GccbError naming the first row that holds a NaN or an
    Inf, or the fold, class and final gradient norm of a problem that did not converge."""
    import torch
    lib = _lib.get()
    _lib.require_device()
    if len(rows.shape) != 2:
        raise ValueError("rows of shape %s: expected a 2-D array" % (tuple(rows.shape),))
    n, d = rows.shape
    c = Y.shape[1]
    _check_shapes(n, d, c, Y.shape[0], folds.shape[0])
    dev = rows.device if isinstance(rows, torch.Tensor) and rows.is_cuda else torch.device("cuda",
                                                                                          torch.cuda.current_device())
    with torch.cuda.device(dev):
        batch = check_memory(n, d, c, n_folds, batch, dev)
        x, y, fo = _device_inputs(rows, Y, folds, dev)
        P = n_folds * c
        ws_bytes = lib.gccb_probe_workspace(n, d, c, n_folds, batch)
        if ws_bytes == 0:
            raise ValueError("gccb_probe_fit refuses n=%d d=%d c=%d folds=%d" % (n, d, c, n_folds))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        w = torch.empty((P, d + 1), dtype=torch.float64, device=dev)
        z = torch.empty((n, c), dtype=torch.float64, device=dev)
        counts = torch.empty((n_folds, 3), dtype=torch.int64, device=dev)
        status = torch.empty(P, dtype=torch.int32, device=dev)
        gnorm = torch.empty(P, dtype=torch.float64, device=dev)
        iters = torch.empty(P, dtype=torch.int32, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        D = _lib.dptr
        _lib.check(lib.gccb_probe_fit(D(x), n, d, D(y), c, D(fo), n_folds, float(C), max_iter, batch, D(w), D(z),
                                      D(counts), D(status), D(gnorm), D(iters), D(flags), D(ws), ws_bytes,
                                      _lib.stream_ptr()), "gccb_probe_fit")
        fl = int(flags.item())
        if fl & _capi.FLAG_NONFINITE:
            bad = torch.nonzero(~torch.isfinite(x).all(dim=1))
            raise _lib.GccbError("linear probe: row %d holds a NaN or an Inf" % int(bad[0, 0]) if bad.numel()
                                 else "gccb_probe_fit reported a NaN or an Inf in its input")
        st = status.cpu().numpy()
        if fl & _capi.FLAG_PROBE_NOCONV:
            gn = gnorm.cpu().numpy()
            it = iters.cpu().numpy()
            failed = (_capi.GCCB_PROBE_NOCONV, _capi.GCCB_PROBE_LS_FAIL, _capi.GCCB_PROBE_NOT_PD)
            p = int(np.nonzero(np.isin(st, failed))[0][0])
            raise _lib.GccbError("linear probe: the problem of fold %d, class %d did not converge (%s) after %d "
                                 "Newton iterations; final gradient norm %.3e"
                                 % (p // c, p % c, _capi.PROBE_STATUS[int(st[p])], it[p], gn[p]))
        cnt = counts.cpu().numpy()
        tp, fp, fn = cnt[:, 0], cnt[:, 1], cnt[:, 2]
        den = 2 * tp + fp + fn
        f1 = np.where(den > 0, 2 * tp / np.maximum(den, 1), 0.0)
        return ProbeResult(w.cpu().numpy().reshape(n_folds, c, d + 1), z.cpu().numpy(), f1,
                           iters.cpu().numpy().reshape(n_folds, c), st.reshape(n_folds, c))


# ---- datasets and command line --------------------------------------------------------------------------------------

def load_task(dataset, emb_path, root="data"):
    """(rows [n, d] float32, Y [n, c] uint8) of `dataset` with the rows of emb_path, resolved by the existing readers:
    a named node dataset, an .npz with y (finetune format), or what graph_classification.graph_labels accepts."""
    from ..datasets.downstream import NODE_DSETS, create_node_classification_dataset
    from . import edge_nodes
    from .graph_classification import graph_labels
    emb = np.load(emb_path, mmap_mode="r")
    if emb.ndim != 2:
        raise ValueError("%s: expected a 2-D array of rows, got shape %s" % (emb_path, emb.shape))
    if dataset in NODE_DSETS:
        data = create_node_classification_dataset(dataset, root).data
        Y = label_matrix(data.y.numpy())
        nodes = edge_nodes(data.edge_index.numpy())
        if len(emb) <= int(nodes.max()):
            raise ValueError("%d embedding rows for the %d nodes of %s" % (len(emb), len(Y), dataset))
        rows = np.zeros((len(Y), emb.shape[1]), np.float32)
        rows[nodes] = emb[nodes]
        return rows, Y
    if dataset.endswith(".npz"):
        with np.load(dataset) as z:
            has_y = "y" in z.files
            y = z["y"] if has_y else None
        if has_y:
            Y = label_matrix(y)
            if len(emb) != len(Y):
                raise ValueError("%d embedding rows for %d label rows in %s" % (len(emb), len(Y), dataset))
            return np.ascontiguousarray(emb, np.float32), Y
    labels = graph_labels(dataset, root)
    if len(emb) != len(labels):
        raise ValueError("%d embedding rows for %d graph labels: the rows must be one per graph, in order"
                         % (len(emb), len(labels)))
    return np.ascontiguousarray(emb, np.float32), label_matrix(labels)


def main(argv=None):
    import torch
    args = parse_args(argv)
    rows, Y = load_task(args.dataset, args.emb_path, args.root)
    folds = fold_ids(Y, args.seed)
    torch.cuda.set_device(args.gpu)
    res = fit_probe(rows, Y, folds)
    ret = {"Micro-F1": float(np.mean(res.f1))}
    print(json.dumps(ret))
    return ret


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--emb-path", type=str, required=True, help="rows: a 2-D float .npy (e.g. generate.py's)")
    ap.add_argument("--dataset", type=str, required=True,
                    help="a named node dataset, an .npz with y, a graph dataset name, TU directory or .npz with "
                         "graph_labels")
    ap.add_argument("--seed", type=int, default=0, help="random_state of the stratified 10-fold split")
    ap.add_argument("--gpu", type=int, default=0, help="GPU id")
    ap.add_argument("--root", type=str, default="data", help="directory of the named datasets")
    return ap.parse_args(argv)


if __name__ == "__main__":
    main()
