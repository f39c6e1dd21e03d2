"""Time the linear probe (gcc_b200.tasks.linear_probe.fit_probe, csrc/probe.cu) at ogbn-products-like sizes, and one
fold of the reference's host evaluator on the same machine.

    python profiles/linear_probe_time.py [--n 2000000] [--sklearn 64x47,128x10] [--out linear_probe_time.json]

Seeded rows with a noisy linear signal per class.  For each shape (n x 64 with 47 classes, n x 128 with 10 classes):
the full 10-fold fit timed with CUDA events (after a warm-up fit of the same width on 50k rows), its Newton
iterations, the seconds of each probe kernel in that fit (torch.profiler, a second identical fit), and the Hessian pass (probe_gram_kernel) alone from torch.profiler over one gccb_probe_system call on
every problem: its time per Newton iteration and its FP64 rate, counted as the useful upper-triangle work
P n_train d1 (d1 + 1) and as the work the tensor cores execute (the padded 8 x 8 blocks), each against the
67 TFLOP/s FP64 tensor-core figure of the H100 SXM data sheet.  --sklearn WxC,... also times ONE fold of the default
reference evaluator (OneVsRestClassifier(LogisticRegression(C=1000)), lbfgs) at n rows of that shape on the host CPU
("none" skips it).  The card's name, power limit and clocks are read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gcc_b200 import _lib  # noqa: E402
from gcc_b200.tasks import linear_probe as lp  # noqa: E402

PEAK_FP64_TC = 67e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out.splitlines()[0] if out else "unavailable"


def make(n, d, c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn((n, d), device="cuda", generator=g)
    U = torch.randn((d, c), device="cuda", generator=g) / d ** 0.5
    S = X @ U * 3.0 + torch.randn((n, c), device="cuda", generator=g)
    Y = np.zeros((n, c), np.uint8)
    Y[np.arange(n), S.argmax(1).cpu().numpy()] = 1
    return X, Y


def gram_time(X, Y, folds):
    """Seconds of probe_gram_kernel in one gccb_probe_system call over every problem (w = 0)."""
    lib = _lib.get()
    n, d = X.shape
    c = Y.shape[1]
    P = 10 * c
    y = torch.from_numpy(Y).cuda()
    fo = torch.from_numpy(folds).cuda()
    ws_b = lib.gccb_probe_workspace(n, d, c, 10, 0)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    w = torch.zeros((P, d + 1), dtype=torch.float64, device="cuda")
    g = torch.empty_like(w)
    H = torch.empty((P, d + 1, d + 1), dtype=torch.float64, device="cuda")
    st = torch.empty_like(w)
    f = torch.empty(P, dtype=torch.float64, device="cuda")
    status = torch.empty(P, dtype=torch.int32, device="cuda")
    D = _lib.dptr

    def call():
        _lib.check(lib.gccb_probe_system(D(X), n, d, D(y), c, D(fo), 10, 1000.0, 0, D(w), D(g), D(H), D(st), D(f),
                                         D(status), D(ws), ws_b, _lib.stream_ptr()), "gccb_probe_system")
    call()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "probe_gram_kernel" in e.key)
    solve = sum(e.device_time_total for e in prof.key_averages() if "probe_solve_kernel" in e.key)
    return us / 1e6, solve / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2_000_000)
    ap.add_argument("--sklearn", type=str, default="64x47,128x10",
                    help="comma-separated WxC shapes for which to time one host fold, or none")
    ap.add_argument("--out", type=str, default=None, help="also write the JSON summary here")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _lib.require_device()
    res = {"gpu": gpu_info(), "n": args.n, "runs": []}
    print(res["gpu"], flush=True)
    for d, c in ((64, 47), (128, 10)):
        X, Y = make(args.n, d, c, d)
        folds = lp.fold_ids(Y, 0)
        lp.fit_probe(X[:50000], Y[:50000], folds[:50000])                  # warm-up at the same width
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        r = lp.fit_probe(X, Y, folds)
        b.record()
        torch.cuda.synchronize()
        t = a.elapsed_time(b) / 1e3
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            lp.fit_probe(X, Y, folds)                                        # the same fit, kernel by kernel
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if "probe_" in e.key:
                name = e.key.split("probe_")[1].split("_kernel")[0]
                kernels[name] = kernels.get(name, 0.0) + e.device_time_total / 1e6
        P, d1 = 10 * c, d + 1
        n_train = args.n * 0.9
        tg, ts = gram_time(X, Y, folds)
        nb = (d1 + 7) // 8
        useful = P * n_train * d1 * (d1 + 1)
        executed = P * args.n * nb * (nb + 1) / 2 * 64 * 2
        row = {"n": args.n, "d": d, "classes": c, "problems": P, "fit_s": t,
               "newton_iterations_max": int(r.iters.max()), "newton_iterations_mean": float(r.iters.mean()),
               "fit_s_per_iteration": t / max(1, int(r.iters.max())), "micro_f1": float(r.f1.mean()),
               "kernel_s_in_fit": kernels, "gram_pass_s_all_problems": tg, "solve_pass_s_all_problems": ts,
               "gram_useful_tflops": useful / tg / 1e12, "gram_useful_share_of_fp64_tc": useful / tg / PEAK_FP64_TC,
               "gram_executed_tflops": executed / tg / 1e12,
               "gram_executed_share_of_fp64_tc": executed / tg / PEAK_FP64_TC}
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
        if "%dx%d" % (d, c) in args.sklearn.split(","):
            from sklearn.linear_model import LogisticRegression
            from sklearn.multiclass import OneVsRestClassifier
            Xh = X.cpu().numpy()
            tr = folds != 0
            t0 = time.perf_counter()
            OneVsRestClassifier(LogisticRegression(C=1000)).fit(Xh[tr], Y[tr].astype(np.float32))
            th = time.perf_counter() - t0
            row = {"sklearn_one_fold_of_ten_s": th, "d": d, "classes": c, "train_rows": int(tr.sum()),
                   "cpu_count": os.cpu_count()}
            res["runs"].append(row)
            print(json.dumps(row), flush=True)
        del X
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
