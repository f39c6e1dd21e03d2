"""Time the exact cosine top-k (gcc_b200.tasks.knn.topk_cosine, csrc/knn.cu) on C2-sized inputs against a chunked
torch.mm + torch.topk baseline on the same GPU.

    python profiles/knn_time.py [--nc 1000000] [--out knn_time.json]

Seeded random rows (C2 is about a million nodes).  For each width: the search of `nq` queries against `nc`
candidates (k = 20), timed with CUDA events after a warm-up call of the same shapes on fewer queries; achieved FP32
FLOP/s from 2 nq nc d4 against the 67 TFLOP/s data-sheet peak; and the baseline -- fp32 torch.mm (TF32 off) of
`base_q`-query chunks against the normalised candidates, then torch.topk -- on `base_q` queries, compared per query.
Also checks that the baseline's top-k ids agree with the kernel's on the timed queries except at near-ties.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gcc_b200.tasks import knn  # noqa: E402

PEAK_FP32 = 67e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out.splitlines()[0] if out else "unavailable"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, out


def baseline(q, cn, k, chunk):
    """Chunked fp32 torch.mm + torch.topk over normalised rows."""
    qn = torch.nn.functional.normalize(q, dim=1)
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device=q.device)
    for lo in range(0, q.shape[0], chunk):
        s = torch.mm(qn[lo:lo + chunk], cn.T)
        ids[lo:lo + chunk] = torch.topk(s, k, dim=1).indices
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nc", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--base-q", type=int, default=65536)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON summary here")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_info(), "nc": args.nc, "k": args.k, "runs": []}
    print(res["gpu"], flush=True)
    for d, nq in ((64, args.nc), (256, args.nc // 4)):
        c = torch.randn((args.nc, d), device="cuda", generator=g)
        q = c[:nq]
        knn.topk_cosine(q[:4096], c, args.k)                                    # warm-up
        t, (ids, _) = timed(lambda: knn.topk_cosine(q, c, args.k))
        d4 = (d + 3) // 4 * 4
        flops = 2.0 * nq * args.nc * d4
        cn = torch.nn.functional.normalize(c, dim=1)
        bq = min(args.base_q, nq)
        chunk = max(1, (8 << 30) // (4 * args.nc))                              # 8 GB of scores per chunk
        baseline(q[:chunk], cn, args.k, chunk)                                  # warm-up
        tb, bids = timed(lambda: baseline(q[:bq], cn, args.k, chunk))
        agree = float((torch.sort(bids, 1).values == torch.sort(ids[:bq], 1).values).all(1).float().mean())
        row = {"d": d, "nq": nq, "kernel_s": t, "tflops": flops / t / 1e12, "share_of_peak": flops / t / PEAK_FP32,
               "baseline_q": bq, "baseline_s": tb, "kernel_us_per_query": 1e6 * t / nq,
               "baseline_us_per_query": 1e6 * tb / bq, "speedup": (tb / bq) / (t / nq),
               "baseline_same_id_sets": agree}
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
        del c, q, cn, ids, bids
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
