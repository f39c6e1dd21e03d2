"""Wall time of `train.py --finetune --cv`: the serial fold loop (train.finetune_cv_serial: main_finetune for each
fold in turn, each building its dataset) against the concurrent driver (train.main_finetune_cv: one dataset per
GPU, the folds' steps interleaved on their own streams), alternating, in one call (DESIGN.md §5d).

    python profiles/cv_time.py [--epochs 30] [--reps 3] [--gpus 0 1]

Workloads: the two synthetic sets of profiles/finetune_time.py -- a usa_airport-sized node set (1,190 vertices,
rw_hops 256) and a REDDIT-BINARY-sized whole-graph set (2,000 graphs of about 446 vertices) -- at batch 32, GIN
5 layers at hidden 64 (SIMT) and hidden 128 (tensor cores), Adam, the reference's --print-freq 10.  Both arms include
building the datasets (and the whole-graph feature cache; the synthetic graphs are generated once) and write their checkpoints and TensorBoard files to a
temporary directory.  With --gpus 0 1 the concurrent arm spreads the folds over both GPUs; the serial arm runs on
the first.  Prints one JSON line per workload and hidden size with the card's name, power limit and SM clock.
"""
import argparse
import contextlib
import copy
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from finetune_time import card, graph_set, node_set  # noqa: E402


def dataset_maker(make, cls_name):
    """dev -> the labeled dataset `make` builds, with the synthetic graphs generated once: only the dataset's own
    construction (device upload, seed-first relabelling, union CSR) is repeated, as a user's runs repeat it."""
    from gcc_b200.datasets import labeled
    cls = getattr(labeled, cls_name)
    setattr(labeled, cls_name, lambda data, **kw: (data, kw))
    try:
        data, kw = make(None)
    finally:
        setattr(labeled, cls_name, cls)
    return lambda dev: cls(data, **dict(kw, device=dev))


def run(name, make, H, gpus, epochs, reps, tmp):
    import torch
    import train
    args = train.parse_option(["--finetune", "--cv", "--epochs", str(epochs), "--batch-size", "32",
                               "--hidden-size", str(H), "--rw-hops", "256", "--dataset", name,
                               "--model-path", os.path.join(tmp, "m"), "--tb-path", os.path.join(tmp, "tb"),
                               "--gpu"] + [str(g) for g in gpus])
    times, f1 = {"serial": [], "concurrent": []}, {}
    for rep in range(reps):
        for arm in ("serial", "concurrent"):
            torch.cuda.synchronize()
            t0 = time.time()
            with contextlib.redirect_stdout(io.StringIO()):
                if arm == "serial":
                    r = train.finetune_cv_serial(copy.deepcopy(args), make_dataset=make)
                else:
                    r = train.main_finetune_cv(copy.deepcopy(args),
                                               datasets={g: make(torch.device("cuda", g)) for g in set(gpus)})
            for g in set(gpus):
                torch.cuda.synchronize(g)
            times[arm].append(time.time() - t0)
            f1[arm] = r
    return dict(workload=name, hidden=H, gpus=list(gpus), epochs=epochs,
                serial_s=[round(t, 2) for t in times["serial"]],
                concurrent_s=[round(t, 2) for t in times["concurrent"]],
                speedup=round(float(np.median(times["serial"]) / np.median(times["concurrent"])), 2),
                same_f1=f1["serial"] == f1["concurrent"], card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gpus", type=int, nargs="+", default=[0])
    ap.add_argument("--hidden", type=int, nargs="+", default=[64, 128])
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(a.gpus[0])
    with tempfile.TemporaryDirectory() as tmp:
        for name, make, cls in (("nodes", node_set, "NodeClassificationDatasetLabeled"),
                                ("graphs", graph_set, "GraphClassificationDatasetLabeled")):
            make = dataset_maker(make, cls)
            for H in a.hidden:
                print(json.dumps(run(name, make, H, a.gpus, a.epochs, a.reps, tmp)), flush=True)


if __name__ == "__main__":
    main()
