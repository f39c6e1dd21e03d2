"""GPU: the concurrent --finetune --cv driver (train.main_finetune_cv) against main_finetune run alone for each fold.
Every fold uses the existing kernels on its own stream, with its own batch buffers, sampler counter, encoder, head,
optimiser state and RandomState, so each fold must reproduce its solo run: weights, BatchNorm running statistics,
optimiser state, per-step losses and correct counts, validation F1, the printed blocks and the checkpoints on disk.

The engine is not bit-reproducible from one run to the next: the encoder's BatchNorm and pooling sums are float64
atomics and the degree-embedding gradient (and GAT's attention-vector gradients) float atomics (DESIGN §4d, §5d), so
their order of additions varies between runs.  On an H100 two solo runs of the same fold (node set, GIN hidden 64,
Adam) first differed at step 6 of two epochs, by 5e-5 in a weight at the end.  So the folds are held to the bars of test_gpu_finetune_engine.py (rtol 2e-3,
atol 5e-5 on weights, 1e-3 on losses, the chaotic pre-BatchNorm biases skipped), a correct count may move by one row,
and the validation F1 by one item; with tensor cores and Adam, whose runs diverge (that file's docstring), every
parameter is held to the step bound used there instead."""
import copy
import os
import re

import numpy as np
import pytest
import torch

from gcc_b200.utils.misc import warmup_linear

pytestmark = pytest.mark.gpu

EPOCHS = 2
LR = 0.005


def _node_set(dev=0, **kw):
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.labeled import NodeClassificationDatasetLabeled
    g = synthetic.chung_lu(600, 3000, 0.5, seed=4)
    deg = np.diff(g.indptr)
    y = np.digitize(deg, np.quantile(deg, [1 / 3, 2 / 3]))                 # three degree buckets
    return NodeClassificationDatasetLabeled((g, y), rw_hops=32, batch_size=32, device=torch.device("cuda", dev), **kw)


def _graph_set(dev=0):
    from gcc_b200.datasets.labeled import GraphClassificationDatasetLabeled
    from test_gpu_finetune_engine import _two_class_graphs
    return GraphClassificationDatasetLabeled(_two_class_graphs(100, seed=6), batch_size=16,
                                             device=torch.device("cuda", dev))


SETS = {"nodes": _node_set, "graphs": _graph_set}


def _args(tmp, tag, model, H, optimizer, gpus=(0,), batch_size=32):
    import train
    return train.parse_option([
        "--finetune", "--cv", "--epochs", str(EPOCHS), "--batch-size", str(batch_size), "--hidden-size", str(H),
        "--num-layer", "3", "--rw-hops", "32", "--model", model, "--optimizer", optimizer, "--print-freq", "5",
        "--model-path", str(tmp / tag / "m"), "--tb-path", str(tmp / tag / "tb"), "--dataset", "synthetic",
        "--gpu"] + [str(g) for g in gpus])


def _snapshot(fold):
    eng = fold.engine
    sd = {k: v.detach().cpu().clone() for k, v in fold.model.state_dict().items()}
    sd["head"] = eng.head_flat.cpu().clone()
    for name, opt in (("enc", eng.enc_opt), ("head", eng.head_opt)):
        for a in ("m", "v", "state"):
            if getattr(opt, a) is not None:
                sd["%s_opt.%s" % (name, a)] = getattr(opt, a).cpu().clone()
    return sd


@pytest.fixture
def recorded_folds(monkeypatch):
    """Every _FinetuneFold built, with its per-epoch snapshots and per-step (loss, correct, rows)."""
    import train
    made = []

    class Recording(train._FinetuneFold):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.snaps, self.steps = [], []
            self.init_head = self.engine.head_flat.detach().cpu().clone()
            inner = self.engine.train_epoch_steps

            def steps(*a, **kw):
                r = yield from inner(*a, **kw)
                self.snaps.append(_snapshot(self))
                self.steps += [(s[0], round(s[1] * s[2]), s[2]) for s in self.engine.last_steps]
                return r
            self.engine.train_epoch_steps = steps
            made.append(self)

    monkeypatch.setattr(train, "_FinetuneFold", Recording)
    return made


def _solo(args, make_set, made):
    """train.finetune_cv_serial: main_finetune for each fold, alone, one after another, each with a dataset of its own.
    Returns the F1 list and {fold: recorded fold}."""
    import train
    n = len(made)
    f1 = train.finetune_cv_serial(args, make_dataset=lambda dev: make_set(dev.index))
    assert len(made) == n + 10
    return f1, dict(enumerate(made[n:]))


def _assert_same(a, b, where, bound=None):
    """The weight bars of test_gpu_finetune_engine.py; with `bound`, parameters within it and statistics skipped."""
    from test_gpu_finetune_engine import _chaotic
    assert a.keys() == b.keys(), where
    for k in a:
        if _chaotic(k) or k.endswith("num_batches_tracked"):
            continue
        x, y = a[k].double(), b[k].double()
        if bound is None:
            assert torch.allclose(x, y, rtol=2e-3, atol=5e-5), (where, k, (x - y).abs().max())
        elif not k.endswith(("running_mean", "running_var", "_opt.v", "_opt.m", "_opt.state", "exp_avg", "exp_avg_sq")):
            assert (x - y).abs().max() <= bound, (where, k, (x - y).abs().max(), bound)


def _same_steps(a, b, where, chaotic):
    assert len(a) == len(b), where
    for i, ((la, ca, ra), (lb, cb, rb)) in enumerate(zip(a, b)):
        assert ra == rb, (where, i)
        if chaotic and i:
            continue
        assert np.isclose(la, lb, rtol=1e-3, atol=1e-4) and abs(ca - cb) <= 1, (where, i, la, lb, ca, cb)


def _shape(text):
    """The printed lines with every number masked: which line of which fold comes where."""
    return re.sub(r"-?[0-9][0-9.e+-]*", "#", text)


def _load(path):
    return torch.load(path, map_location="cpu", weights_only=False)


def _assert_same_checkpoint(p, q, bound):
    a, b = _load(p), _load(q)
    assert a["epoch"] == b["epoch"] and a["opt"].fold_idx == b["opt"].fold_idx == 9
    _assert_same(a["model"], b["model"], p, bound)
    sa, sb = a["optimizer"]["state"], b["optimizer"]["state"]
    assert sa.keys() == sb.keys()
    if bound is None:
        for i in sa:
            _assert_same({k: v for k, v in sa[i].items() if torch.is_tensor(v)},
                         {k: v for k, v in sb[i].items() if torch.is_tensor(v)}, (p, i))


def _check_cv(tmp_path, recorded_folds, capsys, set_name, model, H, optimizer, gpus=(0,)):
    import train
    made = recorded_folds
    make_set = SETS[set_name]
    bs = 32 if set_name == "nodes" else 16
    serial = _args(tmp_path, "serial", model, H, optimizer, batch_size=bs)
    f1_solo, solo = _solo(serial, make_set, made)
    out_solo = capsys.readouterr().out
    conc = _args(tmp_path, "conc", model, H, optimizer, gpus, batch_size=bs)
    n = len(made)
    f1 = train.main_finetune_cv(conc, datasets={g: make_set(g) for g in set(gpus)})
    folds = made[n:]
    assert [f.args.fold_idx for f in folds] == list(range(10))
    chaotic = model == "gin" and H >= 128 and optimizer != "sgd"
    lr_sum = 0.0
    for e in range(EPOCHS):
        nb = len(folds[0].steps) // EPOCHS
        lr_sum += sum(LR * warmup_linear(((e + 1) * nb + i) / (EPOCHS * nb), 0.1) for i in range(nb))
    bound = 2 * 3.17 * lr_sum if chaotic else None
    for f, run in enumerate(folds):
        s = solo[f]
        assert len(run.snaps) == len(s.snaps) == EPOCHS
        for e in range(EPOCHS):
            _assert_same(run.snaps[e], s.snaps[e], "fold %d epoch %d" % (f, e + 1), bound)
        _same_steps(run.steps, s.steps, f, chaotic)
        if not chaotic:
            assert abs(f1[f] - f1_solo[f]) <= 1.0 / len(run.test_idx) + 1e-12, (f, f1[f], f1_solo[f])
    out = capsys.readouterr().out
    assert out.count("Epoch %d, loss" % EPOCHS) == 10
    assert _shape(out) == _shape(out_solo)                       # one block per fold, in fold order
    folder, serial_folder = folds[0].args.model_folder, solo[0].args.model_folder
    assert folder != serial_folder
    for name in ["current.pth"] + ["ckpt_epoch_%d.pth" % e for e in range(1, EPOCHS + 1)]:
        _assert_same_checkpoint(os.path.join(serial_folder, name), os.path.join(folder, name), bound)
    return folds


CONFIGS = [("gin", 64), ("gin", 128), ("gat", 64)]


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
@pytest.mark.parametrize("model,H", CONFIGS, ids=["gin64", "gin128-tc", "gat64"])
@pytest.mark.parametrize("set_name", ["nodes", "graphs"])
def test_concurrent_folds_equal_their_solo_runs(tmp_path, recorded_folds, capsys, set_name, model, H, optimizer):
    _check_cv(tmp_path, recorded_folds, capsys, set_name, model, H, optimizer)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("set_name", ["nodes", "graphs"])
def test_concurrent_folds_on_two_gpus(tmp_path, recorded_folds, capsys, set_name):
    folds = _check_cv(tmp_path, recorded_folds, capsys, set_name, "gin", 64, "adam", gpus=(0, 1))
    assert [f.model.flat_params.device.index for f in folds] == [i % 2 for i in range(10)]


def test_concurrent_epoch_issues_no_host_sync(tmp_path, monkeypatch):
    """The round-robin epoch of every fold runs with no host sync when the print and TensorBoard steps lie beyond the
    epoch; each fold's step log is read afterwards."""
    import train
    deferred, inner = [], train._cv_epoch

    def epoch_without_reads(folds, epoch, epochs):
        for f in folds:
            read = f.run.engine._read
            f.run.engine._read = (lambda log, a, z, what, f=f, read=read:
                                  deferred.append((f, read, log, a, z, what)) or np.zeros((0, 6), np.float32))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            inner(folds, epoch, epochs)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        for f in folds:
            del f.run.engine._read
        assert sorted(d[0].idx for d in deferred) == list(range(10))   # the end of each fold's epoch only
        for f, read, log, a, z, what in deferred:
            with torch.cuda.stream(f.stream):
                rows = read(log, a, z, what)
            assert len(rows) == z - a and np.all(rows[:, 2] > 0)

    monkeypatch.setattr(train, "_cv_epoch", epoch_without_reads)
    for make_set in (_node_set, _graph_set):
        deferred.clear()
        args = _args(tmp_path, make_set.__name__, "gin", 64, "adam")
        args.epochs, args.print_freq = 1, 10 ** 6
        train.main_finetune_cv(args, datasets={0: make_set()})


def test_overflowing_fold_is_skipped_alone(tmp_path, recorded_folds, capsys):
    """Fold 3's batches overflow its edge capacity: its steps are skipped on the device, the driver raises naming the
    fold and the step, and every other fold holds the weights of its solo run after the epoch."""
    import train
    from gcc_b200 import _lib
    made = recorded_folds
    _, solo = _solo(_args(tmp_path, "serial", "gin", 64, "adam"), _node_set, made)
    ds = _node_set()
    views, fold_view = [], ds.fold_view

    def small_fold_3():
        v = fold_view()
        if len(views) == 3:
            v._caps = (None, 64)
        views.append(v)
        return v
    ds.fold_view = small_fold_3
    n = len(made)
    with pytest.raises(_lib.GccbError, match=r"^fold 3: epoch 1: finetune step batch 0 exceeded its buffers"):
        train.main_finetune_cv(_args(tmp_path, "conc", "gin", 64, "adam"), datasets={0: ds})
    folds = made[n:]
    assert len(folds) == 10 and not folds[3].snaps
    assert torch.equal(folds[3].engine.head_opt.m, torch.zeros_like(folds[3].engine.head_opt.m))   # never stepped
    for f, run in enumerate(folds):
        if f != 3:
            assert len(run.snaps) == 1
            _assert_same(run.snaps[0], solo[f].snaps[0], "fold %d" % f)
            _same_steps(run.steps, solo[f].steps[:len(run.steps)], f, False)


def test_resumed_folds_are_seeded_as_their_solo_runs(tmp_path, recorded_folds, capsys):
    """--resume replaces the options by the pretraining checkpoint's, whose seed differs from --seed: every fold still
    draws its head and dropout key from the command line's seed, as main_finetune --fold-idx i does."""
    import train
    made = recorded_folds
    pre = train.parse_option(["--seed", "7", "--hidden-size", "64", "--num-layer", "3", "--rw-hops", "32",
                              "--model-path", str(tmp_path / "m"), "--tb-path", str(tmp_path / "tb")])
    torch.manual_seed(11)
    ckpt = tmp_path / "pretrained.pth"
    torch.save({"opt": pre, "model": train._make_encoder(pre).state_dict()}, ckpt)
    args = _args(tmp_path, "resume", "gin", 64, "adam")
    args.resume, args.seed, args.epochs = str(ckpt), 3, 1
    _, solo = _solo(args, _node_set, made)
    n = len(made)
    train.main_finetune_cv(copy.deepcopy(args), datasets={0: _node_set()})
    folds = made[n:]
    assert "=> loading checkpoint" in capsys.readouterr().out
    for f, run in enumerate(folds):
        s = solo[f]
        assert run.args.seed == s.args.seed == 7                  # the checkpoint's options, as before
        assert run.model.dropout_key == s.model.dropout_key == 0x9E3779B97F4A7C15 ^ 3
        assert torch.equal(run.init_head, s.init_head), f
        _assert_same(run.snaps[0], s.snaps[0], "fold %d" % f)
