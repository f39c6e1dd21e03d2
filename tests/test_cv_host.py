"""CPU: the concurrent --finetune --cv driver of train.py (main_finetune_cv) with the device parts stubbed out -- the
reference's fold placement, per-fold dataset state over one shared dataset, and the order of the printed blocks
and of the checkpoint writes."""
import contextlib
import copy
import types

import numpy as np
import pytest
import torch

import train
from gcc_b200.datasets import labeled


@pytest.mark.parametrize("gpus,want", [
    ([0], [0] * 10),
    ([0, 1, 2], [0, 1, 2, 0, 1, 2, 0, 1, 2, 0]),
    ([4, 5, 6, 7], [4, 5, 6, 7, 4, 5, 6, 7, 4, 5]),
    (None, [0] * 10),
])
def test_fold_placement_follows_the_reference(gpus, want):
    assert train.fold_gpus(gpus) == want


# ---- per-fold dataset state -------------------------------------------------------------------------------------
def _node_dataset():
    """A NodeClassificationDatasetLabeled as its constructor leaves it, without the device graph."""
    ds = object.__new__(labeled.NodeClassificationDatasetLabeled)
    ds.labels = np.arange(50) % 3
    ds.length = ds.total = 50
    ds.batch_size = 8
    ds._caps = (None, None)
    ds._bufs = {}
    ds.next_sample = 0
    ds.graph = object()                                        # shared read-only state: the same object in a view
    return ds


@pytest.fixture
def recorded_batches(monkeypatch):
    calls = []

    def sample_pairs(ds, buf, first_sample, seeds=None):
        calls.append((id(ds), first_sample, seeds.tolist(), buf))
        return buf

    monkeypatch.setattr(labeled, "sample_pairs", sample_pairs)
    monkeypatch.setattr(labeled.NodeClassificationDatasetLabeled, "_new_buffers",
                        lambda self, B: types.SimpleNamespace(B=B, flags=torch.zeros(1, dtype=torch.int32),
                                                              posenc=lambda: None))
    return calls


def _draw(ds, calls, orders):
    """The (sample id of the first walk, item ids) of device_batch over `orders`, and the buffers used."""
    start = len(calls)
    for o in orders:
        ds.device_batch(torch.as_tensor(o, dtype=torch.int64))
    return [(c[1], c[2]) for c in calls[start:]], [c[3] for c in calls[start:]]


def test_fold_views_draw_what_fresh_datasets_draw(recorded_batches):
    calls = recorded_batches
    rng = np.random.RandomState(0)
    orders = [[rng.permutation(50)[:8] for _ in range(3)] + [rng.permutation(50)[:5]] for _ in range(2)]
    fresh = [_draw(_node_dataset(), calls, o) for o in orders]
    shared = _node_dataset()
    shared.next_sample = 77                                    # a used dataset: views still start as fresh ones
    views = [shared.fold_view(), shared.fold_view()]
    # interleaved, as the driver issues them: one batch of each fold in turn
    got = [([], []), ([], [])]
    for i in range(len(orders[0])):
        for f in range(2):
            d, b = _draw(views[f], calls, [orders[f][i]])
            got[f][0].extend(d)
            got[f][1].extend(b)
    for f in range(2):
        assert got[f][0] == fresh[f][0]
        assert views[f].graph is shared.graph and views[f].labels is shared.labels
    bufs0, bufs1 = {id(b) for b in got[0][1]}, {id(b) for b in got[1][1]}
    assert bufs0.isdisjoint(bufs1) and not shared._bufs            # own buffers, own flag words
    assert shared.next_sample == 77
    assert views[0].next_sample == views[1].next_sample == 3 * 8 + 5


def test_graph_fold_views_share_the_feature_cache():
    ds = object.__new__(labeled.GraphClassificationDatasetLabeled)
    ds._bufs = {8: "the base's buffers"}
    ds.positional_embedding_size, ds.batch_size = 32, 8
    built = []
    gs = ds.graph_set = types.SimpleNamespace(features=None)      # DeviceGraphSet without the device

    def feature_cache(pos_dim, B):
        if gs.features is None:
            built.append((pos_dim, B))
            gs.features = torch.zeros(3)
        return gs.features
    gs.feature_cache = feature_cache
    a, b = ds.fold_view(), ds.fold_view()
    assert built == [(32, 8)]                                   # built by the first fold_view, before any fold used it
    assert a.feature_cache() is b.feature_cache() is ds.feature_cache() is gs.features
    assert len(built) == 1 and a.graph_set is b.graph_set is gs
    assert a._bufs == {} and b._bufs == {} and a._bufs is not b._bufs


# ---- the driver with a stub engine ------------------------------------------------------------------------------
class _StubEngine:
    """Prints like FinetuneEngine: a line per step, then the validation line."""

    def __init__(self, idx):
        self.idx, self.out, self.steps_done = idx, None, 0

    def train_epoch_steps(self, epoch, order, epochs, sw=None, print_freq=10, tb_freq=250):
        for i in range(2 + self.idx % 3):                      # folds of different lengths
            self.steps_done += 1
            print("fold %d epoch %d step %d" % (self.idx, epoch, i), file=self.out)
            yield
        return 0.5 + self.idx, 0.25

    def evaluate(self, epoch, indices, sw=None):
        print("Epoch %d, valid of fold %d" % (epoch, self.idx), file=self.out)
        return 0.0, self.idx / 10.0

    def optimizer_state_dict(self):
        return {"steps": self.steps_done}


class _StubFold:
    def __init__(self, args, checkpoint, dataset, dev):
        self.args, self.test_idx, self.sw = args, [], None
        self.engine = _StubEngine(args.fold_idx)
        self.model = torch.nn.Linear(2, 2)

    def epoch_order(self):
        return np.arange(4)


class _StubStream:
    def __init__(self, device=None):
        pass

    def wait_stream(self, other):
        pass

    def synchronize(self):
        pass


@pytest.fixture
def stub_driver(monkeypatch, tmp_path):
    saved = []
    monkeypatch.setattr(torch.cuda, "Stream", _StubStream)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: _StubStream())
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "manual_seed", lambda s: None)
    monkeypatch.setattr(train, "_FinetuneFold", _StubFold)
    monkeypatch.setattr(train, "_finetune_options", lambda a: (print("options of fold %d" % a.fold_idx) or a, None))
    monkeypatch.setattr(train, "_labeled_dataset", lambda a, dev: types.SimpleNamespace(fold_view=lambda: None))
    monkeypatch.setattr(train, "_save_finetune_state",
                        lambda a, state, epoch: saved.append((a.fold_idx, epoch, state["optimizer"]["steps"])))
    return saved


@pytest.mark.parametrize("gpus", [[0], [0, 1, 2]])
def test_blocks_and_checkpoints_in_fold_order(stub_driver, capsys, gpus):
    saved = stub_driver
    args = types.SimpleNamespace(gpu=gpus, epochs=2, seed=0, fold_idx=0, print_freq=10, tb_freq=250)
    f1 = train.main_finetune_cv(args)
    assert f1 == [i / 10.0 for i in range(10)]
    want = []
    for f in range(10):
        want.append("options of fold %d" % f)
        for e in (1, 2):
            want += ["fold %d epoch %d step %d" % (f, e, i) for i in range(2 + f % 3)]
            want.append("epoch %d, loss %.4f, total time " % (e, 0.5 + f))
        want.append("Epoch 2, valid of fold %d" % f)
    lines = capsys.readouterr().out.splitlines()
    assert len(lines) == len(want)
    for got, w in zip(lines, want):
        assert got.startswith(w), (got, w)
    # each epoch's checkpoints in fold order, with the state of that epoch's end
    assert saved == [(f, e, e * (2 + f % 3)) for e in (1, 2) for f in range(10)]


def test_a_failing_fold_is_named_and_ends_the_run(stub_driver, capsys, monkeypatch):
    from gcc_b200 import _lib

    class Failing(_StubEngine):
        def train_epoch_steps(self, epoch, order, epochs, sw=None, print_freq=10, tb_freq=250):
            if self.idx != 3:
                return (yield from super().train_epoch_steps(epoch, order, epochs, sw, print_freq, tb_freq))
            yield
            raise _lib.GccbError("epoch %d: finetune step batch 1 exceeded its buffers" % epoch)

    class Fold(_StubFold):
        def __init__(self, *a):
            super().__init__(*a)
            self.engine = Failing(self.args.fold_idx)

    monkeypatch.setattr(train, "_FinetuneFold", Fold)
    args = types.SimpleNamespace(gpu=[0], epochs=2, seed=0, fold_idx=0, print_freq=10, tb_freq=250)
    with pytest.raises(_lib.GccbError, match=r"^fold 3: epoch 1: finetune step batch 1 exceeded"):
        train.main_finetune_cv(args)
    out = capsys.readouterr().out
    assert "options of fold 3" in out and "options of fold 4" not in out
    assert "fold 2 epoch 1 step 3" in out                         # the other folds finished the epoch
    assert not stub_driver                                        # no epoch was complete on every fold


def test_folds_are_seeded_with_the_command_line_seed(stub_driver, monkeypatch):
    """--resume swaps in the checkpoint's options (another seed); main_finetune seeds torch before that swap."""
    seeds = []
    monkeypatch.setattr(torch, "manual_seed", seeds.append)

    def options(a):
        a = copy.copy(a)
        a.seed = 99
        return a, None
    monkeypatch.setattr(train, "_finetune_options", options)
    args = types.SimpleNamespace(gpu=[0], epochs=1, seed=5, fold_idx=0, print_freq=10, tb_freq=250)
    train.main_finetune_cv(args)
    assert seeds == [5] * 10


def test_failures_still_write_the_blocks(stub_driver, capsys, monkeypatch):
    """A fold's GccbError in validation is named like one in training; any other exception still writes every block."""
    from gcc_b200 import _lib

    class BadValidation(_StubEngine):
        def evaluate(self, epoch, indices, sw=None):
            if self.idx == 2:
                raise _lib.GccbError("evaluation batch 0 exceeded its buffers")
            return super().evaluate(epoch, indices, sw)

    class Crash(_StubEngine):
        def train_epoch_steps(self, *a, **kw):
            if self.idx == 5:
                raise RuntimeError("host bug")
            return (yield from super().train_epoch_steps(*a, **kw))

    args = types.SimpleNamespace(gpu=[0], epochs=1, seed=0, fold_idx=0, print_freq=10, tb_freq=250)
    for engine, error, last, done in ((BadValidation, r"^fold 2: evaluation batch 0", 2, "Epoch 1, valid of fold 1"),
                                      (Crash, "host bug", 9, "fold 4 epoch 1 step 0")):
        class Fold(_StubFold):
            def __init__(self, *a):
                super().__init__(*a)
                self.engine = engine(self.args.fold_idx)
        monkeypatch.setattr(train, "_FinetuneFold", Fold)
        with pytest.raises((_lib.GccbError, RuntimeError), match=error):
            train.main_finetune_cv(args)
        out = capsys.readouterr().out
        assert "options of fold %d" % last in out and "options of fold %d" % (last + 1) not in out
        assert done in out
