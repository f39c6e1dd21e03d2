"""Host: pretraining on a downstream node or graph dataset -- the epoch order, the short last batch and the LR
schedule of train_moco (reference train.py:350-434: n_batch = total // B, global_step = epoch * n_batch + idx
over every batch), and the single-GPU rule.  The engine is a stub that records its step() calls."""
import types

import pytest

import train
from gcc_b200.datasets.graph_dataset import GraphClassificationDataset, NodeClassificationDataset
from gcc_b200.engine import PretrainEngine
from gcc_b200.utils.misc import warmup_linear


class _StubEngine:
    def __init__(self, ds):
        self.ds, self.world, self.global_step = ds, 1, 0
        self.lrs, self.unread = [], 0

    def step(self, lr=None):
        self.lrs.append(lr)
        self.global_step += 1
        self.unread += 1

    def read_stats(self):
        w, self.unread = self.unread, 0
        B = self.ds.batch_size
        return dict(loss=1.0, prob=0.5, grad_norm=1.0, nodes_q=4 * B, nodes_k=4 * B, edges_q=8 * B, edges_k=8 * B,
                    batch_size=B, window_steps=w, window_pairs=w * B, window_loss=1.0, window_prob=0.5,
                    window_grad_norm=1.0)


def _host_dataset(cls, total, B):
    """The dataset's epoch logic without its device state."""
    ds = object.__new__(cls)
    ds.total, ds.batch_size, ds.next_batch = total, B, 0
    return ds


@pytest.mark.parametrize("cls", [NodeClassificationDataset, GraphClassificationDataset])
def test_train_moco_trains_the_short_batch_with_the_reference_lr(cls):
    total, B, epochs = 37, 8, 3                      # total mod B = 5
    opt = train.parse_option(["--batch-size", str(B), "--epochs", str(epochs), "--print-freq", "2"])
    eng = _StubEngine(_host_dataset(cls, total, B))
    for epoch in range(1, epochs + 1):
        train.train_moco(epoch, eng, None, opt, False)
    n_batch = total // B
    steps = -(-total // B)
    assert len(eng.lrs) == epochs * steps == 15
    want = [opt.learning_rate * warmup_linear((e * n_batch + idx) / (epochs * n_batch), 0.1)
            for e in range(1, epochs + 1) for idx in range(steps)]      # idx reaches n_batch
    assert eng.lrs == want


def test_sampled_dataset_keeps_its_step_count():
    opt = train.parse_option(["--batch-size", "8", "--epochs", "2", "--print-freq", "3"])
    eng = _StubEngine(types.SimpleNamespace(total=37, batch_size=8))
    train.train_moco(1, eng, None, opt, False)
    assert len(eng.lrs) == 37 // 8


@pytest.mark.parametrize("cls", [NodeClassificationDataset, GraphClassificationDataset])
def test_epoch_order_of_the_engine_batches(cls):
    ds = _host_dataset(cls, 37, 8)
    got = [ds._locate(j * 8) for j in range(11)]
    order = [(0, 8), (8, 8), (16, 8), (24, 8), (32, 5)]
    assert got == [(e, a, b) for e in range(3) for a, b in order][:11]
    assert [ds._locate(None) for _ in range(6)] == got[:6]                 # unnumbered calls count batches


@pytest.mark.parametrize("cls", [NodeClassificationDataset, GraphClassificationDataset])
def test_multi_gpu_is_refused_for_downstream_datasets(cls):
    with pytest.raises(ValueError, match="one GPU"):
        PretrainEngine(_host_dataset(cls, 37, 8), None, None, None, world_size=2, rank=1)


def test_dgl_names_the_reference_corpus():
    args = train.parse_option(["--dataset", "dgl"])
    assert train.build_graph(args, None) == "./data/small.bin"
