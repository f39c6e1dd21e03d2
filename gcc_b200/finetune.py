"""FinetuneEngine: the supervised finetune loop (train.py:175-337 of the reference, this repository's
train.train_finetune / test_finetune) as a fixed sequence of libgccb200 launches per step with no host sync:

  the epoch's order (one pinned H2D copy) -> the batch of the next item ids           (datasets/labeled.py)
    node sets: sampler walks from the ids + positional features
    graph sets: union gather + cached whole-graph features
  -> encoder forward (BatchNorm in train mode, dropout on)                             (models/graph_encoder.py)
  -> classification head: logits, cross-entropy, first-max correct count, dfeat, dW, db (csrc/finetune.cu)
  -> encoder backward into a flat gradient
  -> clip_grad_value_(1) + the encoder's --optimizer, and clip_grad_value_(1) + Adam for the head

train_finetune / test_finetune stay the module-level path with torch ops; this engine computes the same steps on the
same batches (the order comes from the same RandomState, node walks from the dataset's next_sample counter, dropout
masks from model._drop_step).  Per-step statistics (loss, correct, rows, nodes, edges, flags) stay in a device log
that the host reads at the print and TensorBoard steps and at the end of an epoch.
"""
import ctypes as C
import time

import numpy as np
import torch

from . import _capi, _lib
from .datasets.data_util import BatchedSubgraphs
from .engine import ADAGRAD_EPS, FlatOptimizer
from .utils.misc import AverageMeter, warmup_linear

OVERFLOW = _capi.FLAG_NODE_OVERFLOW | _capi.FLAG_EDGE_OVERFLOW
LOSS, CORRECT, ROWS, NODES, EDGES, FLAGS = range(6)       # columns of the step log


class FinetuneEngine:
    def __init__(self, dataset, model, output_layer, optimizer="adam", lr=0.005, betas=(0.9, 0.999),
                 weight_decay=1e-5, momentum=0.9, lr_decay=0.0, clip_value=1.0, batch_size=None):
        """dataset: a labeled dataset of datasets/labeled.py (device_batch, labels_dev); output_layer: the
        torch.nn.Linear(hidden, num_classes) head, whose weight and bias become views of one flat buffer.  The
        encoder is updated by `optimizer` (adam, sgd or adagrad, as train.make_optimizer builds it), the head by Adam
        (the reference's output_layer_optimizer), both after clip_grad_value_(clip_value)."""
        _lib.require_device()
        self.lib = _lib.get()
        dev = model.flat_params.device
        self.dev = dev
        self.ds, self.model, self.head = dataset, model, output_layer
        self.B = int(batch_size or dataset.batch_size)
        self.H, self.C = model.cfg.hidden, output_layer.out_features
        if output_layer.in_features != self.H:
            raise ValueError("output layer takes %d features, the encoder gives %d" % (output_layer.in_features, self.H))
        if int(dataset.labels.max()) >= self.C or int(dataset.labels.min()) < 0:
            raise ValueError("labels must lie in [0, %d)" % self.C)
        self.clip = float(clip_value)
        CH = self.C * self.H
        flat = torch.empty(CH + self.C, dtype=torch.float32, device=dev)
        with torch.no_grad():
            flat[:CH].copy_(output_layer.weight.detach().reshape(-1))
            flat[CH:].copy_(output_layer.bias.detach())
        output_layer.weight.data = flat[:CH].view(self.C, self.H)
        output_layer.bias.data = flat[CH:]
        self.head_flat = flat
        self.enc_opt = FlatOptimizer(optimizer, model.n_live, dev, lr, betas, 1e-8, weight_decay, momentum, lr_decay)
        self.head_opt = FlatOptimizer("adam", CH + self.C, dev, lr, betas, 1e-8, weight_decay)
        f32 = dict(dtype=torch.float32, device=dev)
        self.grads = torch.zeros(model.n_live, **f32)
        self.head_grads = torch.zeros(CH + self.C, **f32)
        self.feat = torch.zeros(self.B, self.H, **f32)
        self.dfeat = torch.zeros(self.B, self.H, **f32)
        self.head_ws = torch.empty(self.lib.gccb_ft_head_workspace(self.B, self.C), dtype=torch.uint8, device=dev)
        self._scratch = {}
        n = len(dataset)
        self.order_dev = torch.zeros(n, dtype=torch.int64, device=dev)
        self.order_host = [torch.zeros(n, dtype=torch.int64).pin_memory() for _ in range(2)]
        self._order_slot = 0
        self.global_step = 0                           # training steps issued, over every epoch
        if hasattr(dataset, "feature_cache"):
            dataset.feature_cache()                    # computed once, before the first step
        self.last_steps = None                         # per-step (loss, f1, rows, nodes, edges) of the last epoch
        self.out = None                                # where the engine prints (None: sys.stdout)

    # -------------------------------------------------------------------------------------------
    def _buffers_scratch(self, buf):
        key = (buf.B, buf.node_cap)
        if key not in self._scratch:
            m = self.model
            self._scratch[key] = (torch.empty(m.acts_bytes(buf.B, buf.node_cap), dtype=torch.uint8, device=self.dev),
                                  torch.empty(m.backward_workspace_bytes(buf.B, buf.node_cap), dtype=torch.uint8,
                                              device=self.dev))
        return self._scratch[key]

    def _load_order(self, indices):
        """Copy an epoch's item order to the device from pinned memory, without a host sync."""
        n = len(indices)
        host = self.order_host[self._order_slot]
        self._order_slot ^= 1
        host[:n].numpy()[:] = np.asarray(indices, dtype=np.int64)
        self.order_dev[:n].copy_(host[:n], non_blocking=True)
        return n

    def _head(self, b, ids, log_row, eval_):
        CH = self.C * self.H
        hg = self.head_grads
        _lib.check(self.lib.gccb_ft_head(
            _lib.dptr(self.feat), self.B, b, self.H, self.C, _lib.dptr(self.head_flat),
            C.c_void_p(self.head_flat.data_ptr() + CH * 4), _lib.dptr(ids), _lib.dptr(self.ds.labels_dev),
            len(self.ds.labels), 1 if eval_ else 0, _lib.dptr(self.dfeat), _lib.dptr(hg),
            C.c_void_p(hg.data_ptr() + CH * 4), C.c_void_p(log_row.data_ptr()), _lib.dptr(self.head_ws),
            self.head_ws.numel(), _lib.stream_ptr()), "gccb_ft_head")

    @staticmethod
    def _log_sizes(log_row, buf, b):
        log_row[NODES].copy_(buf.node_off[0, b])
        log_row[EDGES].copy_(buf.edge_off[0, b])
        log_row[FLAGS].copy_(buf.flags[0])

    def _step(self, ids, lr, log_row):
        """One training step on the items `ids` (device int64 [b]): no host sync."""
        lib, st, model = self.lib, _lib.stream_ptr(), self.model
        b = ids.numel()
        buf = self.ds.device_batch(ids)
        g = BatchedSubgraphs(buf, 0)
        acts, ws = self._buffers_scratch(buf)
        step = getattr(model, "_drop_step", 0)
        _, _, saved = model._run_forward(g, True, step=step, dropout=True, acts=acts, feat=self.feat,
                                         all_outputs=False, bn_train=True)
        if hasattr(model, "_drop_step"):
            model._drop_step += 1                      # as the module-level forward advances it
        self._head(b, ids, log_row, eval_=False)
        self.grads.zero_()
        model._run_backward(g, saved, self.dfeat, grads_flat=self.grads, ws=ws)
        # a batch published empty (capacity overflow) must not train: both updates skip it on the device
        skip = _lib.dptr(buf.flags)
        eo, ho = self.enc_opt, self.head_opt
        eo.next_step(lr)
        ho.next_step(lr)
        p_, g_ = _lib.dptr(model.flat_params), _lib.dptr(self.grads)
        if eo.kind == "adam":
            _lib.check(lib.gccb_clip_value_adam(p_, g_, _lib.dptr(eo.m), _lib.dptr(eo.v), model.n_live,
                                                _lib.dptr(eo.hyper), eo.betas[0], eo.betas[1], eo.eps, eo.wd,
                                                self.clip, skip, OVERFLOW, st), "gccb_clip_value_adam")
        elif eo.kind == "sgd":
            _lib.check(lib.gccb_clip_value_sgd(p_, g_, _lib.dptr(eo.state), model.n_live, _lib.dptr(eo.hyper),
                                               eo.momentum, eo.wd, self.clip, skip, OVERFLOW, st),
                       "gccb_clip_value_sgd")
        else:
            _lib.check(lib.gccb_clip_value_adagrad(p_, g_, _lib.dptr(eo.state), model.n_live, _lib.dptr(eo.hyper),
                                                   ADAGRAD_EPS, eo.wd, self.clip, skip, OVERFLOW, st),
                       "gccb_clip_value_adagrad")
        _lib.check(lib.gccb_clip_value_adam(_lib.dptr(self.head_flat), _lib.dptr(self.head_grads), _lib.dptr(ho.m),
                                            _lib.dptr(ho.v), self.head_flat.numel(), _lib.dptr(ho.hyper),
                                            ho.betas[0], ho.betas[1], ho.eps, ho.wd, self.clip, skip, OVERFLOW, st),
                   "gccb_clip_value_adam")
        self._log_sizes(log_row, buf, b)
        self.global_step += 1

    def _read(self, log, a, z, what):
        """Host sync: rows a..z-1 of a step log; raises GccbError naming the first step whose batch overflowed."""
        rows = log[a:z].cpu().numpy()
        bad = np.flatnonzero(rows[:, FLAGS].astype(np.int64) & OVERFLOW)
        for buf in getattr(self.ds, "_bufs", {}).values():
            if bad.size:
                buf.flags.zero_()
            else:
                buf.check_flags()                      # the eigensolver's non-convergence warning, other faults
        if bad.size:
            f = int(rows[bad[0], FLAGS])
            raise _lib.GccbError("%s batch %d exceeded its buffers (%s): the step was skipped" % (
                what, a + int(bad[0]), "; ".join(n for k, n in _capi.FLAG_NAMES.items() if f & k)))
        return rows

    # -------------------------------------------------------------------------------------------
    def train_epoch(self, epoch, order, n_epochs, sw=None, print_freq=10, tb_freq=250):
        """One epoch over `order` (the epoch's shuffled train indices) in batches of B, the last one short; the LR of
        batch idx is lr * warmup_linear((epoch * n_batch + idx) / (n_epochs * n_batch), 0.1).  Prints and logs what
        train.train_finetune does; returns (epoch loss, epoch micro-F1)."""
        steps = self.train_epoch_steps(epoch, order, n_epochs, sw, print_freq, tb_freq)
        while True:
            try:
                next(steps)
            except StopIteration as done:
                return done.value

    def train_epoch_steps(self, epoch, order, n_epochs, sw=None, print_freq=10, tb_freq=250):
        """train_epoch as a generator that yields after issuing each step (and after the reads and prints due at
        that step), so that one host thread can interleave the steps of several engines on their own streams; its
        return value is train_epoch's.  Every call to next() must run on the stream of the first."""
        B = self.B
        n = self._load_order(order)
        n_batch = (n + B - 1) // B
        log = torch.zeros(n_batch, 6, dtype=torch.float32, device=self.dev)
        batch_time, loss_meter, f1_meter = AverageMeter(), AverageMeter(), AverageMeter()
        epoch_loss_meter, epoch_f1_meter, graph_size = AverageMeter(), AverageMeter(), AverageMeter()
        max_num_nodes = max_num_edges = 0
        steps, read_upto = [], 0
        end = time.time()
        for idx in range(n_batch):
            a = idx * B
            global_step = epoch * n_batch + idx
            lr_this_step = self.enc_opt.lr0 * warmup_linear(global_step / (n_epochs * n_batch), 0.1)
            self._step(self.order_dev[a:min(a + B, n)], lr_this_step, log[idx])
            printing, logging = (idx + 1) % print_freq == 0, sw is not None and (idx + 1) % tb_freq == 0
            if not (printing or logging or idx + 1 == n_batch):
                yield
                continue
            rows = self._read(log, read_upto, idx + 1, "epoch %d: finetune step" % epoch)
            bt = (time.time() - end) / max(len(rows), 1)
            end = time.time()
            for r in rows:                             # the meters of train_finetune, one update per step
                bsz = int(r[ROWS])
                f1 = float(r[CORRECT]) / bsz
                f1_meter.update(f1, bsz)
                epoch_f1_meter.update(f1, bsz)
                loss_meter.update(float(r[LOSS]), bsz)
                epoch_loss_meter.update(float(r[LOSS]), bsz)
                graph_size.update(float(r[NODES]) / bsz, bsz)
                max_num_nodes = max(max_num_nodes, int(r[NODES]))
                max_num_edges = max(max_num_edges, int(r[EDGES]))
                batch_time.update(bt)
                steps.append((float(r[LOSS]), f1, bsz, int(r[NODES]), int(r[EDGES])))
            read_upto = idx + 1
            if printing:
                print("Train: [{0}][{1}/{2}]\tBT {bt.val:.3f} ({bt.avg:.3f})\tloss {loss.val:.3f} ({loss.avg:.3f})\t"
                      "f1 {f1.val:.3f} ({f1.avg:.3f})\tGS {gs.val:.3f} ({gs.avg:.3f})".format(
                          epoch, idx + 1, n_batch, bt=batch_time, loss=loss_meter, f1=f1_meter, gs=graph_size),
                      file=self.out)
            if logging:
                sw.add_scalar("ft_loss", loss_meter.avg, global_step)
                sw.add_scalar("ft_f1", f1_meter.avg, global_step)
                sw.add_scalar("graph_size", graph_size.avg, global_step)
                sw.add_scalar("lr", lr_this_step, global_step)
                sw.add_scalar("graph_size/max", max_num_nodes, global_step)
                sw.add_scalar("graph_size/max_edges", max_num_edges, global_step)
                loss_meter.reset()
                f1_meter.reset()
                graph_size.reset()
                max_num_nodes = max_num_edges = 0
            yield
        self.last_steps = steps
        return epoch_loss_meter.avg, epoch_f1_meter.avg

    def evaluate(self, epoch, indices, sw=None):
        """test_finetune: the eval-mode encoder (running statistics, no dropout) and the head's forward over
        `indices` in order, in batches of B.  Prints and logs what test_finetune does; returns (loss, micro-F1)."""
        B, model = self.B, self.model
        n = self._load_order(indices)
        n_batch = (n + B - 1) // B
        log = torch.zeros(n_batch, 6, dtype=torch.float32, device=self.dev)
        for idx in range(n_batch):
            ids = self.order_dev[idx * B:min(idx * B + B, n)]
            buf = self.ds.device_batch(ids)
            acts, _ = self._buffers_scratch(buf)
            model._run_forward(BatchedSubgraphs(buf, 0), False, step=0, dropout=False, acts=acts, feat=self.feat,
                               all_outputs=False, bn_train=False)
            self._head(ids.numel(), ids, log[idx], eval_=True)
            self._log_sizes(log[idx], buf, ids.numel())
        rows = self._read(log, 0, n_batch, "evaluation")
        epoch_loss_meter, epoch_f1_meter = AverageMeter(), AverageMeter()
        for r in rows:
            bsz = int(r[ROWS])
            epoch_loss_meter.update(float(r[LOSS]), bsz)
            epoch_f1_meter.update(float(r[CORRECT]) / bsz, bsz)
        global_step = (epoch + 1) * n_batch
        if sw is not None:
            sw.add_scalar("ft_loss/valid", epoch_loss_meter.avg, global_step)
            sw.add_scalar("ft_f1/valid", epoch_f1_meter.avg, global_step)
        print(f"Epoch {epoch}, loss {epoch_loss_meter.avg:.3f}, f1 {epoch_f1_meter.avg:.3f}", file=self.out)
        return epoch_loss_meter.avg, epoch_f1_meter.avg

    def optimizer_state_dict(self):
        """The encoder optimiser's state in the layout of torch.optim.<--optimizer>(model.parameters()).state_dict()."""
        return self.enc_opt.state_dict(self.model)
