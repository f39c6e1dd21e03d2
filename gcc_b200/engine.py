"""PretrainEngine: one MoCo / E2E pretraining step (train.py:378-434 + the DataLoader work that
feeds it) as a fixed sequence of libgccb200 kernel launches with no host synchronisation:

  draw seeds -> RWR walk / induce / batch -> positional features           (datasets/)
  -> encoder forward q (model) and k (model_ema, BN in train mode, train.py:357-365)
  -> fused InfoNCE (loss, dq; logits never materialised)                     (memory_moco.py, criterions.py)
  -> encoder backward -> [all-gather of keys+grads when world > 1]
  -> clip + optimiser step (Adam, SGD or Adagrad) + momentum update on flat buffers (train.py:409-417,430-431)
  -> FIFO enqueue of the keys (memory_moco.py:55-61)

The module-level API (GraphEncoder.forward + autograd, MemoryMoCo.forward, NCESoftmaxLoss) runs
the same kernels piecewise and stays drop-in for the reference's train_moco; this engine is what
train.py / bench.py drive.  Scalars the reference reads with .item() every step (train.py:420-422)
live in a device stats buffer read on demand.
"""
import ctypes as C
import math

import torch

from . import _capi, _lib
from .datasets.data_util import BatchedSubgraphs
from .parallel import StepExchange, first_sample_id

ADAGRAD_EPS = 1e-10                                    # torch.optim.Adagrad's default; train.py never sets it


class FlatOptimizer:
    """The state of one torch.optim.{Adam,SGD,Adagrad} over a flat fp32 buffer of n live entries, for the flat optimiser
    kernels (csrc/optim.cu, csrc/finetune.cu): the moment / sum buffers, the step count t and the per-step `hyper`
    scalars.  adam: betas, eps; sgd: momentum (dampening 0, no Nesterov); adagrad: lr_decay, eps 1e-10."""

    def __init__(self, kind, n, device, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5, momentum=0.9,
                 lr_decay=0.0):
        if kind not in ("adam", "sgd", "adagrad"):
            raise ValueError("optimizer must be adam, sgd or adagrad, not %r" % (kind,))
        self.kind, self.lr0, self.betas, self.eps, self.wd = kind, lr, betas, eps, weight_decay
        self.momentum, self.lr_decay = momentum, lr_decay
        f32 = dict(dtype=torch.float32, device=device)
        self.m = self.v = self.state = None
        if kind == "adam":
            self.m = torch.zeros(n, **f32)
            self.v = torch.zeros(n, **f32)
        elif kind == "adagrad" or momentum != 0:
            # SGD's momentum_buffer or Adagrad's sum; zero is also torch's starting point (Adagrad's
            # initial_accumulator_value 0; SGD's first-step copy, see csrc/optim_rules.cuh)
            self.state = torch.zeros(n, **f32)
        self.t = 0                                     # steps issued (skipped ones included)
        self.hyper = torch.zeros(4, **f32)
        # ring of pinned slots: the host enqueues several steps ahead of the device, and an async H2D copy
        # reads its pinned source when it EXECUTES, so each step needs a slot of its own
        self.hyper_host = torch.zeros(256, 4, dtype=torch.float32).pin_memory()

    def next_step(self, lr):
        """Count one more step and enqueue its scalars (LR at step t, bias corrections) into `hyper`, without a
        host sync."""
        self.t += 1
        slot = self.hyper_host[self.t % self.hyper_host.shape[0]]
        if self.kind == "adam":
            b1, b2 = self.betas
            slot[0] = lr
            slot[1] = 1.0 - b1 ** self.t
            slot[2] = math.sqrt(1.0 - b2 ** self.t)
        elif self.kind == "sgd":
            slot[0] = lr
        else:                                          # torch.optim.Adagrad's clr, in double
            slot[0] = lr / (1.0 + (self.t - 1) * self.lr_decay)
        self.hyper.copy_(slot, non_blocking=True)

    def state_dict(self, model):
        """The flat buffers in the layout of torch.optim.{Adam,SGD,Adagrad}(model.parameters()).state_dict()
        (train.py:659-678,752).  Adam: exp_avg / exp_avg_sq / step for the parameters that receive gradients (the
        GIN path); the unused set2set / lin_readout tensors have no state, as in the reference where they never get
        a gradient.  SGD: momentum_buffer for those parameters once a step has run, and no state without momentum.
        Adagrad: state for every parameter, as torch creates it at construction -- the unused tensors keep step 0
        and a zero sum."""
        names = [n for n, _ in model.named_parameters()]
        state = {}
        for i, (n, prm) in enumerate(model.named_parameters()):
            if n in model._slices:
                o, shape = model._slices[n]
                cnt = 1
                for d_ in shape:
                    cnt *= d_
                if self.kind == "adam":
                    state[i] = {"step": torch.tensor(float(self.t)),
                                "exp_avg": self.m[o:o + cnt].view(shape).clone(),
                                "exp_avg_sq": self.v[o:o + cnt].view(shape).clone()}
                elif self.kind == "sgd":
                    if self.state is not None and self.t > 0:
                        state[i] = {"momentum_buffer": self.state[o:o + cnt].view(shape).clone()}
                else:
                    state[i] = {"step": torch.tensor(float(self.t)),
                                "sum": self.state[o:o + cnt].view(shape).clone()}
            elif self.kind == "adagrad":
                state[i] = {"step": torch.tensor(0.0), "sum": torch.zeros_like(prm.detach())}
        params = list(range(len(names)))
        if self.kind == "adam":
            group = {"lr": self.lr0, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.wd,
                     "amsgrad": False, "maximize": False, "foreach": None, "capturable": False,
                     "differentiable": False, "fused": None, "params": params}
        elif self.kind == "sgd":
            group = {"lr": self.lr0, "momentum": self.momentum, "dampening": 0, "weight_decay": self.wd,
                     "nesterov": False, "maximize": False, "foreach": None, "differentiable": False, "fused": None,
                     "params": params}
        else:
            group = {"lr": self.lr0, "lr_decay": self.lr_decay, "eps": ADAGRAD_EPS, "weight_decay": self.wd,
                     "initial_accumulator_value": 0, "foreach": None, "maximize": False, "differentiable": False,
                     "fused": None, "params": params}
        return {"state": state, "param_groups": [group]}


class PretrainEngine:
    def __init__(self, dataset, model, model_ema, contrast, moco=True, learning_rate=0.005,
                 betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5, clip_norm=1.0, alpha=0.999,
                 nce_t=0.07, rank=0, world_size=1, process_group=None, prefetch=4, optimizer="adam",
                 momentum=0.9, lr_decay=0.0):
        """optimizer: "adam" (betas, eps), "sgd" (momentum; dampening 0, no Nesterov) or "adagrad" (lr_decay;
        eps 1e-10), as train.py:659-678 builds them over model.parameters()."""
        if optimizer not in ("adam", "sgd", "adagrad"):
            raise ValueError("optimizer must be adam, sgd or adagrad, not %r" % (optimizer,))
        if world_size > 1 and getattr(dataset, "epoch_ordered", False):
            raise ValueError("%s: the reference trains node and graph datasets on one GPU; use world_size 1"
                             % type(dataset).__name__)
        _lib.require_device()
        self.lib = _lib.get()
        self.ds, self.model, self.model_ema, self.contrast = dataset, model, model_ema, contrast
        self.moco, self.lr0, self.betas, self.eps = moco, learning_rate, betas, eps
        self.wd, self.clip, self.alpha, self.T = weight_decay, clip_norm, alpha, nce_t
        self.rank, self.world, self.pg = rank, world_size, process_group
        self.optimizer, self.momentum, self.lr_decay = optimizer, momentum, lr_decay
        dev = model.flat_params.device
        self.dev = dev
        B, H, L = dataset.batch_size, model.cfg.hidden, model.cfg.num_layers
        self.B, self.H, self.L = B, H, L
        f32 = dict(dtype=torch.float32, device=dev)
        n_live = model.n_live
        self.xch = None
        if world_size > 1:
            # data-parallel exchange (SURVEY 8e): ONE all-gather per step of [keys | gradient | stats].  The
            # key encoder, the backward and the loss kernels write straight into the send buffer: no packing
            self.xch = StepExchange(B, H, n_live, world_size, dev, process_group)
            self.payload = self.xch.payload
        self.grads = self.xch.grads_send if self.xch else torch.zeros(n_live, **f32)
        self.opt = FlatOptimizer(optimizer, n_live, dev, learning_rate, betas, eps, weight_decay, momentum, lr_decay)
        # loss, prob, grad_norm(pre-clip), overflow marker of this rank's batch (multi-GPU skip protocol)
        self.stats = self.xch.stats_send if self.xch else torch.zeros(4, **f32)
        self.stats_acc = torch.zeros(4, dtype=torch.float64, device=dev)   # per-step sums since the last read_stats()
        self.steps_acc = 0
        self.pairs_acc = 0                             # pairs trained since the last read_stats()
        self.norm_ws = torch.zeros(1, dtype=torch.float64, device=dev)
        self.any_skip = torch.zeros(1, dtype=torch.int32, device=dev)
        self.feat_q = torch.zeros(B, H, **f32)
        self.feat_k = self.xch.keys_send if self.xch else torch.zeros(B, H, **f32)
        self.dq = torch.zeros(B, H, **f32)
        self.dk = torch.zeros(B, H, **f32)
        self.aux_stream = self._new_stream(0, -1)      # key encoder, concurrent with the query encoder
        cap = dataset.node_cap
        acts_bytes = model.acts_bytes(B, cap)
        self.acts_q = torch.empty(acts_bytes, dtype=torch.uint8, device=dev)
        self.acts_k = torch.empty(acts_bytes, dtype=torch.uint8, device=dev)
        self.bwd_ws = torch.empty(model.backward_workspace_bytes(B, cap), dtype=torch.uint8, device=dev)
        K = contrast.queueSize
        self.K = K
        self.nce_ws = torch.empty(max(self.lib.gccb_infonce_workspace(B, H, K), B * B * 4, 8),
                                  dtype=torch.uint8, device=dev)
        self.index_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.index_dev.fill_(contrast.index)
        self.global_step = 0
        if world_size > 1 and moco and K % (world_size * B) != 0:
            raise ValueError("queue size must be a multiple of world_size*batch (identical queues)")
        self.launches_per_step = None
        # Loader run-ahead (the reference's DataLoader workers prepare later batches while the
        # model trains on batch t, train.py:577-586): sampler + eigensolver of batches t+1..t+S run
        # on S data streams into a ring of S+1 batch buffers and overlap this step's encoder.  The
        # eigensolver's critical path is a few very large ego-nets, so S=4 batches in flight fill
        # the SMs that one batch leaves idle.  prefetch=0 runs everything on the caller's stream.
        self.prefetch = 4 if prefetch is True else int(prefetch)
        self.count_acc = None                          # optional float64[4]: sums of buf.counters
        self.timing = None                             # optional list collecting per-batch events
        self.timing_main = None                        # same for the training stream
        if self.prefetch:
            from .datasets.graph_dataset import BatchBuffers
            ds = dataset
            S = self.prefetch
            self.depth = S + 1
            self.bufs = [ds.buffers] + [BatchBuffers(B, ds.node_cap, ds.edge_cap, ds.buffers.pos_dim,
                                                     ds.buffers.max_budget, dev) for _ in range(S)]
            self.slot_bufs = list(self.bufs)           # what each slot holds: its buffers, or them narrowed
            self.data_streams = [self._new_stream(1, 0) for _ in range(S)]
            self.ready = [torch.cuda.Event() for _ in range(self.depth)]
            self.consumed = [torch.cuda.Event() for _ in range(self.depth)]
            self.prepared = 0                          # batches issued to the data streams so far
            # the training kernels are short and dependent: a high-priority stream lets their CTAs
            # go ahead of the queued sampler / eigensolver CTAs whenever an SM slot frees up
            self.train_stream = self._new_stream(0, -1)
        self.cur_buf = dataset.buffers
        self._seed_ev = None

    # -------------------------------------------------------------------------------------------
    def _new_stream(self, group, priority):
        return torch.cuda.Stream(device=self.dev, priority=priority)

    # the optimiser state under its historical names (tests and tools read them)
    adam_m = property(lambda self: self.opt.m)
    adam_v = property(lambda self: self.opt.v)
    opt_state = property(lambda self: self.opt.state)
    adam_t = property(lambda self: self.opt.t)
    hyper = property(lambda self: self.opt.hyper)

    def _prepare(self, seeds):
        """Issue sampler + eigensolver of batch number `self.prepared` on the data stream."""
        j = self.prepared
        slot = j % self.depth
        buf = self.bufs[slot]
        main = torch.cuda.current_stream(self.dev)
        ds_ = self.data_streams[j % self.prefetch]
        if j >= self.depth:
            ds_.wait_event(self.consumed[slot])        # the step that read this slot has finished with it
        else:
            ds_.wait_stream(main)
        if seeds is not None:
            # only the caller's H2D copy of the seeds has to be ordered before the sampler -- NOT the training
            # stream's backlog (waiting on `main` here would hold the next batch's data path behind the
            # previous step's training part and give the run-ahead away)
            if self._seed_ev is not None:
                ds_.wait_event(self._seed_ev)
            else:
                ds_.wait_stream(main)
            seeds.record_stream(ds_)
        with torch.cuda.stream(ds_):
            t = None
            if self.timing is not None:
                t = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                t[0].record()
            first = first_sample_id(j, self.world, self.rank, self.B)
            buf = self.ds.sample_batch(first_sample=first, seeds=seeds, buffers=buf, posenc=False)
            self.slot_bufs[slot] = buf                 # an epoch's short last batch: fewer pairs, same memory
            if t:
                t[1].record()
            self.ds.posenc(buf)
            if t:
                t[2].record()
                self.timing.append(t)
            self.ready[slot].record()
        self.prepared = j + 1

    def step(self, lr=None, seeds=None, _presampled=False):
        """One optimisation step (see _step); with prefetch on, the training part runs on the
        engine's high-priority stream, ordered after and before the caller's current stream."""
        if not self.prefetch or _presampled:
            return self._step(lr, seeds, _presampled)
        caller = torch.cuda.current_stream(self.dev)
        self.train_stream.wait_stream(caller)
        self._seed_ev = None
        if seeds is not None:
            seeds.record_stream(self.train_stream)
            self._seed_ev = torch.cuda.Event()
            self._seed_ev.record(caller)               # after the caller's copy into `seeds`
        with torch.cuda.stream(self.train_stream):
            self._step(lr, seeds, False)
        caller.wait_stream(self.train_stream)

    def _step(self, lr=None, seeds=None, _presampled=False):
        """One optimisation step.  `seeds`: optional int64 CUDA tensor [B] (else drawn on device
        from the Philox stream); with prefetch on they seed the batch being PREPARED by this call
        (consumed `prefetch` steps later), like a DataLoader running ahead -- the first call
        prepares prefetch+1 batches, of which only the first uses `seeds` (the rest are drawn on the
        device).  Out-of-range seeds are clamped by the sampler.  Returns nothing; read_stats() syncs."""
        lib, st = self.lib, _lib.stream_ptr()
        ds, model, ema = self.ds, self.model, self.model_ema
        B, H, L = self.B, self.H, self.L
        lr = self.lr0 if lr is None else lr
        if _presampled:
            buf = ds.buffers
        elif self.prefetch:
            while self.prepared < self.global_step + self.depth:
                self._prepare(seeds)
                seeds = None        # warm-up: only the first batch of a multi-batch fill takes the caller's seeds,
                                    # the others are drawn on the device (no duplicated batches)
            slot = self.global_step % self.depth
            buf = self.slot_bufs[slot]
            torch.cuda.current_stream(self.dev).wait_event(self.ready[slot])
        else:
            first = first_sample_id(self.global_step, self.world, self.rank, B)
            buf = ds.sample_batch(first_sample=first, seeds=seeds)
        self.cur_buf = buf
        if self.timing_main is not None:
            tm = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            tm[0].record()
        if self.count_acc is not None:
            self.count_acc += buf.counters.double().sum(0)
        gq, gk = BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1)
        # pairs in this batch: B, or fewer in the last batch of an epoch of a node / graph dataset.  The feature and
        # gradient buffers are [B][H]; the kernels use their first b rows
        b = buf.B
        step = self.global_step
        if self.moco:
            # the key encoder (model_ema, its own weights and running statistics) is independent of
            # the query encoder until the head: run it on a second stream
            cur = torch.cuda.current_stream(self.dev)
            self.aux_stream.wait_stream(cur)
            with torch.cuda.stream(self.aux_stream):
                ema._run_forward(gk, False, step=step, dropout=False, acts=self.acts_k, feat=self.feat_k,
                                 all_outputs=False, bn_train=True)
        _, _, saved_q = model._run_forward(gq, True, step=step, dropout=True, acts=self.acts_q, feat=self.feat_q,
                                           all_outputs=False, bn_train=True)
        self.grads.zero_()
        if self.moco:
            cur.wait_stream(self.aux_stream)
            _lib.check(lib.gccb_infonce_fused(_lib.dptr(self.feat_q), _lib.dptr(self.feat_k),
                                              _lib.dptr(self.contrast.memory), b, H, self.K, self.T,
                                              _lib.dptr(self.stats), _lib.dptr(self.dq),
                                              _lib.dptr(self.nce_ws), self.nce_ws.numel(), st),
                       "gccb_infonce_fused")
            model._run_backward(gq, saved_q, self.dq, grads_flat=self.grads, ws=self.bwd_ws)
        else:
            _, _, saved_k = model._run_forward(gk, True, step=step, dropout=True, acts=self.acts_k, feat=self.feat_k,
                                               all_outputs=False, bn_train=True)
            _lib.check(lib.gccb_e2e_nce(_lib.dptr(self.feat_q), _lib.dptr(self.feat_k), b, H, self.T,
                                        _lib.dptr(self.stats), _lib.dptr(self.dq), _lib.dptr(self.dk),
                                        _lib.dptr(self.nce_ws), self.nce_ws.numel(), st), "gccb_e2e_nce")
            model._run_backward(gq, saved_q, self.dq, grads_flat=self.grads, ws=self.bwd_ws)
            model._run_backward(gk, saved_k, self.dk, grads_flat=self.grads, ws=self.bwd_ws)
        if self.prefetch and not _presampled:
            self.consumed[self.global_step % self.depth].record()
        grads, scale = self.grads, 1.0
        # a batch published empty (capacity overflow; the flag is raised for the host) must not train:
        # optimiser / EMA / enqueue skip the step on the device, the flags reach the host in read_stats()
        OVERFLOW = _capi.FLAG_NODE_OVERFLOW | _capi.FLAG_EDGE_OVERFLOW
        skip_word, skip_mask = _lib.dptr(buf.flags), OVERFLOW
        if self.world > 1:
            # the ONE collective of the step: keys + gradients + stats, then a fixed-rank-order sum
            n_live = model.n_live
            self.stats[3:4].copy_((buf.flags & OVERFLOW).float())
            gathered = self.xch.all_gather()
            _lib.check(lib.gccb_sum_ranks(C.c_void_p(gathered.data_ptr() + self.xch.grad_offset_bytes()),
                                          self.world, self.payload, n_live, _lib.dptr(self.grads),
                                          n_live + 3, _lib.dptr(self.any_skip), st), "gccb_sum_ranks")
            scale = 1.0 / self.world
            skip_word, skip_mask = _lib.dptr(self.any_skip), -1     # every replica skips the same steps
        self.opt.next_step(lr)
        p_ema, alpha = (_lib.dptr(ema.flat_params), self.alpha) if self.moco else (None, -1.0)
        tail = (p_ema, model.n_live, model._n_all, _lib.dptr(self.hyper))
        common = (self.wd, self.clip, alpha, scale, C.c_void_p(self.stats.data_ptr() + 8), _lib.dptr(self.norm_ws),
                  skip_word, skip_mask, st)
        p_, g_, s_ = _lib.dptr(model.flat_params), _lib.dptr(grads), _lib.dptr(self.opt_state)
        if self.optimizer == "adam":
            _lib.check(lib.gccb_clip_adam_ema(p_, g_, _lib.dptr(self.adam_m), _lib.dptr(self.adam_v), *tail,
                                              self.betas[0], self.betas[1], self.eps, *common), "gccb_clip_adam_ema")
        elif self.optimizer == "sgd":
            _lib.check(lib.gccb_clip_sgd_ema(p_, g_, s_, *tail, self.momentum, *common), "gccb_clip_sgd_ema")
        else:
            _lib.check(lib.gccb_clip_adagrad_ema(p_, g_, s_, *tail, ADAGRAD_EPS, *common), "gccb_clip_adagrad_ema")
        if self.moco:
            # all ranks' keys in rank order with one launch -> identical queues on every rank
            src = self.xch.gathered if self.world > 1 else self.feat_k
            _lib.check(lib.gccb_moco_enqueue(_lib.dptr(self.contrast.memory), _lib.dptr(src), b, H, self.K,
                                             _lib.dptr(self.index_dev), self.world,
                                             self.payload if self.world > 1 else 0, skip_word, skip_mask, st),
                       "gccb_moco_enqueue")
            self.contrast.index = (self.contrast.index + b * self.world) % self.K
        # the reference updates its meters from .item() reads every step (train.py:420-428); here the
        # per-step scalars are summed on the device and read on demand
        if b == B:
            self.stats_acc.add_(self.stats)
        else:                                          # loss and prob weighted by pairs, as the reference's meters
            self.stats_acc[:2].add_(self.stats[:2], alpha=b / B)
            self.stats_acc[2:].add_(self.stats[2:])
        self.steps_acc += 1
        self.pairs_acc += b
        if self.timing_main is not None:
            tm[1].record()
            self.timing_main.append(tm)
        self.global_step += 1

    def wait_data_streams(self):
        """Order the caller's current stream after everything issued so far on the run-ahead data streams
        (no host sync).  Benchmarks close their timed window with it so that the window holds as many data
        parts as training parts."""
        if self.prefetch:
            cur = torch.cuda.current_stream(self.dev)
            for ds_ in self.data_streams:
                cur.wait_stream(ds_)

    def read_stats(self):
        """Host sync: loss, prob (mean positive logit), pre-clip grad norm, sizes of the batch the last step
        trained on, flags.  window_loss / window_prob average over the window's pairs (window_pairs), the
        grad norm over its steps."""
        buf = self.cur_buf
        torch.cuda.synchronize(self.dev)
        for b_ in (self.bufs if self.prefetch else [buf]):     # every buffer of the run-ahead ring, not only
            b_.check_flags()                                   # the one the last step trained on
        s = self.stats.tolist()
        acc, w = self.stats_acc.tolist(), max(self.steps_acc, 1)
        wp = self.pairs_acc / self.B if self.pairs_acc else 1      # = w when every batch is full
        self.stats_acc.zero_()
        window, pairs = self.steps_acc, self.pairs_acc
        self.steps_acc = self.pairs_acc = 0
        sizes = buf.node_off[:, buf.B].tolist() + buf.edge_off[:, buf.B].tolist()
        return dict(loss=s[0], prob=s[1], grad_norm=s[2], nodes_q=sizes[0], nodes_k=sizes[1],
                    edges_q=sizes[2], edges_k=sizes[3], batch_size=buf.B, window_steps=window,
                    window_pairs=pairs, window_loss=acc[0] / wp, window_prob=acc[1] / wp,
                    window_grad_norm=acc[2] / w)

    def optimizer_state_dict(self):
        """FlatOptimizer.state_dict of the encoder's optimiser."""
        return self.opt.state_dict(self.model)
