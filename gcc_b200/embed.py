"""EmbedEngine: generate.py's embedding pass (the reference's generate.py:33-53) over a node range or id list of a
NodeClassificationDataset, with the data path of later batches running ahead of the encoder (DESIGN §5e).

  batch t+1 .. t+S: seeds -> RWR walk / induce -> positional features    S data streams, ring of S+1 BatchBuffers
  batch t:          encoder(q), encoder(k) in eval mode -> (f(q) + f(k)) / 2 -> pinned host slot   high-priority stream

The row of node v is a pure function of (run seed, v): its Philox sample id is v, BatchNorm uses its running
statistics and dropout is off.  So any split of the ids into shards or subsets needs no communication.

The host waits on one event per batch, when it takes the batch's rows out of their staging slot, just before the slot
is reused.  The batch's device flag word travels with its rows into pinned memory, so reading it costs no further
sync.  Host memory is the staging ring, (S+1) x B x hidden floats, whatever the number of nodes.
"""
import numpy as np
import torch

from . import _lib
from .datasets.data_util import BatchedSubgraphs
from .datasets.graph_dataset import BatchBuffers, sample_pairs


class EmbedEngine:
    def __init__(self, dataset, model, prefetch=4):
        """dataset: a NodeClassificationDataset; model: a GraphEncoder on the dataset's device.  prefetch: S, the
        batches whose data path runs ahead of the encoder; 0 runs every stage of a batch on the caller's stream and
        waits for its rows before the next batch starts (the serial loop)."""
        _lib.require_device()
        self.ds, self.model = dataset, model
        self.dev = model.flat_params.device
        self.B, self.H = B, H = dataset.batch_size, model.cfg.hidden
        self.prefetch = S = int(prefetch)
        if S < 0:
            raise ValueError("prefetch must be >= 0, got %d" % S)
        self.depth = S + 1
        ds = dataset
        self.bufs = [ds.buffers] + [BatchBuffers(B, ds.node_cap, ds.edge_cap, ds.buffers.pos_dim,
                                                 ds.buffers.max_budget, self.dev) for _ in range(S)]
        f32 = dict(dtype=torch.float32, device=self.dev)
        # the encoder stream runs batches one after another, so one set of activations and features serves them all
        self.acts = torch.empty(model.acts_bytes(B, ds.node_cap), dtype=torch.uint8, device=self.dev)
        self.feat_q, self.feat_k, self.avg = (torch.empty(B, H, **f32) for _ in range(3))
        # the host side: one pinned slot of rows and one flag word per ring slot
        self.stage = torch.empty(self.depth, B, H, dtype=torch.float32).pin_memory()
        self.flag_stage = torch.zeros(self.depth, dtype=torch.int32).pin_memory()
        self.ready = [torch.cuda.Event() for _ in range(self.depth)]       # data path of the slot's batch done
        self.consumed = [torch.cuda.Event() for _ in range(self.depth)]    # encoder finished reading the slot
        self.staged = [torch.cuda.Event() for _ in range(self.depth)]      # rows and flags are in host memory
        if S:
            self.data_streams = [torch.cuda.Stream(device=self.dev, priority=0) for _ in range(S)]
            self.enc_stream = torch.cuda.Stream(device=self.dev, priority=-1)
        self.host_waits = 0                            # event synchronisations in the last run()

    def run(self, nodes, out=None):
        """Rows (f(q) + f(k)) / 2 of `nodes` (a range of node ids, or a 1-D int64 sequence of them) written to out[i]
        for the i-th id: a float32 array-like [len(nodes), hidden] such as a numpy memmap, or a new array if None.
        Raises GccbError naming the batch's nodes when a batch's ego-nets overflow their capacity."""
        n_nodes = self.ds.graph.num_nodes
        if isinstance(nodes, range):
            if nodes.step != 1 or (len(nodes) and not 0 <= nodes.start < nodes.stop <= n_nodes):
                raise ValueError("node range %r is not a contiguous part of 0..%d" % (nodes, n_nodes - 1))
            self._first, self._ids = nodes.start, None
        else:
            ids = np.ascontiguousarray(np.asarray(nodes, dtype=np.int64).reshape(-1))
            if ids.size and (ids.min() < 0 or ids.max() >= n_nodes):
                raise ValueError("node ids must lie in 0..%d" % (n_nodes - 1))
            self._ids_host = ids
            self._ids = torch.from_numpy(ids).pin_memory().to(self.dev, non_blocking=True)
        self.n = n = len(nodes)
        if out is None:
            out = np.empty((n, self.H), dtype=np.float32)
        if tuple(out.shape) != (n, self.H):
            raise ValueError("output holds %s rows, %d x %d are needed" % (tuple(out.shape), n, self.H))
        self.out = out
        self.host_waits = 0
        caller = torch.cuda.current_stream(self.dev)
        if self.prefetch:
            for st in self.data_streams + [self.enc_stream]:
                st.wait_stream(caller)                 # the id upload and any earlier work on these buffers
            for st in self.data_streams:
                st.wait_stream(self.enc_stream)        # a run that raised may have left encodes in flight
        n_b = -(-n // self.B)
        prepared = drained = 0
        for t in range(n_b):
            while prepared < min(t + self.depth, n_b):
                self._prepare(prepared)
                prepared += 1
            while drained <= t - self.depth:           # batch t reuses the staging slot of batch t - depth
                self._drain(drained)
                drained += 1
            self._encode(t)
        while drained < n_b:
            self._drain(drained)
            drained += 1
        if self.prefetch:
            caller.wait_stream(self.enc_stream)
        return out

    # -------------------------------------------------------------------------------------------
    def _rows(self, j):
        a = j * self.B
        return a, min(self.B, self.n - a)

    def _prepare(self, j):
        """Seeds, ego-nets and positional features of batch j into slot j mod depth, on data stream j mod S."""
        slot, (a, b) = j % self.depth, self._rows(j)
        buf = self.bufs[slot].narrow(b)
        st = self.data_streams[j % self.prefetch] if self.prefetch else torch.cuda.current_stream(self.dev)
        if j >= self.depth:
            st.wait_event(self.consumed[slot])         # the encoder has finished with the slot's previous batch
        with torch.cuda.stream(st):
            if self._ids is None:
                torch.arange(self._first + a, self._first + a + b, device=self.dev, out=buf.seeds)
            else:
                buf.seeds.copy_(self._ids[a:a + b], non_blocking=True)
            sample_pairs(self.ds, buf, None, buf.seeds, sample_ids=buf.seeds)     # sample id of node v is v
            buf.posenc()
            self.ready[slot].record()

    def _encode(self, t):
        """Both views of batch t through the encoder, their mean and the batch's flag word into pinned slot t mod
        depth."""
        slot, (a, b) = t % self.depth, self._rows(t)
        buf = self.bufs[slot].narrow(b)
        st = self.enc_stream if self.prefetch else torch.cuda.current_stream(self.dev)
        st.wait_event(self.ready[slot])
        with torch.cuda.stream(st):
            fq, fk, avg = self.feat_q[:b], self.feat_k[:b], self.avg[:b]
            for v, feat in ((0, fq), (1, fk)):
                self.model._run_forward(BatchedSubgraphs(buf, v), False, step=0, dropout=False, acts=self.acts,
                                        feat=feat, all_outputs=False, bn_train=False)
            torch.add(fq, fk, out=avg)
            avg.mul_(0.5)                              # = torch.stack([fq, fk]).mean(0), bit for bit
            self.flag_stage[slot:slot + 1].copy_(buf.flags, non_blocking=True)
            buf.flags.zero_()
            self.consumed[slot].record()
            self.stage[slot, :b].copy_(avg, non_blocking=True)
            self.staged[slot].record()

    def _drain(self, t):
        """Host: wait for batch t's slot, check its flags, copy its rows to the output."""
        slot, (a, b) = t % self.depth, self._rows(t)
        self.staged[slot].synchronize()
        self.host_waits += 1
        f = int(self.flag_stage[slot])
        if f:
            if self._ids is None:
                where = "batch of nodes %d..%d: " % (self._first + a, self._first + a + b - 1)
            else:
                where = "batch of rows %d..%d (node ids %d..%d in the given order): " % (
                    a, a + b - 1, self._ids_host[a], self._ids_host[a + b - 1])
            self.bufs[slot].raise_flags(f, where)
        self.out[a:a + b] = self.stage[slot, :b].numpy()
