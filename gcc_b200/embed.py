"""EmbedEngine: generate.py's embedding pass (the reference's generate.py:33-53) over a node range or id list of a
NodeClassificationDataset, with the data path of later batches running ahead of the encoder (DESIGN §5e).

  batch t+1 .. t+S: seeds -> RWR walk / induce -> positional features    S data streams, ring of S+1 BatchBuffers
  batch t:          encoder(q), encoder(k) in eval mode -> (f(q) + f(k)) / 2 -> pinned host slot   high-priority stream

The row of node v is a pure function of (run seed, v): its Philox sample id is v, BatchNorm uses its running
statistics and dropout is off.  So any split of the ids into shards or subsets needs no communication.

The host waits on one event per batch, when it takes the batch's rows out of their staging slot, just before the slot
is reused.  The batch's device flag word travels with its rows into pinned memory, so reading it costs no further
sync.  Host memory is the staging ring, (S+1) x B x hidden floats, whatever the number of nodes.

A WholeGraphDataset (one row per graph of a corpus, DESIGN §5f) runs through the same ring.  The dataset decides a
batch's data path: the gather of its whole graphs, view 1 marked absent, and the positional features of view 0; the
encoder runs view 0 alone, since q and k are the same graph and (x + x) / 2 == x.  The host knows every graph's
size, so run() sizes the ring's buffers exactly, from the largest batch it will run; a whole-graph batch never
overflows and is never re-run.

A batch whose ego-nets overflow a dataset of the default capacity is re-run after the ring has drained, on spill
buffers of the engine's own (DESIGN §5e): sampled again with the same sample ids, so with the same walks, its
counters read (one host sync), and its ego-nets cut into consecutive groups that fit (spill_groups).
"""
import numpy as np
import torch

from . import _capi, _lib
from .datasets.data_util import BatchedSubgraphs
from .datasets.graph_dataset import BatchBuffers, sample_pairs

SPILL_PASSES = 4            # sampling passes that may measure an overflowed batch before it is given up
INT32_MAX = 2 ** 31 - 1     # the batch layout's offsets are int32


def spill_groups(sizes, exact, node_cap, edge_cap):
    """The re-run plan of a batch whose ego-nets overflowed buffers of node_cap vertices and edge_cap edge slots per
    view.  sizes: [b, 4] per ego-net pair, (n_q, m_q, n_k, m_k) as the sampler counted them; exact: [b] bools, False
    where a pair's counts are only lower bounds.  Returns (groups, remeasure).  remeasure lists the pairs that must be
    sampled again before they can be sized; groups is None while it is not empty.  Otherwise groups cuts pairs
    0..b-1, in order, into consecutive runs (lo, hi, node_cap, edge_cap): pairs whose q views and whose k views each
    fit the given capacity, or a single pair that does not fit it alone, with the capacity of its larger view."""
    sizes = np.asarray(sizes, dtype=np.int64).reshape(-1, 4)
    remeasure = [i for i in range(len(sizes)) if not exact[i]]
    if remeasure:
        return None, remeasure
    caps = np.array([node_cap, edge_cap, node_cap, edge_cap], dtype=np.int64)
    groups, lo, tot = [], 0, np.zeros(4, dtype=np.int64)
    for i, s in enumerate(sizes):
        if (s > caps).any():                            # too large for any group: alone, on buffers of its size
            if lo < i:
                groups.append((lo, i, int(node_cap), int(edge_cap)))
            groups.append((i, i + 1, int(max(s[0], s[2])), int(max(s[1], s[3]))))
            lo, tot = i + 1, np.zeros(4, dtype=np.int64)
            continue
        if (tot + s > caps).any():
            groups.append((lo, i, int(node_cap), int(edge_cap)))
            lo, tot = i, np.zeros(4, dtype=np.int64)
        tot += s
    if lo < len(sizes):
        groups.append((lo, len(sizes), int(node_cap), int(edge_cap)))
    return groups, []


class EmbedEngine:
    def __init__(self, dataset, model, prefetch=4):
        """dataset: a NodeClassificationDataset or a WholeGraphDataset; model: a GraphEncoder on the dataset's
        device.  prefetch: S, the
        batches whose data path runs ahead of the encoder; 0 runs every stage of a batch on the caller's stream and
        waits for its rows before the next batch starts (the serial loop)."""
        _lib.require_device()
        self.ds, self.model = dataset, model
        self.whole = getattr(dataset, "whole_graphs", False)
        self.item = "graph" if self.whole else "node"
        # a caller who gave the dataset a capacity has set a memory limit: an overflowing batch raises
        self.replan = not self.whole and not dataset.caps_given
        self.dev = model.flat_params.device
        self.B, self.H = B, H = dataset.batch_size, model.cfg.hidden
        self.prefetch = S = int(prefetch)
        if S < 0:
            raise ValueError("prefetch must be >= 0, got %d" % S)
        self.depth = S + 1
        ds = dataset
        if self.whole:
            self.bufs = self.acts = None               # sized by run() from the batches it runs (_size_ring)
            self.node_cap = self.edge_cap = 0
        else:
            self.bufs = [ds.buffers] + [BatchBuffers(B, ds.node_cap, ds.edge_cap, ds.buffers.pos_dim,
                                                     ds.buffers.max_budget, self.dev) for _ in range(S)]
            # the encoder stream runs batches one after another, so one set of activations serves them all
            self.acts = torch.empty(model.acts_bytes(B, ds.node_cap), dtype=torch.uint8, device=self.dev)
        f32 = dict(dtype=torch.float32, device=self.dev)
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
        self.replanned = 0                             # batches of the last run() re-run on spill buffers
        self.largest_egonet = (0, 0)                   # (vertices, edges) of the largest ego-net they held
        self._spill = self._spill_big = None

    def run(self, nodes, out=None):
        """Rows (f(q) + f(k)) / 2 of `nodes` (a range of node ids, or a 1-D int64 sequence of them) written to out[i]
        for the i-th id: a float32 array-like [len(nodes), hidden] such as a numpy memmap, or a new array if None.
        A batch whose ego-nets overflow the dataset's default capacity is re-run after the others on buffers sized from
        them (_replan); when the caller gave the dataset its capacity, GccbError is raised naming the batch's nodes.
        On a WholeGraphDataset, `nodes` are graph ids and a row is f(graph)."""
        n_nodes = self.ds.total if self.whole else self.ds.graph.num_nodes
        if isinstance(nodes, range):
            if nodes.step != 1 or (len(nodes) and not 0 <= nodes.start < nodes.stop <= n_nodes):
                raise ValueError("%s range %r is not a contiguous part of 0..%d" % (self.item, nodes, n_nodes - 1))
            self._first, self._ids = nodes.start, None
        else:
            ids = np.ascontiguousarray(np.asarray(nodes, dtype=np.int64).reshape(-1))
            if ids.size and (ids.min() < 0 or ids.max() >= n_nodes):
                raise ValueError("%s ids must lie in 0..%d" % (self.item, n_nodes - 1))
            self._ids_host = ids
            self._ids = torch.from_numpy(ids).pin_memory().to(self.dev, non_blocking=True)
        self.n = n = len(nodes)
        if self.whole:
            self._size_ring(np.arange(nodes.start, nodes.stop) if self._ids is None else self._ids_host)
        if out is None:
            out = np.empty((n, self.H), dtype=np.float32)
        if tuple(out.shape) != (n, self.H):
            raise ValueError("output holds %s rows, %d x %d are needed" % (tuple(out.shape), n, self.H))
        self.out = out
        self.host_waits = self.replanned = 0
        self.largest_egonet = (0, 0)
        self._overflowed = []
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
        try:
            for t in self._overflowed:                 # off the ring: its buffers, streams and stash are not touched
                self._replan(t)
        finally:
            self._spill = self._spill_big = None
        return out

    # -------------------------------------------------------------------------------------------
    def _size_ring(self, ids):
        """Whole graphs: the ring's buffers and activations sized for the largest batch of `ids` (the dataset's plan),
        reallocated when the plan changes."""
        caps = self.ds.plan(ids)
        if self.bufs is not None and caps == (self.node_cap, self.edge_cap):
            return
        if self.bufs is not None and self.prefetch:
            torch.cuda.current_stream(self.dev).wait_stream(self.enc_stream)   # an earlier run's work on them
        self.bufs = self.acts = None                   # freed before the new ones are allocated
        self.node_cap, self.edge_cap = caps
        self.bufs = [self.ds.buffers(*caps) for _ in range(self.depth)]
        self.acts = torch.empty(self.model.acts_bytes(self.B, caps[0]), dtype=torch.uint8, device=self.dev)

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
            if self.whole:
                self.ds.prepare(buf, buf.seeds)
            else:
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
            if self.whole:                             # q = k = the graph: (f + f) / 2 = f, bit for bit
                avg = self._forward_view(buf, 0, self.acts, self.feat_q[:b])
            else:
                avg = self._forward_mean(buf, self.acts, self.feat_q[:b], self.feat_k[:b], self.avg[:b])
            self.flag_stage[slot:slot + 1].copy_(buf.flags, non_blocking=True)
            buf.flags.zero_()
            self.consumed[slot].record()
            self.stage[slot, :b].copy_(avg, non_blocking=True)
            self.staged[slot].record()

    def _forward_view(self, buf, v, acts, feat):
        """View v of the batch in buf through the encoder in eval mode, into feat."""
        self.model._run_forward(BatchedSubgraphs(buf, v), False, step=0, dropout=False, acts=acts,
                                feat=feat, all_outputs=False, bn_train=False)
        return feat

    def _forward_mean(self, buf, acts, fq, fk, avg):
        """Both views of the batch in buf through the encoder in eval mode, then avg = (fq + fk) / 2."""
        for v, feat in ((0, fq), (1, fk)):
            self._forward_view(buf, v, acts, feat)
        torch.add(fq, fk, out=avg)
        avg.mul_(0.5)                                  # = torch.stack([fq, fk]).mean(0), bit for bit
        return avg

    def _where(self, t):
        a, b = self._rows(t)
        if self._ids is None:
            return "batch of %ss %d..%d: " % (self.item, self._first + a, self._first + a + b - 1)
        return "batch of rows %d..%d (%s ids %d..%d in the given order): " % (
            a, a + b - 1, self.item, self._ids_host[a], self._ids_host[a + b - 1])

    def _drain(self, t):
        """Host: wait for batch t's slot, check its flags, copy its rows to the output, or record the batch for a
        re-run if it overflowed a default capacity."""
        slot, (a, b) = t % self.depth, self._rows(t)
        self.staged[slot].synchronize()
        self.host_waits += 1
        f = int(self.flag_stage[slot])
        over = f & (_capi.FLAG_NODE_OVERFLOW | _capi.FLAG_EDGE_OVERFLOW) if self.replan else 0
        if f & ~over:
            self.bufs[slot].raise_flags(f & ~over, self._where(t))
        if over:
            self._overflowed.append(t)
        else:
            self.out[a:a + b] = self.stage[slot, :b].numpy()

    # -- the re-run of an overflowed batch, on the caller's stream, after the ring has drained ---------------------
    def _node_ids(self, t):
        a, b = self._rows(t)
        if self._ids is None:
            return torch.arange(self._first + a, self._first + a + b, device=self.dev)
        return self._ids[a:a + b]

    def _node_id(self, t, i):
        a = self._rows(t)[0] + i
        return self._first + a if self._ids is None else int(self._ids_host[a])

    def _buffers(self, B, node_cap, edge_cap, node_id):
        """Spill BatchBuffers for B pairs and an activation stash for them, or GccbError naming node_id."""
        what = "node %d: buffers of %d vertices and %d edges per view" % (node_id, node_cap, edge_cap)
        if max(node_cap, edge_cap) > INT32_MAX:
            raise _lib.GccbError(what + " exceed the batch layout's int32 offsets")
        try:
            buf = BatchBuffers(B, node_cap, edge_cap, self.ds.buffers.pos_dim, self.ds.buffers.max_budget, self.dev)
            acts = torch.empty(self.model.acts_bytes(B, node_cap), dtype=torch.uint8, device=self.dev)
        except torch.cuda.OutOfMemoryError:
            raise _lib.GccbError(what + " do not fit in device memory") from None
        return buf, acts

    def _big(self, node_cap, edge_cap, node_id):
        """The one-pair spill buffers, grown (never shrunk) to hold node_cap vertices and edge_cap edges per view."""
        if self._spill_big is not None:
            have = self._spill_big[0]
            if node_cap <= have.node_cap and edge_cap <= have.edge_cap:
                return self._spill_big
            node_cap, edge_cap = max(node_cap, have.node_cap), max(edge_cap, have.edge_cap)
            self._spill_big = have = None              # freed before the larger ones are allocated
        self._spill_big = self._buffers(1, node_cap, edge_cap, node_id)
        return self._spill_big

    def _sample(self, buf, seeds):
        """Both views of the pairs seeded by `seeds` (sample id = node id) into buf narrowed to them."""
        buf = buf.narrow(len(seeds))
        buf.seeds.copy_(seeds)
        return sample_pairs(self.ds, buf, None, buf.seeds, sample_ids=buf.seeds)

    def _measure(self, buf, seeds):
        """Host sync: sample the pairs of `seeds` into buf and read their counts -> (sizes [b, 4] as (n_q, m_q, n_k,
        m_k), exact [b]).  An ego-net above the walk budget of shared memory that found no room in its view's wide
        region is counted with m = n - 1, a lower bound, and a sum of degrees of 0, which no other ego-net has (every
        vertex has a neighbour); every other count is exact, also in an overflowing view (an exhausted induction pool
        only makes the fill pass scan a row again)."""
        b = len(seeds)
        c = self._sample(buf, seeds).counters.view(2, b, 4).cpu().numpy()
        buf.flags.zero_()                              # the overflow this measurement expects
        sizes = np.stack([c[0, :, 0], c[0, :, 1], c[1, :, 0], c[1, :, 1]], axis=1)
        return sizes, (c[0, :, 3] > 0) & (c[1, :, 3] > 0)

    def _replan(self, t):
        """Rows of overflowed batch t, from groups of its ego-nets that fit (spill_groups)."""
        ds, (a, b) = self.ds, self._rows(t)
        seeds = self._node_ids(t)
        if self._spill is None:
            self._spill = self._buffers(self.B, ds.node_cap, ds.edge_cap, self._node_id(t, 0))
        sizes, exact = self._measure(self._spill[0], seeds)
        for _ in range(SPILL_PASSES):
            groups, remeasure = spill_groups(sizes, exact, ds.node_cap, ds.edge_cap)
            if groups is not None:
                break
            for i in remeasure:                        # room for its node set (the wide region: edge_cap + 1)
                n = int(max(sizes[i, 0], sizes[i, 2]))
                big = self._big(n, 16 * n, self._node_id(t, i))[0]
                s, e = self._measure(big, seeds[i:i + 1])
                sizes[i], exact[i] = s[0], e[0]
        else:
            raise _lib.GccbError(self._where(t) + "ego-net sizes still unknown after %d sampling passes"
                                 % SPILL_PASSES)
        self.replanned += 1
        i = int(np.argmax(np.maximum(sizes[:, 0], sizes[:, 2])))
        v = 0 if sizes[i, 0] >= sizes[i, 2] else 2
        self.largest_egonet = max(self.largest_egonet, (int(sizes[i, v]), int(sizes[i, v + 1])))
        for lo, hi, node_cap, edge_cap in groups:
            if node_cap <= ds.node_cap and edge_cap <= ds.edge_cap:
                buf, acts = self._spill
            else:
                buf, acts = self._big(node_cap, edge_cap, self._node_id(t, lo))
            buf = self._sample(buf, seeds[lo:hi])
            buf.posenc()
            fq, fk, avg = (torch.empty(hi - lo, self.H, dtype=torch.float32, device=self.dev) for _ in range(3))
            rows = self._forward_mean(buf, acts, fq, fk, avg).cpu().numpy()
            f = int(buf.flags.item())
            buf.flags.zero_()
            if f & (_capi.FLAG_NODE_OVERFLOW | _capi.FLAG_EDGE_OVERFLOW):
                raise _lib.GccbError(self._where(t) + "pairs %d..%d overflowed the buffers sized from their "
                                     "measured ego-nets" % (lo, hi - 1))
            buf.raise_flags(f, self._where(t))
            self.out[a + lo:a + hi] = rows
