"""GraphEncoder with the reference's constructor, forward signature and state_dict keys
(gcc/models/graph_encoder.py:19-200, gin branch; SURVEY.md section 8b), executing as
hand-written sm_90a kernels through libgccb200 (csrc/gin_fwd.cu, csrc/gin_bwd.cu).

All live parameters are views into ONE flat fp32 buffer (models/layout.py) followed by the
unused-but-present tensors of the reference module (set2set.*, lin_readout.*), so that
  * checkpoints stay key-compatible (load_state_dict / state_dict as in train.py:690-694,750-758),
  * Adam / clipping / the momentum update are single flat kernels (csrc/optim.cu),
  * the multi-GPU gradient exchange is one buffer.
Parameter initialisation draws from torch's RNG in the same order as the reference's
constructor, so torch.manual_seed(s) gives identical initial weights.
"""
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib
from . import layout as glayout


class _Holder(nn.Module):
    """Anonymous container used to reproduce the reference's nested state_dict keys."""


class _BatchNormHolder(_Holder):
    """Class name contains 'BatchNorm' on purpose: train.py:360-365 (set_bn_train) switches
    modules to train mode by class name, and the finetune branch resets the statistics the same way
    (clear_bn, train.py:648-653)."""

    def reset_running_stats(self):
        # in place: the buffers are views of the encoder's flat running-statistics arrays
        self._buffers["running_mean"].zero_()
        self._buffers["running_var"].fill_(1.0)
        self._buffers["num_batches_tracked"].zero_()


def _child(mod, name, cls=_Holder):
    if name not in mod._modules:
        mod.add_module(name, cls())
    return mod._modules[name]


class _GinEncodeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, g, need_grad, *params):
        # (grad mode is always off inside Function.forward; the caller decides)
        feat, pooled, saved = module._run_forward(g, keep_for_backward=need_grad)
        ctx.module, ctx.g, ctx.saved = module, g, saved
        ctx.mark_non_differentiable(pooled)
        return feat, pooled

    @staticmethod
    def backward(ctx, dfeat, _dpooled):
        grads = ctx.module._run_backward(ctx.g, ctx.saved, dfeat.contiguous())
        ctx.saved = None
        return (None, None, None) + tuple(grads)


class GraphEncoder(nn.Module):
    def __init__(self, positional_embedding_size=32, max_node_freq=8, max_edge_freq=8, max_degree=128,
                 freq_embedding_size=32, degree_embedding_size=32, output_dim=32, node_hidden_dim=32,
                 edge_hidden_dim=32, num_layers=6, num_heads=4, num_step_set2set=6,
                 num_layer_set2set=3, norm=False, gnn_model="mpnn", degree_input=False,
                 lstm_as_gate=False):
        super(GraphEncoder, self).__init__()
        if gnn_model != "gin":
            raise NotImplementedError("only gnn_model='gin' (train.py:77 default, the north-star path) "
                                      "is implemented; mpnn/gat are out of scope (SURVEY.md section 2)")
        if not degree_input:
            raise NotImplementedError("degree_input=False is never used by train.py (:618)")
        if output_dim != node_hidden_dim:
            raise NotImplementedError("output_dim must equal node_hidden_dim (train.py:612-613)")
        self.gnn_model, self.norm, self.degree_input = gnn_model, norm, degree_input
        self.max_node_freq, self.max_edge_freq, self.max_degree = max_node_freq, max_edge_freq, max_degree
        H, L = node_hidden_dim, num_layers
        self.cfg = glayout.make_cfg(num_layers=L, hidden=H, pos_dim=positional_embedding_size,
                                    deg_dim=degree_embedding_size, max_degree=max_degree, norm=norm)
        self._slices, self._n_live = glayout.param_slices(self.cfg)
        self._rslices, self._n_run = glayout.running_slices(self.cfg)
        din = positional_embedding_size + degree_embedding_size + 1
        # ---- draw initial values in the reference's construction order (gin.py:152-197,
        #      graph_encoder.py:92-130) so that a given torch seed yields the same weights
        init = {}
        for l in range(L - 1):
            p = "gnn.ginlayers.%d.apply_func." % l
            lin0 = nn.Linear(din if l == 0 else H, H)
            lin1 = nn.Linear(H, H)
            init[p + "mlp.linears.0.weight"], init[p + "mlp.linears.0.bias"] = lin0.weight, lin0.bias
            init[p + "mlp.linears.1.weight"], init[p + "mlp.linears.1.bias"] = lin1.weight, lin1.bias
        for l in range(L):
            lp = nn.Linear(din if l == 0 else H, output_dim)
            init["gnn.linears_prediction.%d.weight" % l] = lp.weight
            init["gnn.linears_prediction.%d.bias" % l] = lp.bias
        init["degree_embedding.weight"] = nn.Embedding(max_degree + 1, degree_embedding_size).weight
        lstm = nn.LSTM(2 * H, H, num_layer_set2set)                 # dgl Set2Set's only parameters
        ro0, ro2 = nn.Linear(2 * H, H), nn.Linear(H, output_dim)
        dead = [("set2set.lstm." + n, p_) for n, p_ in lstm.named_parameters()]
        dead += [("lin_readout.0.weight", ro0.weight), ("lin_readout.0.bias", ro0.bias),
                 ("lin_readout.2.weight", ro2.weight), ("lin_readout.2.bias", ro2.bias)]
        self._dead_slices, off = {}, self._n_live
        for name, p_ in dead:
            self._dead_slices[name] = (off, tuple(p_.shape))
            off += p_.numel()
        self._n_all = off
        flat = torch.zeros(self._n_all)
        for key, (o, shape) in self._slices.items():
            n = 1
            for s in shape:
                n *= s
            if key in init:
                flat[o:o + n] = init[key].detach().reshape(-1)
            elif key.endswith("weight"):
                flat[o:o + n] = 1.0                                  # BatchNorm gamma
        for name, p_ in dead:
            o, shape = self._dead_slices[name]
            flat[o:o + p_.numel()] = p_.detach().reshape(-1)
        running = torch.zeros(self._n_run)
        for key, (o, shape) in self._rslices.items():
            if key.endswith("running_var"):
                running[o:o + shape[0]] = 1.0
        # ---- module tree with the reference's names ------------------------------------------------
        gnn = _child(self, "gnn")
        ginlayers = _child(gnn, "ginlayers")
        for l in range(L - 1):
            conv = _child(ginlayers, str(l))
            apply_func = _child(conv, "apply_func")
            conv.register_buffer("eps", torch.zeros(1))              # GINConv(learn_eps=False, init_eps=0)
            mlp = _child(apply_func, "mlp")
            _child(_child(mlp, "linears"), "0")
            _child(_child(mlp, "linears"), "1")
            _child(_child(mlp, "batch_norms"), "0", _BatchNormHolder)
            _child(apply_func, "bn", _BatchNormHolder)
        gbn = _child(gnn, "batch_norms")
        for l in range(L - 1):
            _child(gbn, str(l), _BatchNormHolder)
        lp = _child(gnn, "linears_prediction")
        for l in range(L):
            _child(lp, str(l))
        gnn.add_module("drop", nn.Dropout(0.5))                      # gin.py:202 final_dropout
        _child(self, "degree_embedding")
        _child(_child(self, "set2set"), "lstm")
        ro = _child(self, "lin_readout")
        _child(ro, "0")
        ro.add_module("1", nn.ReLU())
        _child(ro, "2")
        self._flat = flat
        self._running = running
        self._nbt = torch.zeros(3 * (L - 1), dtype=torch.long)
        self._param_list = []
        self._bind_views(register=True)
        self.dropout_key = 0x9E3779B97F4A7C15 ^ (torch.initial_seed() & 0xFFFFFFFFFFFF)
        self._drop_step = 0
        self._scratch = {}

    # ---------------------------------------------------------------------------------------------
    def _resolve(self, key):
        mod = self
        parts = key.split(".")
        for p in parts[:-1]:
            mod = mod._modules[p]
        return mod, parts[-1]

    def _bind_views(self, register=False):
        """(Re)point every named parameter / buffer at its slice of the flat buffers."""
        self._param_list = []
        allp = list(self._slices.items()) + list(self._dead_slices.items())
        order = {}
        for key, (o, shape) in allp:
            n = 1
            for s in shape:
                n *= s
            view = self._flat[o:o + n].view(shape)
            mod, leaf = self._resolve(key)
            if register:
                mod.register_parameter(leaf, nn.Parameter(view))
            else:
                mod._parameters[leaf].data = view
            order[key] = mod._parameters[leaf]
        for key, (o, shape) in self._rslices.items():
            mod, leaf = self._resolve(key)
            view = self._running[o:o + shape[0]]
            if register:
                mod.register_buffer(leaf, view)
            else:
                mod._buffers[leaf] = view
        for i, key in enumerate(glayout.nbt_keys(self.cfg)):
            mod, leaf = self._resolve(key)
            if register:
                mod.register_buffer(leaf, self._nbt[i])
            else:
                mod._buffers[leaf] = self._nbt[i]
        self._live_params = [order[k] for k in self._slices]

    def _apply(self, fn, *a, **kw):
        super()._apply(fn, *a, **kw)
        # parameters were moved one by one: gather them back into flat buffers on the new device
        dev = next(iter(self.parameters())).device
        flat = torch.empty(self._n_all, dtype=torch.float32, device=dev)
        for key, (o, shape) in list(self._slices.items()) + list(self._dead_slices.items()):
            mod, leaf = self._resolve(key)
            flat[o:o + mod._parameters[leaf].numel()] = mod._parameters[leaf].data.reshape(-1).float()
        running = torch.empty(self._n_run, dtype=torch.float32, device=dev)
        for key, (o, shape) in self._rslices.items():
            mod, leaf = self._resolve(key)
            running[o:o + shape[0]] = mod._buffers[leaf].float()
        nbt = torch.empty(len(self._nbt), dtype=torch.long, device=dev)
        for i, key in enumerate(glayout.nbt_keys(self.cfg)):
            mod, leaf = self._resolve(key)
            nbt[i] = mod._buffers[leaf]
        self._flat, self._running, self._nbt = flat, running, nbt
        self._bind_views(register=False)
        self._scratch = {}
        return self

    def load_state_dict(self, state_dict, strict=True, **kw):
        res = super().load_state_dict(state_dict, strict=strict, **kw)   # copies INTO the views
        return res

    # flat views used by the engine / optimiser kernels
    @property
    def flat_params(self):
        return self._flat

    @property
    def n_live(self):
        return self._n_live

    @property
    def bn_train(self):
        return self.gnn.batch_norms._modules["0"].training

    # ---------------------------------------------------------------------------------------------
    def _acts_buffer(self, g, fresh):
        lib = _lib.get()
        nbytes = lib.gccb_gin_acts_bytes(C.byref(self.cfg), g.buffers.B, g.buffers.node_cap)
        if fresh:
            return torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
        key = ("acts", nbytes)
        if key not in self._scratch:
            self._scratch[key] = torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
        return self._scratch[key]

    def _run_forward(self, g, keep_for_backward, drop_step=None, drop_base=None, acts=None, feat=None,
                     pooled=None, bn_train=None):
        lib = _lib.get()
        buf = g.buffers
        dev = self._flat.device
        B, H, L = buf.B, self.cfg.hidden, self.cfg.num_layers
        if acts is None:
            acts = self._acts_buffer(g, fresh=keep_for_backward)
        if feat is None:
            feat = torch.empty(B, H, dtype=torch.float32, device=dev)
        if pooled is None:
            pooled = torch.empty(L - 1, B, H, dtype=torch.float32, device=dev)
        if drop_base is None:
            if self.gnn.drop.training:
                # mask layer ids: q view 0..L-1, k view L..2L-1 (E2E runs both views through this
                # module); the step index advances with every q-view forward
                drop_base = g.view * L
                if g.view == 0:
                    drop_step = self._drop_step
                    self._drop_step += 1
                else:
                    drop_step = max(self._drop_step - 1, 0)
            else:
                drop_base, drop_step = -1, 0
        rc = lib.gccb_gin_forward(C.byref(self.cfg), C.byref(buf.c), g.view, _lib.dptr(buf.pos),
                                  _lib.dptr(self._flat), _lib.dptr(self._running), _lib.dptr(self._nbt),
                                  1 if (self.bn_train if bn_train is None else bn_train) else 0,
                                  self.dropout_key, int(drop_step), int(drop_base),
                                  _lib.dptr(acts), acts.numel(), _lib.dptr(feat), _lib.dptr(pooled),
                                  _lib.stream_ptr())
        _lib.check(rc, "gccb_gin_forward")
        return feat, pooled, (acts, int(drop_step), int(drop_base))

    def _run_backward(self, g, saved, dfeat, grads_flat=None, ws=None):
        lib = _lib.get()
        acts, drop_step, drop_base = saved
        buf = g.buffers
        dev = self._flat.device
        own = grads_flat is None
        if own:
            # a fresh buffer per backward: autograd may keep the returned views as p.grad (or accumulate into
            # them), so a buffer must never be recycled by a later backward
            grads_flat = torch.zeros(self._n_live, dtype=torch.float32, device=dev)
        if ws is None:
            nbytes = lib.gccb_gin_backward_workspace(C.byref(self.cfg), buf.B, buf.node_cap)
            key = ("bwd", nbytes)
            if key not in self._scratch:
                self._scratch[key] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            ws = self._scratch[key]
        rc = lib.gccb_gin_backward(C.byref(self.cfg), C.byref(buf.c), g.view, _lib.dptr(self._flat),
                                   _lib.dptr(acts), _lib.dptr(dfeat), _lib.dptr(grads_flat), self.dropout_key,
                                   drop_step, drop_base, _lib.dptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "gccb_gin_backward")
        if not own:
            return None
        out = []
        for key, (o, shape) in self._slices.items():
            n = 1
            for s in shape:
                n *= s
            out.append(grads_flat[o:o + n].view(shape))
        return out

    def forward(self, g, return_all_outputs=False):
        """g: gcc_b200.datasets.BatchedSubgraphs (the batched DGLGraph stand-in).
        Returns Tensor[B, output_dim] or (x, [L-1 x Tensor[B, hidden]]) (graph_encoder.py:197-200)."""
        _lib.require_device()
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self._live_params)
        x, pooled = _GinEncodeFn.apply(self, g, need_grad, *self._live_params)
        if return_all_outputs:
            return x, [pooled[i] for i in range(pooled.shape[0])]
        return x
