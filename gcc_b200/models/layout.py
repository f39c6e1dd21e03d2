"""Flat parameter layout of the GIN encoder <-> the reference's state_dict keys.

The CUDA kernels read every live parameter from ONE flat fp32 buffer
(include/gccb200.h: gccb_gin_layout_t, built by gccb_gin_param_layout).  This
module maps the reference's state_dict keys (SURVEY.md section 8b;
gcc/models/graph_encoder.py:44-130, gcc/models/gin.py:119-211) onto slices of
that buffer, so checkpoints stay key-compatible while Adam / EMA / gradient
exchange operate on a single contiguous array.
"""
import ctypes as C
from collections import OrderedDict

from .. import _capi


def make_cfg(num_layers=5, hidden=64, pos_dim=32, deg_dim=16, max_degree=512, norm=True,
             bn_eps=1e-5, bn_momentum=0.1, norm_eps=1e-5, dropout_p=0.5, tensor_cores=None):
    """tensor_cores: None = on for hidden >= 128 (the fp32 SIMT path stays selectable with tensor_cores=0)."""
    if tensor_cores is None:
        tensor_cores = hidden >= 128
    return _capi.GinCfg(num_layers, hidden, pos_dim, deg_dim, max_degree, int(bool(norm)),
                        bn_eps, bn_momentum, norm_eps, dropout_p, int(bool(tensor_cores)), 0)


def param_slices(cfg):
    """OrderedDict key -> (offset, shape) for the live parameters, in flat-buffer order.
    Pure-Python mirror of make_param_layout() in csrc/gin_common.cuh (tests compare the
    two through gccb_gin_param_layout)."""
    L, H = cfg.num_layers, cfg.hidden
    din = cfg.pos_dim + cfg.deg_dim + 1
    out = OrderedDict()
    off = 0

    def take(key, shape):
        nonlocal off
        n = 1
        for s in shape:
            n *= s
        out[key] = (off, tuple(shape))
        off += n

    for l in range(L - 1):
        inf = din if l == 0 else H
        p = "gnn.ginlayers.%d.apply_func." % l
        take(p + "mlp.linears.0.weight", (H, inf))
        take(p + "mlp.linears.0.bias", (H,))
        take(p + "mlp.batch_norms.0.weight", (H,))
        take(p + "mlp.batch_norms.0.bias", (H,))
        take(p + "mlp.linears.1.weight", (H, H))
        take(p + "mlp.linears.1.bias", (H,))
        take(p + "bn.weight", (H,))
        take(p + "bn.bias", (H,))
        take("gnn.batch_norms.%d.weight" % l, (H,))
        take("gnn.batch_norms.%d.bias" % l, (H,))
    for l in range(L):
        inf = din if l == 0 else H
        take("gnn.linears_prediction.%d.weight" % l, (H, inf))
        take("gnn.linears_prediction.%d.bias" % l, (H,))
    take("degree_embedding.weight", (cfg.max_degree + 1, cfg.deg_dim))
    return out, off


def running_slices(cfg):
    """key -> (offset, shape) into the flat running-statistics buffer
    [layer][bn: mlp.batch_norms.0, apply_func.bn, gnn.batch_norms][mean|var][H]."""
    L, H = cfg.num_layers, cfg.hidden
    out = OrderedDict()
    for l in range(L - 1):
        names = ("gnn.ginlayers.%d.apply_func.mlp.batch_norms.0." % l,
                 "gnn.ginlayers.%d.apply_func.bn." % l, "gnn.batch_norms.%d." % l)
        for b, name in enumerate(names):
            base = ((l * 3 + b) * 2) * H
            out[name + "running_mean"] = (base, (H,))
            out[name + "running_var"] = (base + H, (H,))
    return out, (L - 1) * 3 * 2 * H


def nbt_keys(cfg):
    keys = []
    for l in range(cfg.num_layers - 1):
        keys += ["gnn.ginlayers.%d.apply_func.mlp.batch_norms.0.num_batches_tracked" % l,
                 "gnn.ginlayers.%d.apply_func.bn.num_batches_tracked" % l,
                 "gnn.batch_norms.%d.num_batches_tracked" % l]
    return keys


def c_layout(lib, cfg):
    lay = _capi.GinLayout()
    rc = lib.gccb_gin_param_layout(C.byref(cfg), C.byref(lay))
    if rc:
        raise ValueError(lib.gccb_last_error().decode())
    return lay


# ---- GAT encoder (gnn_model="gat"; include/gccb200.h: gccb_gat_layout_t) --------------------------------------
def make_gat_cfg(num_layers=5, hidden=64, num_heads=4, pos_dim=32, deg_dim=16, max_degree=512, set2set_iter=6,
                 set2set_layers=3, norm=True, norm_eps=1e-5):
    return _capi.GatCfg(num_layers, hidden, num_heads, pos_dim, deg_dim, max_degree, set2set_iter, set2set_layers,
                        int(bool(norm)), norm_eps)


def gat_param_slices(cfg):
    """OrderedDict key -> (offset, shape) of every GAT-encoder parameter, in flat-buffer order.  Pure-Python mirror
    of gat_param_layout() in csrc/gat.cu (tests compare the two through gccb_gat_param_layout).  Keys are the
    reference's: gnn.layers.{i}.gnn.* (dgl GATLayer wrapping GATConv), degree_embedding, set2set.lstm.*,
    lin_readout.{0,2}.*."""
    L, H, nh = cfg.num_layers, cfg.hidden, cfg.num_heads
    din = cfg.pos_dim + cfg.deg_dim + 1
    out = OrderedDict()
    off = 0

    def take(key, shape):
        nonlocal off
        n = 1
        for s in shape:
            n *= s
        out[key] = (off, tuple(shape))
        off += n

    for i in range(L):
        p = "gnn.layers.%d.gnn." % i
        take(p + "fc.weight", (H, din if i == 0 else H))
        take(p + "attn_l", (1, nh, H // nh))
        take(p + "attn_r", (1, nh, H // nh))
    take("degree_embedding.weight", (cfg.max_degree + 1, cfg.deg_dim))
    for k in range(cfg.set2set_layers):
        take("set2set.lstm.weight_ih_l%d" % k, (4 * H, 2 * H if k == 0 else H))
        take("set2set.lstm.weight_hh_l%d" % k, (4 * H, H))
        take("set2set.lstm.bias_ih_l%d" % k, (4 * H,))
        take("set2set.lstm.bias_hh_l%d" % k, (4 * H,))
    take("lin_readout.0.weight", (H, 2 * H))
    take("lin_readout.0.bias", (H,))
    take("lin_readout.2.weight", (H, H))
    take("lin_readout.2.bias", (H,))
    return out, off


def gat_c_layout(lib, cfg):
    lay = _capi.GatLayout()
    rc = lib.gccb_gat_param_layout(C.byref(cfg), C.byref(lay))
    if rc:
        raise ValueError(lib.gccb_last_error().decode())
    return lay
