"""Oracle (test infrastructure): GIN encoder, MoCo head, InfoNCE, optimiser.

Torch-CPU restatement (autograd supplies the backward oracle) of:
  gcc/models/graph_encoder.py:152-196  feature assembly, GIN dispatch, L2 norm
  gcc/models/gin.py:42-58,107-116,213-232  ApplyNodeFunc / MLP / UnsupervisedGIN
  DGL GINConv('sum', eps=0 buffer) and SumPooling   [M: documented semantics]
  gcc/contrastive/memory_moco.py:26-63  logits + FIFO enqueue
  gcc/contrastive/criterions.py:5-33    NCESoftmaxLoss / NCESoftmaxLossNS
  train.py:169-172   moment_update (EMA, parameters only)
  train.py:340-347,409  clip_grad_norm ; train.py:411-417,667-672 Adam step
  gcc/utils/misc.py:5-10  warmup_linear
Parameter names are the reference's state_dict keys (SURVEY.md section 8b).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def param_shapes(num_layers=5, hidden=64, pos_size=32, deg_emb=16, max_degree=512,
                 output_dim=None):
    """Ordered {state_dict key: shape} of the GIN-path parameters + buffers."""
    out_dim = output_dim or hidden
    d_in = pos_size + deg_emb + 1
    shapes = {}
    for i in range(num_layers - 1):
        din = d_in if i == 0 else hidden
        p = "gnn.ginlayers.%d." % i
        shapes[p + "eps"] = (1,)
        shapes[p + "apply_func.mlp.linears.0.weight"] = (hidden, din)
        shapes[p + "apply_func.mlp.linears.0.bias"] = (hidden,)
        shapes[p + "apply_func.mlp.linears.1.weight"] = (hidden, hidden)
        shapes[p + "apply_func.mlp.linears.1.bias"] = (hidden,)
        for bn in (p + "apply_func.mlp.batch_norms.0.", p + "apply_func.bn.",
                   "gnn.batch_norms.%d." % i):
            shapes[bn + "weight"] = (hidden,)
            shapes[bn + "bias"] = (hidden,)
            shapes[bn + "running_mean"] = (hidden,)
            shapes[bn + "running_var"] = (hidden,)
            shapes[bn + "num_batches_tracked"] = ()
    for i in range(num_layers):
        din = d_in if i == 0 else hidden
        shapes["gnn.linears_prediction.%d.weight" % i] = (out_dim, din)
        shapes["gnn.linears_prediction.%d.bias" % i] = (out_dim,)
    shapes["degree_embedding.weight"] = (max_degree + 1, deg_emb)
    return shapes


def _bn_train(x, weight, bias, eps=1e-5):
    mean = x.mean(dim=0)
    var = x.var(dim=0, unbiased=False)
    return (x - mean) / torch.sqrt(var + eps) * weight + bias, mean, var


def _bn(x, params, key, train, stats_out, momentum=0.1, eps=1e-5):
    w, b = params[key + "weight"], params[key + "bias"]
    if train:
        y, mean, var = _bn_train(x, w, b, eps)
        n = x.shape[0]
        stats_out[key] = (mean.detach(), (var * n / max(n - 1, 1)).detach())
        return y
    rm, rv = params[key + "running_mean"], params[key + "running_var"]
    return (x - rm) / torch.sqrt(rv + eps) * w + b


def _round_operand(x, dt):
    """Round a GEMM operand to `dt` (bf16: what the tensor-core path feeds wgmma) in the forward only
    (straight-through for autograd); accumulation stays in the oracle's precision."""
    if dt is None:
        return x
    return x + (x.detach().to(dt).to(x.dtype) - x.detach())


def gin_encoder_forward(params, indptr, indices, pos, seed_flag, sub_deg, node_off,
                        num_layers=5, max_degree=512, norm=True, bn_train=True,
                        dropout_keep=None, dropout_p=0.5, gemm_operand_dtype=None):
    """graph_encoder.py:132-200 (gin branch) on a batched graph.

    indptr/indices: batched CSR with global row ids; node_off: [B+1] offsets.
    dropout_keep: None (eval-mode dropout) or list of num_layers bool [B,out]
    masks (the Philox mask spec) -> x * keep / (1-p).
    Returns (feat[B,out], all_outputs list, bn batch stats dict)."""
    dt = pos.dtype
    N = pos.shape[0]
    B = len(node_off) - 1
    emb = params["degree_embedding.weight"]
    deg = torch.as_tensor(np.asarray(sub_deg), dtype=torch.long).clamp(0, max_degree)
    h = torch.cat([pos, emb[deg], torch.as_tensor(np.asarray(seed_flag)).to(dt).unsqueeze(1)],
                  dim=-1)                                   # graph_encoder.py:158-165
    row = torch.repeat_interleave(torch.arange(N), torch.as_tensor(np.diff(indptr)).long())
    col = torch.as_tensor(np.asarray(indices)).long()
    gid = torch.repeat_interleave(torch.arange(B), torch.as_tensor(np.diff(node_off)).long())
    stats = {}
    hidden_rep = [h]
    for i in range(num_layers - 1):
        p = "gnn.ginlayers.%d." % i
        # DGL GINConv 'sum': rst = (1 + eps) * feat + sum_{u in N(v)} feat_u   [M]
        neigh = torch.zeros_like(h).index_add_(0, row, h[col])
        a = (1.0 + params[p + "eps"].to(dt)) * h + neigh
        gd = gemm_operand_dtype
        z1 = F.linear(_round_operand(a, gd), _round_operand(params[p + "apply_func.mlp.linears.0.weight"], gd),
                      params[p + "apply_func.mlp.linears.0.bias"])      # gin.py:113-115
        x1 = F.relu(_bn(z1, params, p + "apply_func.mlp.batch_norms.0.", bn_train, stats))
        z2 = F.linear(_round_operand(x1, gd), _round_operand(params[p + "apply_func.mlp.linears.1.weight"], gd),
                      params[p + "apply_func.mlp.linears.1.bias"])      # gin.py:116
        y = F.relu(_bn(z2, params, p + "apply_func.bn.", bn_train, stats))   # gin.py:55-57
        h = F.relu(_bn(y, params, "gnn.batch_norms.%d." % i, bn_train, stats))  # gin.py:219-220
        hidden_rep.append(h)
    score = 0
    all_outputs = []
    for i, hh in enumerate(hidden_rep):
        pooled = torch.zeros(B, hh.shape[1], dtype=dt).index_add_(0, gid, hh)  # SumPooling [M]
        all_outputs.append(pooled)
        s = F.linear(pooled, params["gnn.linears_prediction.%d.weight" % i],
                     params["gnn.linears_prediction.%d.bias" % i])
        if dropout_keep is not None:
            s = s * torch.as_tensor(dropout_keep[i]).to(dt) / (1.0 - dropout_p)
        score = score + s                                               # gin.py:227-230
    x = score
    if norm:
        x = F.normalize(x, p=2, dim=-1, eps=1e-5)                       # graph_encoder.py:196
    return x, all_outputs[1:], stats


def moco_logits(q, k, memory, T):
    """memory_moco.py:33-44, use_softmax branch: [q.k | q.queue^T] / T."""
    l_pos = (q * k.detach()).sum(dim=1, keepdim=True)
    l_neg = q @ memory.detach().t()
    return torch.cat([l_pos, l_neg], dim=1) / T


def moco_enqueue(memory, k, index):
    """memory_moco.py:55-61.  Returns new index; memory updated in place."""
    K = memory.shape[0]
    B = k.shape[0]
    ids = torch.fmod(torch.arange(B) + index, K).long()
    memory.index_copy_(0, ids, k.detach())
    return (index + B) % K


def nce_softmax_loss(out):
    """criterions.py:12-17: CE against label 0."""
    return F.cross_entropy(out, torch.zeros(out.shape[0], dtype=torch.long))


def nce_softmax_loss_ns(out):
    """criterions.py:27-33: CE against label arange(B)."""
    return F.cross_entropy(out, torch.arange(out.shape[0]))


def warmup_linear(x, warmup=0.002):
    """misc.py:5-10."""
    if x < warmup:
        return x / warmup
    return max((x - 1.0) / (warmup - 1.0), 0)


def clip_adam_ema(p, g, m, v, p_ema, step, lr, beta1=0.9, beta2=0.999, eps=1e-8,
                  weight_decay=1e-5, clip_norm=1.0, alpha=0.999, n_live=None):
    """Flat float64/32 numpy restatement of train.py:409 (clip_grad_norm_),
    :417 Adam(L2 weight decay) and :169-172 moment_update.
    p/g/m/v: live parameters [n_live]; p_ema covers [n_all >= n_live] and p_all is
    p for the first n_live entries.  `step` is the 1-based Adam step count.
    Returns grad_norm; arrays updated in place."""
    gnorm = float(np.sqrt((g.astype(np.float64) ** 2).sum()))
    coef = clip_norm / (gnorm + 1e-6)
    if coef < 1.0:
        g *= g.dtype.type(coef)
    g += g.dtype.type(weight_decay) * p
    m *= beta1
    m += (1 - beta1) * g
    v *= beta2
    v += (1 - beta2) * g * g
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = np.sqrt(v) / math.sqrt(bc2) + eps
    p -= (lr / bc1) * (m / denom)
    return gnorm


def ema_update(p_ema, p, alpha):
    """train.py:169-172: p_ema = alpha * p_ema + (1 - alpha) * p."""
    p_ema *= alpha
    p_ema += (1 - alpha) * p
