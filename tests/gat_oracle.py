"""Float64 restatement of the GAT encoder (test infrastructure): GraphEncoder(gnn_model="gat") of the reference
(gcc/models/gat.py UnsupervisedGAT of dgl GATLayers, dgl Set2Set, lin_readout; graph_encoder.py:152-196) in torch on
the CPU, autograd supplying the backward.  DGL 0.4.3 cannot run here, so the DGL parts are restated from their
documented semantics (DESIGN.md, GAT section):
  GATConv (feat_drop = attn_drop = 0, no residual): z = X W^T viewed [N, nh, F]; el = sum_f z attn_l, er likewise;
  e(u->v) = leaky_relu(el_u + er_v, 0.2); a = softmax of e over the in-edges of v (row v of the CSR; parallel edges
  and self loops are separate terms); out_v = sum a z_u, 0 without in-edges; flatten; leaky_relu(0.01) except after
  the last layer.
  Set2Set: q* = 0, (h, c) = 0; n_iters times q, (h, c) = LSTM(q*, (h, c)) (the real torch.nn.LSTM),
  e_i = <x_i, q_b>, alpha = softmax over b's nodes, r_b = sum alpha_i x_i, q* = [q | r].
The input X0 is the GIN path's, as in oracle/model.py.  The step (train_step below) is oracle/step.py's with this
encoder in place of the GIN one."""
import numpy as np
import torch
import torch.nn.functional as F
from torch.func import functional_call


def gat_encoder_forward(params, indptr, indices, pos, seed_flag, sub_deg, node_off, num_layers, num_heads,
                        set2set_iter, set2set_layers, max_degree=512, norm=True, record=None):
    """params: {state_dict key: tensor} (float64); indptr / indices: batched CSR with global row ids;
    node_off: [B+1].  record (optional dict) receives the intermediates the kernels stash.  Returns feat [B, H]."""
    dt = pos.dtype
    N = pos.shape[0]
    B = len(node_off) - 1
    emb = params["degree_embedding.weight"]
    deg = torch.as_tensor(np.asarray(sub_deg), dtype=torch.long).clamp(0, max_degree)
    h = torch.cat([pos, emb[deg], torch.as_tensor(np.asarray(seed_flag)).to(dt).unsqueeze(1)], dim=-1)
    row = torch.repeat_interleave(torch.arange(N), torch.as_tensor(np.diff(indptr)).long())    # destination v
    col = torch.as_tensor(np.asarray(indices)).long()                                          # source u
    rec = record if record is not None else {}
    rec["x0"] = h
    for i in range(num_layers):
        p = "gnn.layers.%d.gnn." % i
        W = params[p + "fc.weight"]
        H = W.shape[0]
        nh = num_heads
        z = (h @ W.t()).view(N, nh, H // nh)
        el = (z * params[p + "attn_l"]).sum(-1)
        er = (z * params[p + "attn_r"]).sum(-1)
        e = F.leaky_relu(el[col] + er[row], 0.2)
        emax = torch.full((N, nh), -torch.inf, dtype=dt).scatter_reduce(0, row[:, None].expand(-1, nh), e.detach(),
                                                                         "amax")
        ex = torch.exp(e - emax[row])
        den = torch.zeros(N, nh, dtype=dt).index_add(0, row, ex)
        a = ex / den[row]
        out = torch.zeros(N, nh, H // nh, dtype=dt).index_add(0, row, a[:, :, None] * z[col]).reshape(N, H)
        if i < num_layers - 1:
            out = F.leaky_relu(out, 0.01)
        rec.setdefault("z", []).append(z.reshape(N, H))
        rec.setdefault("el", []).append(el)
        rec.setdefault("er", []).append(er)
        rec.setdefault("den", []).append(den)
        rec.setdefault("h", []).append(out)
        h = out
    x = h
    H = x.shape[1]
    lstm = torch.nn.LSTM(2 * H, H, set2set_layers).to(dt)
    lsd = {n: params["set2set.lstm." + n] for n, _ in lstm.named_parameters()}
    gid = torch.repeat_interleave(torch.arange(B), torch.as_tensor(np.diff(node_off)).long())
    hc = (torch.zeros(set2set_layers, B, H, dtype=dt), torch.zeros(set2set_layers, B, H, dtype=dt))
    q_star = torch.zeros(B, 2 * H, dtype=dt)
    for _ in range(set2set_iter):
        q, hc = functional_call(lstm, lsd, (q_star.unsqueeze(0), hc))
        q = q.view(B, H)
        e = (x * q[gid]).sum(-1)
        emax = torch.full((B,), -torch.inf, dtype=dt).scatter_reduce(0, gid, e.detach(), "amax")
        ex = torch.exp(e - emax[gid])
        den = torch.zeros(B, dtype=dt).index_add(0, gid, ex)
        alpha = ex / den[gid]
        r = torch.zeros(B, H, dtype=dt).index_add(0, gid, alpha[:, None] * x)
        q_star = torch.cat([q, r], dim=-1)
        rec.setdefault("alpha", []).append(alpha)
        rec.setdefault("qstar", []).append(q_star)
    y = F.relu(q_star @ params["lin_readout.0.weight"].t() + params["lin_readout.0.bias"])
    s = y @ params["lin_readout.2.weight"].t() + params["lin_readout.2.bias"]
    rec["y1"], rec["score"] = y, s
    if norm:
        s = F.normalize(s, p=2, dim=-1, eps=1e-5)
    return s


class _GATConv(torch.nn.Module):
    """dgl.nn.pytorch.GATConv (0.4.3) as UnsupervisedGAT builds it: in_feats an int, residual=False, dropouts 0 --
    only its parameters and their initialisation."""

    def __init__(self, in_feats, out_feats, num_heads):
        super().__init__()
        self.fc = torch.nn.Linear(in_feats, out_feats * num_heads, bias=False)
        self.attn_l = torch.nn.Parameter(torch.FloatTensor(size=(1, num_heads, out_feats)))
        self.attn_r = torch.nn.Parameter(torch.FloatTensor(size=(1, num_heads, out_feats)))
        self.reset_parameters()

    def reset_parameters(self):
        gain = torch.nn.init.calculate_gain("relu")
        torch.nn.init.xavier_normal_(self.fc.weight, gain=gain)
        torch.nn.init.xavier_normal_(self.attn_l, gain=gain)
        torch.nn.init.xavier_normal_(self.attn_r, gain=gain)


class _GATLayer(torch.nn.Module):
    """dgl.model_zoo.chem.gnn.GATLayer: a GATConv named `gnn`."""

    def __init__(self, in_feats, out_feats, num_heads):
        super().__init__()
        self.gnn = _GATConv(in_feats, out_feats, num_heads)


class _Set2Set(torch.nn.Module):
    """dgl.nn.pytorch.glob.Set2Set (0.4.3): the LSTM, then reset_parameters() from the constructor."""

    def __init__(self, input_dim, n_iters, n_layers):
        super().__init__()
        self.lstm = torch.nn.LSTM(2 * input_dim, input_dim, n_layers)
        self.reset_parameters()

    def reset_parameters(self):
        self.lstm.reset_parameters()


class _ReferenceGAT(torch.nn.Module):
    """GraphEncoder.__init__ with gnn_model="gat", degree_input=True (graph_encoder.py:44-130): gnn, then
    degree_embedding, set2set, lin_readout."""

    def __init__(self, num_layers, hidden, num_heads, din, max_degree, deg_dim, set2set_iter, set2set_layers):
        super().__init__()
        self.gnn = torch.nn.Module()
        self.gnn.layers = torch.nn.ModuleList([_GATLayer(din if i == 0 else hidden, hidden // num_heads, num_heads)
                                              for i in range(num_layers)])
        self.degree_embedding = torch.nn.Embedding(max_degree + 1, deg_dim)
        self.set2set = _Set2Set(hidden, set2set_iter, set2set_layers)
        self.lin_readout = torch.nn.Sequential(torch.nn.Linear(2 * hidden, hidden), torch.nn.ReLU(),
                                               torch.nn.Linear(hidden, hidden))


def reference_init(num_layers, hidden, num_heads, din, max_degree, deg_dim, set2set_layers, set2set_iter=6):
    """state_dict of a plain-torch construction with the reference's module structure and order (above)."""
    return {k: v.detach() for k, v in _ReferenceGAT(num_layers, hidden, num_heads, din, max_degree, deg_dim,
                                                    set2set_iter, set2set_layers).state_dict().items()}


def train_step(state, batch_q, batch_k, *, num_layers, num_heads, set2set_iter, set2set_layers, moco=True, T=0.07,
               lr=0.005, alpha=0.999, clip_norm=1.0, weight_decay=1e-5, beta1=0.9, beta2=0.999, max_degree=512):
    """One MoCo / E2E step (train.py:378-434) with the GAT encoder: oracle/step.py's train_step with the encoder
    forward replaced by gat_encoder_forward and nothing else -- the head, loss, clip, Adam, EMA and enqueue are the
    project's oracle functions (oracle/model.py, oracle/step.py).  The GAT encoder has no BatchNorm and no dropout.
    batch_* = dict(indptr, indices, pos, seed, sub_deg, node_off).  Returns dict(loss, grad_norm, feat_q, feat_k)."""
    from oracle import model as om
    from oracle import step as ostep
    params = state["params"]
    live = [k for k in params if not ostep.is_buffer(k)]
    for k in live:
        params[k] = params[k].detach().clone().requires_grad_(True)

    def enc(p, b):
        return gat_encoder_forward(p, b["indptr"], b["indices"], torch.as_tensor(b["pos"]).double(), b["seed"],
                                   b["sub_deg"], b["node_off"], num_layers, num_heads, set2set_iter, set2set_layers,
                                   max_degree=max_degree, norm=True)

    feat_q = enc(params, batch_q)
    if moco:
        with torch.no_grad():
            feat_k = enc(state["ema"], batch_k)
        loss = om.nce_softmax_loss(om.moco_logits(feat_q, feat_k, state["memory"], T))
    else:
        feat_k = enc(params, batch_k)
        loss = om.nce_softmax_loss_ns(feat_k @ feat_q.t() / T)
    grads = torch.autograd.grad(loss, [params[k] for k in live], allow_unused=True)
    gdict = {k: g for k, g in zip(live, grads) if g is not None}
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in gdict.values()))
    coef = clip_norm / (float(total) + 1e-6)
    state["adam_t"] = state.get("adam_t", 0) + 1
    t = state["adam_t"]
    with torch.no_grad():
        for k, g in gdict.items():
            params[k] = ostep._adam(state, k, params[k], g * coef if coef < 1.0 else g, lr, t, weight_decay, beta1,
                                    beta2)
        for k in live:
            params[k] = params[k].detach()
        if moco:
            for k in live:
                state["ema"][k] = state["ema"][k] * alpha + (1 - alpha) * params[k]
            state["index"] = om.moco_enqueue(state["memory"], feat_k, state["index"])
    return dict(loss=float(loss.detach()), grad_norm=float(total), feat_q=feat_q.detach(), feat_k=feat_k.detach())
