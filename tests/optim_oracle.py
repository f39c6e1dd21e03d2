"""Oracle (test infrastructure): one pretraining step with torch.optim.SGD or torch.optim.Adagrad as the
optimiser (train.py:659-678), in float64 on CPU.

oracle.step.train_step does the forward, loss, backward, BatchNorm statistics and enqueue; it is called with its
own update turned into the identity (Adam with lr = 0 leaves every parameter as it was, alpha = 1 leaves the
EMA as it was), and the clip, the named optimiser and moment_update are then applied here to the gradients it
returns.  State: the dict of oracle.step (params, ema, memory, index) plus
  t            -- steps taken (the reference's Adagrad counts it per parameter; all live ones step together)
  sgd_buf      -- {key: momentum_buffer}
  adagrad_sum  -- {key: sum}
"""
from oracle import step as ostep

ADAGRAD_EPS = 1e-10


def train_step(state, batch_q, batch_k, *, optimizer, num_layers, moco=True, lr=0.005, alpha=0.999, clip_norm=1.0,
               weight_decay=1e-5, momentum=0.9, lr_decay=0.0, **kw):
    """optimizer: "sgd" (momentum, dampening 0, no Nesterov) or "adagrad" (lr_decay, eps 1e-10); **kw go to
    oracle.step.train_step (T, dropout_key, step_index, max_degree).  Returns its result dict."""
    if optimizer not in ("sgd", "adagrad"):
        raise ValueError("optimizer must be sgd or adagrad, not %r" % (optimizer,))
    inner = dict(state, adam_m={}, adam_v={}, adam_t=0)
    r = ostep.train_step(inner, batch_q, batch_k, num_layers=num_layers, moco=moco, lr=0.0, alpha=1.0,
                         clip_norm=clip_norm, **kw)
    state["index"] = inner["index"]
    params = state["params"]
    state["t"] = t = state.get("t", 0) + 1
    coef = clip_norm / (r["grad_norm"] + 1e-6)                 # clip_grad_norm_ (train.py:409)
    for k, g in r["grads"].items():
        g = g.detach()
        if coef < 1.0:
            g = g * coef
        p = params[k]
        d = g + weight_decay * p
        if optimizer == "sgd":
            if momentum != 0:
                buf = state.setdefault("sgd_buf", {}).get(k)
                d = d.clone() if buf is None else buf.mul_(momentum).add_(d)     # first step: buf = d
                state["sgd_buf"][k] = d
            params[k] = p - lr * d
        else:
            s = state.setdefault("adagrad_sum", {}).get(k)
            s = d * d if s is None else s.addcmul_(d, d)
            state["adagrad_sum"][k] = s
            clr = lr / (1 + (t - 1) * lr_decay)
            params[k] = p - clr * d / (s.sqrt() + ADAGRAD_EPS)
    if moco:                                                    # moment_update (train.py:169-172,430-431)
        for k in params:
            if not ostep.is_buffer(k):
                state["ema"][k] = state["ema"][k] * alpha + (1 - alpha) * params[k]
    return r
