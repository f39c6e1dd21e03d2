#!/usr/bin/env python
"""Generate tests/golden/train_moco_{sgd,adagrad}_golden.npz by executing the REAL reference train_moco
(train.py:350-478) with the other optimisers of train.py:659-678: torch.optim.SGD(momentum=0.9) and
torch.optim.Adagrad(lr_decay=0.01; non-zero so that the step count shows in the result).

The run is the one make_golden.py records in train_moco_golden.npz -- same batches, same initial weights
(torch.manual_seed(11)), same 3 steps and warm-up LR -- with only the optimiser changed, so the fixtures keep
just what differs and stay small:
  losses, post_clip_gnorms, s<step>_memory, final_index      every step / the end of the run
  idx/<param>                                                  a fixed sample of flat indices of each parameter
                                                               that receives gradients (all of it when small)
  model/<param>, ema/<param>, state/<param>/<field>            final weights, EMA weights and optimiser state
                                                               (momentum_buffer or sum) at those indices
  state_present, state_step, state_sum_absmax                  per parameter in param_order: whether the
                                                               optimiser holds state for it, Adagrad's step, and
                                                               the largest |sum| (0 for the unused tensors)
The tests read batches and initial weights from train_moco_golden.npz.

Run:  GCC_REFERENCE=<checkout of THUDM/GCC> python tests/golden/make_golden_optim.py
"""
import os
import types

import numpy as np
import torch

import make_golden as mg          # sets up the reference checkout, the DGL stub and the import paths

SAMPLE = 128


def golden_optim(kind, make_optimizer, num_layer=5, hidden=64, B=8, K=32, num_steps=3):
    import train as ref_train
    from oracle import rwr as orwr
    from gcc_b200.datasets import synthetic
    # golden_train("moco", ...) of make_golden.py up to the optimiser
    torch.manual_seed(11)
    g = synthetic.erdos_renyi(400, 1600, seed=9)
    cdf = orwr.seed_cdf(g.indptr)
    bt = orwr.budget_table(int(np.diff(g.indptr).max()), 48, 0.8)
    rt = orwr.restart_threshold(0.8)
    batches = mg._make_batches(num_steps, B, 48, g, cdf, bt, rt)

    def mk():
        return mg.ref_ge.GraphEncoder(positional_embedding_size=32, max_node_freq=16, max_edge_freq=16,
                                      max_degree=512, freq_embedding_size=16, degree_embedding_size=16,
                                      output_dim=hidden, node_hidden_dim=hidden, edge_hidden_dim=hidden,
                                      num_layers=num_layer, num_step_set2set=6, num_layer_set2set=3, norm=True,
                                      gnn_model="gin", degree_input=True)

    model, model_ema = mk(), mk()
    drop = mg._MaskDrop(mg.KEY, hidden)
    model.gnn.drop = drop
    ref_train.moment_update(model, model_ema, 0)
    contrast = mg.ref_moco.MemoryMoCo(hidden, None, K, 0.07, use_softmax=True)
    base = np.load(os.path.join(mg.HERE, "train_moco_golden.npz"))
    for k_, v in model.state_dict().items():
        assert np.array_equal(v.numpy(), base["init/" + k_]), k_
    assert np.array_equal(contrast.memory.numpy(), base["init_memory"])
    criterion = mg.ref_crit.NCESoftmaxLoss()
    optimizer = make_optimizer(model.parameters())
    opt = types.SimpleNamespace(batch_size=B, gpu="cpu", moco=True, clip_norm=1.0, learning_rate=0.005, epochs=2,
                                alpha=0.999, print_freq=1000, tb_freq=1000, nce_t=0.07, hidden_size=hidden)
    out = {"optimizer": np.array(kind)}
    losses, gnorms = [], []
    for st, (bq, bk) in enumerate(batches):
        for name, bg in (("q", bq), ("k", bk)):
            assert np.array_equal(bg.batched_csr()[1], base["s%d_%s_indices" % (st, name)])
        drop.step, drop.layer = st, 0
        sw = types.SimpleNamespace(add_scalar=lambda *a, **k: None)

        class _OneStep:
            dataset = types.SimpleNamespace(total=num_steps * B)

            def __iter__(self_inner):
                return iter([(bq, bk)])

        # global_step == st, as in golden_train
        losses.append(ref_train.train_moco(st / float(num_steps), _OneStep(), model, model_ema, contrast, criterion,
                                           optimizer, sw, opt))
        gnorms.append(float(torch.sqrt(sum((p.grad.detach() ** 2).sum() for p in model.parameters()
                                           if p.grad is not None))))
        out["s%d_memory" % st] = contrast.memory.numpy().copy()
    out["losses"], out["post_clip_gnorms"] = np.array(losses), np.array(gnorms)
    out["final_index"] = np.array(contrast.index)
    rng = np.random.default_rng(0)
    ema = dict(model_ema.named_parameters())
    names = [n for n, _ in model.named_parameters()]
    state = optimizer.state_dict()["state"]
    present, steps, sum_max = [], [], []
    for i, (n, p) in enumerate(model.named_parameters()):
        st_ = state.get(i, {})
        present.append(bool(st_))
        steps.append(float(st_["step"]) if "step" in st_ else -1.0)
        sum_max.append(float(st_["sum"].abs().max()) if "sum" in st_ else -1.0)
        if p.grad is None:
            continue
        size = p.numel()
        idx = np.arange(size) if size <= SAMPLE else np.sort(rng.choice(size, SAMPLE, replace=False))
        out["idx/" + n] = idx.astype(np.int32)
        out["model/" + n] = p.detach().reshape(-1).numpy()[idx].copy()
        out["ema/" + n] = ema[n].detach().reshape(-1).numpy()[idx].copy()
        for f, v in st_.items():
            if f != "step":
                out["state/%s/%s" % (n, f)] = v.reshape(-1).numpy()[idx].copy()
    out["param_order"] = np.array(names)
    out["state_present"], out["state_step"] = np.array(present), np.array(steps)
    out["state_sum_absmax"] = np.array(sum_max)
    mg.save("train_moco_%s_golden.npz" % kind, **out)


def main():
    golden_optim("sgd", lambda ps: torch.optim.SGD(ps, lr=0.005, momentum=0.9, weight_decay=1e-5))
    golden_optim("adagrad", lambda ps: torch.optim.Adagrad(ps, lr=0.005, lr_decay=0.01, weight_decay=1e-5))


if __name__ == "__main__":
    main()
