"""CPU: tests/optim_oracle.py:train_step with optimizer="sgd" / "adagrad" reproduces the REAL reference train_moco
(train.py:350-478) run with torch.optim.SGD(momentum=0.9) and torch.optim.Adagrad(lr_decay=0.01)
(train.py:659-678) by tests/golden/make_golden_optim.py: losses, queue, updated weights, EMA weights and
optimiser state.  Batches and initial weights are those of train_moco_golden.npz."""
import os

import numpy as np
import pytest
import torch

import optim_oracle
from oracle import model as om

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OPTIM = {"sgd": dict(momentum=0.9), "adagrad": dict(lr_decay=0.01)}


def _load_batch(z, st, name):
    indptr = z["s%d_%s_indptr" % (st, name)]
    nn = z["s%d_%s_num_nodes" % (st, name)]
    return dict(indptr=indptr, indices=z["s%d_%s_indices" % (st, name)],
                pos=z["s%d_%s_pos" % (st, name)], seed=z["s%d_%s_seed" % (st, name)],
                sub_deg=np.diff(indptr), node_off=np.concatenate([[0], np.cumsum(nn)]))


def _chaotic(name):
    # a bias feeding a train-mode BatchNorm has an exactly-zero true gradient; Adagrad's first step d/sqrt(d^2)
    # is sign-like and moves it by +-lr on fp32 noise, in the reference too (see test_train_step_golden)
    return "mlp.linears" in name and name.endswith("bias")


@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_train_step_golden_other_optimizers(kind):
    base = np.load(os.path.join(G, "train_moco_golden.npz"))
    z = np.load(os.path.join(G, "train_moco_%s_golden.npz" % kind))
    assert str(z["optimizer"]) == kind and list(z["param_order"]) == list(base["param_order"])
    L, S = int(base["num_layer"]), int(base["num_steps"])
    init = {k[5:]: torch.from_numpy(base[k].copy()) for k in base.files if k.startswith("init/")}
    state = dict(params={k: v.clone() for k, v in init.items()}, ema={k: v.clone() for k, v in init.items()},
                 memory=torch.from_numpy(base["init_memory"].copy()), index=0)
    for st in range(S):
        lr = 0.005 * om.warmup_linear(st / (2.0 * S), 0.1)        # train.py:411-416, epochs=2
        r = optim_oracle.train_step(state, _load_batch(base, st, "q"), _load_batch(base, st, "k"), optimizer=kind,
                                    num_layers=L, moco=True, T=0.07, lr=lr, dropout_key=int(base["key"]),
                                    step_index=st, **OPTIM[kind])
        assert np.isclose(r["loss"], z["losses"][st], rtol=2e-5), (st, r["loss"], z["losses"][st])
        coef = min(1.0, 1.0 / (r["grad_norm"] + 1e-6))
        assert np.isclose(r["grad_norm"] * coef, z["post_clip_gnorms"][st], rtol=1e-4)
        assert np.allclose(state["memory"].numpy(), z["s%d_memory" % st], atol=2e-6)
    assert state["index"] == int(z["final_index"]) and state["t"] == S
    # final weights, EMA weights and optimiser state at the sampled entries of every trained parameter
    trained = [k[4:] for k in z.files if k.startswith("idx/")]
    assert len(trained) == len(state["sgd_buf" if kind == "sgd" else "adagrad_sum"]) > 40
    biases = 0
    for n in trained:
        idx = z["idx/" + n]
        if kind == "adagrad" and _chaotic(n):
            continue
        # SGD moves the BatchNorm-fed biases by lr * (their ~1e-9 gradient), so they are compared like the rest
        biases += _chaotic(n)
        got = state["params"][n].reshape(-1).numpy()[idx]
        assert np.allclose(got, z["model/" + n], rtol=1e-3, atol=2e-5), (n, np.abs(got - z["model/" + n]).max())
        got = state["ema"][n].reshape(-1).numpy()[idx]
        assert np.allclose(got, z["ema/" + n], rtol=1e-4, atol=2e-6), n
        if kind == "sgd":
            got, want = state["sgd_buf"][n].reshape(-1).numpy()[idx], z["state/%s/momentum_buffer" % n]
        else:
            got, want = state["adagrad_sum"][n].reshape(-1).numpy()[idx], z["state/%s/sum" % n]
        assert np.allclose(got, want, rtol=2e-3, atol=2e-5 if kind == "sgd" else 1e-10), n
    assert biases == (2 * (L - 1) if kind == "sgd" else 0)
    # which parameters torch holds state for: SGD the trained ones; Adagrad every one (step 0, zero sum unused)
    live = [str(n) in trained for n in z["param_order"]]
    if kind == "sgd":
        assert list(z["state_present"]) == live
    else:
        assert z["state_present"].all()
        assert list(z["state_step"]) == [float(S) if x else 0.0 for x in live]
        assert all((m > 0) == x for m, x in zip(z["state_sum_absmax"], live))
