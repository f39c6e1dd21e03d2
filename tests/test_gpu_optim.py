"""GPU (H100): the SGD and Adagrad optimisers (--optimizer sgd|adagrad, train.py:659-678) through the module
API, PretrainEngine and train.py, against the golden fixtures of the real reference, the CPU oracle step, the
float64 update formula and real torch.optim optimisers; and the default Adam step against its float64 formula."""
import os

import numpy as np
import pytest
import torch

from test_gpu_finetune import _two_class_graphs
from test_gpu_parity import _dataset, _golden_batch

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KINDS = ["sgd", "adagrad"]
HYPER = {"sgd": dict(momentum=0.9), "adagrad": dict(lr_decay=0.01)}


def _torch_opt(kind, params, lr=0.005):
    if kind == "sgd":
        return torch.optim.SGD(params, lr=lr, momentum=0.9, weight_decay=1e-5)
    return torch.optim.Adagrad(params, lr=lr, lr_decay=0.01, weight_decay=1e-5)


def _chaotic(name):
    # a bias feeding a train-mode BatchNorm has an exactly-zero true gradient; a sign-like first step (Adam,
    # Adagrad) moves it by +-lr on fp32 noise, in the reference too (see test_train_step_golden)
    return ("mlp.linears" in name and name.endswith("bias")) or (name.endswith("running_mean") and "apply_func" in name)


@pytest.mark.parametrize("kind", KINDS)
def test_module_api_vs_reference_golden(kind):
    """GraphEncoder + MemoryMoCo + NCESoftmaxLoss + torch.optim.SGD / Adagrad, wired like the reference's
    train_moco, reproduce train_moco_{sgd,adagrad}_golden.npz (the run of train_moco_golden.npz with the other
    optimiser): losses, queue at every step, final weights and EMA weights at the sampled entries."""
    from gcc_b200.contrastive.criterions import NCESoftmaxLoss
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.datasets.data_util import BatchedSubgraphs
    from gcc_b200.models import GraphEncoder
    from gcc_b200.utils.misc import warmup_linear
    base = np.load(os.path.join(G, "train_moco_golden.npz"))
    z = np.load(os.path.join(G, "train_moco_%s_golden.npz" % kind))
    L, H, S, K = int(base["num_layer"]), int(base["hidden"]), int(base["num_steps"]), int(base["K"])

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_node_freq=16, max_edge_freq=16, max_degree=512,
                            freq_embedding_size=16, degree_embedding_size=16, output_dim=H, node_hidden_dim=H,
                            edge_hidden_dim=H, num_layers=L, num_step_set2set=6, num_layer_set2set=3,
                            norm=True, gnn_model="gin", degree_input=True)

    model, model_ema = mk(), mk()
    init = {k[5:]: torch.from_numpy(base[k]) for k in base.files if k.startswith("init/")}
    model.load_state_dict(init)
    model_ema.load_state_dict(init)
    model, model_ema = model.cuda(), model_ema.cuda()
    model.dropout_key = int(base["key"])
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).cuda()
    contrast.memory.copy_(torch.from_numpy(base["init_memory"]))
    criterion = NCESoftmaxLoss()
    opt = _torch_opt(kind, model.parameters())
    model.train()
    model_ema.eval()
    for m in model_ema.modules():                          # train.py:360-365
        if m.__class__.__name__.find("BatchNorm") != -1:
            m.train()
    for st in range(S):
        buf = _golden_batch(base, st)
        gq, gk = BatchedSubgraphs(buf, 0), BatchedSubgraphs(buf, 1)
        feat_q = model(gq)
        with torch.no_grad():
            feat_k = model_ema(gk)
        out = contrast(feat_q, feat_k)
        opt.zero_grad()
        loss = criterion(out)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        for pg in opt.param_groups:
            pg["lr"] = 0.005 * warmup_linear(st / (2.0 * S), 0.1)
        opt.step()
        for p1, p2 in zip(model.parameters(), model_ema.parameters()):
            p2.data.mul_(0.999).add_(p1.detach().data, alpha=1 - 0.999)
        assert np.isclose(loss.item(), z["losses"][st], rtol=1e-3), (st, loss.item(), z["losses"][st])
        assert np.allclose(contrast.memory.cpu().numpy(), z["s%d_memory" % st], atol=5e-5)
    assert contrast.index == int(z["final_index"])
    params, ema_params = dict(model.named_parameters()), dict(model_ema.named_parameters())
    trained = [k[4:] for k in z.files if k.startswith("idx/")]
    assert len(trained) > 40
    for n in trained:
        if kind == "adagrad" and _chaotic(n):
            continue
        idx = torch.from_numpy(z["idx/" + n].astype(np.int64))
        got = params[n].detach().reshape(-1).cpu()[idx].numpy()
        assert np.allclose(got, z["model/" + n], rtol=2e-3, atol=5e-5), (n, np.abs(got - z["model/" + n]).max())
        got = ema_params[n].detach().reshape(-1).cpu()[idx].numpy()
        assert np.allclose(got, z["ema/" + n], rtol=2e-3, atol=5e-5), n


def _engine(kind, moco, H, L, B=16, K=64, prefetch=0, opt_kw=None, **ds_kw):
    from gcc_b200.contrastive.memory_moco import MemoryMoCo
    from gcc_b200.datasets import synthetic
    from gcc_b200.engine import PretrainEngine
    from gcc_b200.models import GraphEncoder
    torch.manual_seed(3)
    ds = _dataset(synthetic.chung_lu(5000, 40000, seed=4), B, 48, seed=9, **ds_kw)

    def mk():
        return GraphEncoder(positional_embedding_size=32, max_degree=512, degree_embedding_size=16, output_dim=H,
                            node_hidden_dim=H, num_layers=L, norm=True, gnn_model="gin", degree_input=True)

    model, ema = mk(), mk()
    ema.load_state_dict(model.state_dict())
    model, ema = model.cuda(), ema.cuda()
    contrast = MemoryMoCo(H, None, K, 0.07, use_softmax=True).cuda()
    eng = PretrainEngine(ds, model, ema, contrast, moco=moco, prefetch=prefetch, optimizer=kind,
                         **(HYPER[kind] if opt_kw is None else opt_kw))
    return eng, model, ema, contrast


def _view(buf, v, B):
    n, m = int(buf.node_off[v, B]), int(buf.edge_off[v, B])
    noff = buf.node_off[v].cpu().numpy().astype(np.int64)
    seed = np.zeros(n, np.int64)
    seed[noff[:B]] = 1
    return dict(indptr=buf.indptr[v, :n + 1].cpu().numpy().astype(np.int64),
                indices=buf.indices[v, :m].cpu().numpy().astype(np.int64),
                pos=buf.pos[v, :n].cpu().double().numpy(), seed=seed,
                sub_deg=buf.sub_deg[v, :n].cpu().numpy(), node_off=noff)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("moco,H,L", [(True, 64, 5), (False, 32, 2)], ids=["moco", "e2e"])
def test_engine_steps_match_oracle(kind, moco, H, L):
    """PretrainEngine(optimizer=kind) against optim_oracle.train_step over several steps on the same
    device-sampled batches.  Before every step the oracle starts from the engine's own state (weights, EMA,
    queue, optimiser buffers, step count), so each step is compared from equal inputs and the optimiser state
    carried between steps is part of what is checked."""
    import optim_oracle
    B = 16
    eng, model, ema, contrast = _engine(kind, moco, H, L, B=B)
    lr = 0.005
    for step in range(3):
        state = dict(params={k: v.detach().cpu().double().clone() for k, v in model.state_dict().items()},
                     ema={k: v.detach().cpu().double().clone() for k, v in ema.state_dict().items()},
                     memory=contrast.memory.detach().cpu().double().clone(), index=int(eng.index_dev.item()),
                     t=eng.adam_t)
        flat = eng.opt_state.cpu().double()
        state["sgd_buf" if kind == "sgd" else "adagrad_sum"] = {
            k: flat[o:o + int(np.prod(shape))].view(shape).clone() for k, (o, shape) in model._slices.items()}
        eng.step(lr=lr)
        s = eng.read_stats()
        buf = eng.cur_buf
        r = optim_oracle.train_step(state, _view(buf, 0, B), _view(buf, 1, B), optimizer=kind, num_layers=L,
                                    moco=moco, T=0.07, lr=lr, dropout_key=model.dropout_key, step_index=step,
                                    **HYPER[kind])
        assert np.isclose(s["loss"], r["loss"], rtol=1e-3), (step, s["loss"], r["loss"])
        assert np.isclose(s["grad_norm"], r["grad_norm"], rtol=2e-3), (step, s["grad_norm"], r["grad_norm"])
        clr = lr / (1 + step * HYPER[kind].get("lr_decay", 0.0))
        sd1 = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
        for k, v in state["params"].items():
            if k.endswith("num_batches_tracked") or k.endswith(".eps"):
                continue
            if kind == "sgd":
                atol = 1e-4 if "running" in k else 2e-5
                assert np.allclose(sd1[k], v.numpy(), rtol=1e-3, atol=atol), (step, k, np.abs(sd1[k] - v.numpy()).max())
            elif not _chaotic(k):
                # Adagrad's step d / sqrt(sum) is sign-like while sum is small: entries whose gradient is
                # eps-sized are ill-conditioned in the reference too; require agreement elsewhere
                diff = np.abs(sd1[k] - v.numpy())
                assert diff.max() <= 2 * clr + 1e-6, (step, k, diff.max())
                assert (diff > 5e-5).mean() < 0.02, (step, k, (diff > 5e-5).mean())
        if moco:
            assert np.allclose(contrast.memory.cpu().numpy(), state["memory"].numpy(), atol=1e-4)
            assert int(eng.index_dev.item()) == state["index"]
            sde = {k: v.detach().cpu().numpy() for k, v in ema.state_dict().items()}
            for k in model._slices:
                if not _chaotic(k):
                    assert np.allclose(sde[k], state["ema"][k].numpy(), rtol=1e-3, atol=2e-5), (step, k)
    assert eng.adam_t == 3


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("moco,H,L", [(True, 64, 5), (True, 256, 3), (False, 32, 2)], ids=["fp32", "wgmma", "e2e"])
def test_engine_update_matches_float64_formula(kind, moco, H, L):
    """The update the engine applies, checked against the float64 formula computed from its own gradient buffer
    and its pre-step weights, optimiser state and EMA: clip, L2 decay, SGD / Adagrad step, EMA over every entry
    (the unused set2set / lin_readout tail moves by the EMA only), at rtol 1e-5."""
    eng, model, ema, contrast = _engine(kind, moco, H, L, prefetch=4)
    assert bool(model.cfg.tensor_cores) == (H >= 128)
    n_live, n_all = model.n_live, model._n_all
    assert n_all > n_live
    lr = 0.005
    for step in range(4):
        torch.cuda.synchronize()
        p0 = model.flat_params[:n_all].double().cpu().numpy()
        e0 = ema.flat_params[:n_all].double().cpu().numpy()
        s0 = eng.opt_state.double().cpu().numpy()
        eng.step(lr=lr)
        s = eng.read_stats()
        g = eng.grads.double().cpu().numpy()
        total = np.sqrt((g ** 2).sum())
        assert np.isclose(s["grad_norm"], total, rtol=1e-5)
        d = min(1.0, 1.0 / (total + 1e-6)) * g + 1e-5 * p0[:n_live]
        if kind == "sgd":
            s1 = 0.9 * s0 + d
            p1_live = p0[:n_live] - lr * s1
        else:
            s1 = s0 + d * d
            p1_live = p0[:n_live] - lr / (1 + step * 0.01) * d / (np.sqrt(s1) + 1e-10)
        p1 = np.concatenate([p1_live, p0[n_live:]])
        got_p = model.flat_params[:n_all].double().cpu().numpy()
        assert np.allclose(eng.opt_state.double().cpu().numpy(), s1, rtol=1e-5, atol=1e-12 if kind == "adagrad"
                           else 1e-8), step
        assert np.allclose(got_p, p1, rtol=1e-5, atol=1e-7), (step, np.abs(got_p - p1).max())
        assert np.array_equal(got_p[n_live:], p0[n_live:])
        got_e = ema.flat_params[:n_all].double().cpu().numpy()
        if moco:
            assert np.allclose(got_e, 0.999 * e0 + 0.001 * p1, rtol=1e-5, atol=1e-7), step
        else:
            assert np.array_equal(got_e, e0)                 # E2E: no momentum encoder
    assert eng.adam_t == 4


@pytest.mark.parametrize("moco,H,L", [(True, 64, 5), (True, 256, 3)], ids=["fp32", "wgmma"])
def test_engine_adam_update_matches_float64_formula(moco, H, L):
    """The default optimiser: the Adam update the engine applies against the float64 formula computed from its own
    gradient buffer and its pre-step weights, adam_m, adam_v and EMA, with the step's lr and bias corrections read
    from `hyper` (which must hold lr, 1 - beta1^t and sqrt(1 - beta2^t) in fp32).  Each entry is held to a bound
    from the fp32 arithmetic of AdamRule: 16 U on the clipped, decayed gradient (the clip coefficient comes from a
    rounded norm), 8 U on each moment's terms, their propagation through m / (sqrt(v) / sbc2 + eps), 8 U on the step
    and on the weight."""
    U = 2.0 ** -24
    eng, model, ema, contrast = _engine("adam", moco, H, L, prefetch=4, opt_kw={})
    assert bool(model.cfg.tensor_cores) == (H >= 128)
    n_live, n_all = model.n_live, model._n_all
    lr = 0.005
    # the betas, eps and the EMA alpha as the kernel receives them (fp32); 1 - beta is exact in fp32 (Sterbenz)
    b1, b2, eps, alpha = (float(np.float32(x)) for x in (0.9, 0.999, 1e-8, 0.999))
    for step in range(4):
        torch.cuda.synchronize()
        p0 = model.flat_params[:n_all].double()
        e0 = ema.flat_params[:n_all].double()
        m0, v0 = eng.adam_m.double(), eng.adam_v.double()
        eng.step(lr=lr)
        s = eng.read_stats()
        torch.cuda.synchronize()
        t = step + 1
        hyper = eng.hyper.double().cpu().numpy()
        assert hyper[0] == np.float32(lr) and hyper[1] == np.float32(1 - 0.9 ** t)
        assert hyper[2] == np.float32(np.sqrt(1 - 0.999 ** t))
        lr_h, bc1, sbc2 = (float(x) for x in hyper[:3])
        g = eng.grads.double()
        total = float(torch.sqrt((g * g).sum()))
        assert np.isclose(s["grad_norm"], total, rtol=1e-5)
        coef = min(1.0, 1.0 / (total + 1e-6))
        pl = p0[:n_live]
        d = coef * g + 1e-5 * pl
        ad = coef * g.abs() + 1e-5 * pl.abs()
        err_d = 16 * U * ad
        m1 = b1 * m0 + (1 - b1) * d
        v1 = b2 * v0 + (1 - b2) * d * d
        err_m = (1 - b1) * err_d + 8 * U * (b1 * m0.abs() + (1 - b1) * ad)
        err_v = (1 - b2) * 2 * ad * err_d + 8 * U * (b2 * v0 + (1 - b2) * ad * ad)
        den = v1.sqrt() / sbc2 + eps
        stp = lr_h / bc1 * m1 / den
        rel_sqrt = torch.where(v1 > 0, err_v / (2 * v1), torch.zeros_like(v1))
        err_p = 8 * U * (pl.abs() + stp.abs()) + lr_h / bc1 * (err_m + m1.abs() * rel_sqrt) / den
        p1 = torch.cat([pl - stp, p0[n_live:]])
        got_m, got_v = eng.adam_m.double(), eng.adam_v.double()
        got_p = model.flat_params[:n_all].double()
        for name, got, want, bound in (("m", got_m, m1, err_m), ("v", got_v, v1, err_v),
                                       ("p", got_p[:n_live], p1[:n_live], err_p)):
            ratio = float(((got - want).abs() / (bound + 1e-30)).max())
            print("adam %s step %d %s: worst |err| / bound = %.3g" % ("fp32" if H < 128 else "wgmma", step, name,
                                                                      ratio))
            assert ratio <= 1.0, (step, name, ratio)
        assert torch.equal(got_p[n_live:], p0[n_live:])
        got_e = ema.flat_params[:n_all].double()
        want_e = alpha * e0 + (1 - alpha) * got_p
        assert ((got_e - want_e).abs() <= 4 * U * (alpha * e0.abs() + (1 - alpha) * got_p.abs()) + 1e-30).all(), step
    assert eng.adam_t == 4


@pytest.mark.parametrize("kind", KINDS)
def test_overflowed_batch_is_skipped_under_prefetch(kind):
    """An overflowed batch (published empty) under run-ahead leaves weights, optimiser state, EMA, queue and
    BatchNorm running statistics bit-identical, and read_stats() raises."""
    from gcc_b200 import _lib
    eng, model, ema, contrast = _engine(kind, True, 64, 3, prefetch=4, node_cap=100, edge_cap=100000)
    snap = [t.detach().clone() for t in (model.flat_params, ema.flat_params, contrast.memory, model._running,
                                          ema._running, eng.opt_state)]
    for _ in range(7):                                           # steps land on several ring slots
        eng.step(lr=0.005)
    torch.cuda.synchronize()
    now = (model.flat_params, ema.flat_params, contrast.memory, model._running, ema._running, eng.opt_state)
    for a, b in zip(snap, now):
        assert torch.equal(a, b)
    assert int(eng.index_dev.item()) == 0 and eng.adam_t == 7
    with pytest.raises(_lib.GccbError):
        eng.read_stats()


def _structure(sd):
    return ({i: {k: tuple(v.shape) for k, v in st.items()} for i, st in sd["state"].items()},
            [sorted(g) for g in sd["param_groups"]], [g["params"] for g in sd["param_groups"]])


@pytest.mark.parametrize("kind", KINDS)
def test_train_py_pretraining_checkpoint_holds_a_torch_optimizer_state(kind, tmp_path, monkeypatch):
    """train.py --moco --optimizer sgd|adagrad --max-steps 3 writes a checkpoint whose "optimizer" loads into
    the torch optimiser of that kind, has the structure of one stepped on the same module, and holds the
    engine's buffers."""
    import train
    from gcc_b200.engine import PretrainEngine
    engines = []

    class Capture(PretrainEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            engines.append(self)

    monkeypatch.setattr(train, "PretrainEngine", Capture)
    args = train.parse_option(["--moco", "--optimizer", kind, "--max-steps", "3", "--dataset", "synthetic-er",
                               "--graph-nodes", "2000", "--graph-edges", "10000", "--batch-size", "16",
                               "--num-workers", "1", "--num-copies", "1", "--num-samples", "64", "--epochs", "1",
                               "--nce-k", "64",
                               "--hidden-size", "64", "--num-layer", "3", "--rw-hops", "32", "--print-freq", "1000",
                               "--lr_decay_rate", "0.01", "--model-path", str(tmp_path / "m"),
                               "--tb-path", str(tmp_path / "tb")])
    train.main(args)
    (eng,) = engines
    assert eng.optimizer == kind and eng.adam_t == 3
    ckpt = torch.load(os.path.join(args.model_folder, "current.pth"), map_location="cpu", weights_only=False)
    saved = ckpt["optimizer"]
    model = train._make_encoder(args)
    real = train.make_optimizer(args, model.parameters())
    real.load_state_dict(saved)                              # loads into the torch optimiser of that kind
    # a real optimiser stepped on the same module, with gradients on the parameters the engine trains
    ref_model = train._make_encoder(args)
    ref = train.make_optimizer(args, ref_model.parameters())
    for n, p in ref_model.named_parameters():
        if n in eng.model._slices:
            p.grad = torch.ones_like(p)
    ref.step()
    assert _structure(saved) == _structure(ref.state_dict())
    assert saved["param_groups"][0]["weight_decay"] == args.weight_decay
    names = [n for n, _ in eng.model.named_parameters()]
    for i, n in enumerate(names):
        if n not in eng.model._slices:
            if kind == "adagrad":
                assert float(saved["state"][i]["step"]) == 0 and not saved["state"][i]["sum"].any()
            continue
        o, shape = eng.model._slices[n]
        want = eng.opt_state[o:o + int(np.prod(shape))].view(shape).cpu()
        if kind == "sgd":
            assert torch.equal(saved["state"][i]["momentum_buffer"], want), n
            assert saved["param_groups"][0]["momentum"] == 0.9
        else:
            assert torch.equal(saved["state"][i]["sum"], want) and float(saved["state"][i]["step"]) == 3, n
            assert saved["param_groups"][0]["lr_decay"] == 0.01


def test_sgd_without_momentum_has_no_state():
    """SGD with momentum 0 allocates no optimiser buffer, still trains, and saves no per-parameter state, like
    torch.optim.SGD(momentum=0)."""
    eng0, model, ema, contrast = _engine("sgd", True, 64, 3, opt_kw=dict(momentum=0.0))
    assert eng0.opt_state is None and eng0.adam_m is None and eng0.adam_v is None
    p0 = model.flat_params.clone()
    eng0.step(lr=0.005)
    s = eng0.read_stats()
    assert np.isfinite(s["loss"]) and not torch.equal(model.flat_params, p0)
    sd = eng0.optimizer_state_dict()
    assert sd["state"] == {} and sd["param_groups"][0]["momentum"] == 0.0
    torch.optim.SGD(model.parameters(), lr=0.005, momentum=0.0).load_state_dict(sd)


@pytest.mark.parametrize("kind", KINDS)
def test_finetune_uses_the_chosen_optimizer(kind, tmp_path):
    """train.py --finetune --optimizer sgd|adagrad runs an epoch and saves that optimiser's state_dict; the
    output layer keeps Adam (train.py:645-650)."""
    import train
    from gcc_b200.datasets.labeled import GraphClassificationDatasetLabeled
    graphs, labels = _two_class_graphs(60, seed=1)
    args = train.parse_option(["--finetune", "--optimizer", kind, "--epochs", "1", "--batch-size", "16",
                               "--hidden-size", "32", "--num-layer", "3", "--rw-hops", "32",
                               "--model-path", str(tmp_path / "m"), "--tb-path", str(tmp_path / "tb"),
                               "--dataset", "synthetic-graphs", "--gpu", "0", "--print-freq", "1000"])
    f1 = train.main_finetune(args, dataset=GraphClassificationDatasetLabeled((graphs, labels), batch_size=16))
    assert 0.0 <= f1 <= 1.0
    saved = torch.load(os.path.join(args.model_folder, "current.pth"), map_location="cpu", weights_only=False)
    model = train._make_encoder(args)
    want = train.make_optimizer(args, model.parameters())
    assert type(want).__name__ == {"sgd": "SGD", "adagrad": "Adagrad"}[kind]
    assert sorted(saved["optimizer"]["param_groups"][0]) == sorted(want.state_dict()["param_groups"][0])
    st = next(iter(saved["optimizer"]["state"].values()))
    assert set(st) == ({"momentum_buffer"} if kind == "sgd" else {"step", "sum"})
    want.load_state_dict(saved["optimizer"])
