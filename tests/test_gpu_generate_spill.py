"""GPU (H100): EmbedEngine re-runs a batch that overflows the default capacity on buffers sized from its measured
ego-nets.  The reference for every row is the same engine on a dataset given a capacity large enough that nothing
overflows: the ordinary path.  GAT rows must match bit for bit; GIN rows to 1e-6 of their norm, because GIN's sum
pooling rounds by an ego-net's position in its batch (test_gpu_generate.py, DESIGN §5e) and a re-run batch is cut
into groups."""
import argparse
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WALK_BUDGET_MAX = 32768 - 64
KINDS = {"gin64": ("gin", 64), "gin128": ("gin", 128), "gat64": ("gat", 64)}
GIN_TOL = 1e-6


def _opt(kind, folder=".", rw_hops=64):
    gnn, H = KINDS[kind]
    return argparse.Namespace(positional_embedding_size=32, max_node_freq=8, max_edge_freq=8, max_degree=512,
                              freq_embedding_size=16, degree_embedding_size=16, hidden_size=H, num_layer=5,
                              set2set_iter=6, set2set_lstm_layer=3, model=gnn, norm=True, rw_hops=rw_hops,
                              subgraph_size=128, restart_prob=0.8, seed=5, model_folder=str(folder))


def _model(kind):
    import generate
    from gcc_b200.models import GraphEncoder
    opt = _opt(kind)
    torch.manual_seed(1)
    enc = GraphEncoder(degree_input=True, **{kw: getattr(opt, a) for kw, a in generate.ENCODER_KWARGS.items()})
    return enc.cuda().eval()


def _dataset(g, B, rw_hops=64, **kw):
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    return NodeClassificationDataset(dataset=g, rw_hops=rw_hops, subgraph_size=128, restart_prob=0.8,
                                     positional_embedding_size=32, device="cuda", seed=5, batch_size=B, **kw)


def _roomy(g, B, node_cap, edge_cap, rw_hops=64):
    """The reference: a dataset given a capacity that the test's batches fit (it raises if one does not)."""
    return _dataset(g, B, rw_hops, node_cap=node_cap, edge_cap=edge_cap)


def _powerlaw():
    """Chung-Lu, w_i ~ (i+1)^-0.5: its hubs are the lowest ids, so the first batch of 64 holds 64 consecutive hubs
    (ego-nets of up to ~1,900 vertices, ~36k vertices and ~720k edge slots per view against a default capacity of
    24,181 and 386,896); later batches fit.  Its largest walk budget, 3,637, keeps the sampler's shared-memory key
    array at 16 KB (DESIGN §9)."""
    from gcc_b200.datasets import synthetic
    return synthetic.chung_lu(6000, 190_000, exponent=0.5, seed=11)


def _same_bytes(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _assert_rows_match(kind, got, want, what):
    assert np.isfinite(want).all() and np.isfinite(got).all()
    err = float((np.abs(got - want).max(axis=1) / np.linalg.norm(want, axis=1)).max())
    print("%s %s: bitwise %s, max |diff| / |row| = %.3g" % (what, kind, _same_bytes(got, want), err))
    if KINDS[kind][0] == "gat":
        assert _same_bytes(got, want), (what, err)
    else:
        assert err <= GIN_TOL, (what, err)


def _flags_of_batch(ds, nodes):
    """The flag word of sampling `nodes` once into the dataset's own buffers (cleared afterwards)."""
    from gcc_b200.datasets.graph_dataset import sample_pairs
    buf = ds.buffers.narrow(len(nodes)) if len(nodes) < ds.buffers.B else ds.buffers
    buf.seeds.copy_(torch.as_tensor(nodes, dtype=torch.int64, device="cuda"))
    sample_pairs(ds, buf, None, buf.seeds, sample_ids=buf.seeds)
    f = int(buf.flags.item())
    buf.flags.zero_()
    return f


@pytest.mark.parametrize("kind", list(KINDS))
def test_overflowing_hub_batches_are_replanned_and_match_the_roomy_reference(kind):
    from gcc_b200 import _capi
    from gcc_b200.embed import EmbedEngine
    g, B = _powerlaw(), 64
    nodes = range(0, 10 * B + 17)                               # the hub batch, nine that fit, a short last one
    ds, ref = _dataset(g, B), _roomy(g, B, 300_000, 8_000_000)
    assert not ds.caps_given and ref.caps_given
    assert _flags_of_batch(ds, np.arange(B)) & (_capi.FLAG_NODE_OVERFLOW | _capi.FLAG_EDGE_OVERFLOW)
    model = _model(kind)
    want = EmbedEngine(ref, model, prefetch=4).run(nodes)
    for prefetch in (0, 4):
        eng = EmbedEngine(ds, model, prefetch=prefetch)
        got = eng.run(nodes)
        assert eng.replanned >= 1 and eng.largest_egonet[0] > 320
        _assert_rows_match(kind, got, want, "prefetch %d" % prefetch)
        assert eng._spill is None and eng._spill_big is None     # freed when run() returns
        # the ids in another order and with repeats: the same batches spill or not by their nodes alone
        ids = np.concatenate([np.arange(40, 0, -1), np.arange(200, 260), [3, 3, 7]])
        _assert_rows_match(kind, eng.run(ids), want[ids], "ids prefetch %d" % prefetch)


def test_an_edge_only_overflow_is_replanned():
    """Nodes 0..127 are a 128-clique: at B = 128 and rw_hops 256 its batch holds ~16k vertices (the default node_cap
    is 41,280) and ~2.1M edge slots (edge_cap 660,480).  Nodes 128.. are a sparse graph whose batches fit."""
    from gcc_b200 import _capi
    from gcc_b200.datasets import synthetic
    from gcc_b200.embed import EmbedEngine
    er = synthetic.erdos_renyi(700, 2800, seed=2)
    iu, ju = np.triu_indices(128, 1)
    src = np.concatenate([iu, np.repeat(np.arange(700), np.diff(er.indptr)) + 128])
    dst = np.concatenate([ju, er.indices.astype(np.int64) + 128])
    g = synthetic.from_pairs(src, dst, 828, "clique+er")
    B = 128
    ds, ref = _dataset(g, B, 256), _roomy(g, B, 41_280, 4_000_000, 256)
    assert (ds.node_cap, ds.edge_cap) == (41_280, 660_480)
    assert _flags_of_batch(ds, np.arange(B)) == _capi.FLAG_EDGE_OVERFLOW
    for kind in KINDS:
        model = _model(kind)
        want = EmbedEngine(ref, model, prefetch=4).run(range(g.num_nodes))
        for prefetch in (0, 4):
            eng = EmbedEngine(ds, model, prefetch=prefetch)
            got = eng.run(range(g.num_nodes))
            assert eng.replanned == 1 and eng.largest_egonet[0] <= 128
            _assert_rows_match(kind, got, want, "edge-only prefetch %d" % prefetch)


def _wide_hub():
    """Vertex 0 joined to 20,000 others that form a random graph of average degree 100: its plain-degree walk budget
    (39,549) takes the sampler's wide path, and its ego-net (~17,300 vertices, ~1.5M edge slots) does not fit the
    default edge capacity at B = 64 (961,488) on its own."""
    from gcc_b200.datasets import synthetic
    H = 20_000
    er = synthetic.erdos_renyi(H, 1_000_000, seed=3)
    src = np.repeat(np.arange(H, dtype=np.int64), np.diff(er.indptr)) + 1
    dst = er.indices.astype(np.int64) + 1
    hub = np.arange(1, H + 1, dtype=np.int64)
    return synthetic.from_pairs(np.concatenate([src, np.zeros_like(hub)]), np.concatenate([dst, hub]), H + 1, "hub")


def test_a_wide_egonet_above_the_default_capacity_is_embedded_alone():
    from gcc_b200.embed import EmbedEngine
    g, B = _wide_hub(), 64
    ds, ref = _dataset(g, B), _roomy(g, B, 120_000, 4_000_000)
    assert ds.graph.max_budget > WALK_BUDGET_MAX
    nodes = range(0, 2 * B)
    for kind in ("gat64", "gin64"):
        model = _model(kind)
        want = EmbedEngine(ref, model, prefetch=0).run(nodes)
        eng = EmbedEngine(ds, model, prefetch=4)
        got = eng.run(nodes)
        n, m = eng.largest_egonet
        print("hub ego-net: %d vertices, %d edge slots; default capacity %d / %d" % (n, m, ds.node_cap, ds.edge_cap))
        assert eng.replanned == 1 and m > ds.edge_cap
        _assert_rows_match(kind, got[:1], want[:1], "hub row")
        _assert_rows_match(kind, got, want, "hub batches")


def _ckpt(tmp_path, kind):
    path = str(tmp_path / ("%s.pth" % kind))
    torch.save({"opt": _opt(kind, tmp_path), "model": _model(kind).cpu().state_dict(), "epoch": 1}, path)
    return path


def _main(ckpt, dataset, gpu, B=64, **kw):
    import generate
    return generate.main(types.SimpleNamespace(load_path=ckpt, dataset=dataset, graph_nodes=0, graph_edges=0,
                                               batch_size=B, gpu=gpu, **kw))


@pytest.mark.parametrize("kind", ["gin64", "gat64"])
def test_generate_at_the_defaults_shards_and_subsets_agree(tmp_path, capsys, kind):
    g = _powerlaw()
    npz, out = str(tmp_path / "pl.npz"), str(tmp_path / "pl.npy")
    np.savez(npz, indptr=g.indptr, indices=g.indices)
    ckpt = _ckpt(tmp_path, kind)
    line = lambda: [s for s in capsys.readouterr().out.splitlines() if s.startswith("re-planned")]
    _main(ckpt, npz, [0])
    printed = line()
    assert len(printed) == 1 and "re-planned 0 of" not in printed[0] and "largest ego-net met" in printed[0]
    one = np.load(out).copy()
    _main(ckpt, npz, [0, 0])
    assert _same_bytes(np.load(out), one)
    assert line() == printed                                    # the shards re-plan the batches one run re-plans
    ids = np.random.RandomState(2).randint(0, g.num_nodes, size=300)
    ids[:70] = np.arange(70)[::-1]                              # hubs, in another order and other batches
    (tmp_path / "ids.txt").write_text("\n".join(map(str, ids)) + "\n")
    for gpu in ([0], [0, 0]):
        _main(ckpt, npz, gpu, nodes=str(tmp_path / "ids.txt"))
        _assert_rows_match(kind, np.load(out), one[ids], "--nodes on %s" % gpu)
