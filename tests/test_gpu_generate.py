"""GPU (H100): generate.py's node export on EmbedEngine -- the run-ahead ring against the serial loop byte for byte
(GIN hidden 64 and 128, GAT, a short last batch, a hub above the shared-memory walk budget, a multigraph), shards
against one run, `--nodes` subsets against the full run, no host sync per batch, the bounded staging ring, the
failure paths and `.bin` input."""
import argparse
import multiprocessing
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WALK_BUDGET_MAX = 32768 - 64
KINDS = {"gin64": ("gin", 64), "gin128": ("gin", 128), "gat64": ("gat", 64)}


def _opt(kind, folder="."):
    gnn, H = KINDS[kind]
    return argparse.Namespace(positional_embedding_size=32, max_node_freq=8, max_edge_freq=8, max_degree=512,
                              freq_embedding_size=16, degree_embedding_size=16, hidden_size=H, num_layer=5,
                              set2set_iter=6, set2set_lstm_layer=3, model=gnn, norm=True, rw_hops=64,
                              subgraph_size=128, restart_prob=0.8, seed=5, model_folder=str(folder))


def _model(kind):
    import generate
    from gcc_b200.models import GraphEncoder
    opt = _opt(kind)
    torch.manual_seed(1)
    return GraphEncoder(degree_input=True, **{kw: getattr(opt, a) for kw, a in generate.ENCODER_KWARGS.items()})


def _ckpt(tmp_path, kind):
    path = str(tmp_path / ("%s.pth" % kind))
    torch.save({"opt": _opt(kind, tmp_path), "model": _model(kind).state_dict(), "epoch": 1}, path)
    return path


def _dataset(g, B, **kw):
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    return NodeClassificationDataset(dataset=g, rw_hops=64, subgraph_size=128, restart_prob=0.8,
                                     positional_embedding_size=32, device="cuda", seed=5, batch_size=B, **kw)


def _er():
    from gcc_b200.datasets import synthetic
    return synthetic.erdos_renyi(1000, 5000, seed=3)


def _hub():
    """Vertex 0 joined to 17,000 others (plain-degree walk budget about 33,600, above the shared-memory budget),
    beside a Chung-Lu graph on them."""
    from gcc_b200.datasets import synthetic
    g = synthetic.chung_lu(17000, 50000, exponent=0.5, seed=4)
    src = np.repeat(np.arange(g.num_nodes, dtype=np.int64), np.diff(g.indptr)) + 1
    dst = g.indices.astype(np.int64) + 1
    hub = np.arange(1, 17001, dtype=np.int64)
    return synthetic.from_pairs(np.concatenate([src, np.zeros_like(hub)]), np.concatenate([dst, hub]), 17001, "hub")


def _multigraph():
    """Two hubs joined to 500 leaves by 1..5 parallel edges each, a sparse leaf layer and a self loop."""
    from gcc_b200.datasets import downstream
    rng = np.random.RandomState(7)
    src, dst = [], []
    for h in (0, 1):
        for leaf in range(2, 502):
            t = int(rng.randint(1, 6))
            src += [h] * t
            dst += [leaf] * t
    e = rng.randint(2, 502, size=(800, 2))
    src += e[:, 0].tolist() + [0]
    dst += e[:, 1].tolist() + [0]
    return downstream.multigraph_from_edge_index(np.array([src, dst]), "multi")


def _same_bytes(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


CASES = [("er", "gin64", 64), ("er", "gin128", 64), ("er", "gat64", 64), ("hub", "gin64", 256),
         ("multi", "gin64", 64), ("multi", "gat64", 64)]


@pytest.mark.parametrize("graph,kind,B", CASES)
def test_run_ahead_equals_the_serial_loop_byte_for_byte(graph, kind, B):
    import generate
    from gcc_b200.embed import EmbedEngine
    g = {"er": _er, "hub": _hub, "multi": _multigraph}[graph]()
    assert g.num_nodes % B != 0                                  # a short last batch
    ds = _dataset(g, B)
    if graph == "hub":
        assert ds.graph.max_budget > WALK_BUDGET_MAX
    model = _model(kind).cuda().eval()
    want = generate.test_moco(ds, model, argparse.Namespace(hidden_size=KINDS[kind][1])).numpy()
    assert want.shape == (g.num_nodes, KINDS[kind][1]) and np.isfinite(want).all()
    for prefetch in (0, 1, 4):
        got = EmbedEngine(ds, model, prefetch=prefetch).run(range(g.num_nodes))
        assert _same_bytes(got, want), (prefetch, float(np.abs(got - want).max()))


@pytest.mark.parametrize("kind", list(KINDS))
def test_subset_rows_equal_the_same_rows_of_the_full_run(kind):
    """A row does not depend on which other nodes are requested, up to the order of a float sum.  GAT rows are equal
    byte for byte: every stage is per row or, for Set2Set, one CTA per ego-net indexed from the ego-net's first row.
    GIN rows are held to 1e-6 of their norm: gccb_gin_forward's sum pooling adds each ego-net's rows in fp32 runs
    cut at the batch's fixed 16-row tiles (gin_fwd.cu, pool_acc), so where an ego-net starts relative to a tile --
    which the ego-nets before it in the batch decide -- changes the rounding of its pooled sum."""
    from gcc_b200.embed import EmbedEngine
    g = _er()
    ds = _dataset(g, 64)
    model = _model(kind).cuda().eval()
    eng = EmbedEngine(ds, model, prefetch=4)
    full = eng.run(range(g.num_nodes)).copy()
    rng = np.random.RandomState(0)
    ids = rng.randint(0, g.num_nodes, size=300)                  # shuffled, with repeats
    ids[:5] = ids[5]                                             # one node six times, at different tile offsets
    sub = eng.run(ids)
    want = full[ids]
    err = np.abs(sub - want).max(axis=1) / np.linalg.norm(want, axis=1)
    print("%s: subset rows bitwise equal: %s, max |diff| / |row| = %.3g" % (kind, _same_bytes(sub, want), err.max()))
    if KINDS[kind][0] == "gat":
        assert _same_bytes(sub, want)
    else:
        assert err.max() <= 1e-6


def test_no_host_sync_per_batch_and_the_staging_ring_is_bounded():
    from gcc_b200.embed import EmbedEngine
    g = _er()
    B, S = 64, 4
    ds = _dataset(g, B)
    model = _model("gin64").cuda().eval()
    eng = EmbedEngine(ds, model, prefetch=S)
    ids = np.arange(g.num_nodes)[::-1].copy()
    torch.cuda.synchronize()
    n_b = -(-g.num_nodes // B)
    assert n_b >= 8
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = eng.run(range(g.num_nodes))
        assert eng.host_waits == n_b                             # one slot event per batch, nothing else
        b = eng.run(ids)
        assert eng.host_waits == n_b
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _same_bytes(b, a[ids]) or np.abs(b - a[ids]).max() <= 1e-6
    staging = [t for t in vars(eng).values() if torch.is_tensor(t) and not t.is_cuda]
    assert sum(t.numel() for t in staging if t.is_floating_point()) <= (S + 1) * B * model.cfg.hidden
    assert all(t.is_pinned() for t in staging)


@pytest.mark.parametrize("prefetch", [0, 4])
def test_an_overflowing_batch_raises_naming_its_nodes(prefetch):
    """Nodes 0..191 are 96 separate edges (ego-nets of 2 vertices), nodes 192..255 a 64-clique: with room for 1,000
    vertices per view, only the fourth batch of 64 overflows."""
    from gcc_b200 import _lib
    from gcc_b200.datasets import synthetic
    from gcc_b200.embed import EmbedEngine
    src = list(range(0, 192, 2))
    dst = list(range(1, 192, 2))
    for u in range(192, 256):
        for v in range(u + 1, 256):
            src.append(u)
            dst.append(v)
    g = synthetic.from_pairs(np.array(src), np.array(dst), 256, "matching+clique")
    ds = _dataset(g, 64, node_cap=1000)
    eng = EmbedEngine(ds, _model("gin64").cuda().eval(), prefetch=prefetch)
    with pytest.raises(_lib.GccbError, match=r"nodes 192\.\.255"):
        eng.run(range(256))
    torch.cuda.synchronize()
    rows = EmbedEngine(ds, _model("gin64").cuda().eval(), prefetch=prefetch).run(range(192))
    assert np.isfinite(rows).all()                               # the batches that fit


def _save_npz(path, g, sizes=None):
    kw = {} if sizes is None else {"graph_sizes": np.array(sizes, dtype=np.int64)}
    np.savez(path, indptr=g.indptr, indices=g.indices, **kw)


def _main(ckpt, dataset, gpu, B=64, **kw):
    import generate
    return generate.main(types.SimpleNamespace(load_path=ckpt, dataset=dataset, graph_nodes=0, graph_edges=0,
                                               batch_size=B, gpu=gpu, **kw))


def test_shards_write_the_file_one_run_writes(tmp_path):
    ckpt = _ckpt(tmp_path, "gin64")
    g = _er()
    _save_npz(str(tmp_path / "er.npz"), g)
    out = str(tmp_path / "er.npy")
    one = _main(ckpt, str(tmp_path / "er.npz"), [0])
    assert tuple(one.shape) == (g.num_nodes, 64)
    want = np.load(out).copy()
    os.remove(out)
    _main(ckpt, str(tmp_path / "er.npz"), [0, 0, 0])                # 16 batches: 6 + 5 + 5, the last one short
    assert multiprocessing.active_children() == []
    got = np.load(out, mmap_mode="r")
    assert isinstance(got, np.memmap) and got.dtype == np.float32
    assert _same_bytes(got, want)
    os.remove(out)
    _main(ckpt, str(tmp_path / "er.npz"), [0, 0], prefetch=0)       # the serial loop, sharded
    assert _same_bytes(np.load(out), want)


def test_nodes_file_writes_those_rows_in_its_order(tmp_path):
    ckpt = _ckpt(tmp_path, "gat64")
    g = _er()
    _save_npz(str(tmp_path / "er.npz"), g)
    _main(ckpt, str(tmp_path / "er.npz"), 0)
    full = np.load(str(tmp_path / "er.npy"))
    ids = np.random.RandomState(1).randint(0, g.num_nodes, size=150)
    (tmp_path / "ids.txt").write_text("\n".join(map(str, ids)) + "\n")
    for gpu in ([0], [0, 0]):
        _main(ckpt, str(tmp_path / "er.npz"), gpu, nodes=str(tmp_path / "ids.txt"))
        assert _same_bytes(np.load(str(tmp_path / "er.npy")), full[ids])     # GAT rows: see the subset test


def test_a_failing_shard_fails_the_command_and_leaves_nothing_behind(tmp_path):
    """The second shard names a device that does not exist: a host-side argument error in that worker."""
    ckpt = _ckpt(tmp_path, "gin64")
    _save_npz(str(tmp_path / "er.npz"), _er())
    with pytest.raises(RuntimeError, match="shard 1"):
        _main(ckpt, str(tmp_path / "er.npz"), [0, torch.cuda.device_count(), 0])
    assert not os.path.exists(str(tmp_path / "er.npy"))
    assert multiprocessing.active_children() == []


def test_bin_corpus_embeds_like_the_equivalent_npz(tmp_path):
    from gcc_b200.datasets import dgl_bin, synthetic
    ckpt = _ckpt(tmp_path, "gin64")
    graphs = [synthetic.erdos_renyi(600, 3000, seed=1), synthetic.erdos_renyi(400, 2000, seed=2)]
    dgl_bin.write_dgl_bin(str(tmp_path / "two.bin"), graphs)
    _save_npz(str(tmp_path / "two_u.npz"), synthetic.disjoint_union(graphs), [600, 400])
    _main(ckpt, str(tmp_path / "two.bin"), 0)
    _main(ckpt, str(tmp_path / "two_u.npz"), 0)
    a, b = np.load(str(tmp_path / "two.npy")), np.load(str(tmp_path / "two_u.npy"))
    assert a.shape == (1000, 64) and _same_bytes(a, b)
