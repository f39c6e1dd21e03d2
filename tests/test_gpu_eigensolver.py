"""GPU: the eigensolver (gcc_b200/csrc/posenc.cu) against float64 on the structure set of tests/eig_structures.py --
every size class from the dense solver (n <= 96) to the L2 ChFSI class (n > 3584), whole graphs with components and
isolated vertices, multigraphs, degenerate spectra, hub-heavy dense graphs whose cluster slabs overflow the hub-row
list -- under the shipped dispatch and under GCCB200_DENSE_MAX=228, at pos_dim 2, 5, 16, 31 and 32; through explicit
batches and through the two producers (a node dataset's sampler on a multigraph, a graph dataset's
gccb_gather_graphs).  The checks are in tests/eig_checks.py.  Then placement invariance: a graph's output bits depend
on the graph alone -- not on its slot, view, batch composition, node_cap or, where its class stays, the dispatch.
Run with -s for the worst error / bound ratio per class and per check."""
import ctypes as C

import numpy as np
import pytest
import torch

import eig_checks as ec
import eig_structures as es
from test_gpu_parity import _fill_batch, _split

pytestmark = pytest.mark.gpu
POS_DIMS = (2, 5, 16, 31, 32)


@pytest.fixture(params=["default", "dense"])
def solver(request, monkeypatch):
    """gccb_posenc reads GCCB200_DENSE_MAX on every call: unset is the shipped dispatch, 228 sends every graph up
    to 228 vertices to the dense solver."""
    if request.param == "dense":
        monkeypatch.setenv("GCCB200_DENSE_MAX", "228")
    else:
        monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
    return request.param


@pytest.fixture(scope="module")
def structs():
    graphs = es.structures()
    return graphs, {g["name"]: ec.reference(g) for g in graphs}


def _batch(views, pos_dim, node_cap=None):
    from gcc_b200.datasets.graph_dataset import BatchBuffers
    B = len(views[0])
    assert len(views[1]) == B
    N = max(sum(g["n"] for g in v) for v in views)
    E = max(sum(g["m"] for g in v) for v in views)
    buf = BatchBuffers(B, node_cap or N + 8, E + 8, pos_dim, 64, "cuda")
    _fill_batch(buf, views)
    return buf


def _posenc(buf, pos_dim, normalize):
    """gccb_posenc on buffers prefilled with NaN: (pos, eigvals, kernel-side residual per slot, flags)."""
    from gcc_b200 import _lib
    buf.pos.fill_(float("nan"))
    buf.eigvals.fill_(float("nan"))
    buf.flags.zero_()
    _lib.check(_lib.get().gccb_posenc(C.byref(buf.c), pos_dim, normalize, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals),
                                      _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    it, res = buf.eig_debug()
    buf.last_iters = it.cpu().numpy()
    return buf.pos.cpu().numpy().copy(), buf.eigvals.cpu().numpy().copy(), res.cpu().numpy(), int(buf.flags.item())


def _noconv(buf, views, kres):
    """Graphs that ran all GCCB_CF_MAXIT = 8 outer iterations, with their last residual (the NOCONV candidates)."""
    return [(g["name"], float(kres[v * buf.B + gi])) for v in (0, 1) for gi, g in enumerate(views[v])
            if buf.last_iters[v * buf.B + gi] >= 8]


def _halves(graphs):
    """Both views of a batch: the graphs alternately, the shorter view padded with copies of the first graph."""
    a, b = graphs[0::2], graphs[1::2]
    b = b + a[:len(a) - len(b)]
    return [a, b]


def _outputs(buf, views, raw, eig):
    """{name: (rows bytes, eigenvalues bytes)} of every slot of the batch (the first occurrence of a name)."""
    noff = buf.node_off.cpu().numpy()
    out = {}
    for v in (0, 1):
        for gi, g in enumerate(views[v]):
            out.setdefault(g["name"], (raw[v, noff[v, gi]:noff[v, gi + 1]].tobytes(), eig[v * buf.B + gi].tobytes()))
    return out


@pytest.mark.parametrize("pos_dim", POS_DIMS)
def test_structures_match_float64(structs, solver, pos_dim):
    """Checks 1-5 of eig_checks on every graph of the set in one batch: normalize = 0 against float64, normalize = 1
    against the row-normalised normalize = 0 output of the same call, rows outside the batch untouched."""
    graphs, refs = structs
    views = _halves(graphs)
    buf = _batch(views, pos_dim)
    raw, eig, kres, flags = _posenc(buf, pos_dim, 0)
    assert flags == 0, (flags, _noconv(buf, views, kres))           # GCCB_FLAG_EIG_NOCONV among them
    nrm, eig1, _, flags1 = _posenc(buf, pos_dim, 1)
    assert flags1 == 0 and np.array_equal(eig, eig1)
    noff = buf.node_off.cpu().numpy()
    worst = {}
    for v in (0, 1):
        end = noff[v, buf.B]
        assert np.all(np.isfinite(raw[v, :end])) and np.all(np.isnan(raw[v, end:])), v
        assert np.all(np.isnan(nrm[v, end:])), v
        for gi, g in enumerate(views[v]):
            a, z = noff[v, gi], noff[v, gi + 1]
            cls = es.eig_class(g["n"], solver)
            w = worst.setdefault(cls, {})
            ec.check(g, refs[g["name"]], raw[v, a:z], eig[v * buf.B + gi], pos_dim, cls.startswith("dense"),
                     float(kres[v * buf.B + gi]), w)
            ec.check_normalized(g, raw[v, a:z], nrm[v, a:z], w)
    want = set(es.CLASS_ORDER) - ({"dense<=144", "dense<=228"} if solver == "default" else {"chfsi<=160"})
    assert set(worst) == want
    ec.report("eigensolver [%s], pos_dim %d: worst error / bound per class" % (solver, pos_dim),
              {c: worst[c] for c in es.CLASS_ORDER if c in worst})


def test_placement_invariance_per_class(structs, solver):
    """One representative per class and every hub-heavy graph: every slot of both views holds a copy; all 2B outputs
    are bit-identical to each other and to a B = 1 call.  The Philox start block depends on (entry, n) only, and
    the cluster kernel's hub-row list is the first 16 heavy rows in row order, so nothing else may matter."""
    graphs, _ = structs
    reps = es.representatives(graphs, solver)
    assert {es.eig_class(g["n"], solver) for g in reps} >= set(es.CLASS_ORDER) - {"dense<=144", "dense<=228",
                                                                                 "chfsi<=160"}
    assert sum(g["family"] == "hub_heavy" for g in reps) == 3
    for g in reps:
        B = 4 if g["n"] <= 1600 else 2
        buf = _batch([[g] * B, [g] * B], 32)
        raw, eig, _, flags = _posenc(buf, 32, 1)
        assert flags == 0, g["name"]
        n = g["n"]
        rows = [raw[v, i * n:(i + 1) * n].tobytes() for v in (0, 1) for i in range(B)]
        assert len(set(rows)) == 1 and len({eig[s].tobytes() for s in range(2 * B)}) == 1, g["name"]
        one = _batch([[g], [g]], 32)
        raw1, eig1, _, _ = _posenc(one, 32, 1)
        assert raw1[0, :n].tobytes() == rows[0] and raw1[1, :n].tobytes() == rows[0], g["name"]
        assert eig1[0].tobytes() == eig[0].tobytes(), g["name"]
    print("placement invariance [%s]: %s" % (solver, ", ".join("%s (%s)" % (g["name"], es.eig_class(g["n"], solver))
                                                              for g in reps)))


def test_other_composition_same_bits(structs, solver):
    """The whole set in a second batch -- reversed order, the other view, other slots, a larger node_cap -- gives the
    same bits for every graph."""
    graphs, _ = structs
    views = _halves(graphs)
    buf = _batch(views, 32)
    raw, eig, _, flags = _posenc(buf, 32, 0)
    first = _outputs(buf, views, raw, eig)
    rev = graphs[::-1]
    views2 = _halves(rev)[::-1]
    buf2 = _batch(views2, 32, node_cap=buf.node_cap + 1000)
    raw2, eig2, _, flags2 = _posenc(buf2, 32, 0)
    assert flags == 0 and flags2 == 0
    second = _outputs(buf2, views2, raw2, eig2)
    bad = [name for name in first if first[name] != second[name]]
    assert not bad, bad


def test_dense_max_keeps_the_other_classes(structs, monkeypatch):
    """Graphs whose class GCCB200_DENSE_MAX does not change (n <= 96 and n > 228) have the same bits under both
    settings."""
    graphs, _ = structs
    views = _halves(graphs)
    buf = _batch(views, 32)
    out = {}
    for setting in (None, "228"):
        if setting is None:
            monkeypatch.delenv("GCCB200_DENSE_MAX", raising=False)
        else:
            monkeypatch.setenv("GCCB200_DENSE_MAX", setting)
        raw, eig, _, flags = _posenc(buf, 32, 1)
        assert flags == 0
        out[setting] = _outputs(buf, views, raw, eig)
    same = [g["name"] for g in graphs if es.eig_class(g["n"]) == es.eig_class(g["n"], "dense")]
    assert len(same) > 30
    bad = [name for name in same if out[None][name] != out["228"][name]]
    assert not bad, bad


def _check_buffers(buf, subs, pos_dim, solver, refs_by_index, title):
    raw, eig, kres, flags = _posenc(buf, pos_dim, 0)
    assert flags == 0, flags
    noff = buf.node_off.cpu().numpy()
    worst = {}
    for v in (0, 1):
        for gi, s in enumerate(subs[v]):
            a, z = noff[v, gi], noff[v, gi + 1]
            cls = es.eig_class(s["n"], solver)
            ec.check(s, refs_by_index(v, gi, s), raw[v, a:z], eig[v * buf.B + gi], pos_dim, cls.startswith("dense"),
                     float(kres[v * buf.B + gi]), worst.setdefault(cls, {}))
    ec.report(title, {c: worst[c] for c in es.CLASS_ORDER if c in worst})
    return worst


@pytest.mark.parametrize("pos_dim", [16, 32])
def test_node_dataset_on_a_multigraph(structs, solver, pos_dim):
    """NodeClassificationDataset on the set's largest multigraph plus hubs: the sampler induces ego-nets with
    parallel edges and self loops and computes sub_deg itself; each ego-net against float64."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import NodeClassificationDataset
    graphs, _ = structs
    g = next(g for g in graphs if g["name"] == "multi_900")
    csr = synthetic.CSRGraph(g["indptr"].astype(np.int64), g["indices"], g["n"], g["name"])
    ds = NodeClassificationDataset(csr, rw_hops=256, positional_embedding_size=pos_dim, device="cuda", seed=3,
                                   batch_size=48)
    buf = ds.sample_batch(first_sample=0, posenc=False)
    torch.cuda.synchronize()
    buf.check_flags()
    subs = [_split(buf, v) for v in (0, 1)]
    for v in (0, 1):
        for gi, s in enumerate(subs[v]):
            s["name"] = "multi_900 ego %d/%d" % (v, gi)
            s["m"] = len(s["indices"])
    dup = sum(len(s["indices"]) - len(np.unique(np.repeat(np.arange(s["n"]), np.diff(s["indptr"])) * s["n"] +
                                                s["indices"])) for v in (0, 1) for s in subs[v])
    assert dup > 0                                                  # the ego-nets do hold parallel edges
    assert np.array_equal(buf.sub_deg[0, :int(buf.node_off[0, buf.B])].cpu().numpy(),
                          np.diff(buf.indptr[0, :int(buf.node_off[0, buf.B]) + 1].cpu().numpy()))
    _check_buffers(buf, subs, pos_dim, solver, lambda v, gi, s: ec.reference(s),
                   "node dataset on a multigraph [%s], pos_dim %d" % (solver, pos_dim))


@pytest.mark.parametrize("pos_dim", [5, 32])
def test_graph_dataset_whole_graphs(structs, solver, pos_dim):
    """GraphClassificationDataset over the set's whole graphs (components and isolated vertices, more than 48
    components, all isolated, cliques, dense ER, multigraphs): gccb_gather_graphs relabels each seed first; each
    relabelled graph against float64."""
    from gcc_b200.datasets import synthetic
    from gcc_b200.datasets.graph_dataset import GraphClassificationDataset
    graphs, _ = structs
    whole = [g for g in graphs if g["family"] in ("components", "many_components", "isolated", "cliques", "er_dense",
                                                   "multi") and g["n"] > 2]
    csrs = [synthetic.CSRGraph(g["indptr"].astype(np.int64), g["indices"], g["n"], g["name"]) for g in whole]
    B = len(whole)
    ds = GraphClassificationDataset(csrs, positional_embedding_size=pos_dim, device="cuda", batch_size=B)
    buf = ds.sample_batch(first_sample=0, posenc=False)
    torch.cuda.synchronize()
    subs = []
    for v in (0, 1):
        subs.append([])
        for gi in range(B):
            ip, ix = ds.items[gi]
            subs[v].append(dict(name=whole[gi]["name"], n=len(ip) - 1, m=len(ix), indptr=np.asarray(ip, np.int32),
                                indices=np.asarray(ix, np.int32)))
    got = _split(buf, 0)
    for gi in range(B):
        assert np.array_equal(got[gi]["indptr"], subs[0][gi]["indptr"]), gi
        assert np.array_equal(got[gi]["indices"], subs[0][gi]["indices"]), gi
    refs = [ec.reference(s) for s in subs[0]]
    _check_buffers(buf, subs, pos_dim, solver, lambda v, gi, s: refs[gi],
                   "graph dataset, whole graphs [%s], pos_dim %d" % (solver, pos_dim))
