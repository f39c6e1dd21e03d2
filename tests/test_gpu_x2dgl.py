"""GPU: the corpus builder (datasets/x2dgl.py, csrc/edgelist.cu) against the reference's own x2dgl run
(tests/golden/x2dgl_golden.npz) and the host path (numpy parse + synthetic.from_pairs) on ~10M-line files of both
formats; the written corpus read back and trained on; and the device generators after their cleaning moved into
synthetic.from_keys_device, against a copy of the inline sequence they had."""
import os

import numpy as np
import pytest
import torch

import x2dgl_oracle as oracle
from gcc_b200 import _lib
from gcc_b200.datasets import dgl_bin, synthetic, x2dgl
from gcc_b200.datasets.graph_dataset import load_graphs

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "x2dgl_golden.npz")


def _same(g, indptr, indices):
    np.testing.assert_array_equal(g.indptr.cpu().numpy(), indptr)
    np.testing.assert_array_equal(g.indices.cpu().numpy(), indices)
    assert g.indices.dtype == torch.int32 and g.num_nodes == len(indptr) - 1


@pytest.fixture(scope="module")
def kdd17(tmp_path_factory):
    z = np.load(GOLDEN)
    d = tmp_path_factory.mktemp("kdd17")
    for k in z.files:
        if k.startswith("text_"):
            (d / k[5:]).write_bytes(z[k].tobytes())
    return z, d


def test_build_graph_equals_reference_x2dgl(kdd17):
    z, d = kdd17
    for i in range(int(z["count"])):
        for chunk in (x2dgl.DEFAULT_CHUNK, 64):
            _same(x2dgl.build_graph(d / z["file%d" % i].item(), chunk_bytes=chunk), z["indptr%d" % i],
                  z["indices%d" % i])


def test_cli_writes_the_reference_corpus(kdd17, tmp_path):
    z, d = kdd17
    out = str(tmp_path / "small.bin")
    x2dgl.main(["--graph-dir", str(d), "--save-file", out])
    graphs, labels = dgl_bin.read_dgl_bin(out)
    np.testing.assert_array_equal(labels["graph_sizes"], z["graph_sizes"])
    for i, g in enumerate(graphs):
        np.testing.assert_array_equal(g.indptr, z["indptr%d" % i])
        np.testing.assert_array_equal(g.indices, z["indices%d" % i])


def _write_big(tmp, rng, n, m):
    """A seeded ~m-line .lscc file and the plain edge list of the same edges (self loops and duplicates kept)."""
    w = (np.arange(n) + 1.0) ** -0.5
    cdf = np.cumsum(w) / w.sum()
    u = np.minimum(np.searchsorted(cdf, rng.random(m), side="right"), n - 1)
    v = np.minimum(np.searchsorted(cdf, rng.random(m), side="right"), n - 1)
    edges = "\n".join("%d %d" % e for e in zip(u.tolist(), v.tolist()))
    lscc, plain = tmp / "big.lscc", tmp / "big.txt"
    with open(lscc, "w") as f:
        f.write("n %d\n" % n)
        f.write("\n".join("%d %d" % (i, i) for i in range(n)))
        f.write("\nm %d\n" % m)
        f.write(" 1\n".join(edges.split("\n")) + " 1\n")
    with open(plain, "w") as f:
        f.write("# seeded Chung-Lu test graph\n" + edges + "\n")
    return lscc, plain


def test_ten_million_lines_equal_host_path(tmp_path):
    lscc, plain = _write_big(tmp_path, np.random.default_rng(7), 1_000_000, 10_000_000)
    for path in (lscc, plain):
        ref = oracle.host_build(path)
        for chunk in (x2dgl.DEFAULT_CHUNK, 64 << 10):
            a = x2dgl.build_graph(path, chunk_bytes=chunk)
            _same(a, ref.indptr, ref.indices)
            b = x2dgl.build_graph(path, chunk_bytes=chunk)
            assert torch.equal(a.indptr, b.indptr) and torch.equal(a.indices, b.indices)


def test_errors_name_file_and_line(tmp_path):
    p = tmp_path / "bad.lscc"
    p.write_bytes(b"n 3\n0\n1\n2\nm 2\n0 1 1\n1 7 1\n")
    with pytest.raises(_lib.GccbError, match=r"bad\.lscc:7: vertex id out of range"):
        x2dgl.build_graph(p)
    p = tmp_path / "long.txt"
    p.write_bytes(b"0 1\n" * 40 + b"1" * 100 + b" 2\n")
    with pytest.raises(_lib.GccbError, match=r"long\.txt:41: line longer than the 64-byte staging chunk"):
        x2dgl.build_graph(p, chunk_bytes=64)


def test_corpus_reads_back_and_trains(kdd17, tmp_path, monkeypatch):
    z, d = kdd17
    rng = np.random.default_rng(11)
    extra = tmp_path / "extra.txt"
    src, dst = rng.integers(0, 500, 4000), rng.integers(0, 500, 4000)
    extra.write_text("% comment\n" + "".join("%d\t%d\n" % e for e in zip(src, dst)))
    files = [d / z["file%d" % i].item() for i in range(int(z["count"]))] + [extra]
    out = str(tmp_path / "corpus.bin")
    x2dgl.main(["--graph-dir", str(d), "--save-file", out, "--embed-dim", "64", "--graph-files", str(extra)])
    union, sizes = load_graphs(out)
    built = [x2dgl.build_graph(f) for f in files]
    built = [synthetic.CSRGraph(g.indptr.cpu().numpy(), g.indices.cpu().numpy(), g.num_nodes, g.name) for g in built]
    built.sort(key=lambda g: g.num_nodes, reverse=True)
    ref = synthetic.disjoint_union(built)
    assert sizes == [g.num_nodes for g in built]
    np.testing.assert_array_equal(union.indptr, ref.indptr)
    np.testing.assert_array_equal(union.indices, ref.indices)

    import train
    monkeypatch.chdir(tmp_path)
    args = train.parse_option(["--moco", "--dataset", out, "--max-steps", "2", "--batch-size", "16", "--nce-k", "64",
                               "--num-workers", "1", "--num-copies", "1", "--num-samples", "64", "--epochs", "1",
                               "--model-path", str(tmp_path / "m"), "--tb-path", str(tmp_path / "tb")])
    train.main(args)
    assert os.path.exists(os.path.join(args.model_folder, "current.pth"))


# ---- the device generators: the inline cleaning they had, kept here as the reference ----------------------------
def _old_chung_lu_device(n, n_pairs, exponent=0.5, seed=0, device="cuda"):
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    w = (torch.arange(n, device=device, dtype=torch.float64) + 1.0) ** (-exponent)
    cdf = torch.cumsum(w, 0)
    cdf = cdf / cdf[-1]
    keys = []
    left, chunk = n_pairs, 1 << 24
    while left > 0:
        c = min(left, chunk)
        src = torch.searchsorted(cdf, torch.rand(c, generator=gen, device=device, dtype=torch.float64), right=True).clamp_(max=n - 1)
        dst = torch.searchsorted(cdf, torch.rand(c, generator=gen, device=device, dtype=torch.float64), right=True).clamp_(max=n - 1)
        keep = src != dst
        src, dst = src[keep], dst[keep]
        keys.append(src * n + dst)
        keys.append(dst * n + src)
        left -= c
    key = torch.unique(torch.cat(keys), sorted=True)
    del keys
    s, d = key // n, key % n
    deg = torch.bincount(s, minlength=n)
    alive = deg > 0
    n2 = int(alive.sum())
    if n2 != n:
        remap = torch.cumsum(alive.long(), 0) - 1
        d = remap[d]
        deg = deg[alive]
    indptr = torch.zeros(n2 + 1, dtype=torch.int64, device=device)
    torch.cumsum(deg, 0, out=indptr[1:])
    return synthetic.CSRGraph(indptr, d.to(torch.int32), n2, "chunglu_dev_n%d_p%d" % (n, n_pairs))


def _old_rmat_device(scale, n_pairs, abcd=(0.57, 0.19, 0.19, 0.05), seed=0, device="cuda"):
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    a, b, c, _ = abcd
    n = 1 << scale
    keys = []
    left, chunk = n_pairs, 1 << 24
    while left > 0:
        m = min(left, chunk)
        src = torch.zeros(m, dtype=torch.int64, device=device)
        dst = torch.zeros(m, dtype=torch.int64, device=device)
        for _bit in range(scale):
            r = torch.rand(m, generator=gen, device=device)
            sbit = (r >= a + b).long()
            dbit = (((r >= a) & (r < a + b)) | (r >= a + b + c)).long()
            src = (src << 1) | sbit
            dst = (dst << 1) | dbit
        keep = src != dst
        src, dst = src[keep], dst[keep]
        keys.append(src * n + dst)
        keys.append(dst * n + src)
        left -= m
    key = torch.unique(torch.cat(keys), sorted=True)
    del keys
    s, d = key // n, key % n
    del key
    deg = torch.bincount(s, minlength=n)
    del s
    alive = deg > 0
    n2 = int(alive.sum())
    remap = torch.cumsum(alive.long(), 0) - 1
    d = remap[d].to(torch.int32)
    deg = deg[alive]
    indptr = torch.zeros(n2 + 1, dtype=torch.int64, device=device)
    torch.cumsum(deg, 0, out=indptr[1:])
    return synthetic.CSRGraph(indptr, d, n2, "rmat_dev_s%d_p%d" % (scale, n_pairs))


@pytest.mark.parametrize("which", ["chung_lu", "rmat"])
def test_generators_unchanged(which):
    if which == "chung_lu":
        new, old = synthetic.chung_lu_device(1_000_000, 20_000_000, 0.5, seed=0), _old_chung_lu_device(1_000_000, 20_000_000)
    else:
        new, old = synthetic.rmat_device(20, 20_000_000, seed=3), _old_rmat_device(20, 20_000_000, seed=3)
    assert new.num_nodes == old.num_nodes and new.name == old.name
    assert torch.equal(new.indptr, old.indptr) and torch.equal(new.indices, old.indices)
    assert new.indices.dtype == old.indices.dtype == torch.int32
