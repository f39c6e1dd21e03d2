"""Synthetic input graphs for BASELINE.json's configs (SURVEY.md section 8d).

Every generator returns a ``CSRGraph`` that satisfies the invariants the
reference's data preparation enforces (gcc/utils/x2dgl.py:40-62): symmetric,
no self loops, de-duplicated, zero-degree nodes removed and ids compacted.
"edges" in BASELINE.json are undirected pairs; CSR nnz = 2 x pairs (minus
duplicates).  indptr is int64, indices int32, neighbour lists ascending.
"""
from collections import namedtuple

import numpy as np

CSRGraph = namedtuple("CSRGraph", ["indptr", "indices", "num_nodes", "name"])


def _sort_unique_i64(key):
    """Sorted unique of an int64 key array; on a CUDA box the sort runs on the
    device (setup only -- not part of the timed path), same result either way."""
    try:
        import torch
        if torch.cuda.is_available() and key.size > (1 << 22):
            t = torch.from_numpy(key).cuda()
            return torch.unique(t, sorted=True).cpu().numpy()
    except ImportError:  # pragma: no cover
        pass
    return np.unique(key)


def from_pairs(src, dst, n, name="graph"):
    """Symmetrise / clean an edge list exactly like x2dgl.py does."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    keep = src != dst                       # x2dgl.py: remove self loops
    src, dst = src[keep], dst[keep]
    # symmetrise + de-duplicate: unique over directed keys s*n+d of both directions
    key = _sort_unique_i64(np.concatenate([src * n + dst, dst * n + src]))
    s, d = key // n, key % n
    deg = np.bincount(s, minlength=n)
    alive = deg > 0                         # x2dgl.py:61 zero-degree removal
    n2 = int(alive.sum())
    if n2 != n:
        remap = np.cumsum(alive) - 1        # monotone: keeps (s, d) order sorted
        s, d = remap[s], remap[d]
        deg = deg[alive]
    indptr = np.zeros(n2 + 1, dtype=np.int64)
    np.cumsum(deg, out=indptr[1:])
    return CSRGraph(indptr, d.astype(np.int32), n2, name)


def from_keys_device(keys, n, name="graph"):
    """The cleaning of x2dgl.py:52-62 on directed keys s*n + d that hold both orientations of every edge and no
    self loop, with torch on the keys' device: tocsr() (duplicates merged into one entry), then remove_nodes
    (in_degrees == 0) with the remaining vertices kept in order.  Neighbour lists come out ascending.
    keys: an int64 tensor or a list of them; a list is emptied here, so that its tensors are freed as soon as
    the de-duplicated copy exists (BASELINE config 5 holds 400M keys)."""
    import torch
    if isinstance(keys, list):
        key = keys[0] if len(keys) == 1 else torch.cat(keys)
        keys.clear()
    else:
        key = keys
    del keys
    key = torch.unique(key, sorted=True)
    s, d = key // n, key % n
    device = key.device
    del key
    deg = torch.bincount(s, minlength=n)
    del s
    alive = deg > 0
    n2 = int(alive.sum())
    if n2 != n:
        remap = torch.cumsum(alive.long(), 0) - 1
        d = remap[d]
        deg = deg[alive]
    indptr = torch.zeros(n2 + 1, dtype=torch.int64, device=device)
    torch.cumsum(deg, 0, out=indptr[1:])
    return CSRGraph(indptr, d.to(torch.int32), n2, name)


def erdos_renyi(n=1000, n_pairs=5000, seed=0):
    """C1: ER G(n, pairs)."""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, size=n_pairs, dtype=np.int64)
    dst = rng.integers(0, n, size=n_pairs, dtype=np.int64)
    return from_pairs(src, dst, n, "er_n%d_p%d" % (n, n_pairs))


def chung_lu(n=1_000_000, n_pairs=20_000_000, exponent=0.5, seed=0, chunk=1 << 24):
    """C2/C3/C4: Chung-Lu power-law graph, w_i ~ (i+1)^-exponent."""
    rng = np.random.default_rng(seed)
    w = (np.arange(n, dtype=np.float64) + 1.0) ** (-exponent)
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    srcs, dsts = [], []
    left = n_pairs
    while left > 0:
        c = min(left, chunk)
        srcs.append(np.searchsorted(cdf, rng.random(c), side="right"))
        dsts.append(np.searchsorted(cdf, rng.random(c), side="right"))
        left -= c
    src = np.minimum(np.concatenate(srcs), n - 1)
    dst = np.minimum(np.concatenate(dsts), n - 1)
    return from_pairs(src, dst, n, "chunglu_n%d_p%d" % (n, n_pairs))


def rmat(scale=20, n_pairs=1 << 24, a=0.57, b=0.19, c=0.19, d=0.05, seed=0):
    """C5: R-MAT(a,b,c,d) on 2^scale nodes."""
    rng = np.random.default_rng(seed)
    n = 1 << scale
    src = np.zeros(n_pairs, dtype=np.int64)
    dst = np.zeros(n_pairs, dtype=np.int64)
    for _ in range(scale):
        r = rng.random(n_pairs)
        src = (src << 1) | (r >= a + b)
        dst = (dst << 1) | (((r >= a) & (r < a + b)) | (r >= a + b + c))
    return from_pairs(src, dst, n, "rmat_s%d_p%d" % (scale, n_pairs))


def path_graph(n):
    i = np.arange(n - 1)
    return from_pairs(i, i + 1, n, "path%d" % n)


def star_graph(n_leaves):
    return from_pairs(np.zeros(n_leaves, dtype=np.int64),
                      np.arange(1, n_leaves + 1), n_leaves + 1, "star%d" % n_leaves)


def triangle_tail(tail=3):
    src = [0, 1, 2] + list(range(2, 2 + tail))
    dst = [1, 2, 0] + list(range(3, 3 + tail))
    return from_pairs(src, dst, 3 + tail, "tri_tail%d" % tail)


def disjoint_union(graphs, name="union"):
    """Block-diagonal union (a multi-graph corpus as one CSR; global node id =
    the reference's concatenated idx, graph_dataset.py:95-102)."""
    indptrs, indices, off, eoff = [np.zeros(1, dtype=np.int64)], [], 0, 0
    for g in graphs:
        indptrs.append(g.indptr[1:] + eoff)
        indices.append(g.indices.astype(np.int64) + off)
        off += g.num_nodes
        eoff += int(g.indptr[-1])
    return CSRGraph(np.concatenate(indptrs), np.concatenate(indices).astype(np.int32),
                    off, name)


def chung_lu_device(n=1_000_000, n_pairs=20_000_000, exponent=0.5, seed=0, device="cuda"):
    """C2-size Chung-Lu graph generated ON the GPU with torch (setup, not the timed path): the
    same construction as chung_lu()/from_pairs() -- sample endpoints ~ w, drop self loops,
    symmetrise, de-duplicate, drop zero-degree vertices -- with tensors left on the device.
    (torch's CUDA RNG stream differs from numpy's, so the edge set differs from chung_lu(seed).)"""
    import torch
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
    return from_keys_device(keys, n, "chunglu_dev_n%d_p%d" % (n, n_pairs))


def rmat_device(scale=24, n_pairs=200_000_000, abcd=(0.57, 0.19, 0.19, 0.05), seed=0, device="cuda"):
    """RMAT graph generated with torch on `device` (setup, not the timed path): 2^scale candidate
    vertices, n_pairs sampled (src, dst) pairs by recursive quadrant choice, then the x2dgl.py:40-62
    invariants -- self loops dropped, symmetrised, de-duplicated, zero-degree vertices removed and
    ids compacted.  BASELINE config 5 (10M-node / 200M-pair RMAT) is scale=24."""
    import torch
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
            sbit = (r >= a + b).long()                          # quadrants c, d: lower half of the rows
            dbit = (((r >= a) & (r < a + b)) | (r >= a + b + c)).long()   # quadrants b, d: right half
            src = (src << 1) | sbit
            dst = (dst << 1) | dbit
        keep = src != dst
        src, dst = src[keep], dst[keep]
        keys.append(src * n + dst)
        keys.append(dst * n + src)
        left -= m
    return from_keys_device(keys, n, "rmat_dev_s%d_p%d" % (scale, n_pairs))
