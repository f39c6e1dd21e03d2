"""Oracle (test infrastructure) of the reference's other views: the step_dist key seed and neighbour-sampled
ego-nets (aug="ns"), restated from DESIGN.md section 3 (the bullet on the reference's other views) with the
Philox counters of the kernels (sampler.cu).

DGL's semantics are choices here (DGL is absent):
  * random_walk(g, [s], 1, step)[0][0][-1] is the end of a `step`-hop uniform walk from s (the trace holds s first);
  * a vertex without neighbours ends that walk where it is;
  * a layer samples num_neighbors distinct neighbour ENTRIES without replacement (parallel edges are separate entries
    and collapse in the de-duplication), and takes all of them when there are no more;
  * layers are not reduced by the earlier ones; only the final union is.
The paired RWR view reuses oracle/rwr.py's walk with the k seed and the q seed's budget."""
import numpy as np

from oracle import rwr as orwr

TAG_STEP, TAG_KHOP, TAG_NS = 4, 5, 6
M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox_np(c0, c1, c2, c3, key):
    """Philox4x32-10 over arrays of counters (uint64 holding 32-bit words); returns word x."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & MASK for c in (c0, c1, c2, c3))
    k0, k1 = key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0)) & MASK, p1 & MASK, \
            ((p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1)) & MASK, p0 & MASK
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c0


def step_cdf(step_dist):
    cdf = np.cumsum(np.asarray(step_dist, dtype=np.float64))
    return cdf / cdf[-1]


def draw_step(cdf, key, sample):
    w = orwr._philox_at(key, sample, 0, 0, 0, TAG_STEP)
    u = float((w[0] << 21) | (w[1] >> 11)) / 9007199254740992.0
    return min(int(np.searchsorted(cdf, u, side="right")), len(cdf) - 1)


def pair_seed(indptr, indices, key, sample, seed_q, cdf):
    """(step, k seed) of one sample."""
    step = draw_step(cdf, key, sample)
    cur = int(seed_q)
    for h in range(1, step + 1):
        beg, deg = int(indptr[cur]), int(indptr[cur + 1] - indptr[cur])
        if deg == 0:
            break
        w = orwr._philox_at(key, sample, 0, h, 0, TAG_KHOP)
        cur = int(indices[beg + ((w[1] * deg) >> 32)])
    return step, cur


def pairs_batch(indptr, indices, key, sample_ids, seeds_q, seeds_k, btable, restart_thresh):
    """RWR views with separate seeds, both budgets from the q seed: [view][i] dicts as orwr.rwr_subgraph."""
    deg = np.diff(np.asarray(indptr, dtype=np.int64))
    out = [[], []]
    for s, q, k in zip(sample_ids, seeds_q, seeds_k):
        budget = int(btable[min(int(deg[q]), len(btable) - 1)])
        for v, seed in ((0, q), (1, k)):
            out[v].append(orwr.rwr_subgraph(indptr, indices, key, int(s), v, int(seed), budget, restart_thresh))
    return out


def _floyd(words, d, k):
    """k distinct positions of [0, d): draw t picks r = umulhi(words[t], j + 1) in [0, j], j = d - k + t, or j when
    r was taken already."""
    chosen = []
    for t in range(k):
        j = d - k + t
        r = (int(words[t]) * (j + 1)) >> 32
        chosen.append(j if r in chosen else r)
    return chosen


def ns_nodes(indptr, indices, key, sample, view, seed, hops, k):
    """Node set [seed, rest ascending] after all `hops` layers (no early stop)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    union, layer = {int(seed)}, [int(seed)]
    for hop in range(1, hops + 1):
        if not layer:
            break
        degs = np.array([indptr[u + 1] - indptr[u] for u in layer], dtype=np.int64)
        hubs = np.flatnonzero(degs > k)
        words = None
        if len(hubs):
            p = np.repeat(hubs, k).astype(np.uint64)
            t = np.tile(np.arange(k), len(hubs)).astype(np.uint64)
            c3 = (hop & 0xFF) | (view << 8) | ((TAG_NS | ((hop >> 8) << 8)) << 16)
            words = philox_np(np.full(len(p), sample & 0xFFFFFFFF), np.full(len(p), sample >> 32),
                              p | (t << np.uint64(16)), np.full(len(p), c3), key).reshape(len(hubs), k)
        cand = []
        hub_row = {int(h): r for r, h in enumerate(hubs)}
        for pos, u in enumerate(layer):
            beg, d = int(indptr[u]), int(degs[pos])
            if d <= k:
                cand.extend(int(x) for x in indices[beg:beg + d])
            else:
                cand.extend(int(indices[beg + c]) for c in _floyd(words[hub_row[pos]], d, k))
        layer = sorted(set(cand))
        union.update(layer)
    return [int(seed)] + sorted(union - {int(seed)})


def induce_np(indptr, indices, subv):
    """g.subgraph(subv) (subv = [seed, rest ascending], local ids in subv order): every neighbour entry of every
    row that lies in subv, in row order, parallel edges kept.  orwr.induce_py's arithmetic, one row at a time in
    numpy (ego-nets of thousands of vertices)."""
    sv = np.asarray(subv, dtype=np.int64)
    order = np.argsort(sv, kind="stable")
    ids = sv[order]
    sp, si = [0], []
    for v in sv:
        row = np.asarray(indices[int(indptr[v]):int(indptr[v + 1])], dtype=np.int64)
        pos = np.minimum(np.searchsorted(ids, row), len(ids) - 1)
        hit = ids[pos] == row
        si.append(order[pos[hit]])
        sp.append(sp[-1] + int(hit.sum()))
    si = np.concatenate(si) if si else np.zeros(0, np.int64)
    return sv.astype(np.int32), np.array(sp, dtype=np.int32), si.astype(np.int32)


def ns_subgraph(indptr, indices, key, sample, view, seed, hops, k):
    subv = ns_nodes(indptr, indices, key, sample, view, seed, hops, k)
    sv, sp, si = induce_np(indptr, indices, subv) if len(subv) > 64 else \
        orwr.induce_py(indptr, indices, int(seed), [subv])
    sumdeg = int(np.sum(np.diff(np.asarray(indptr, dtype=np.int64))[sv]))
    return dict(subv=sv, indptr=sp, indices=si, n=len(sv), m=len(si), sumdeg=sumdeg)


def ns_batch(indptr, indices, key, sample_ids, seeds_q, seeds_k, hops, k):
    return [[ns_subgraph(indptr, indices, key, int(s), v, int(seed), hops, k)
             for s, seed in zip(sample_ids, seeds)] for v, seeds in ((0, seeds_q), (1, seeds_k))]
