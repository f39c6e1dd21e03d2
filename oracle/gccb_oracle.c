/*
 * gccb_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C restatement of the integer part of the THUDM/GCC pretraining hot
 * path: seed draw, random walk with restart, ego-subgraph induction.  Only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this file.  The product (gcc_b200/) never does.
 *
 * PARITY STATUS: "parity unpinned" against DGL.  The arithmetic of these
 * functions lives in DGL 0.4.3 (dgl.contrib.sampling.random_walk_with_restart,
 * DGLGraph.subgraph), which is not part of the reference and was not installable
 * where this oracle was written
 * (SURVEY.md section 8c).  What IS followed line by line is the reference's own
 * glue around those calls:
 *   - seed draw p ~ in_deg^0.75         gcc/datasets/graph_dataset.py:85-92
 *   - walk budget max(rw_hops, ...)     gcc/datasets/graph_dataset.py:113-124
 *   - RWR call with seeds=[s, s]        gcc/datasets/graph_dataset.py:125-130
 *   - subv=[seed]+sorted(unique(trace)\{seed}), induced subgraph, seed=row 0
 *                                       gcc/datasets/data_util.py:218-239
 * The DGL semantics chosen here (documented in DESIGN.md "RWR-Philox v1"):
 *   per seed, traces restart from the seed; inside a trace hop 0 is always
 *   taken, at hop h>0 the trace ends with probability restart_prob, otherwise
 *   a uniformly random out-neighbour is taken and recorded; traces exclude the
 *   seed; sampling stops after the first trace at which the cumulative number
 *   of recorded nodes reaches max_nodes_per_seed.
 * DGL's sequential thread-local RNG cannot be reproduced (and the reference
 * never seeds it in workers, graph_dataset.py:30), so randomness is a
 * counter-based Philox4x32-10 stream: identical integers on CPU and GPU.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define GCCB_O_HOPCAP 64u      /* hard cap on hops inside one trace            */
#define GCCB_O_TAG_WALK 0u
#define GCCB_O_TAG_SEED 1u
#define GCCB_O_TAG_DROPOUT 2u

/* ---- Philox4x32-10 (Salmon et al., SC'11; Random123 reference constants) ---- */
void gccb_o_philox4x32_10(const uint32_t ctr_in[4], const uint32_t key_in[2],
                          uint32_t out[4]) {
  uint32_t c0 = ctr_in[0], c1 = ctr_in[1], c2 = ctr_in[2], c3 = ctr_in[3];
  uint32_t k0 = key_in[0], k1 = key_in[1];
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

static void philox_at(uint64_t key, uint64_t sample, uint32_t trace, uint32_t hop,
                      uint32_t view, uint32_t tag, uint32_t out[4]) {
  uint32_t ctr[4] = {(uint32_t)sample, (uint32_t)(sample >> 32), trace,
                     hop | (view << 8) | (tag << 16)};
  uint32_t k[2] = {(uint32_t)key, (uint32_t)(key >> 32)};
  gccb_o_philox4x32_10(ctr, k, out);
}

/* Seed draw (graph_dataset.py:85-92): node = first i with cdf[i] > u, where
 * cdf is the host-built float64 cumulative sum of in_deg^0.75 / total and
 * u = 53 random bits * 2^-53.  Mirrors np.random.choice's searchsorted(right). */
int64_t gccb_o_draw_seed(const double *cdf, int64_t n, uint64_t key,
                         uint64_t sample) {
  uint32_t w[4];
  philox_at(key, sample, 0, 0, 0, GCCB_O_TAG_SEED, w);
  uint64_t u53 = ((uint64_t)w[0] << 21) | (uint64_t)(w[1] >> 11);
  double u = (double)u53 * (1.0 / 9007199254740992.0);
  int64_t lo = 0, hi = n; /* first index with cdf[i] > u */
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  return lo < n ? lo : n - 1;
}

static int cmp_i32(const void *a, const void *b) {
  int32_t x = *(const int32_t *)a, y = *(const int32_t *)b;
  return (x > y) - (x < y);
}

/*
 * One ego-subgraph: RWR walk from `seed` (graph_dataset.py:125-130), then the
 * node order / induction of data_util.py:218-239.
 * counters[0]=n  [1]=m (directed edges)  [2]=recorded walk steps  [3]=traces
 * counters[4]=sum over subv of parent degree (induction read volume).
 * Returns 0, -2 on capacity overflow (n > cap_n, m > cap_m, steps > cap_walk),
 * -1 on bad input (zero-degree node hit: DGL would LOG(FATAL) here).
 */
int gccb_o_rwr_subgraph(const int64_t *indptr, const int32_t *indices,
                        int64_t n_nodes, uint64_t key, uint64_t sample, int view,
                        int64_t seed, int64_t budget, uint32_t restart_thresh,
                        int32_t *subv, int32_t cap_n, int32_t *sub_indptr,
                        int32_t *sub_indices, int64_t cap_m, int64_t *counters) {
  if (seed < 0 || seed >= n_nodes || budget < 1) return -1;
  int64_t cap_walk = budget + GCCB_O_HOPCAP;
  int32_t *visited = (int32_t *)malloc(sizeof(int32_t) * (size_t)cap_walk);
  if (!visited) return -2;
  int64_t total = 0;
  uint32_t trace = 0;
  while (total < budget) {
    int64_t cur = seed;
    for (uint32_t hop = 0; hop < GCCB_O_HOPCAP; ++hop) {
      uint32_t w[4];
      philox_at(key, sample, trace, hop, (uint32_t)view, GCCB_O_TAG_WALK, w);
      if (hop > 0 && w[0] < restart_thresh) break;
      int64_t beg = indptr[cur], deg = indptr[cur + 1] - beg;
      if (deg <= 0) { free(visited); return -1; }
      uint32_t pick = (uint32_t)(((uint64_t)w[1] * (uint64_t)(uint32_t)deg) >> 32);
      cur = indices[beg + pick];
      visited[total++] = (int32_t)cur;
    }
    ++trace;
  }
  counters[2] = total;
  counters[3] = trace;
  /* subv = [seed] + sorted(unique(visited) \ {seed})   (data_util.py:221-226) */
  qsort(visited, (size_t)total, sizeof(int32_t), cmp_i32);
  int64_t n = 0;
  if (cap_n < 1) { free(visited); return -2; }
  subv[n++] = (int32_t)seed;
  for (int64_t i = 0; i < total; ++i) {
    int32_t v = visited[i];
    if (v == (int32_t)seed) continue;
    if (i > 0 && visited[i - 1] == v) continue;
    if (n >= cap_n) { free(visited); return -2; }
    subv[n++] = v;
  }
  free(visited);
  /* induced subgraph, new ids follow subv order (seed = 0; data_util.py:230,238).
   * Row i lists the neighbours of subv[i] that are inside subv, in the parent's
   * adjacency order, multiplicity kept. */
  int64_t m = 0, sumdeg = 0;
  sub_indptr[0] = 0;
  for (int64_t i = 0; i < n; ++i) {
    int64_t v = subv[i];
    int64_t beg = indptr[v], end = indptr[v + 1];
    sumdeg += end - beg;
    for (int64_t e = beg; e < end; ++e) {
      int32_t u = indices[e];
      int64_t j = -1;
      if (u == (int32_t)seed) {
        j = 0;
      } else { /* binary search in subv[1..n) */
        int64_t lo = 1, hi = n;
        while (lo < hi) {
          int64_t mid = (lo + hi) >> 1;
          if (subv[mid] < u) lo = mid + 1; else hi = mid;
        }
        if (lo < n && subv[lo] == u) j = lo;
      }
      if (j >= 0) {
        if (m >= cap_m) return -2;
        sub_indices[m++] = (int32_t)j;
      }
    }
    sub_indptr[i + 1] = (int32_t)m;
  }
  counters[0] = n;
  counters[1] = m;
  counters[4] = sumdeg;
  return 0;
}

/* Dropout keep-mask bits (gin.py:202,230; Dropout(0.5) on the q branch).
 * Torch's RNG stream is not reproducible across devices, so the mask is a
 * Philox stream: element e of prediction layer `layer` at optimisation step
 * `step` is kept iff word (e & 3) of philox(key,(step, e>>2, layer|tag)) has
 * its top bit clear... i.e. keep iff w < keep_thresh.                     */
void gccb_o_dropout_mask(uint64_t key, uint64_t step, uint32_t layer,
                         int64_t count, uint32_t keep_thresh, uint8_t *keep) {
  for (int64_t e = 0; e < count; e += 4) {
    uint32_t w[4];
    philox_at(key, step, (uint32_t)(e >> 2), 0, layer, GCCB_O_TAG_DROPOUT, w);
    for (int j = 0; j < 4 && e + j < count; ++j) keep[e + j] = w[j] < keep_thresh;
  }
}

/* A whole batch for timing (cpu_baseline): B samples x 2 views, outputs packed. */
int gccb_o_rwr_batch(const int64_t *indptr, const int32_t *indices, int64_t n_nodes,
                     uint64_t key, const int64_t *sample_ids, const int64_t *seeds,
                     const int32_t *budget_table, int64_t budget_table_len,
                     uint32_t restart_thresh, int64_t count, int32_t cap_n,
                     int64_t cap_m, int32_t *subv_out, int32_t *indptr_out,
                     int32_t *indices_out, int64_t *counters_out) {
  /* outputs: per (sample, view) slot s = 2*i+view: subv_out[s*cap_n..],
   * indptr_out[s*(cap_n+1)..], indices_out[s*cap_m..], counters_out[s*5..] */
  for (int64_t i = 0; i < count; ++i) {
    int64_t seed = seeds[i];
    int64_t deg = indptr[seed + 1] - indptr[seed];
    int64_t bi = deg < budget_table_len ? deg : budget_table_len - 1;
    for (int view = 0; view < 2; ++view) {
      int64_t s = 2 * i + view;
      int rc = gccb_o_rwr_subgraph(indptr, indices, n_nodes, key,
                                   (uint64_t)sample_ids[i], view, seed,
                                   budget_table[bi], restart_thresh,
                                   subv_out + s * cap_n, cap_n,
                                   indptr_out + s * (cap_n + 1),
                                   indices_out + s * cap_m, cap_m,
                                   counters_out + s * 5);
      if (rc) return rc;
    }
  }
  return 0;
}
