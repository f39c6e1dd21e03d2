// gather.cu -- whole-graph batches: both views of B pairs copied from a device-resident set of graphs.
//
// Replaces (reference file:line):
//   GraphClassificationDataset.__getitem__ with entire_graph=True  gcc/datasets/graph_dataset.py:311-340
//     (q and k are both the whole graph; the seed one-hot sits on the first maximum-degree vertex)
//   batcher() / dgl.batch                                          gcc/datasets/data_util.py:26-32
//
// The graphs are relabelled seed-first once (gccb_seed_first_union, below) and kept as one union CSR,
// so a batch is a copy with its offsets shifted into the view-local numbering: no walk, no induction, no host
// work per step.  Rows are copied as listed: parallel edges, self loops and isolated vertices are kept.
#include "common.cuh"

namespace gccb {

// Pass 1: per-view exclusive scans of the picked graphs' sizes -> node_off / edge_off, counters (n, m, 0, 0) and
// the capacity check (batch_offsets_kernel's contract: on overflow the view is published empty).
// grid = 2 (views), block = 256.
__global__ void __launch_bounds__(256)
gather_offsets_kernel(const int64_t* __restrict__ g_node_off, const int64_t* __restrict__ g_edge_off,
                      int64_t n_graphs, const int64_t* __restrict__ graph_ids, int B, int node_cap, int edge_cap,
                      int32_t* __restrict__ node_off, int32_t* __restrict__ edge_off,
                      int64_t* __restrict__ counters, int32_t* __restrict__ flags) {
  __shared__ int scan_scratch[33];
  const int view = blockIdx.x, tid = threadIdx.x;
  long long nbase = 0, ebase = 0;
  for (int b0 = 0; b0 < B; b0 += 256) {
    const int g = b0 + tid;
    int n = 0, m = 0;
    if (g < B) {
      const int64_t id = clamp_graph(graph_ids[g], n_graphs);
      n = (int)(g_node_off[id + 1] - g_node_off[id]);
      m = (int)(g_edge_off[id + 1] - g_edge_off[id]);
      int64_t* c = counters + (size_t)(view * B + g) * 4;
      c[0] = n;
      c[1] = m;
      c[2] = 0;
      c[3] = 0;
    }
    int tn, tm;
    const int en = block_scan_excl(n, scan_scratch, &tn);
    const int em = block_scan_excl(m, scan_scratch, &tm);
    if (g < B) {
      const long long no = nbase + en, eo = ebase + em;
      node_off[view * (B + 1) + g] = (int)(no > 0x7fffffffLL ? 0x7fffffffLL : no);
      edge_off[view * (B + 1) + g] = (int)(eo > 0x7fffffffLL ? 0x7fffffffLL : eo);
    }
    nbase += tn;
    ebase += tm;
  }
  if (tid == 0) {
    int f = 0;
    if (nbase > node_cap) f |= GCCB_FLAG_NODE_OVERFLOW;
    if (ebase > edge_cap) f |= GCCB_FLAG_EDGE_OVERFLOW;
    node_off[view * (B + 1) + B] = f ? -1 : (int)nbase;
    edge_off[view * (B + 1) + B] = f ? -1 : (int)ebase;
    if (f) atomicOr(flags, f);
  }
}

// Pass 2: copy graph g into view v.  grid = (B, 2), block = 256.
__global__ void __launch_bounds__(256)
gather_fill_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const int64_t* __restrict__ g_node_off, const int64_t* __restrict__ g_edge_off, int64_t n_graphs,
                   const int64_t* __restrict__ graph_ids, int B, int node_cap, int edge_cap,
                   const int32_t* __restrict__ node_off, const int32_t* __restrict__ edge_off,
                   int32_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices,
                   int32_t* __restrict__ out_subdeg, int32_t* __restrict__ out_graph_id,
                   int32_t* __restrict__ out_orig_id) {
  const int g = blockIdx.x, view = blockIdx.y, tid = threadIdx.x;
  if (node_off[view * (B + 1) + B] < 0) return;        // view overflowed: published empty
  const int64_t id = clamp_graph(graph_ids[g], n_graphs);
  const int64_t v0 = g_node_off[id], e0 = g_edge_off[id];
  const int n = (int)(g_node_off[id + 1] - v0);
  const int m = (int)(g_edge_off[id + 1] - e0);
  const int noff = node_off[view * (B + 1) + g];
  const int eoff = edge_off[view * (B + 1) + g];
  int32_t* v_indptr = out_indptr + (size_t)view * (node_cap + 1);
  int32_t* v_indices = out_indices + (size_t)view * edge_cap;
  const size_t nb = (size_t)view * node_cap + noff;
  for (int i = tid; i < n; i += blockDim.x) {
    const int64_t r = indptr[v0 + i];
    v_indptr[noff + i] = eoff + (int)(r - e0);
    out_subdeg[nb + i] = (int)(indptr[v0 + i + 1] - r);
    out_graph_id[nb + i] = g;
    out_orig_id[nb + i] = noff + i;                      // the row itself: a whole graph has no parent graph
  }
  if (g == B - 1 && tid == 0) v_indptr[noff + n] = eoff + m;   // closing entry = E_v
  for (int e = tid; e < m; e += blockDim.x) v_indices[eoff + e] = noff + (int)(indices[e0 + e] - v0);
}

// ---- the whole-graph set relabelled seed first (gccb_seed_first_union) ------------------------------------------
// Graph g's seed s is its first vertex of maximum row length.  The new row order is [s, 0..s-1, s+1..n-1] and old
// local id u becomes 0 (u == s), u + 1 (u < s) or u (u > s).  That map is monotone except at s, so a non-decreasing
// row stays non-decreasing once its entries equal to s (all of them: parallel edges) move to its front; rows after
// the seed keep their offsets and rows 1..s shift by the seed's row length.  One read and one write of the CSR.
//
// The seed is found as the maximum of a packed key, (row length << 32) | (2^32 - 1 - local id): a longer row wins,
// and among equal lengths the lower id.  seeds[] holds the keys until seed_finish_kernel turns them into local ids.

// last i in [lo, hi] with off[i] <= x (off non-decreasing, off[lo] <= x): the graph of a vertex (off = node_off),
// or the row of an entry (off = indptr); empty graphs and rows are skipped.
template <class T>
__device__ __forceinline__ int64_t find_segment(const T* __restrict__ off, int64_t lo, int64_t hi, int64_t x) {
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if ((int64_t)off[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// first i in [lo, hi) with a[i] >= x (upper = false) or a[i] > x (upper = true); hi if none
__device__ __forceinline__ int64_t row_bound(const int32_t* __restrict__ a, int64_t lo, int64_t hi, int32_t x,
                                             bool upper) {
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (a[mid] < x || (upper && a[mid] == x)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The graphs [*g_lo, *g_hi] that hold the items first .. last of this block (thread 0 searches, the block reads).
template <class T>
__device__ __forceinline__ void block_segments(const T* __restrict__ off, int64_t n_seg, int64_t first, int64_t last,
                                               int64_t* s_range) {
  if (threadIdx.x == 0) {
    s_range[0] = find_segment(off, 0, n_seg - 1, first);
    s_range[1] = find_segment(off, s_range[0], n_seg - 1, last);
  }
  __syncthreads();
}

// Pass 1: one thread per vertex; keys[g] = max over graph g's vertices of the packed key.  A warp inside one graph
// reduces first; keys are only raised, so a stale read only costs an extra atomic.  grid = ceil(V / 256), block 256.
__global__ void __launch_bounds__(256)
seed_keys_kernel(const int64_t* __restrict__ indptr, const int64_t* __restrict__ node_off, int64_t n_graphs,
                 int64_t n_nodes, unsigned long long* keys) {
  __shared__ int64_t s_range[2];
  const int64_t first = (int64_t)blockIdx.x * blockDim.x;
  const int64_t last = (first + blockDim.x < n_nodes ? first + blockDim.x : n_nodes) - 1;
  block_segments(node_off, n_graphs, first, last, s_range);
  const int64_t v = first + threadIdx.x;
  long long g = -1;
  unsigned long long key = 0;
  if (v < n_nodes) {
    g = find_segment(node_off, s_range[0], s_range[1], v);
    const unsigned long long len = (unsigned long long)(indptr[v + 1] - indptr[v]);
    key = (len << 32) | (0xffffffffull - (unsigned long long)(v - node_off[g]));
  }
  const long long g0 = __shfl_sync(0xffffffffu, g, 0);
  if (__all_sync(0xffffffffu, g == g0)) {
    for (int o = 16; o; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
      key = other > key ? other : key;
    }
    if ((threadIdx.x & 31) == 0 && g >= 0 && key > keys[g]) atomicMax(keys + g, key);
  } else if (g >= 0 && key > keys[g]) {
    atomicMax(keys + g, key);
  }
}

// Pass 2: key -> local seed id, in place.  A graph without vertices keeps seed 0.  grid = ceil(G / 256), block 256.
__global__ void __launch_bounds__(256) seed_finish_kernel(int64_t n_graphs, unsigned long long* keys) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_graphs) return;
  const unsigned long long k = keys[g];
  keys[g] = k ? 0xffffffffull - (k & 0xffffffffull) : 0;
}

// Pass 3: one thread per old row (and one for the closing entry): its offset at its new position.
// grid = ceil((V + 1) / 256), block 256.
__global__ void __launch_bounds__(256)
relabel_indptr_kernel(const int64_t* __restrict__ indptr, const int64_t* __restrict__ node_off, int64_t n_graphs,
                      int64_t n_nodes, const int64_t* __restrict__ seeds, int64_t* __restrict__ out_indptr) {
  __shared__ int64_t s_range[2];
  const int64_t first = (int64_t)blockIdx.x * blockDim.x;
  const int64_t last = (first + blockDim.x < n_nodes ? first + blockDim.x : n_nodes) - 1;
  if (first < n_nodes) block_segments(node_off, n_graphs, first, last, s_range);
  const int64_t v = first + threadIdx.x;
  if (v == n_nodes) out_indptr[v] = indptr[v];
  if (v >= n_nodes) return;
  const int64_t g = find_segment(node_off, s_range[0], s_range[1], v);
  const int64_t v0 = node_off[g], s = seeds[g], u = v - v0;
  if (u == s) out_indptr[v0] = indptr[v0];
  else if (u < s) out_indptr[v + 1] = indptr[v] + (indptr[v0 + s + 1] - indptr[v0 + s]);
  else out_indptr[v] = indptr[v];
}

// Pass 4: one thread per entry: its new position and id, and the row contract (non-decreasing, ids inside the
// graph).  An entry equal to the seed S moves to (its index among the S entries); one below S moves past the row's
// S entries; one above S stays.  Every position stays inside its row, whatever the input.
// grid = ceil(E / 256), block 256.
__global__ void __launch_bounds__(256)
relabel_indices_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                       const int64_t* __restrict__ node_off, int64_t n_graphs, int64_t n_nodes, int64_t n_edges,
                       const int64_t* __restrict__ seeds, int32_t* __restrict__ out_indices,
                       int32_t* __restrict__ flags) {
  __shared__ int64_t s_rows[2], s_graphs[2];
  const int64_t first = (int64_t)blockIdx.x * blockDim.x;
  const int64_t last = (first + blockDim.x < n_edges ? first + blockDim.x : n_edges) - 1;
  block_segments(indptr, n_nodes, first, last, s_rows);
  block_segments(node_off, n_graphs, s_rows[0], s_rows[1], s_graphs);
  const int64_t e = first + threadIdx.x;
  if (e >= n_edges) return;
  const int64_t r = find_segment(indptr, s_rows[0], s_rows[1], e);
  const int64_t g = find_segment(node_off, s_graphs[0], s_graphs[1], r);
  const int64_t v0 = node_off[g], s = seeds[g], u = r - v0;
  const int64_t rs = indptr[r], re = indptr[r + 1], j = e - rs;
  const int32_t S = (int32_t)(v0 + s), w = indices[e];
  if (w < v0 || w >= node_off[g + 1] || (j > 0 && indices[e - 1] > w)) atomicOr(flags, GCCB_FLAG_BAD_ROW);
  const int64_t base = u == s ? indptr[v0] : (u < s ? rs + (indptr[S + 1] - indptr[S]) : rs);
  int64_t pos;
  int32_t id;
  if (w == S) {
    pos = e - row_bound(indices, rs, e, S, false);
    id = (int32_t)v0;
  } else if (w < S) {
    pos = j + row_bound(indices, e + 1, re, S, true) - row_bound(indices, e + 1, re, S, false);
    id = w + 1;
  } else {
    pos = j;
    id = w;
  }
  out_indices[base + pos] = id;
}

}  // namespace gccb

using namespace gccb;

extern "C" int gccb_seed_first_union(const gccb_graph_set_t* set, int64_t n_nodes, int64_t n_edges, int64_t* seeds,
                                     int64_t* out_indptr, int32_t* out_indices, int32_t* flags, gccb_stream_t stream) {
  if (!set || set->n_graphs <= 0 || !set->indptr || !set->node_off || !seeds || !out_indptr || !flags ||
      n_nodes < 0 || n_nodes > 0x80000000LL || n_edges < 0 || (n_edges > 0 && (!set->indices || !out_indices))) {
    set_last_error("gccb_seed_first_union: bad argument");
    return GCCB_ERR_BADARG;
  }
  const int64_t G = set->n_graphs;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(seeds);
  cudaMemsetAsync(seeds, 0, (size_t)G * sizeof(int64_t), (cudaStream_t)stream);
  if (n_nodes > 0)
    GCCB_LAUNCH(seed_keys_kernel, (unsigned)((n_nodes + 255) / 256), 256, 0, stream, set->indptr, set->node_off, G,
                n_nodes, keys);
  GCCB_LAUNCH(seed_finish_kernel, (unsigned)((G + 255) / 256), 256, 0, stream, G, keys);
  GCCB_LAUNCH(relabel_indptr_kernel, (unsigned)((n_nodes + 256) / 256), 256, 0, stream, set->indptr, set->node_off,
              G, n_nodes, (const int64_t*)seeds, out_indptr);
  if (n_edges > 0)
    GCCB_LAUNCH(relabel_indices_kernel, (unsigned)((n_edges + 255) / 256), 256, 0, stream, set->indptr, set->indices,
                set->node_off, G, n_nodes, n_edges, (const int64_t*)seeds, out_indices, flags);
  return check_launch("gccb_seed_first_union");
}

extern "C" int gccb_gather_graphs(const gccb_graph_set_t* set, const int64_t* graph_ids, const gccb_batch_t* batch,
                                  gccb_stream_t stream) {
  if (!set || !batch || !graph_ids || batch->batch <= 0 || set->n_graphs <= 0 || !set->indptr || !set->indices ||
      !set->node_off || !set->edge_off) {
    set_last_error("gccb_gather_graphs: bad argument");
    return GCCB_ERR_BADARG;
  }
  const int B = batch->batch;
  GCCB_LAUNCH(gather_offsets_kernel, 2, 256, 0, stream, set->node_off, set->edge_off, set->n_graphs, graph_ids, B,
              batch->node_cap, batch->edge_cap, batch->node_off, batch->edge_off, batch->counters, batch->flags);
  GCCB_LAUNCH(gather_fill_kernel, dim3(B, 2), 256, 0, stream, set->indptr, set->indices, set->node_off,
              set->edge_off, set->n_graphs, graph_ids, B, batch->node_cap, batch->edge_cap, batch->node_off,
              batch->edge_off, batch->indptr, batch->indices, batch->sub_deg, batch->graph_id, batch->orig_id);
  return check_launch("gccb_gather_graphs");
}
