// gather.cu -- whole-graph batches: both views of B pairs copied from a device-resident set of graphs.
//
// Replaces (reference file:line):
//   GraphClassificationDataset.__getitem__ with entire_graph=True  gcc/datasets/graph_dataset.py:311-340
//     (q and k are both the whole graph; the seed one-hot sits on the first maximum-degree vertex)
//   batcher() / dgl.batch                                          gcc/datasets/data_util.py:26-32
//
// The graphs are relabelled seed-first once on the host (datasets/labeled.seed_first) and kept as one union CSR,
// so a batch is a copy with its offsets shifted into the view-local numbering: no walk, no induction, no host
// work per step.  Rows are copied as listed: parallel edges, self loops and isolated vertices are kept.
#include "common.cuh"

namespace gccb {

__device__ __forceinline__ int64_t clamp_graph(int64_t id, int64_t n_graphs) {
  return id < 0 ? 0 : (id >= n_graphs ? n_graphs - 1 : id);     // caller-supplied ids: never read out of bounds
}

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

}  // namespace gccb

using namespace gccb;

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
