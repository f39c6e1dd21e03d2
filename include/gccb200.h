/*
 * gccb200.h -- C ABI of libgccb200.so: the Hopper (sm_90a) implementation of the
 * THUDM/GCC pretraining hot path (SURVEY.md section 8).
 *
 * The reference has no FFI of its own (it is Python calling DGL / PyTorch), so
 * each entry point cites the reference call site it replaces.  Conventions:
 *   - every pointer is a CALLER-ALLOCATED DEVICE pointer unless marked "host";
 *   - the library never allocates, frees, synchronises or throws; it enqueues
 *     kernels on `stream` (a cudaStream_t passed as void*) and returns
 *     GCCB_OK or a negative gccb_status;  gccb_last_error() gives the text;
 *   - data-dependent failures (capacity overflow, zero-degree vertex, eigen
 *     non-convergence) are reported through a device-side flag word
 *     (gccb_batch_t.flags, GCCB_FLAG_*), so calls stay CUDA-graph capturable;
 *   - stateless, thread-safe per stream.
 * There is no CPU fallback: on a machine without an sm_90 device every compute
 * entry point returns GCCB_ERR_CUDA / GCCB_ERR_ARCH.
 */
#ifndef GCCB200_H_
#define GCCB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GCCB_VERSION 200 /* round 2 */

typedef void* gccb_stream_t; /* cudaStream_t */

typedef enum {
  GCCB_OK = 0,
  GCCB_ERR_BADARG = -1,
  GCCB_ERR_CAPACITY = -2,
  GCCB_ERR_ARCH = -3,
  GCCB_ERR_CUDA = -4
} gccb_status;

/* bits of the device-side flag word */
#define GCCB_FLAG_NODE_OVERFLOW 1   /* batched nodes of a view exceed node_cap          */
#define GCCB_FLAG_EDGE_OVERFLOW 2   /* batched edges of a view exceed edge_cap          */
#define GCCB_FLAG_ZERO_DEGREE 4     /* walk hit a vertex without successors (DGL: FATAL) */
#define GCCB_FLAG_EIG_NOCONV 8      /* eigensolver hit its sweep/iteration limit        */
#define GCCB_FLAG_EIG_TOOBIG 16     /* ego-net larger than the eigensolver supports     */
#define GCCB_FLAG_NONFINITE 32      /* gccb_knn: an input row holds a NaN or an Inf     */
#define GCCB_FLAG_BAD_ROW 64        /* gccb_seed_first_union: a row is not non-decreasing
                                       or names a vertex outside its graph              */
#define GCCB_FLAG_PROBE_NOCONV 128  /* gccb_probe_fit: a problem did not converge
                                       (iteration limit, line search or a non-positive pivot) */

int gccb_version(void);
/* compute capability (major*10+minor) of the current device, or a negative status */
int gccb_arch(void);
const char* gccb_last_error(void);
/* number of kernels this library has enqueued so far in this process (host counter) */
unsigned long long gccb_launch_count(void);

/* ---- parent graph + sampler constants (host struct, device pointers inside) --------
 * Row v of the CSR lists the heads of v's out-edges, NON-DECREASING: a neighbour repeated c
 * times is c parallel edges (a DGL multigraph keeps them).  A walk step picks each entry with
 * equal probability, so u with probability c/deg(v); the induced ego-net keeps all c copies,
 * in the order a scan of the row meets them, and sub_deg counts them.  Self loops are allowed
 * and kept.  Every vertex needs an out-edge.                                               */
typedef struct {
  const int64_t* indptr;       /* [n_nodes+1] CSR row offsets                                */
  const int32_t* indices;      /* [nnz] neighbour ids, non-decreasing per row (see above)    */
  int64_t n_nodes;
  const int32_t* budget_table; /* [budget_table_len] max_nodes_per_seed by seed degree:
                                  graph_dataset.py:113-124, built on the host               */
  int32_t budget_table_len;
  int32_t max_budget;          /* max over budget_table (sizes shared memory / scratch)      */
  uint32_t restart_thresh;     /* floor(restart_prob * 2^32)                                 */
  uint32_t _pad;
  uint64_t key;                /* Philox key = run seed (train.py:118 --seed)                */
} gccb_graph_t;

/* ---- a batch of ego-subgraphs: B (q,k) pairs = two views of B graphs each ----------
 * Replaces the pair of batched DGLGraphs produced by batcher() (data_util.py:26-32).
 * View v occupies rows [v*node_cap, v*node_cap + N_v) of every per-node array and
 * entries [v*edge_cap, ...) of `indices`; graph g of view v owns rows
 * node_off[v*(B+1)+g] .. node_off[v*(B+1)+g+1).  Row ids inside `indices` are
 * view-local (0..N_v).  The seed of every graph is its first row
 * (data_util.py:226,238).                                                             */
typedef struct {
  int32_t batch;     /* B */
  int32_t node_cap;  /* per view */
  int32_t edge_cap;  /* per view */
  int32_t _pad;
  int32_t* node_off; /* [2][B+1]  node_off[v][B] = N_v                                   */
  int32_t* edge_off; /* [2][B+1]  edge_off[v][B] = E_v                                   */
  int32_t* indptr;   /* [2][node_cap+1] view-local edge offsets                          */
  int32_t* indices;  /* [2][edge_cap]                                                    */
  int32_t* sub_deg;  /* [2][node_cap] in-degree inside the ego-net (graph_encoder.py:154) */
  int32_t* graph_id; /* [2][node_cap] graph index 0..B-1                                  */
  int32_t* orig_id;  /* [2][node_cap] parent vertex id (subv)                             */
  int64_t* counters; /* [2B][4] per ego-net: n, m, recorded walk steps, sum of parent
                        degrees over subv (the induction read volume); slot = v*B+g      */
  int32_t* flags;    /* [1] GCCB_FLAG_* (OR-accumulated; caller clears)                  */
} gccb_batch_t;

/* A2  seed draw.  Replaces LoadBalanceGraphDataset.__iter__ (graph_dataset.py:85-92):
 * np.random.choice(length, p = in_deg^0.75/sum).  cdf = float64 cumulative p (host-built,
 * device-resident); sample i draws 53 Philox bits -> first index with cdf > u.
 * Writes seeds_out[i], sample_ids_out[i] = first_sample + i.                          */
int gccb_draw_seeds(const double* cdf, int64_t n_nodes, uint64_t key, int64_t first_sample,
                    int32_t count, int64_t* seeds_out, int64_t* sample_ids_out,
                    gccb_stream_t stream);

/* A3+A4+A6  random walk with restart, ego-net induction, batching.  Replaces
 * dgl.contrib.sampling.random_walk_with_restart (graph_dataset.py:125-130),
 * _rwr_trace_to_dgl_graph's unique/sort/subgraph (data_util.py:218-239) and
 * dgl.batch (data_util.py:29) for both views of `batch->batch` samples.
 * seeds/sample_ids: [B] (both views start from the same seed: step_dist=[1,0,0]).
 * Workspace, in int32 words, with cap(b) = (b + 65 + 3) & ~3:
 *   max_budget <= 32704:  3 * 2B * cap(max_budget) + 16 + 2 * edge_cap
 *   above (wide path):    3 * 2B * cap(32704) + 16 + 2 * edge_cap + 6 * R + min(2B, 32) * K
 *     R = min(edge_cap + B, 2^31 - 1)  per view and array, the node sets and rows of the view's wide ego-nets (an RWR
 *                                      ego-net has m >= n - 1, so a view holding more overflows edge_cap anyway),
 *     K = pow2 >= max_budget + 64      the trace of one of the (at most 32) wide walk CTAs in flight.
 * A sample whose budget exceeds 32,704 (its trace does not fit the walk CTA's 128 KiB of shared memory) is walked,
 * sorted and induced from global memory by the wide kernels, selected per sample on the device; outputs are the
 * same.  max_budget + 64 above 2^30 (int32 trace positions) is refused with GCCB_ERR_CAPACITY.                  */
size_t gccb_sample_batch_workspace(int32_t batch, int32_t max_budget, int32_t edge_cap);
int gccb_sample_batch(const gccb_graph_t* graph, const int64_t* seeds,
                      const int64_t* sample_ids, const gccb_batch_t* batch, void* workspace,
                      size_t workspace_bytes, gccb_stream_t stream);

/* Key seeds of step_dist (graph_dataset.py:104-110).  Sample i (Philox sample id sample_ids[i]) draws
 * step = first index with step_cdf > u (u: 53 Philox bits, tag GCCB_TAG_STEP; step_cdf: n_steps <= 3 host
 * doubles, read at the call, last = 1) and writes in seeds_k[i] the end of a `step`-hop uniform walk from
 * seeds_q[i] (hop h drawn with tag GCCB_TAG_KHOP, hop field h); a vertex without neighbours ends the walk.
 * One thread per sample, no workspace, no host sync.                                                      */
int gccb_pair_seeds(const gccb_graph_t* graph, const double* step_cdf, int32_t n_steps, const int64_t* seeds_q,
                    const int64_t* sample_ids, int32_t count, int64_t* seeds_k, gccb_stream_t stream);

/* gccb_sample_batch with separate view seeds (graph_dataset.py:113-130 with step > 0): view 0 walks from
 * and induces around seeds_q[i], view 1 around seeds_k[i] (its row 0); BOTH walk budgets come from
 * seeds_q[i]'s degree.  Workspace: gccb_sample_batch_workspace.                                            */
int gccb_sample_batch_pairs(const gccb_graph_t* graph, const int64_t* seeds_q, const int64_t* seeds_k,
                            const int64_t* sample_ids, const gccb_batch_t* batch, void* workspace,
                            size_t workspace_bytes, gccb_stream_t stream);

/* Neighbour-sampled ego-nets (aug="ns", graph_dataset.py:131-162).  View 0 from seeds_q[i], view 1 from
 * seeds_k[i] (pass seeds_q twice for step_dist [1,0,0]).  Layer 0 = {seed}; layer h = the de-duplicated
 * union over the vertices u of layer h-1 of all neighbour entries of u if deg(u) <= num_neighbors, else
 * num_neighbors distinct entries drawn uniformly without replacement, for num_hops layers (early stop when a
 * layer is empty or the union is closed under neighbourhood).  Node set = [seed, union minus seed ascending],
 * then the same induced sub-CSR, sub_deg, graph_id, orig_id and flags as gccb_sample_batch; counters =
 * (n, m, layers expanded, sum of parent degrees).  An ego-net holds at most gccb_ns_ego_cap(num_neighbors)
 * vertices (shared memory: 4096 at num_neighbors = 5); a larger one, like a view over node_cap / edge_cap,
 * raises GCCB_FLAG_NODE_OVERFLOW and its view is published empty.  node_cap <= 2^31 / 256 - 2.  The graph's
 * budget table and restart threshold are not read.                                                        */
int32_t gccb_ns_ego_cap(int32_t num_neighbors);
size_t gccb_ns_batch_workspace(int32_t batch, int32_t num_neighbors, int32_t edge_cap);
int gccb_ns_batch(const gccb_graph_t* graph, const int64_t* seeds_q, const int64_t* seeds_k,
                  const int64_t* sample_ids, int32_t num_hops, int32_t num_neighbors, const gccb_batch_t* batch,
                  void* workspace, size_t workspace_bytes, gccb_stream_t stream);

/* Whole-graph batches (entire_graph=True, graph_dataset.py:311-340; dgl.batch, data_util.py:26-32).
 * A set of graphs as one union CSR: graph i owns vertices node_off[i] .. node_off[i+1) and entries
 * edge_off[i] .. edge_off[i+1) (= indptr[node_off[i]] ..), rows as listed (parallel edges, self loops and
 * isolated vertices are kept), `indices` holding union vertex ids.  Each graph must already be relabelled
 * seed first: row 0 is the seed.                                                                          */
typedef struct {
  const int64_t* indptr;   /* [n_nodes+1] union CSR row offsets      */
  const int32_t* indices;  /* [nnz] union vertex ids                 */
  const int64_t* node_off; /* [n_graphs+1] first vertex of graph i   */
  const int64_t* edge_off; /* [n_graphs+1] first entry of graph i    */
  int64_t n_graphs;
} gccb_graph_set_t;

/* Both views of `batch` = the graphs graph_ids[0..B) (device int64, clamped to the set), identical:
 * node_off / edge_off, view-local indptr / indices, sub_deg = row length, graph_id, orig_id = the view-local
 * row, counters (n, m, 0, 0).  A view that exceeds node_cap / edge_cap raises GCCB_FLAG_NODE_OVERFLOW /
 * GCCB_FLAG_EDGE_OVERFLOW and is published empty (node_off[v][B] = edge_off[v][B] = -1), as in
 * gccb_sample_batch.  No workspace, no host sync.                                                       */
int gccb_gather_graphs(const gccb_graph_set_t* set, const int64_t* graph_ids, const gccb_batch_t* batch,
                       gccb_stream_t stream);

/* The graph set relabelled seed first, from `set` as given (indptr, indices, node_off read; edge_off is not: the
 * output keeps the input's edge offsets).  n_nodes = node_off[n_graphs] <= 2^31 and n_edges = indptr[n_nodes] are
 * the caller's host copies.  Per graph of n vertices: the seed s is its first vertex of maximum row length (parallel
 * edges and self loops count); the new row order is [s, 0..s-1, s+1..n-1]; old local id u becomes 0 if u == s, u + 1
 * if u < s and u otherwise.  Writes seeds[n_graphs] (local ids; 0 for a graph without vertices), out_indptr
 * [n_nodes+1] and out_indices[n_edges], in union ids.  Rows must be non-decreasing (gccb_graph_t) and name vertices
 * of their own graph; the relabelled rows are then non-decreasing too, byte for byte what relabelling each graph and
 * sorting its rows gives.  A row that breaks this raises GCCB_FLAG_BAD_ROW in *flags (caller clears), and the
 * output is undefined but written inside its rows.  One read and one write of the CSR; no workspace, no host sync. */
int gccb_seed_first_union(const gccb_graph_set_t* set, int64_t n_nodes, int64_t n_edges, int64_t* seeds,
                          int64_t* out_indptr, int32_t* out_indices, int32_t* flags, gccb_stream_t stream);

/* A5  Laplacian positional features.  Replaces
 * _add_undirected_graph_positional_embedding + eigen_decomposision
 * (data_util.py:242-281): top-k (k = min(n-2, pos_dim)) eigenvectors of
 * D^-1/2 A D^-1/2, ascending, row-L2 normalised, zero-padded to pos_dim.
 * pos: [2][node_cap][pos_dim]; eigvals (optional, may be NULL): [2B][pos_dim]
 * ascending top-k eigenvalues (padding = 0).  normalize=0 returns the raw unit
 * eigenvectors (used by the spectral parity tests).
 * Solvers by ego-net size (device-built work lists, csrc/posenc.cu): a dense tridiagonal
 * solver (Householder -> multisection -> inverse iteration; a direct method) for n <= 96,
 * Chebyshev-filtered subspace iteration above.  The environment variable
 * GCCB200_DENSE_MAX (96 .. 228, read on every call; smaller values act as 96) raises that
 * boundary: 228 = direct-method accuracy up to 228 vertices.
 * workspace: gccb_posenc_workspace(B, node_cap) bytes, 8-byte aligned.
 * Results are deterministic run to run for a given setting.                              */
size_t gccb_posenc_workspace(int32_t batch, int32_t node_cap);
int gccb_posenc(const gccb_batch_t* batch, int32_t pos_dim, int32_t normalize, float* pos,
                float* eigvals, void* workspace, size_t workspace_bytes,
                gccb_stream_t stream);

/* ---- GIN encoder ----------------------------------------------------------------------
 * Replaces GraphEncoder.forward / UnsupervisedGIN.forward (graph_encoder.py:132-200,
 * gin.py:213-232) incl. DGL GINConv('sum', eps buffer = 0) and SumPooling.
 * Parameters live in ONE flat fp32 buffer; gccb_gin_param_layout gives the layout
 * (the Python module maps the reference's state_dict keys onto slices of it).          */
typedef struct {
  int32_t num_layers;  /* L (GIN layers = L-1, prediction heads = L)  train.py:79 */
  int32_t hidden;      /* node_hidden_dim = output_dim                 train.py:90 */
  int32_t pos_dim;     /* positional_embedding_size (32)                            */
  int32_t deg_dim;     /* degree_embedding_size (16)                                */
  int32_t max_degree;  /* 512                                                       */
  int32_t norm;        /* F.normalize on the output (graph_encoder.py:195-196)     */
  float bn_eps;        /* 1e-5 */
  float bn_momentum;   /* 0.1  */
  float norm_eps;      /* 1e-5 */
  float dropout_p;     /* 0.5 (gin.py:202)                                          */
  int32_t tensor_cores; /* 1: the Linear layers of the MLP (gin.py:107-116) and their input / weight
                           gradients run on wgmma tensor cores with bf16 operands and fp32
                           accumulation (hidden >= 128 only; BASELINE config 4); 0: fp32 SIMT  */
  int32_t _pad;
} gccb_gin_cfg_t;

/* offsets (in floats) into the flat parameter buffer; arrays sized for L <= 8 */
typedef struct {
  int64_t w1[8], b1[8], bn1_w[8], bn1_b[8], w2[8], b2[8], bna_w[8], bna_b[8], bnb_w[8], bnb_b[8];
  int64_t wp[8], bp[8];
  int64_t emb;
  int64_t total;     /* number of live floats */
  /* running statistics buffer (separate flat buffer): [layer][bn 0..2][mean|var][hidden] */
  int64_t run_total;
} gccb_gin_layout_t;
int gccb_gin_param_layout(const gccb_gin_cfg_t* cfg, gccb_gin_layout_t* out /* host */);

/* bytes of the activation stash one forward needs for its backward */
size_t gccb_gin_acts_bytes(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap);

/* forward of ONE view.  bn_running/num_batches_tracked are updated (train-mode BN,
 * train.py:357-365) unless bn_train == 0.  dropout: mask layer ids
 * dropout_layer_base+i, Philox (key, step); dropout_layer_base < 0 = eval dropout.
 * feat: [B][hidden]; pooled_out (optional): [L][B][hidden] (all_outputs).               */
int gccb_gin_forward(const gccb_gin_cfg_t* cfg, const gccb_batch_t* batch, int32_t view,
                     const float* pos, const float* params, float* bn_running,
                     int64_t* num_batches_tracked, int32_t bn_train, uint64_t dropout_key,
                     uint64_t dropout_step, int32_t dropout_layer_base, void* acts,
                     size_t acts_bytes, float* feat, float* pooled_out, gccb_stream_t stream);

/* backward of ONE view (loss.backward(), train.py:408): grads += d loss / d params
 * (flat, same layout; caller zeroes before the first view).  The dropout arguments must
 * repeat the forward's.                                                                 */
size_t gccb_gin_backward_workspace(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap);
int gccb_gin_backward(const gccb_gin_cfg_t* cfg, const gccb_batch_t* batch, int32_t view,
                      const float* params, const void* acts, const float* dfeat, float* grads,
                      uint64_t dropout_key, uint64_t dropout_step, int32_t dropout_layer_base,
                      void* workspace, size_t workspace_bytes, gccb_stream_t stream);

/* Where the intermediates live, for tests and diagnostics (host-only query, no device work).
 * Forward fields: byte offsets into the activation stash of gccb_gin_forward (x0 float [node_cap][64];
 * a[l] float [node_cap][64 (l = 0) or hidden]; z1/z2/h[l] float [node_cap][hidden]; stats double
 * [L-1][3][2][hidden]; pooled float [L][B][PW]; a16 bf16 = a of the last layer run; x16 bf16 = its
 * relu(bn1(z1)); w16[l] bf16 W1 [hidden][KW] | W2 | W1^T [KW][hidden] | W2^T, KW = 64 (l = 0) or hidden).
 * Backward fields: byte offsets into the workspace of gccb_gin_backward (dh, da float [node_cap][DW];
 * g1/dz2[l & 1] float [node_cap][hidden], g1 ends as dz1; dpool float [L][B][DW]; coef1 float
 * [L-1][sc | sh][hidden]; dz16 bf16 [node_cap][hidden]; tA bf16 [hidden][cap_pad], tB bf16 [DW][cap_pad]).
 * A field the configuration does not have is -1 (every tensor-core field when cfg selects the fp32 path). */
typedef struct {
  int64_t x0, a[8], z1[8], z2[8], h[8], stats, pooled, a16, x16, w16[8];
  int64_t dh, g1[2], dz2[2], da, dpool, coef1, dz16, tA, tB;
  int32_t cap_pad;   /* rows of the transposed weight-gradient operands (node_cap rounded up to 64) */
  int32_t splits;    /* split-K partitions of the weight-gradient GEMMs                            */
  int32_t DW;        /* row width of dh / da / dpool = max(hidden, 64)                             */
  int32_t PW;        /* row width of pooled = max(hidden, 64)                                      */
} gccb_gin_stash_t;
int gccb_gin_stash_layout(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap,
                          gccb_gin_stash_t* out /* host */);

/* ---- GAT encoder (--model gat) ----------------------------------------------------------
 * Replaces GraphEncoder.forward with gnn_model="gat" (graph_encoder.py:132-200): UnsupervisedGAT
 * (gat.py: num_layers DGL GATLayers, flatten, leaky_relu(0.01) between layers), dgl Set2Set and
 * lin_readout, fp32.  The input X0 is the GIN path's.  Semantics as restated in DESIGN.md (GAT section).
 * Every graph of the batch must be symmetric: the in-edges of v are row v of the batch CSR, and the
 * backward reads the out-edges of u from row u.                                                       */
typedef struct {
  int32_t num_layers;      /* GAT layers, 1..8                        train.py --num-layer         */
  int32_t hidden;          /* H = output_dim, 32 / 64 / 128 / 256                                  */
  int32_t num_heads;       /* 1..8, H % num_heads == 0 (gat.py:20)                                 */
  int32_t pos_dim;         /* as gccb_gin_cfg_t                                                    */
  int32_t deg_dim;
  int32_t max_degree;
  int32_t set2set_iter;    /* Set2Set n_iters >= 1                    --set2set-iter               */
  int32_t set2set_layers;  /* LSTM layers 1..8                        --set2set-lstm-layer         */
  int32_t norm;            /* F.normalize on the output                                            */
  float norm_eps;          /* 1e-5                                                                 */
} gccb_gat_cfg_t;

/* offsets (in floats) into the flat parameter buffer, in this order: per layer fc.weight [H][in],
 * attn_l [nh][F], attn_r; degree_embedding; per LSTM layer weight_ih [4H][in], weight_hh [4H][H],
 * bias_ih [4H], bias_hh [4H] (gate order i, f, g, o); lin_readout.0 weight [H][2H], bias; .2 weight
 * [H][H], bias.  Unused entries are -1.                                                              */
typedef struct {
  int64_t fc[8], attn_l[8], attn_r[8];
  int64_t emb;
  int64_t w_ih[8], w_hh[8], b_ih[8], b_hh[8];
  int64_t ro0_w, ro0_b, ro2_w, ro2_b;
  int64_t total;           /* number of floats, all live */
} gccb_gat_layout_t;
int gccb_gat_param_layout(const gccb_gat_cfg_t* cfg, gccb_gat_layout_t* out /* host */);

/* bytes of the activation stash one forward needs for its backward */
size_t gccb_gat_acts_bytes(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap);
/* forward of ONE view; feat: [B][hidden].  No running state, no dropout.                            */
int gccb_gat_forward(const gccb_gat_cfg_t* cfg, const gccb_batch_t* batch, int32_t view, const float* pos,
                     const float* params, void* acts, size_t acts_bytes, float* feat, gccb_stream_t stream);
/* backward of ONE view: grads += d loss / d params (flat, same layout; caller zeroes before the first
 * view).  acts: the stash of the forward of the same view and parameters.                            */
size_t gccb_gat_backward_workspace(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap);
int gccb_gat_backward(const gccb_gat_cfg_t* cfg, const gccb_batch_t* batch, int32_t view, const float* params,
                      const void* acts, const float* dfeat, float* grads, void* workspace, size_t workspace_bytes,
                      gccb_stream_t stream);

/* Where the intermediates live (host-only query).  Forward, byte offsets into the stash: x0 float
 * [node_cap][64]; z[l], h[l] float [node_cap][hidden] (h = the layer's output after its activation);
 * att[l] float [4][node_cap][nh]: el | er | max | denominator of the edge softmax of each (row, head);
 * qstar float [T+1][B][2H] (q* before each iteration, [0] = 0); hs, cs float [T+1][K][B][H] (LSTM h and c
 * after each iteration, [0] = 0); gates float [T][K][B][4H] (i, f, g, o after their activations); alpha
 * float [T][node_cap] (Set2Set attention); y1 float [B][H] (relu of lin_readout.0); score float [B][H]
 * (before the normalisation).  Backward, byte offsets into the workspace: dh float [node_cap][hidden]
 * (gradient of the layer output being processed; of the top layer after the Set2Set backward); dz, dout
 * float [node_cap][hidden]; sv float [2][node_cap][nh] (sum of a * da | gradient of er); dx0 float
 * [node_cap][64]; dgates float [T][K][B][4H] (pre-activation gate gradients); dy float [B][2][H]
 * (lin_readout.0 | .2 output gradients).                                                              */
typedef struct {
  int64_t x0, z[8], h[8], att[8], qstar, hs, cs, gates, alpha, y1, score;
  int64_t dh, dz, dout, sv, dx0, dgates, dy;
} gccb_gat_stash_t;
int gccb_gat_stash_layout(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap,
                          gccb_gat_stash_t* out /* host */);

/* ---- contrastive head ------------------------------------------------------------------ */
/* MemoryMoCo.forward logits (memory_moco.py:33-44): out[B][K+1] = [q.k | q.memory^T] / T */
int gccb_moco_logits(const float* q, const float* k, const float* memory, int32_t B,
                     int32_t d, int32_t K, float T, float* out, gccb_stream_t stream);
/* backward of the above w.r.t. q (k and the queue are detached, memory_moco.py:28,37)    */
int gccb_moco_logits_backward(const float* dout, const float* k, const float* memory,
                              int32_t B, int32_t d, int32_t K, float T, float* dq,
                              gccb_stream_t stream);
/* NCESoftmaxLoss / NCESoftmaxLossNS (criterions.py:12-17, :27-33): mean CE of out[B][C]
 * against label 0 (label_mode 0) or arange(B) (label_mode 1).  dout optional.            */
int gccb_nce_loss(const float* out, int32_t B, int32_t C, int32_t label_mode, float* loss,
                  float* dout, gccb_stream_t stream);
/* fused InfoNCE: loss and dq in one pass over the queue, logits never materialised.
 * stats[0] = loss, stats[1] = mean positive logit ("prob", train.py:394).
 * d must be 32, 64, 128 or 256 (the encoder widths): other widths return GCCB_ERR_BADARG,
 * and gccb_infonce_workspace returns 0 for them.  d >= 128 with B >= 128 and K a multiple
 * of 64 runs on the tensor cores (bf16 operands, fp32 softmax); every other shape runs the
 * fp32 tiled kernel.                                                                     */
size_t gccb_infonce_workspace(int32_t B, int32_t d, int32_t K);
int gccb_infonce_fused(const float* q, const float* k, const float* memory, int32_t B,
                       int32_t d, int32_t K, float T, float* stats, float* dq, void* workspace,
                       size_t workspace_bytes, gccb_stream_t stream);
/* FIFO enqueue (memory_moco.py:55-61): memory[(index+i) % K] = k[i]; the write pointer is
 * a device int64 (*index_dev) advanced by parts*B (mod K).  parts > 1: `parts` blocks of B keys,
 * block r at k + r*part_stride floats (every rank's keys inside the gathered exchange buffer, in
 * rank order -> identical queues on all ranks).  skip_word (optional, device): the call is a no-op
 * when (*skip_word & skip_mask) != 0 -- pass gccb_batch_t.flags with
 * GCCB_FLAG_NODE_OVERFLOW|GCCB_FLAG_EDGE_OVERFLOW so that a batch published empty never reaches
 * the queue.                                                                                      */
int gccb_moco_enqueue(float* memory, const float* k, int32_t B, int32_t d, int32_t K,
                      int64_t* index_dev, int32_t parts, int64_t part_stride,
                      const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream);
/* E2E head (train.py:397-401, criterions.py:27-33): out = k q^T / T, CE vs arange;
 * returns loss, mean diagonal logit, dq and dk.                                          */
int gccb_e2e_nce(const float* q, const float* k, int32_t B, int32_t d, float T, float* stats,
                 float* dq, float* dk, void* workspace /* B*B floats */, size_t workspace_bytes,
                 gccb_stream_t stream);

/* ---- optimiser ------------------------------------------------------------------------- */
/* clip_grad_norm_ (train.py:340-347,409) + Adam with L2 weight decay (train.py:417,667-672)
 * on the first n_live floats, then moment_update (train.py:169-172,430-431) of p_ema over
 * n_all floats (alpha < 0 skips the EMA).  hyper (device, 4 floats): lr, 1-beta1^t,
 * sqrt(1-beta2^t), unused.  grad_norm_out: device float (pre-clip total norm).
 * grad_scale multiplies the gradient first (1/world for data-parallel averaging).
 * skip_word / skip_mask: as for gccb_moco_enqueue -- the whole update (moments, weights, momentum
 * encoder) is a no-op for a step whose batch was published empty.                         */
int gccb_clip_adam_ema(float* p, float* g, float* m, float* v, float* p_ema, int64_t n_live,
                       int64_t n_all, const float* hyper, float beta1, float beta2, float eps,
                       float weight_decay, float clip_norm, float alpha, float grad_scale,
                       float* grad_norm_out, double* workspace /* 1 double */,
                       const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream);
/* The same clip, EMA, grad_scale and skip word with torch.optim.SGD (dampening 0, no Nesterov;
 * train.py:659-665) as the update: d = clipped g + weight_decay * p; buf = momentum * buf + d;
 * p -= lr * buf.  buf (n_live floats) starts at zero, which equals torch's first-step copy of d.
 * With momentum == 0 the update is p -= lr * d and buf may be NULL.  hyper[0] = lr.          */
int gccb_clip_sgd_ema(float* p, float* g, float* buf, float* p_ema, int64_t n_live, int64_t n_all,
                      const float* hyper, float momentum, float weight_decay, float clip_norm, float alpha,
                      float grad_scale, float* grad_norm_out, double* workspace /* 1 double */,
                      const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream);
/* ... with torch.optim.Adagrad (initial_accumulator_value 0; train.py:673-678) as the update:
 * sum += d * d; p -= clr * d / (sqrt(sum) + eps).  sum (n_live floats) starts at zero.
 * hyper[0] = clr = lr / (1 + (t - 1) * lr_decay) for step t.                                  */
int gccb_clip_adagrad_ema(float* p, float* g, float* sum, float* p_ema, int64_t n_live, int64_t n_all,
                          const float* hyper, float eps, float weight_decay, float clip_norm, float alpha,
                          float grad_scale, float* grad_norm_out, double* workspace /* 1 double */,
                          const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream);
/* deterministic rank-ordered sum of `world` gathered gradient buffers: out = sum_r in[r].
 * any_flag_out (optional, device int): set to 1 when gathered[r*stride + flag_index] != 0 for any
 * rank r (a rank whose batch overflowed), else 0 -- the skip word of gccb_moco_enqueue and of the
 * optimiser calls above when
 * world > 1, so that all replicas skip the same steps and stay identical.                    */
int gccb_sum_ranks(const float* gathered, int32_t world, int64_t stride, int64_t n, float* out,
                   int64_t flag_index, int32_t* any_flag_out, gccb_stream_t stream);

/* ---- supervised finetuning (csrc/finetune.cu) ------------------------------------------------------
 * Classification head (train.py:219-241): logits = feat W^T + bias over the first b rows of feat [B][H],
 * W [C][H], bias [C]; row i's label is labels[item_ids[i]] (device int64 tables, ids clamped to n_items).
 * stats (device, 3 floats): mean cross-entropy (max-subtracted log-sum-exp), the count of rows whose FIRST
 * maximum logit is the label (torch.argmax's tie rule; correct / b is the micro-F1), b.  Unless eval != 0 also
 * dlogits = (softmax - onehot(y)) / b, dfeat [b][H] = dlogits W, dW [C][H] = dlogits^T feat, db [C] = column sums
 * of dlogits.  H in {32, 64, 128, 256}, 2 <= C <= 128, 0 < b <= B <= 4096, else GCCB_ERR_BADARG.  No float
 * atomics: every sum over rows runs in a fixed order, so the call is bit-identical from run to run.          */
size_t gccb_ft_head_workspace(int32_t B, int32_t C);
int gccb_ft_head(const float* feat, int32_t B, int32_t b, int32_t H, int32_t C, const float* W, const float* bias,
                 const int64_t* item_ids, const int64_t* labels, int64_t n_items, int32_t eval, float* dfeat,
                 float* dW, float* db, float* stats, void* workspace, size_t workspace_bytes, gccb_stream_t stream);
/* clip_grad_value_(params, clip_value) (train.py:227-228) then the optimiser step over n floats: g is clamped to
 * [-clip_value, clip_value] (g itself is not written), then the update of gccb_clip_{adam,sgd,adagrad}_ema after
 * its norm clip -- the same weight decay, state buffers and `hyper` layout.  No EMA, no norm.  skip_word /
 * skip_mask: as for gccb_moco_enqueue, the call is a no-op for a batch published empty.                      */
int gccb_clip_value_adam(float* p, const float* g, float* m, float* v, int64_t n, const float* hyper, float beta1,
                         float beta2, float eps, float weight_decay, float clip_value, const int32_t* skip_word,
                         int32_t skip_mask, gccb_stream_t stream);
int gccb_clip_value_sgd(float* p, const float* g, float* buf, int64_t n, const float* hyper, float momentum,
                        float weight_decay, float clip_value, const int32_t* skip_word, int32_t skip_mask,
                        gccb_stream_t stream);
int gccb_clip_value_adagrad(float* p, const float* g, float* sum, int64_t n, const float* hyper, float eps,
                            float weight_decay, float clip_value, const int32_t* skip_word, int32_t skip_mask,
                            gccb_stream_t stream);
/* Positional features of a whole-graph batch built by gccb_gather_graphs from `set`, copied from a per-vertex
 * cache [total vertices of set][pos_dim]: row r of batch graph g in view `view` gets cache row
 * set->node_off[graph_ids[g]] + (r - batch->node_off[view][g]).  pos is [2][node_cap][pos_dim].  A view published
 * empty is left alone.  No workspace, no host sync.                                                          */
int gccb_gather_features(const gccb_graph_set_t* set, const int64_t* graph_ids, const gccb_batch_t* batch,
                         int32_t view, const float* cache, int32_t pos_dim, float* pos, gccb_stream_t stream);

/* ---- corpus builder: edge-list text -> directed keys (csrc/edgelist.cu) ------------------------------------
 * Replaces the per-line loop of yuxiao_kdd17_graph_to_dgl (gcc/utils/x2dgl.py:28-47).  The caller streams a file
 * through gccb_edgelist_parse in chunks of whole lines (each chunk ends at a '\n', except the file's last one) and
 * gets, in file line order, two int64 keys per edge line that is not a self loop: min*n + max, then max*n + min.
 * Tokens are runs of characters other than ' ', '\t', '\r'; an integer token is -?[0-9]+ within int64.
 *   GCCB_EL_LSCC:  line 0's second token is n, lines 1..n are skipped, line n+1's second token is m, then m lines
 *                  of exactly three integers "u v w" (w is ignored; an overflow of w is not an error); later lines
 *                  are ignored.  0 <= n < 2^31.  Keys use the multiplier n.
 *   GCCB_EL_PLAIN: every line "u v [anything]"; blank lines and lines whose first token starts with '#' or '%' are
 *                  skipped.  n = 1 + the largest id of an edge that is not a self loop.  The parse uses the
 *                  multiplier 2^31 (ids must be below it); gccb_edgelist_finish rewrites the keys to s*n + d.
 * An id of an edge that is not a self loop must lie in [0, n).  Errors never fault: state.first_error holds
 * (line << 4) | kind of the offending line with the smallest 0-based index, error_flags the OR of 1 << kind.
 * The state lives at the start of the workspace; the caller reads it back after gccb_edgelist_finish.
 * Deterministic: no key's slot depends on an atomic.                                                      */
#define GCCB_EL_LSCC 0
#define GCCB_EL_PLAIN 1
#define GCCB_EL_ERR_TOKENS 1    /* wrong token count (.lscc edge line != 3, header < 2, plain < 2)        */
#define GCCB_EL_ERR_CHAR 2      /* a read token is not -?[0-9]+                                             */
#define GCCB_EL_ERR_RANGE 3     /* id < 0 or >= n (plain: >= 2^31); header n or m < 0 or >= 2^31           */
#define GCCB_EL_ERR_OVERFLOW 4  /* an id outside int64                                                      */
#define GCCB_EL_ERR_SHORT 5     /* .lscc: the header or fewer than m edge lines (line = the first missing)  */
#define GCCB_EL_ERR_CAPACITY 6  /* more keys than keys_cap                                                  */
typedef struct {
  int64_t lines;          /* lines parsed so far                                                    */
  int64_t n;              /* .lscc: header n (-1 unread, -2 bad); plain: 1 + largest id so far     */
  int64_t m;              /* .lscc: header m (-1 unread, -2 bad)                                    */
  int64_t edge_lines;     /* edge lines read, self loops included (.lscc: at most m)                */
  int64_t keys;           /* keys written                                                           */
  uint64_t first_error;   /* (line << 4) | GCCB_EL_ERR_*; all ones = none                           */
  int32_t error_flags;
  int32_t _pad;
} gccb_edgelist_state_t;
/* workspace for chunks of up to chunk_bytes bytes: about 8 * chunk_bytes (a 64-bit offset per possible line) */
size_t gccb_edgelist_workspace(int64_t chunk_bytes);
/* resets the state for a new file */
int gccb_edgelist_begin(int32_t format, void* workspace, size_t workspace_bytes, gccb_stream_t stream);
/* one chunk of nbytes bytes of device text; keys: [keys_cap] output of the whole file, appended at state.keys */
int gccb_edgelist_parse(const char* text, int64_t nbytes, int32_t format, int64_t* keys, int64_t keys_cap,
                        void* workspace, size_t workspace_bytes, gccb_stream_t stream);
/* after the last chunk: .lscc records missing header or edge lines; plain rewrites the keys to s*n + d */
int gccb_edgelist_finish(int32_t format, int64_t* keys, void* workspace, size_t workspace_bytes,
                         gccb_stream_t stream);

/* ---- tensor-core contraction (wgmma + TMA; csrc/tc_gemm.cu) ---------------------------------------
 * The dense products of the path at hidden >= 128 (BASELINE config 4): the GIN MLP's Linear layers
 * (gcc/models/gin.py:107-116) with the BatchNorm column statistics of :115 fused into the epilogue,
 * their input / weight gradients, and the MoCo logits q.queue^T (gcc/contrastive/memory_moco.py:33-44).
 *   out[M x N] = alpha * A[M x K] . B[N x K]^T (+ bias[N])
 * A [M_cap][K] and B [N][K]: bf16, row-major (K contiguous), 16-byte aligned; K % 64 == 0, N % 32 == 0.
 * m_dev (optional): device int with the number of valid rows (<= M_cap), so the row count of a sampled
 * batch never comes back to the host.  out_f32 / out_bf16: [M_cap][ldo] (either may be NULL).
 * colstats (optional): double [2][N], += column sums / sums of squares of the stored values over the
 * valid rows.  splits > 1: split-K over CTAs; the partial products go to `scratch`, which must hold
 * splits * M_cap * N floats (row pitch N), and are added in a fixed order; colstats must be NULL.  A row
 * pitch ldo that is not a multiple of 8 also goes through `scratch` (M_cap * N floats, splits = 1).    */
int gccb_tc_gemm_bf16(const void* A, const void* B, int32_t M_cap, int32_t N, int32_t K,
                      const int32_t* m_dev, const float* bias, float alpha, float* out_f32,
                      void* out_bf16, int32_t ldo, double* colstats, int32_t splits, float* scratch,
                      gccb_stream_t stream);
/* fp32 [rows][lds] -> bf16 [rows_pad][cols_pad] (transpose = 0) or [cols_pad][rows_pad] (transpose = 1),
 * zero padded; rows_dev (optional): device int, rows beyond it are written as zeros.                 */
int gccb_cast_bf16(const float* src, int32_t rows, int32_t cols, int32_t lds, void* dst, int32_t rows_pad,
                   int32_t cols_pad, int32_t transpose, const int32_t* rows_dev, gccb_stream_t stream);

/* ---- embedding baselines in float64 (csrc/baselines.cu) -------------------------------------------
 * GraphWave (gcc/models/emb/_graphwave) and ProNE (gcc/models/emb/prone.py) for the frozen-embedding
 * tasks.  A graph is a symmetric CSR: indptr [n+1], indices [nnz] ascending per row, and vals [nnz]
 * (NULL: each entry weighs 1, a repeated column being a parallel edge).  Dense blocks are n x k
 * row-major with row stride ld.  Blocks whose rows all start on 16 bytes (16-byte aligned base pointers and
 * an even ld) take the 128-bit path, any other layout the 64-bit one; the results are the same.
 *
 * Y = alpha * dr * ((A + sigma I) (dc X)) + beta X + gamma Z; dr, dc, Z may be NULL (1, 1, no term).
 * Y may alias Z, not X.                                                                                */
int gccb_spmm_f64(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n, int32_t k,
                  int64_t ld, double alpha, double sigma, const double* dr, const double* dc, double beta,
                  const double* X, double gamma, const double* Z, double* Y, gccb_stream_t stream);
/* GraphWave's chi [n][4 n_times]: row u holds, per scale s and time point t, (1/n) sum_i cos and sin of
 * times[t] * heat_s[i,u], heat_s = sum_k cheb[s*(order+1)+k] T_k(L - I) with L the normalised Laplacian and
 * entries <= 1e-4/n set to 0.  cheb (host, [2][order+1]) and times (host, [n_times <= 64]) come from the
 * caller.  The heat is built bc identity columns at a time in a workspace of
 * gccb_graphwave_workspace(n, bc) bytes and never held whole; the result does not depend on bc.       */
size_t gccb_graphwave_workspace(int64_t n, int32_t bc);
int gccb_graphwave(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                   const double* cheb, int32_t order, const double* times, int32_t n_times, int32_t bc,
                   void* workspace, size_t workspace_bytes, double* chi, gccb_stream_t stream);
/* ProNE's sparse factorization on A's pattern: F[e] = log(A_ij / d_i) - log(A_ij neg_j) for entry e =
 * (i, j), d the row sums, neg_j = (sum_i A_ij / d_i)^0.75 normalised to sum 1; FT[e] = F_ji, the entries
 * of F^T on the same (symmetric) pattern.                                                            */
size_t gccb_prone_factor_workspace(int64_t n);
int gccb_prone_factor(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                      void* workspace, size_t workspace_bytes, double* F, double* FT, gccb_stream_t stream);
/* out [rows][cols]: standard normals by Box-Muller on Philox counters (row, col, 0, GCCB_TAG_PRONE),
 * key = run seed: the start block of ProNE's randomized SVD.                                         */
int gccb_gaussian_f64(double* out, int64_t rows, int32_t cols, uint64_t key, gccb_stream_t stream);
/* ProNE's spectral propagation of a [n][k] (order >= 2, bessel (host) = I_0 .. I_{order-1} at theta):
 * M = (1 - mu) I - DA with DA = (I + A) row-l1-normalised, Chebyshev terms Lx_i, conv = sum of
 * +-2 I_i Lx_i (I_0 a for i = 0), mm [n][k] = (I + A)(a - conv).                                     */
size_t gccb_prone_propagate_workspace(int64_t n, int32_t k);
int gccb_prone_propagate(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                         const double* a, int32_t k, double mu, const double* bessel, int32_t order,
                         void* workspace, size_t workspace_bytes, double* mm, gccb_stream_t stream);

/* ---- structural similarity search: exact cosine top-k (csrc/knn.cu) ---------------------------------------
 * The reference's evaluator (gcc/tasks/similarity_search.py) ranks with emb_2.dot(v).argsort() on the host; this is
 * the same search at the sizes generate.py writes.  queries [nq][dim], cands [nc][dim]: fp32 rows, 1 <= dim <= 512.
 *   normalisation (once per row): zero-pad to d4 = dim rounded up to 4; s = the sequential fmaf chain of x_j x_j over
 *     j = 0 .. d4-1; x^_j = x_j / sqrtf(s), IEEE correctly rounded.  A row with s = 0 stays all zeros, so it scores 0
 *     against everything (the reference divides by a zero norm and gets NaN).  A row holding a NaN or an Inf ORs
 *     GCCB_FLAG_NONFINITE into *flags (caller clears); the results are then undefined.
 *   score(q, c) = the sequential fmaf chain of q^_j c^_j over j = 0 .. d4-1, starting from +0.
 *   result of query i: the first k candidates under (score descending, candidate index ascending), -0 == +0, never
 *     exclude[i]: out_ids [nq][k] (int64) and out_scores [nq][k] (a score of -0 is written as +0), in that order.
 * The order is strict and a score's bits depend on its two rows alone, so the output is a function of the inputs:
 * it does not depend on `splits`, on how the queries are cut into calls, or on the device.
 * exclude: [nq] device int64 or NULL; -1 (or any id outside 0..nc-1) excludes nothing.  1 <= k <= 128 and
 * k <= nc - (exclude != NULL), else GCCB_ERR_BADARG; nc < 2^31.
 * splits: candidate partitions of the score kernel (1 .. 128); 0 chooses them from (nq, nc) so that the grid fills
 * the GPU.  cands == NULL reuses the normalised candidates an earlier call left at the start of the same workspace
 * (same nc and dim), so a caller cutting its queries into several calls normalises the candidates once.
 * Workspace, in bytes, 16-byte aligned, with ds = d4 rounded up to 32, S = the splits used, A(b) = b rounded up to 256:
 *   A(nc * ds * 4)  normalised candidates  +  A(nq * ds * 4)  normalised queries  +  nq * S * k * 8  split lists.
 * gccb_knn_workspace returns 0 for arguments gccb_knn refuses by shape.                                         */
size_t gccb_knn_workspace(int64_t nq, int64_t nc, int32_t dim, int32_t k, int32_t splits);
int gccb_knn(const float* queries, int64_t nq, const float* cands, int64_t nc, int32_t dim, int32_t k,
             const int64_t* exclude, int32_t splits, int64_t* out_ids, float* out_scores, int32_t* flags, void* ws,
             size_t ws_bytes, gccb_stream_t stream);

/* ---- linear-probe classification: exact one-vs-rest logistic regression (csrc/probe.cu) ------------------------
 * The reference's node evaluator (gcc/tasks/node_classification.py) fits OneVsRestClassifier(LogisticRegression(
 * C=1000)) on the host; this is the same model, solved to a stated tolerance, at the sizes generate.py writes.
 *   x [n][d]: fp32 rows, 1 <= d <= 256, each value used exactly in float64.  y [n][c]: 0/1 bytes, 1 <= c <= 1024.
 *   fold [n]: the test fold of each row, 0 .. folds-1 (1 <= folds <= 64); a row with any other id is in no test set
 *   and trains every problem.
 *   Problem p = f c + j (fold f, class j), on the training rows of f (fold id != f), targets t_i = y[i][j]:
 *     minimise 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w.x_i + b))), s_i = 2 t_i - 1, b not penalised.
 *   If every training row has the same target the problem is a constant predictor: decision value +inf or -inf,
 *   status GCCB_PROBE_CONST_POS / _NEG, w = 0.  Otherwise damped Newton in float64 from w = 0, b = 0: the exact
 *   gradient and Hessian [X 1]^T diag(C p (1-p)) [X 1] + diag(I_d, 0), a Cholesky solve, and the first step length
 *   alpha = 2^-m, m = 0..15, with f(w + alpha dw) <= f(w) + 1e-4 alpha g.dw + 1e-12 |f(w)| (the last term absorbs
 *   the rounding of f itself); a pass evaluates four consecutive lengths, and a problem that needs more continues
 *   along the same step in the next pass.  Stop when |g|_inf <= 1e-10 max(1, |g at w = 0|_inf).  A problem still
 *   active after max_iter passes, that finds no step length or that meets a non-positive pivot ORs
 *   GCCB_FLAG_PROBE_NOCONV into *flags.
 *   z(i, j) = the sequential fma chain of w_k x_ik over k = 0 .. d-1 from +0, plus b, with the weights of problem
 *   (fold[i], j): decision values z [n][c] (float64).  Each test row with k labels predicts the k classes of largest
 *   z, ties to the lower class; counts [folds][3] = (tp, fp, fn) per fold.
 *   w [folds c][d + 1]: the weights, b last.  status, gnorm (the final |g|_inf), iters: [folds c].
 * Every sum has a fixed order that depends only on n, d and the problem (row splits chosen from n and merged in
 * order), so the outputs are a function of the inputs: they do not depend on `batch`, the problems per launch
 * (0: all), or on the device.  A row holding a NaN or an Inf ORs GCCB_FLAG_NONFINITE into *flags and the call
 * returns before fitting.  The call reads the count of active problems back to the host once per pass, so it
 * synchronises `stream` and is not graph-capturable.
 * Workspace, in bytes, 16-byte aligned, with P = folds c, B = the problems per launch, d1 = d + 1, D = d1 rounded
 * up to 8, T = (D/8)(D/8 + 1)/2, S = min(64, ceil(n / 65536)), A(b) = b rounded up to 256:
 *   3 A(4P) + A(8) + A(8P) + A(8 folds) + A(8c) + 3 A(8P) + A(8 P d1) + A(8 S B d1) + A(8 S B) + A(32 S B)
 *   + A(512 S B T) + (d > 128 ? A(8 B d1^2) : 0).
 * gccb_probe_workspace returns 0 for shapes gccb_probe_fit refuses.
 * gccb_probe_system: for every problem at the given weights w, the gradient g_out [P][d1], the Hessian h_out
 * [P][d1][d1], the Newton step step_out [P][d1] and the objective f_out [P], as one Newton iteration forms them
 * (status [P] is written: GCCB_PROBE_NOT_PD where the Cholesky meets a non-positive pivot; the step is then
 * undefined; no flag is raised).                                                                                  */
#define GCCB_PROBE_ACTIVE 0
#define GCCB_PROBE_CONVERGED 1
#define GCCB_PROBE_CONST_POS 2
#define GCCB_PROBE_CONST_NEG 3
#define GCCB_PROBE_NOCONV 4
#define GCCB_PROBE_LS_FAIL 5
#define GCCB_PROBE_NOT_PD 6
size_t gccb_probe_workspace(int64_t n, int32_t d, int32_t c, int32_t folds, int32_t batch);
int gccb_probe_fit(const float* x, int64_t n, int32_t d, const uint8_t* y, int32_t c, const int32_t* fold,
                   int32_t folds, double C, int32_t max_iter, int32_t batch, double* w, double* z, int64_t* counts,
                   int32_t* status, double* gnorm, int32_t* iters, int32_t* flags, void* ws, size_t ws_bytes,
                   gccb_stream_t stream);
int gccb_probe_system(const float* x, int64_t n, int32_t d, const uint8_t* y, int32_t c, const int32_t* fold,
                      int32_t folds, double C, int32_t batch, const double* w, double* g_out, double* h_out,
                      double* step_out, double* f_out, int32_t* status, void* ws, size_t ws_bytes,
                      gccb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GCCB200_H_ */
