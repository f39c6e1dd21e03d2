// gat.cu -- GAT encoder forward / backward for one view of a batch (GraphEncoder with gnn_model="gat").
//
// Replaces UnsupervisedGAT (gcc/models/gat.py), dgl Set2Set and lin_readout (graph_encoder.py:124-129,191-196),
// fp32 SIMT.  Per GAT layer (DGL GATConv, feat_drop = attn_drop = 0, no residual):
//   z = X W^T (no bias), el = sum_f z attn_l, er = sum_f z attn_r        gat_proj_kernel (el / er in the epilogue)
//   e(u->v) = leaky_relu(el_u + er_v, 0.2), a = softmax of e over row v   gat_agg_kernel, one warp per row; rows
//   out_v = sum a z_u, h = leaky_relu(out, 0.01) except the last layer      above GCCB_HUB_DEG by the whole CTA
// Set2Set (n_iters T, LSTM layers K): per iteration one gat_lstm_cell_kernel per LSTM layer over the B graphs,
// then gat_s2s_attend_kernel (score, segment softmax, readout r) per graph; lin_readout + F.normalize in
// gat_readout_kernel.  The backward walks the same chain in reverse: readout, BPTT through the T x K cells from
// the stashed gates and cells, the attention-readout gradient into x after every iteration, and per GAT layer
// the edge-softmax backward (two row passes), dX = dz W and the split-K weight gradient of the GIN path.
// The batch graphs are symmetric: the backward visits the out-edges of u as row u.
#include "gin_common.cuh"

namespace gccb {

#define GAT_MAXH 8            // heads
#define GAT_MAXK 8            // LSTM layers
#define GAT_GB 4              // graphs per CTA of the LSTM / readout kernels
// gat_agg_kernel, gat_bwd_attn_kernel and gat_s2s_attend_bwd_kernel declare a minimum of one CTA per SM in their
// launch bounds: with the thread count alone, ptxas held them to 32-80 registers and spilled loop-carried scalars
// (4-20 bytes) to local memory; with it they take 43-108 registers and spill nothing

struct GatDims {
  int L, H, nh, F, P, D, maxdeg, din, T, K, norm;
  float norm_eps;
};

static int gat_dims(const gccb_gat_cfg_t* c, GatDims* d) {
  if (!c) {
    set_last_error("gat: null configuration");
    return GCCB_ERR_BADARG;
  }
  d->L = c->num_layers; d->H = c->hidden; d->nh = c->num_heads; d->P = c->pos_dim; d->D = c->deg_dim;
  d->maxdeg = c->max_degree; d->din = c->pos_dim + c->deg_dim + 1; d->T = c->set2set_iter;
  d->K = c->set2set_layers; d->norm = c->norm; d->norm_eps = c->norm_eps;
  d->F = d->nh > 0 ? d->H / d->nh : 0;
  if (d->L < 1 || d->L > GCCB_MAX_L || (d->H != 32 && d->H != 64 && d->H != 128 && d->H != 256) || d->nh < 1 ||
      d->nh > GAT_MAXH || d->H % d->nh != 0 || d->din > GCCB_DINP || d->P < 2 || d->P > 32 || d->D < 1 ||
      d->maxdeg < 1 || d->T < 1 || d->K < 1 || d->K > GAT_MAXK) {
    set_last_error("gat: unsupported configuration (L=%d H=%d heads=%d pos=%d deg=%d iter=%d lstm=%d): need "
                   "1<=L<=8, H in {32,64,128,256}, 1<=heads<=8 dividing H, pos+deg+1<=64, pos<=32, iter>=1, "
                   "1<=lstm<=8", d->L, d->H, d->nh, d->P, d->D, d->T, d->K);
    return GCCB_ERR_BADARG;
  }
  return GCCB_OK;
}

static GinDims gin_input_dims(const GatDims& d) {     // what the shared X0 / embedding kernels read
  GinDims g{};
  g.P = d.P; g.D = d.D; g.maxdeg = d.maxdeg; g.din = d.din; g.H = d.H; g.L = d.L;
  return g;
}

static void gat_param_layout(const GatDims& d, gccb_gat_layout_t* o) {
  int64_t off = 0;
  auto take = [&](int64_t n) { int64_t r = off; off += n; return r; };
  for (int l = 0; l < 8; ++l) o->fc[l] = o->attn_l[l] = o->attn_r[l] = o->w_ih[l] = o->w_hh[l] = o->b_ih[l] =
      o->b_hh[l] = -1;
  for (int l = 0; l < d.L; ++l) {
    o->fc[l] = take((int64_t)d.H * (l == 0 ? d.din : d.H));
    o->attn_l[l] = take(d.H);
    o->attn_r[l] = take(d.H);
  }
  o->emb = take((int64_t)(d.maxdeg + 1) * d.D);
  for (int k = 0; k < d.K; ++k) {
    o->w_ih[k] = take((int64_t)4 * d.H * (k == 0 ? 2 * d.H : d.H));
    o->w_hh[k] = take((int64_t)4 * d.H * d.H);
    o->b_ih[k] = take(4 * d.H);
    o->b_hh[k] = take(4 * d.H);
  }
  o->ro0_w = take((int64_t)d.H * 2 * d.H);
  o->ro0_b = take(d.H);
  o->ro2_w = take((int64_t)d.H * d.H);
  o->ro2_b = take(d.H);
  o->total = off;
}

struct GatActs {
  size_t x0, z[GCCB_MAX_L], h[GCCB_MAX_L], att[GCCB_MAX_L], qstar, hs, cs, gates, alpha, y1, score, total;
};

static GatActs gat_acts_layout(const GatDims& d, int B, int cap) {
  GatActs a{};
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  a.x0 = take((size_t)cap * GCCB_DINP * 4);
  for (int l = 0; l < d.L; ++l) {
    a.z[l] = take((size_t)cap * d.H * 4);
    a.h[l] = take((size_t)cap * d.H * 4);
    a.att[l] = take((size_t)4 * cap * d.nh * 4);
  }
  a.qstar = take((size_t)(d.T + 1) * B * 2 * d.H * 4);
  a.hs = take((size_t)(d.T + 1) * d.K * B * d.H * 4);
  a.cs = take((size_t)(d.T + 1) * d.K * B * d.H * 4);
  a.gates = take((size_t)d.T * d.K * B * 4 * d.H * 4);
  a.alpha = take((size_t)d.T * cap * 4);
  a.y1 = take((size_t)B * d.H * 4);
  a.score = take((size_t)B * d.H * 4);
  a.total = off;
  return a;
}

struct GatBwd {
  size_t dh, dz, dout, sv, dx0, dgates, dy, dup[2], dqtop, dhs, dcs, dal, part, gbias, total;
};

static GatBwd gat_bwd_layout(const GatDims& d, int B, int cap) {
  GatBwd b{};
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const int KQ = d.H > GCCB_DINP ? d.H : GCCB_DINP;
  b.dh = take((size_t)cap * d.H * 4);
  b.dz = take((size_t)cap * d.H * 4);
  b.dout = take((size_t)cap * d.H * 4);
  b.sv = take((size_t)2 * cap * d.nh * 4);
  b.dx0 = take((size_t)cap * GCCB_DINP * 4);
  b.dgates = take((size_t)d.T * d.K * B * 4 * d.H * 4);
  b.dy = take((size_t)B * 2 * d.H * 4);
  for (int i = 0; i < 2; ++i) b.dup[i] = take((size_t)B * 2 * d.H * 4);
  b.dqtop = take((size_t)B * d.H * 4);
  b.dhs = take((size_t)d.K * B * d.H * 4);
  b.dcs = take((size_t)d.K * B * d.H * 4);
  b.dal = take((size_t)cap * 4);
  b.part = take((size_t)GCCB_WG_CHUNKS * ((size_t)d.H * KQ + d.H) * 4);
  b.gbias = take((size_t)d.H * 4);
  b.total = off;
  return b;
}

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lrelu(float x, float slope) { return x > 0.f ? x : slope * x; }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// sums over the 8 warps of a 256-thread CTA; every thread gets the result.  v must be warp-uniform or a lane partial
__device__ __forceinline__ float block_sum8(float v, float* sm) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) r += sm[i];
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_max8(float v, float* sm) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sm[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) r = fmaxf(r, sm[i]);
  __syncthreads();
  return r;
}

// Per-lane head totals: v[j] belongs to column c = lane + 32 j of head c / F (F a power of two).  On return v[j] is
// the sum over all columns of that head.
template <int PER>
__device__ __forceinline__ void head_sum(float (&v)[PER], int F) {
#pragma unroll
  for (int j = 0; j < PER; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      if (o < F) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  if (F > 32) {
    const int G = F / 32;                            // 32-column groups per head
    float t[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      t[j] = 0.f;
#pragma unroll
      for (int jj = 0; jj < PER; ++jj)
        if (jj / G == j / G) t[j] += v[jj];
    }
#pragma unroll
    for (int j = 0; j < PER; ++j) v[j] = t[j];
  }
}

// Online max / sum of exp over the edges [beg, end) of row v, lanes across edges, per head; every lane gets the
// warp's result.  erv: er of row v per head (shared memory).
__device__ __forceinline__ void gat_softmax_range(const int32_t* __restrict__ indices, int beg, int end, int lane,
                                                  int nh, const float* __restrict__ el, const float* erv,
                                                  float (&m)[GAT_MAXH], float (&s)[GAT_MAXH]) {
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) { m[h] = -INFINITY; s[h] = 0.f; }
  for (int e = beg + lane; e < end; e += 32) {
    const int u = indices[e];
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < nh) {
        const float x = lrelu(el[(size_t)u * nh + h] + erv[h], 0.2f);
        if (x > m[h]) { s[h] = s[h] * expf(m[h] - x) + 1.f; m[h] = x; }
        else s[h] += expf(x - m[h]);
      }
  }
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h)
    if (h < nh) {
      const float M = warp_max(m[h]);
      s[h] = warp_sum(m[h] == -INFINITY ? 0.f : s[h] * expf(m[h] - M));
      m[h] = M;
    }
}

// acc[j] += sum over [beg, end) of a(u->v) z_u[c]; co: er_v | max | 1/denominator of row v per head (shared)
template <int H>
__device__ __forceinline__ void gat_agg_range(const int32_t* __restrict__ indices, int beg, int end, int lane, int nh,
                                              int F, const float* __restrict__ el, const float* __restrict__ z,
                                              const float* co, float (&acc)[H / 32]) {
  constexpr int PER = H / 32;
  int hd[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) hd[j] = (lane + 32 * j) / F;
  for (int e = beg; e < end; ++e) {
    const int u = indices[e];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int h = hd[j];
      const float a = expf(lrelu(el[(size_t)u * nh + h] + co[h], 0.2f) - co[GAT_MAXH + h]) * co[2 * GAT_MAXH + h];
      acc[j] = fmaf(a, z[(size_t)u * H + lane + 32 * j], acc[j]);
    }
  }
}

// z = X W^T for 64-row tiles (X rows of K floats, W [H][in], in <= K), z stored, then el / er from the tile in
// shared memory.  Dynamic shared memory: As [64][K+1] | Ws [KC][H+4] | Zs [64][H+1].
template <int K, int H>
__global__ void __launch_bounds__(256)
gat_proj_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ X,
                const float* __restrict__ W, int in, const float* __restrict__ attn_l,
                const float* __restrict__ attn_r, int nh, float* __restrict__ z, float* __restrict__ el,
                float* __restrict__ er) {
  using TC = TileCols<H>;
  GCCB_DYN_SMEM(float, sm);
  float* As = sm;
  float* Ws = As + GCCB_TILE_ROWS * (K + 1);
  float* Zs = Ws + GCCB_KC * (H + 4);
  const int N = max(node_off_v[B], 0), F = H / nh;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int row0 = blockIdx.x * GCCB_TILE_ROWS; row0 < N; row0 += gridDim.x * GCCB_TILE_ROWS) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < GCCB_TILE_ROWS * K; idx += blockDim.x) {
      const int r = idx / K, k = idx - r * K;
      As[r * (K + 1) + k] = row0 + r < N ? X[(size_t)(row0 + r) * K + k] : 0.f;
    }
    __syncthreads();
    float acc[4][TC::CPT];
    tile_gemm<H>(As, K + 1, K, Ws, [&](int k, int c) { return k < in ? W[(size_t)c * in + k] : 0.f; }, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) {
        const int col = TC::col(tx, c);
        Zs[r * (H + 1) + col] = acc[i][c];
        if (row0 + r < N) z[(size_t)(row0 + r) * H + col] = acc[i][c];
      }
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < GCCB_TILE_ROWS * nh; idx += blockDim.x) {
      const int r = idx / nh, h = idx - r * nh;
      if (row0 + r >= N) continue;
      float sl = 0.f, sr = 0.f;
      for (int f = 0; f < F; ++f) {
        const float x = Zs[r * (H + 1) + h * F + f];
        sl = fmaf(x, attn_l[h * F + f], sl);
        sr = fmaf(x, attn_r[h * F + f], sr);
      }
      el[(size_t)(row0 + r) * nh + h] = sl;
      er[(size_t)(row0 + r) * nh + h] = sr;
    }
  }
}

// Edge softmax + aggregation, one warp per row; a row with more than GCCB_HUB_DEG entries is split across the 8
// warps of the CTA after the group of 8 rows it belongs to.  mx / den: the softmax max and denominator of every
// (row, head), 0 for a row without entries (whose output is 0).
template <int H>
__global__ void __launch_bounds__(256, 1)
gat_agg_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
               const int32_t* __restrict__ indices, int nh, const float* __restrict__ z, const float* __restrict__ el,
               const float* __restrict__ er, int act, float* __restrict__ mx, float* __restrict__ den,
               float* __restrict__ out) {
  constexpr int PER = H / 32;
  __shared__ float co[8][3 * GAT_MAXH];
  __shared__ float hub[8][2 * GAT_MAXH];
  __shared__ float part[8][H];
  const int N = max(node_off_v[B], 0), F = H / nh;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int g0 = blockIdx.x * 8; g0 < N; g0 += gridDim.x * 8) {
    const int v = g0 + w;
    if (v < N && indptr[v + 1] - indptr[v] <= GCCB_HUB_DEG) {
      const int beg = indptr[v], end = indptr[v + 1];
      if (lane < nh) co[w][lane] = er[(size_t)v * nh + lane];
      __syncwarp();
      float m[GAT_MAXH], s[GAT_MAXH];
      gat_softmax_range(indices, beg, end, lane, nh, el, co[w], m, s);
#pragma unroll
      for (int h = 0; h < GAT_MAXH; ++h)
        if (h < nh && lane == 0) {
          const float M = s[h] > 0.f ? m[h] : 0.f;
          co[w][GAT_MAXH + h] = M;
          co[w][2 * GAT_MAXH + h] = s[h] > 0.f ? 1.f / s[h] : 0.f;
          mx[(size_t)v * nh + h] = M;
          den[(size_t)v * nh + h] = s[h];
        }
      __syncwarp();
      float acc[PER];
#pragma unroll
      for (int j = 0; j < PER; ++j) acc[j] = 0.f;
      gat_agg_range<H>(indices, beg, end, lane, nh, F, el, z, co[w], acc);
#pragma unroll
      for (int j = 0; j < PER; ++j) out[(size_t)v * H + lane + 32 * j] = act ? lrelu(acc[j], 0.01f) : acc[j];
    }
    for (int k = 0; k < 8; ++k) {                    // hub rows of the group, by the whole CTA (uniform branches)
      const int vh = g0 + k;
      if (vh >= N) break;
      const int beg = indptr[vh], end = indptr[vh + 1];
      if (end - beg <= GCCB_HUB_DEG) continue;
      const int per = (end - beg + 7) / 8, b = min(beg + w * per, end), e = min(b + per, end);
      __syncthreads();                               // co / part of the previous row consumed
      if (lane < nh) co[w][lane] = er[(size_t)vh * nh + lane];
      __syncwarp();
      float m[GAT_MAXH], s[GAT_MAXH];
      gat_softmax_range(indices, b, e, lane, nh, el, co[w], m, s);
      if (lane == 0) {
#pragma unroll
        for (int h = 0; h < GAT_MAXH; ++h)
          if (h < nh) { hub[w][h] = m[h]; hub[w][GAT_MAXH + h] = s[h]; }
      }
      __syncthreads();
      if (lane < nh) {
        float M = -INFINITY, S = 0.f;
        for (int ww = 0; ww < 8; ++ww) M = fmaxf(M, hub[ww][lane]);
        for (int ww = 0; ww < 8; ++ww)
          if (hub[ww][lane] != -INFINITY) S += hub[ww][GAT_MAXH + lane] * expf(hub[ww][lane] - M);
        co[w][GAT_MAXH + lane] = M;
        co[w][2 * GAT_MAXH + lane] = 1.f / S;
        if (w == 0) { mx[(size_t)vh * nh + lane] = M; den[(size_t)vh * nh + lane] = S; }
      }
      __syncwarp();
      float acc[PER];
#pragma unroll
      for (int j = 0; j < PER; ++j) acc[j] = 0.f;
      gat_agg_range<H>(indices, b, e, lane, nh, F, el, z, co[w], acc);
#pragma unroll
      for (int j = 0; j < PER; ++j) part[w][lane + 32 * j] = acc[j];
      __syncthreads();
      if ((int)threadIdx.x < H) {
        float t = 0.f;
#pragma unroll
        for (int ww = 0; ww < 8; ++ww) t += part[ww][threadIdx.x];
        out[(size_t)vh * H + threadIdx.x] = act ? lrelu(t, 0.01f) : t;
      }
    }
  }
}

// One LSTM cell over GAT_GB graphs per CTA: gates = W_ih x + b_ih + W_hh h + b_hh (a warp per gate row, lanes
// across the input), then c = f c + i g, h = o tanh(c).  gates_out keeps i, f, g, o after their activations.
template <int H>
__global__ void __launch_bounds__(256)
gat_lstm_cell_kernel(int B, int KI, const float* __restrict__ inp, const float* __restrict__ hprev,
                     const float* __restrict__ cprev, const float* __restrict__ wih, const float* __restrict__ whh,
                     const float* __restrict__ bih, const float* __restrict__ bhh, float* __restrict__ gates_out,
                     float* __restrict__ hout, float* __restrict__ cout) {
  __shared__ float xs[GAT_GB][3 * H];
  __shared__ float gs[GAT_GB][4 * H];
  const int b0 = blockIdx.x * GAT_GB, lane = threadIdx.x & 31, w = threadIdx.x >> 5, KT = KI + H;
  for (int idx = threadIdx.x; idx < GAT_GB * KT; idx += blockDim.x) {
    const int g = idx / KT, k = idx - g * KT, b = b0 + g;
    float v = 0.f;
    if (b < B) v = k < KI ? inp[(size_t)b * KI + k] : hprev[(size_t)b * H + k - KI];
    xs[g][k] = v;
  }
  __syncthreads();
  for (int r = w; r < 4 * H; r += 8) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    for (int k = lane; k < KT; k += 32) {
      const float wv = k < KI ? wih[(size_t)r * KI + k] : whh[(size_t)r * H + k - KI];
#pragma unroll
      for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, xs[g][k], acc[g]);
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) {
      const float t = warp_sum(acc[g]);
      if (lane == 0) gs[g][r] = t + bih[r] + bhh[r];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < GAT_GB * H; idx += blockDim.x) {
    const int g = idx / H, j = idx - g * H, b = b0 + g;
    if (b >= B) continue;
    const float i = sigmoidf_(gs[g][j]), f = sigmoidf_(gs[g][H + j]), gg = tanhf(gs[g][2 * H + j]),
                o = sigmoidf_(gs[g][3 * H + j]);
    const float c = fmaf(f, cprev[(size_t)b * H + j], i * gg);
    float* go = gates_out + (size_t)b * 4 * H;
    go[j] = i; go[H + j] = f; go[2 * H + j] = gg; go[3 * H + j] = o;
    cout[(size_t)b * H + j] = c;
    hout[(size_t)b * H + j] = o * tanhf(c);
  }
}

// Set2Set attention of one iteration, a CTA per graph: e_i = <x_i, q_b>, alpha = softmax over the graph's nodes,
// r_b = sum alpha_i x_i, q*_b = [q_b | r_b].  A graph without nodes gets r = 0.
template <int H>
__global__ void __launch_bounds__(256)
gat_s2s_attend_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ x,
                      const float* __restrict__ q, float* __restrict__ alpha, float* __restrict__ qstar) {
  constexpr int PER = H / 32, RG = 256 / H;
  __shared__ float qs[H];
  __shared__ float red[8];
  __shared__ float part[256];
  const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int beg = node_off_v[b], end = node_off_v[b + 1];
  if (node_off_v[B] < 0) beg = end = 0;               // a view published empty
  for (int c = threadIdx.x; c < H; c += blockDim.x) qs[c] = q[(size_t)b * H + c];
  __syncthreads();
  float mymax = -INFINITY;
  for (int i = beg + w; i < end; i += 8) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j) t = fmaf(x[(size_t)i * H + lane + 32 * j], qs[lane + 32 * j], t);
    t = warp_sum(t);
    if (lane == 0) alpha[i] = t;
    mymax = fmaxf(mymax, t);
  }
  const float M = block_max8(mymax, red);
  float sum = 0.f;
  for (int i = beg + (int)threadIdx.x; i < end; i += blockDim.x) {
    const float ex = expf(alpha[i] - M);
    alpha[i] = ex;
    sum += ex;
  }
  const float S = block_sum8(sum, red);
  const float inv = S > 0.f ? 1.f / S : 0.f;
  for (int i = beg + (int)threadIdx.x; i < end; i += blockDim.x) alpha[i] *= inv;
  __syncthreads();
  const int c = threadIdx.x % H, rg = threadIdx.x / H;
  float r = 0.f;
  for (int i = beg + rg; i < end; i += RG) r = fmaf(alpha[i], x[(size_t)i * H + c], r);
  part[threadIdx.x] = r;
  __syncthreads();
  if ((int)threadIdx.x < H) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < RG; ++g) t += part[g * H + threadIdx.x];
    qstar[(size_t)b * 2 * H + threadIdx.x] = qs[threadIdx.x];
    qstar[(size_t)b * 2 * H + H + threadIdx.x] = t;
  }
}

// lin_readout (Linear(2H, H) -> ReLU -> Linear(H, H)) and F.normalize(eps), GAT_GB graphs per CTA
template <int H>
__global__ void __launch_bounds__(256)
gat_readout_kernel(int B, const float* __restrict__ qs_in, const float* __restrict__ w0, const float* __restrict__ b0,
                   const float* __restrict__ w2, const float* __restrict__ b2, int norm, float eps,
                   float* __restrict__ y1, float* __restrict__ score, float* __restrict__ feat) {
  __shared__ float xs[GAT_GB][2 * H];
  __shared__ float ys[GAT_GB][H];
  __shared__ float ss[GAT_GB][H];
  const int g0 = blockIdx.x * GAT_GB, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int idx = threadIdx.x; idx < GAT_GB * 2 * H; idx += blockDim.x) {
    const int g = idx / (2 * H), k = idx - g * 2 * H;
    xs[g][k] = g0 + g < B ? qs_in[(size_t)(g0 + g) * 2 * H + k] : 0.f;
  }
  __syncthreads();
  for (int r = w; r < H; r += 8) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    for (int k = lane; k < 2 * H; k += 32) {
      const float wv = w0[(size_t)r * 2 * H + k];
#pragma unroll
      for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, xs[g][k], acc[g]);
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) {
      const float t = warp_sum(acc[g]);
      if (lane == 0) ys[g][r] = fmaxf(t + b0[r], 0.f);
    }
  }
  __syncthreads();
  for (int r = w; r < H; r += 8) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    for (int k = lane; k < H; k += 32) {
      const float wv = w2[(size_t)r * H + k];
#pragma unroll
      for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, ys[g][k], acc[g]);
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) {
      const float t = warp_sum(acc[g]);
      if (lane == 0) ss[g][r] = t + b2[r];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < GAT_GB * H; idx += blockDim.x) {
    const int g = idx / H, j = idx - g * H;
    if (g0 + g < B) {
      y1[(size_t)(g0 + g) * H + j] = ys[g][j];
      score[(size_t)(g0 + g) * H + j] = ss[g][j];
    }
  }
  if (w < GAT_GB && g0 + w < B) {
    float t = 0.f;
    for (int j = lane; j < H; j += 32) t = fmaf(ss[w][j], ss[w][j], t);
    const float nrm = fmaxf(sqrtf(warp_sum(t)), eps);
    for (int j = lane; j < H; j += 32) feat[(size_t)(g0 + w) * H + j] = norm ? ss[w][j] / nrm : ss[w][j];
  }
}

// ------------------------------------------------------------------------------------------------ backward
// normalise + lin_readout backward: dy = [d(lin_readout.0 out, before the ReLU) | d(lin_readout.2 out)],
// dqs = d q* of the last iteration
template <int H>
__global__ void __launch_bounds__(256)
gat_readout_bwd_kernel(int B, const float* __restrict__ y1, const float* __restrict__ score,
                       const float* __restrict__ dfeat, const float* __restrict__ w0, const float* __restrict__ w2,
                       int norm, float eps, float* __restrict__ dy, float* __restrict__ dqs) {
  __shared__ float d2[GAT_GB][H];
  __shared__ float d1[GAT_GB][H];
  const int g0 = blockIdx.x * GAT_GB, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (w < GAT_GB) {
    const int b = g0 + w;
    if (b < B) {
      float n2 = 0.f, dot = 0.f;
      for (int j = lane; j < H; j += 32) {
        const float s = score[(size_t)b * H + j];
        n2 = fmaf(s, s, n2);
        dot = fmaf(s, dfeat[(size_t)b * H + j], dot);
      }
      n2 = warp_sum(n2);
      dot = warp_sum(dot);
      const float n = sqrtf(n2);
      for (int j = lane; j < H; j += 32) {
        const float df = dfeat[(size_t)b * H + j];
        float ds = df;
        if (norm) ds = n > eps ? (df - score[(size_t)b * H + j] * (dot / n2)) / n : df / eps;
        d2[w][j] = ds;
      }
    } else {
      for (int j = lane; j < H; j += 32) d2[w][j] = 0.f;
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < H; k += blockDim.x) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    for (int o = 0; o < H; ++o) {
      const float wv = w2[(size_t)o * H + k];
#pragma unroll
      for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, d2[g][o], acc[g]);
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g)
      d1[g][k] = (g0 + g < B && y1[(size_t)(g0 + g) * H + k] > 0.f) ? acc[g] : 0.f;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < 2 * H; k += blockDim.x) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    for (int o = 0; o < H; ++o) {
      const float wv = w0[(size_t)o * 2 * H + k];
#pragma unroll
      for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, d1[g][o], acc[g]);
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g)
      if (g0 + g < B) dqs[(size_t)(g0 + g) * 2 * H + k] = acc[g];
  }
  for (int idx = threadIdx.x; idx < GAT_GB * H; idx += blockDim.x) {
    const int g = idx / H, j = idx - g * H;
    if (g0 + g < B) {
      dy[(size_t)(g0 + g) * 2 * H + j] = d1[g][j];
      dy[(size_t)(g0 + g) * 2 * H + H + j] = d2[g][j];
    }
  }
}

// Weight gradient of a small dense layer over T steps of B rows: gw[o][k] += sum_t sum_b P[t][b][o] Q[t][b][k],
// gb[o] (and gb2[o]) += sum_t sum_b P[t][b][o].  A thread per entry, rows in a fixed order.
__global__ void __launch_bounds__(256)
gat_dense_wgrad_kernel(int T, int B, const float* __restrict__ P, int64_t p_t, int p_ld, const float* __restrict__ Q,
                       int64_t q_t, int q_ld, int O, int KQ, float* __restrict__ gw, float* __restrict__ gb,
                       float* __restrict__ gb2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < O * KQ) {
    const int o = idx / KQ, k = idx - o * KQ;
    float s = 0.f;
    for (int t = 0; t < T; ++t)
      for (int b = 0; b < B; ++b)
        s = fmaf(P[t * p_t + (size_t)b * p_ld + o], Q[t * q_t + (size_t)b * q_ld + k], s);
    gw[idx] += s;
  } else if (gb && idx < O * KQ + O) {
    const int o = idx - O * KQ;
    float s = 0.f;
    for (int t = 0; t < T; ++t)
      for (int b = 0; b < B; ++b) s += P[t * p_t + (size_t)b * p_ld + o];
    gb[o] += s;
    if (gb2) gb2[o] += s;
  }
}

// One LSTM cell backward over GAT_GB graphs per CTA.  dh = above + dhs (the state gradient from the next
// iteration); dcs holds the cell-state gradient and is replaced by the one for the previous iteration, dhs likewise
// by W_hh^T dgates; dinp = W_ih^T dgates (the gradient of this cell's input).
template <int H>
__global__ void __launch_bounds__(256)
gat_lstm_cell_bwd_kernel(int B, int KI, const float* __restrict__ above, float* __restrict__ dhs,
                         float* __restrict__ dcs, const float* __restrict__ gates, const float* __restrict__ c_cur,
                         const float* __restrict__ c_prev, const float* __restrict__ wih, const float* __restrict__ whh,
                         float* __restrict__ dgates, float* __restrict__ dinp) {
  __shared__ float dg[GAT_GB][4 * H];
  const int b0 = blockIdx.x * GAT_GB;
  for (int idx = threadIdx.x; idx < GAT_GB * H; idx += blockDim.x) {
    const int g = idx / H, j = idx - g * H, b = b0 + g;
    float gi = 0.f, gf = 0.f, gg = 0.f, go = 0.f;
    if (b < B) {
      const size_t bj = (size_t)b * H + j;
      const float* ga = gates + (size_t)b * 4 * H;
      const float i = ga[j], f = ga[H + j], gv = ga[2 * H + j], o = ga[3 * H + j];
      const float dh = above[bj] + dhs[bj];
      const float tc = tanhf(c_cur[bj]);
      const float dc = dcs[bj] + dh * o * (1.f - tc * tc);
      gi = dc * gv * i * (1.f - i);
      gf = dc * c_prev[bj] * f * (1.f - f);
      gg = dc * i * (1.f - gv * gv);
      go = dh * tc * o * (1.f - o);
      dcs[bj] = dc * f;
      float* dga = dgates + (size_t)b * 4 * H;
      dga[j] = gi; dga[H + j] = gf; dga[2 * H + j] = gg; dga[3 * H + j] = go;
    }
    dg[g][j] = gi; dg[g][H + j] = gf; dg[g][2 * H + j] = gg; dg[g][3 * H + j] = go;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < KI + H; k += blockDim.x) {
    float acc[GAT_GB];
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) acc[g] = 0.f;
    if (k < KI) {
      for (int r = 0; r < 4 * H; ++r) {
        const float wv = wih[(size_t)r * KI + k];
#pragma unroll
        for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, dg[g][r], acc[g]);
      }
    } else {
      for (int r = 0; r < 4 * H; ++r) {
        const float wv = whh[(size_t)r * H + k - KI];
#pragma unroll
        for (int g = 0; g < GAT_GB; ++g) acc[g] = fmaf(wv, dg[g][r], acc[g]);
      }
    }
#pragma unroll
    for (int g = 0; g < GAT_GB; ++g) {
      const int b = b0 + g;
      if (b >= B) continue;
      if (k < KI) dinp[(size_t)b * KI + k] = acc[g];
      else dhs[(size_t)b * H + k - KI] = acc[g];
    }
  }
}

// Set2Set attention backward of one iteration, a CTA per graph.  dqs = d q* after the iteration: [dq | dr].
// dx_i += alpha_i dr + de_i q with de_i = alpha_i (<dr, x_i> - sum_j alpha_j <dr, x_j>);
// dq_top = dq + sum_i de_i x_i (the gradient of the top LSTM layer's output).
template <int H>
__global__ void __launch_bounds__(256, 1)
gat_s2s_attend_bwd_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ x,
                          const float* __restrict__ q, const float* __restrict__ alpha, const float* __restrict__ dqs,
                          float* __restrict__ dal, float* __restrict__ dx, float* __restrict__ dqtop) {
  constexpr int PER = H / 32, RG = 256 / H;
  __shared__ float qs[H], dr[H];
  __shared__ float red[8];
  __shared__ float part[256];
  const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int beg = node_off_v[b], end = node_off_v[b + 1];
  if (node_off_v[B] < 0) beg = end = 0;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    qs[c] = q[(size_t)b * H + c];
    dr[c] = dqs[(size_t)b * 2 * H + H + c];
  }
  __syncthreads();
  float sacc = 0.f;
  for (int i = beg + w; i < end; i += 8) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j) t = fmaf(x[(size_t)i * H + lane + 32 * j], dr[lane + 32 * j], t);
    t = warp_sum(t);
    if (lane == 0) dal[i] = t;
    sacc = fmaf(alpha[i], t, sacc);
  }
  const float S = block_sum8(lane == 0 ? sacc : 0.f, red);
  for (int i = beg + w; i < end; i += 8) {
    const float a = alpha[i], de = a * (dal[i] - S);
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int c = lane + 32 * j;
      dx[(size_t)i * H + c] += fmaf(a, dr[c], de * qs[c]);
    }
    __syncwarp();
    if (lane == 0) dal[i] = de;
  }
  __syncthreads();
  const int c = threadIdx.x % H, rg = threadIdx.x / H;
  float acc = 0.f;
  for (int i = beg + rg; i < end; i += RG) acc = fmaf(dal[i], x[(size_t)i * H + c], acc);
  part[threadIdx.x] = acc;
  __syncthreads();
  if ((int)threadIdx.x < H) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < RG; ++g) t += part[g * H + threadIdx.x];
    dqtop[(size_t)b * H + threadIdx.x] = dqs[(size_t)b * 2 * H + threadIdx.x] + t;
  }
}

// Over the entries [beg, end) of row v (edges u -> v): with da = <dout_v, z_u> per head,
// S += a da, A += a da slope, Bs += a slope (slope = leaky_relu'(el_u + er_v)); per lane column, head totals.
template <int H>
__device__ __forceinline__ void gat_attn_bwd_range(const int32_t* __restrict__ indices, int beg, int end, int lane,
                                                   int nh, int F, const float* __restrict__ el,
                                                   const float* __restrict__ z, const float* co,
                                                   const float (&dov)[H / 32], float (&S)[H / 32], float (&A)[H / 32],
                                                   float (&Bs)[H / 32]) {
  constexpr int PER = H / 32;
  int hd[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) hd[j] = (lane + 32 * j) / F;
  for (int e = beg; e < end; ++e) {
    const int u = indices[e];
    float da[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) da[j] = dov[j] * z[(size_t)u * H + lane + 32 * j];
    head_sum<PER>(da, F);
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int h = hd[j];
      const float pre = el[(size_t)u * nh + h] + co[h];
      const float a = expf(lrelu(pre, 0.2f) - co[GAT_MAXH + h]) * co[2 * GAT_MAXH + h];
      const float sl = pre > 0.f ? 1.f : 0.2f;
      S[j] = fmaf(a, da[j], S[j]);
      A[j] = fmaf(a * da[j], sl, A[j]);
      Bs[j] = fmaf(a, sl, Bs[j]);
    }
  }
}

// Edge-softmax backward, pass 1 (rows as destinations): dout = dh * activation', and per (v, head)
// sv[0] = S = sum_e a da, sv[1] = der_v = sum_e a (da - S) slope = A - S Bs.
template <int H>
__global__ void __launch_bounds__(256, 1)
gat_bwd_attn_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
                    const int32_t* __restrict__ indices, int nh, int cap, const float* __restrict__ dh,
                    const float* __restrict__ hout, int act, const float* __restrict__ z, const float* __restrict__ att,
                    float* __restrict__ dout, float* __restrict__ sv) {
  constexpr int PER = H / 32;
  __shared__ float co[8][3 * GAT_MAXH];
  __shared__ float hub[8][3][H];
  const int N = max(node_off_v[B], 0), F = H / nh;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const float* el = att;
  const float* er = att + (size_t)cap * nh;
  const float* mx = att + (size_t)2 * cap * nh;
  const float* den = att + (size_t)3 * cap * nh;
  float* Sv = sv;
  float* der = sv + (size_t)cap * nh;
  for (int g0 = blockIdx.x * 8; g0 < N; g0 += gridDim.x * 8) {
    for (int k = -1; k < 8; ++k) {               // k = -1: the warp rows of the group; then its hub rows
      const int v = k < 0 ? g0 + w : g0 + k;
      if (v >= N) { if (k < 0) continue; else break; }
      const int beg = indptr[v], end = indptr[v + 1];
      const bool is_hub = end - beg > GCCB_HUB_DEG;
      if (k < 0 ? is_hub : !is_hub) continue;
      if (k >= 0) __syncthreads();
      if (lane < nh) {
        const float s = den[(size_t)v * nh + lane];
        co[w][lane] = er[(size_t)v * nh + lane];
        co[w][GAT_MAXH + lane] = mx[(size_t)v * nh + lane];
        co[w][2 * GAT_MAXH + lane] = s > 0.f ? 1.f / s : 0.f;
      }
      __syncwarp();
      float dov[PER], S[PER], A[PER], Bs[PER];
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        const size_t i = (size_t)v * H + lane + 32 * j;
        dov[j] = dh[i] * ((act && !(hout[i] > 0.f)) ? 0.01f : 1.f);
        S[j] = A[j] = Bs[j] = 0.f;
      }
      int b = beg, e = end;
      if (k >= 0) {
        const int per = (end - beg + 7) / 8;
        b = min(beg + w * per, end);
        e = min(b + per, end);
      }
      gat_attn_bwd_range<H>(indices, b, e, lane, nh, F, el, z, co[w], dov, S, A, Bs);
      if (k < 0) {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          const int c = lane + 32 * j;
          dout[(size_t)v * H + c] = dov[j];
          if (c % F == 0) {
            Sv[(size_t)v * nh + c / F] = S[j];
            der[(size_t)v * nh + c / F] = A[j] - S[j] * Bs[j];
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          const int c = lane + 32 * j;
          hub[w][0][c] = S[j]; hub[w][1][c] = A[j]; hub[w][2][c] = Bs[j];
          if (w == 0) dout[(size_t)v * H + c] = dov[j];
        }
        __syncthreads();
        const int c = threadIdx.x;
        if (c < H && c % F == 0) {
          float s = 0.f, a = 0.f, bs = 0.f;
          for (int ww = 0; ww < 8; ++ww) { s += hub[ww][0][c]; a += hub[ww][1][c]; bs += hub[ww][2][c]; }
          Sv[(size_t)v * nh + c / F] = s;
          der[(size_t)v * nh + c / F] = a - s * bs;
        }
      }
    }
  }
}

// Edge-softmax backward, pass 2 (rows as sources; row u of a symmetric graph lists the edges u -> v):
// dz_u = sum_v a(u->v) dout_v + del_u attn_l + der_u attn_r with del_u = sum_v a (da - S_v) slope;
// the attention-vector gradients sum del_u z_u and der_u z_u over the rows (CTA partials, one atomic each).
template <int H>
__global__ void __launch_bounds__(256)
gat_bwd_dz_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
                  const int32_t* __restrict__ indices, int nh, int cap, const float* __restrict__ dout,
                  const float* __restrict__ z, const float* __restrict__ att, const float* __restrict__ sv,
                  const float* __restrict__ attn_l, const float* __restrict__ attn_r, float* __restrict__ dz,
                  float* __restrict__ g_attn_l, float* __restrict__ g_attn_r) {
  constexpr int PER = H / 32;
  __shared__ float co[8][2 * GAT_MAXH];
  __shared__ float hub[8][2][H];
  __shared__ float gsum[2][H];
  const int N = max(node_off_v[B], 0), F = H / nh;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const float* el = att;
  const float* er = att + (size_t)cap * nh;
  const float* mx = att + (size_t)2 * cap * nh;
  const float* den = att + (size_t)3 * cap * nh;
  const float* Sv = sv;
  const float* der = sv + (size_t)cap * nh;
  for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) gsum[c / H][c % H] = 0.f;
  float gl[PER], gr[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) gl[j] = gr[j] = 0.f;
  float hgl = 0.f, hgr = 0.f;                      // hub rows: column threadIdx.x
  int hd[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) hd[j] = (lane + 32 * j) / F;
  __syncthreads();
  for (int g0 = blockIdx.x * 8; g0 < N; g0 += gridDim.x * 8) {
    for (int k = -1; k < 8; ++k) {
      const int u = k < 0 ? g0 + w : g0 + k;
      if (u >= N) { if (k < 0) continue; else break; }
      const int beg = indptr[u], end = indptr[u + 1];
      const bool is_hub = end - beg > GCCB_HUB_DEG;
      if (k < 0 ? is_hub : !is_hub) continue;
      if (k >= 0) __syncthreads();
      if (lane < nh) {
        co[w][lane] = el[(size_t)u * nh + lane];
        co[w][GAT_MAXH + lane] = der[(size_t)u * nh + lane];
      }
      __syncwarp();
      float zu[PER], agg[PER], dl[PER];
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        zu[j] = z[(size_t)u * H + lane + 32 * j];
        agg[j] = dl[j] = 0.f;
      }
      int b = beg, e = end;
      if (k >= 0) {
        const int per = (end - beg + 7) / 8;
        b = min(beg + w * per, end);
        e = min(b + per, end);
      }
      for (int ei = b; ei < e; ++ei) {
        const int v = indices[ei];
        float dov[PER], da[PER];
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          dov[j] = dout[(size_t)v * H + lane + 32 * j];
          da[j] = dov[j] * zu[j];
        }
        head_sum<PER>(da, F);
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          const int h = hd[j];
          const float pre = co[w][h] + er[(size_t)v * nh + h];
          const float a = expf(lrelu(pre, 0.2f) - mx[(size_t)v * nh + h]) * (1.f / den[(size_t)v * nh + h]);
          const float dpre = a * (da[j] - Sv[(size_t)v * nh + h]) * (pre > 0.f ? 1.f : 0.2f);
          agg[j] = fmaf(a, dov[j], agg[j]);
          dl[j] += dpre;
        }
      }
      if (k < 0) {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          const int c = lane + 32 * j;
          const float dr_ = co[w][GAT_MAXH + hd[j]];
          dz[(size_t)u * H + c] = agg[j] + dl[j] * attn_l[c] + dr_ * attn_r[c];
          gl[j] = fmaf(dl[j], zu[j], gl[j]);
          gr[j] = fmaf(dr_, zu[j], gr[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          hub[w][0][lane + 32 * j] = agg[j];
          hub[w][1][lane + 32 * j] = dl[j];
        }
        __syncthreads();
        const int c = threadIdx.x;
        if (c < H) {
          float ag = 0.f, d_l = 0.f;
          for (int ww = 0; ww < 8; ++ww) { ag += hub[ww][0][c]; d_l += hub[ww][1][c]; }
          const float dr_ = der[(size_t)u * nh + c / F], zc = z[(size_t)u * H + c];
          dz[(size_t)u * H + c] = ag + d_l * attn_l[c] + dr_ * attn_r[c];
          hgl = fmaf(d_l, zc, hgl);
          hgr = fmaf(dr_, zc, hgr);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    atomicAdd(&gsum[0][lane + 32 * j], gl[j]);
    atomicAdd(&gsum[1][lane + 32 * j], gr[j]);
  }
  if ((int)threadIdx.x < H) {
    atomicAdd(&gsum[0][threadIdx.x], hgl);
    atomicAdd(&gsum[1][threadIdx.x], hgr);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    if (gsum[0][c] != 0.f) atomicAdd(&g_attn_l[c], gsum[0][c]);
    if (gsum[1][c] != 0.f) atomicAdd(&g_attn_r[c], gsum[1][c]);
  }
}

// dX = dz W for 64-row tiles: dz [N][H], W [H][in] -> dx [N][KO] (columns >= in are 0).
// Dynamic shared memory: As [64][H+1] | Ws [KC][KO+4].
template <int H, int KO>
__global__ void __launch_bounds__(256)
gat_bwd_dx_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ dz,
                  const float* __restrict__ W, int in, float* __restrict__ dx) {
  using TC = TileCols<KO>;
  GCCB_DYN_SMEM(float, sm);
  float* As = sm;
  float* Ws = As + GCCB_TILE_ROWS * (H + 1);
  const int N = max(node_off_v[B], 0);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int row0 = blockIdx.x * GCCB_TILE_ROWS; row0 < N; row0 += gridDim.x * GCCB_TILE_ROWS) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < GCCB_TILE_ROWS * H; idx += blockDim.x) {
      const int r = idx / H, k = idx - r * H;
      As[r * (H + 1) + k] = row0 + r < N ? dz[(size_t)(row0 + r) * H + k] : 0.f;
    }
    __syncthreads();
    float acc[4][TC::CPT];
    tile_gemm<KO>(As, H + 1, H, Ws, [&](int o, int c) { return c < in ? W[(size_t)o * in + c] : 0.f; }, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + ty * 4 + i;
      if (r >= N) continue;
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) dx[(size_t)r * KO + TC::col(tx, c)] = acc[i][c];
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
struct GatArgs {
  GatDims d;
  const gccb_batch_t* batch;
  int view;
  const float* pos;
  const float* params;
  gccb_gat_layout_t lay;
  const char* acts;
  GatActs al;
  gccb_stream_t stream;
};

static int row_grid(int cap) {
  const int g = (cap + 7) / 8;
  return g < 8 * GCCB_NUM_SMS ? (g > 0 ? g : 1) : 8 * GCCB_NUM_SMS;
}
static int tile_grid(int cap) {
  const int t = (cap + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  return t < 4 * GCCB_NUM_SMS ? (t > 0 ? t : 1) : 4 * GCCB_NUM_SMS;
}

template <int K, int H>
static void launch_proj(const GatArgs& a, const int32_t* node_off_v, const float* X, int l, float* z, float* el,
                        float* er, int grid) {
  auto k = gat_proj_kernel<K, H>;
  const size_t sm = ((size_t)GCCB_TILE_ROWS * (K + 1) + (size_t)GCCB_KC * (H + 4) + (size_t)GCCB_TILE_ROWS * (H + 1)) * 4;
  ensure_dyn_smem(k, sm);
  GCCB_LAUNCH(k, grid, 256, sm, a.stream, node_off_v, a.batch->batch, X, a.params + a.lay.fc[l],
              l == 0 ? a.d.din : H, a.params + a.lay.attn_l[l], a.params + a.lay.attn_r[l], a.d.nh, z, el, er);
}

template <int H>
static int gat_run_forward(const GatArgs& a, float* feat) {
  const GatDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap, T = d.T, K = d.K, nh = d.nh;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const int32_t* graph_id = a.batch->graph_id + (size_t)a.view * cap;
  char* acts = (char*)a.acts;
  const GatActs& al = a.al;
  float* x0 = (float*)(acts + al.x0);
  float* qstar = (float*)(acts + al.qstar);
  float* hs = (float*)(acts + al.hs);
  float* cs = (float*)(acts + al.cs);
  float* gates = (float*)(acts + al.gates);
  float* alpha = (float*)(acts + al.alpha);
  const float* P = a.params;
  const size_t BH = (size_t)B * H;
  cudaMemsetAsync(qstar, 0, 2 * BH * sizeof(float), (cudaStream_t)a.stream);
  cudaMemsetAsync(hs, 0, K * BH * sizeof(float), (cudaStream_t)a.stream);
  cudaMemsetAsync(cs, 0, K * BH * sizeof(float), (cudaStream_t)a.stream);
  const int tgrid = tile_grid(cap), rgrid = row_grid(cap), ggrid = (B + GAT_GB - 1) / GAT_GB;
  GCCB_LAUNCH(gin_build_x0_kernel, tgrid, 256, 0, a.stream, gin_input_dims(d), node_off_v, B,
              a.pos + (size_t)a.view * cap * d.P, sub_deg, graph_id, P + a.lay.emb, x0, (double*)nullptr, (int64_t)0);
  for (int l = 0; l < d.L; ++l) {
    float* z = (float*)(acts + al.z[l]);
    float* att = (float*)(acts + al.att[l]);
    float* el = att;
    float* er = att + (size_t)cap * nh;
    if (l == 0) launch_proj<GCCB_DINP, H>(a, node_off_v, x0, l, z, el, er, tgrid);
    else launch_proj<H, H>(a, node_off_v, (const float*)(acts + al.h[l - 1]), l, z, el, er, tgrid);
    GCCB_LAUNCH(gat_agg_kernel<H>, rgrid, 256, 0, a.stream, node_off_v, B, indptr, indices, nh, (const float*)z,
                (const float*)el, (const float*)er, l < d.L - 1 ? 1 : 0, att + (size_t)2 * cap * nh,
                att + (size_t)3 * cap * nh, (float*)(acts + al.h[l]));
  }
  const float* x = (const float*)(acts + al.h[d.L - 1]);
  for (int it = 0; it < T; ++it) {
    for (int k = 0; k < K; ++k) {
      const float* inp = k == 0 ? qstar + (size_t)it * 2 * BH : hs + ((size_t)(it + 1) * K + k - 1) * BH;
      GCCB_LAUNCH(gat_lstm_cell_kernel<H>, ggrid, 256, 0, a.stream, B, k == 0 ? 2 * H : H, inp,
                  (const float*)(hs + ((size_t)it * K + k) * BH), (const float*)(cs + ((size_t)it * K + k) * BH),
                  P + a.lay.w_ih[k], P + a.lay.w_hh[k], P + a.lay.b_ih[k], P + a.lay.b_hh[k],
                  gates + ((size_t)it * K + k) * 4 * BH, hs + ((size_t)(it + 1) * K + k) * BH,
                  cs + ((size_t)(it + 1) * K + k) * BH);
    }
    GCCB_LAUNCH(gat_s2s_attend_kernel<H>, B, 256, 0, a.stream, node_off_v, B, x,
                (const float*)(hs + ((size_t)(it + 1) * K + K - 1) * BH), alpha + (size_t)it * cap,
                qstar + (size_t)(it + 1) * 2 * BH);
  }
  GCCB_LAUNCH(gat_readout_kernel<H>, ggrid, 256, 0, a.stream, B, (const float*)(qstar + (size_t)T * 2 * BH),
              P + a.lay.ro0_w, P + a.lay.ro0_b, P + a.lay.ro2_w, P + a.lay.ro2_b, d.norm, d.norm_eps,
              (float*)(acts + al.y1), (float*)(acts + al.score), feat);
  return check_launch("gccb_gat_forward");
}

template <int H>
static int gat_run_backward(const GatArgs& a, const float* dfeat, float* G, char* ws, const GatBwd& bl) {
  const GatDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap, T = d.T, K = d.K, nh = d.nh;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const char* acts = a.acts;
  const GatActs& al = a.al;
  const float* qstar = (const float*)(acts + al.qstar);
  const float* hs = (const float*)(acts + al.hs);
  const float* cs = (const float*)(acts + al.cs);
  const float* gates = (const float*)(acts + al.gates);
  const float* alpha = (const float*)(acts + al.alpha);
  const float* P = a.params;
  float* dh = (float*)(ws + bl.dh);
  float* dz = (float*)(ws + bl.dz);
  float* dout = (float*)(ws + bl.dout);
  float* sv = (float*)(ws + bl.sv);
  float* dx0 = (float*)(ws + bl.dx0);
  float* dgates = (float*)(ws + bl.dgates);
  float* dy = (float*)(ws + bl.dy);
  float* dup[2] = {(float*)(ws + bl.dup[0]), (float*)(ws + bl.dup[1])};
  float* dqtop = (float*)(ws + bl.dqtop);
  float* dhs = (float*)(ws + bl.dhs);
  float* dcs = (float*)(ws + bl.dcs);
  float* dal = (float*)(ws + bl.dal);
  float* part = (float*)(ws + bl.part);
  const size_t BH = (size_t)B * H;
  cudaMemsetAsync(dh, 0, (size_t)cap * H * sizeof(float), (cudaStream_t)a.stream);
  cudaMemsetAsync(dhs, 0, K * BH * sizeof(float), (cudaStream_t)a.stream);
  cudaMemsetAsync(dcs, 0, K * BH * sizeof(float), (cudaStream_t)a.stream);
  // gin_wgrad_reduce_kernel also sums a bias column; fc has no bias, so those sums land in this zeroed scratch
  cudaMemsetAsync(ws + bl.gbias, 0, (size_t)H * sizeof(float), (cudaStream_t)a.stream);
  const int tgrid = tile_grid(cap), rgrid = row_grid(cap), ggrid = (B + GAT_GB - 1) / GAT_GB;
  // readout: dy, d q*(T) -> dup[0]; its weight gradients
  GCCB_LAUNCH(gat_readout_bwd_kernel<H>, ggrid, 256, 0, a.stream, B, (const float*)(acts + al.y1),
              (const float*)(acts + al.score), dfeat, P + a.lay.ro0_w, P + a.lay.ro2_w, d.norm, d.norm_eps, dy,
              dup[0]);
  GCCB_LAUNCH(gat_dense_wgrad_kernel, (H * H + H + 255) / 256, 256, 0, a.stream, 1, B, (const float*)(dy + H),
              (int64_t)0, 2 * H, (const float*)(acts + al.y1), (int64_t)0, H, H, H, G + a.lay.ro2_w,
              G + a.lay.ro2_b, (float*)nullptr);
  GCCB_LAUNCH(gat_dense_wgrad_kernel, (2 * H * H + H + 255) / 256, 256, 0, a.stream, 1, B, (const float*)dy,
              (int64_t)0, 2 * H, qstar + (size_t)T * 2 * BH, (int64_t)0, 2 * H, H, 2 * H, G + a.lay.ro0_w,
              G + a.lay.ro0_b, (float*)nullptr);
  // Set2Set, iterations in reverse: the attention backward (dx += ..., dq of the top LSTM layer), then the cells
  // top down; cell k writes the gradient of its input to dup[k & 1], cell 0's is d q* of the iteration before
  const float* x = (const float*)(acts + al.h[d.L - 1]);
  for (int it = T - 1; it >= 0; --it) {
    GCCB_LAUNCH(gat_s2s_attend_bwd_kernel<H>, B, 256, 0, a.stream, node_off_v, B, x,
                hs + ((size_t)(it + 1) * K + K - 1) * BH, alpha + (size_t)it * cap, (const float*)dup[0], dal, dh,
                dqtop);
    for (int k = K - 1; k >= 0; --k) {
      const float* above = k == K - 1 ? dqtop : dup[(k + 1) & 1];
      GCCB_LAUNCH(gat_lstm_cell_bwd_kernel<H>, ggrid, 256, 0, a.stream, B, k == 0 ? 2 * H : H, above,
                  dhs + k * BH, dcs + k * BH, gates + ((size_t)it * K + k) * 4 * BH,
                  cs + ((size_t)(it + 1) * K + k) * BH, cs + ((size_t)it * K + k) * BH, P + a.lay.w_ih[k],
                  P + a.lay.w_hh[k], dgates + ((size_t)it * K + k) * 4 * BH, dup[k & 1]);
    }
  }
  for (int k = 0; k < K; ++k) {
    const int KI = k == 0 ? 2 * H : H;
    const float* Q = k == 0 ? qstar : hs + ((size_t)K + k - 1) * BH;     // the cell's input at iteration t
    const int64_t q_t = k == 0 ? (int64_t)2 * BH : (int64_t)K * BH;
    GCCB_LAUNCH(gat_dense_wgrad_kernel, (4 * H * KI + 4 * H + 255) / 256, 256, 0, a.stream, T, B,
                (const float*)(dgates + (size_t)k * 4 * BH), (int64_t)K * 4 * BH, 4 * H, Q, q_t, KI, 4 * H, KI,
                G + a.lay.w_ih[k], G + a.lay.b_ih[k], G + a.lay.b_hh[k]);
    GCCB_LAUNCH(gat_dense_wgrad_kernel, (4 * H * H + 255) / 256, 256, 0, a.stream, T, B,
                (const float*)(dgates + (size_t)k * 4 * BH), (int64_t)K * 4 * BH, 4 * H, hs + (size_t)k * BH,
                (int64_t)K * BH, H, 4 * H, H, G + a.lay.w_hh[k], (float*)nullptr, (float*)nullptr);
  }
  // GAT layers, top down; dh holds the gradient of the layer's output
  for (int l = d.L - 1; l >= 0; --l) {
    const float* z = (const float*)(acts + al.z[l]);
    const float* att = (const float*)(acts + al.att[l]);
    GCCB_LAUNCH(gat_bwd_attn_kernel<H>, rgrid, 256, 0, a.stream, node_off_v, B, indptr, indices, nh, cap,
                (const float*)dh, (const float*)(acts + al.h[l]), l < d.L - 1 ? 1 : 0, z, att, dout, sv);
    GCCB_LAUNCH(gat_bwd_dz_kernel<H>, rgrid, 256, 0, a.stream, node_off_v, B, indptr, indices, nh, cap,
                (const float*)dout, z, att, (const float*)sv, P + a.lay.attn_l[l], P + a.lay.attn_r[l], dz,
                G + a.lay.attn_l[l], G + a.lay.attn_r[l]);
    const int KQ = l == 0 ? GCCB_DINP : H, in = l == 0 ? d.din : H;
    const float* X = l == 0 ? (const float*)(acts + al.x0) : (const float*)(acts + al.h[l - 1]);
    dim3 gr(GCCB_WG_CHUNKS, ((H + 63) / 64) * ((KQ + 63) / 64));
    GCCB_LAUNCH(gin_wgrad_kernel, gr, 256, 0, a.stream, node_off_v, B, H, KQ, (const float*)dz, X,
                (const double*)nullptr, (const float*)nullptr, (const float*)nullptr, 0.f, part);
    GCCB_LAUNCH(gin_wgrad_reduce_kernel, (H * KQ + H + 255) / 256, 256, 0, a.stream, H, KQ, in, (const float*)part,
                G + a.lay.fc[l], (float*)(ws + bl.gbias));
    if (l == 0) {
      auto k = gat_bwd_dx_kernel<H, GCCB_DINP>;
      const size_t sm = ((size_t)GCCB_TILE_ROWS * (H + 1) + (size_t)GCCB_KC * (GCCB_DINP + 4)) * 4;
      ensure_dyn_smem(k, sm);
      GCCB_LAUNCH(k, tgrid, 256, sm, a.stream, node_off_v, B, (const float*)dz, P + a.lay.fc[l], in, dx0);
    } else {
      auto k = gat_bwd_dx_kernel<H, H>;
      const size_t sm = ((size_t)GCCB_TILE_ROWS * (H + 1) + (size_t)GCCB_KC * (H + 4)) * 4;
      ensure_dyn_smem(k, sm);
      GCCB_LAUNCH(k, tgrid, 256, sm, a.stream, node_off_v, B, (const float*)dz, P + a.lay.fc[l], in, dh);
    }
  }
  {
    const size_t sm = (size_t)(d.maxdeg + 1) * d.D * sizeof(float);
    auto k = gin_bwd_emb_kernel;
    ensure_dyn_smem(k, sm);
    GCCB_LAUNCH(k, 64, 256, sm, a.stream, gin_input_dims(d), node_off_v, B, sub_deg, (const float*)dx0,
                G + a.lay.emb);
  }
  return check_launch("gccb_gat_backward");
}

static int gat_prepare(const gccb_gat_cfg_t* cfg, const gccb_batch_t* batch, int32_t view, const float* params,
                       const void* acts, size_t acts_bytes, GatArgs* a, const char* what) {
  int rc = gat_dims(cfg, &a->d);
  if (rc) return rc;
  if (!batch || !params || !acts || view < 0 || view > 1 || batch->batch < 1 || batch->node_cap < 1) {
    set_last_error("%s: bad argument", what);
    return GCCB_ERR_BADARG;
  }
  a->al = gat_acts_layout(a->d, batch->batch, batch->node_cap);
  if (acts_bytes < a->al.total) {
    set_last_error("%s: activation stash too small (%zu < %zu)", what, acts_bytes, a->al.total);
    return GCCB_ERR_CAPACITY;
  }
  gat_param_layout(a->d, &a->lay);
  a->batch = batch; a->view = view; a->params = params; a->acts = (const char*)acts;
  return GCCB_OK;
}

}  // namespace gccb

using namespace gccb;

extern "C" int gccb_gat_param_layout(const gccb_gat_cfg_t* cfg, gccb_gat_layout_t* out) {
  GatDims d;
  int rc = gat_dims(cfg, &d);
  if (rc) return rc;
  if (!out) return GCCB_ERR_BADARG;
  gat_param_layout(d, out);
  return GCCB_OK;
}

extern "C" size_t gccb_gat_acts_bytes(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap) {
  GatDims d;
  if (gat_dims(cfg, &d) || batch < 1 || node_cap < 1) return 0;
  return gat_acts_layout(d, batch, node_cap).total;
}

extern "C" size_t gccb_gat_backward_workspace(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap) {
  GatDims d;
  if (gat_dims(cfg, &d) || batch < 1 || node_cap < 1) return 0;
  return gat_bwd_layout(d, batch, node_cap).total;
}

extern "C" int gccb_gat_stash_layout(const gccb_gat_cfg_t* cfg, int32_t batch, int32_t node_cap,
                                     gccb_gat_stash_t* out) {
  GatDims d;
  int rc = gat_dims(cfg, &d);
  if (rc) return rc;
  if (!out || batch < 1 || node_cap < 1) {
    set_last_error("gccb_gat_stash_layout: bad argument");
    return GCCB_ERR_BADARG;
  }
  const GatActs al = gat_acts_layout(d, batch, node_cap);
  const GatBwd bl = gat_bwd_layout(d, batch, node_cap);
  out->x0 = (int64_t)al.x0;
  for (int l = 0; l < 8; ++l) {
    const bool live = l < d.L;
    out->z[l] = live ? (int64_t)al.z[l] : -1;
    out->h[l] = live ? (int64_t)al.h[l] : -1;
    out->att[l] = live ? (int64_t)al.att[l] : -1;
  }
  out->qstar = (int64_t)al.qstar; out->hs = (int64_t)al.hs; out->cs = (int64_t)al.cs;
  out->gates = (int64_t)al.gates; out->alpha = (int64_t)al.alpha; out->y1 = (int64_t)al.y1;
  out->score = (int64_t)al.score;
  out->dh = (int64_t)bl.dh; out->dz = (int64_t)bl.dz; out->dout = (int64_t)bl.dout; out->sv = (int64_t)bl.sv;
  out->dx0 = (int64_t)bl.dx0; out->dgates = (int64_t)bl.dgates; out->dy = (int64_t)bl.dy;
  return GCCB_OK;
}

extern "C" int gccb_gat_forward(const gccb_gat_cfg_t* cfg, const gccb_batch_t* batch, int32_t view, const float* pos,
                                const float* params, void* acts, size_t acts_bytes, float* feat, gccb_stream_t stream) {
  GatArgs a;
  int rc = gat_prepare(cfg, batch, view, params, acts, acts_bytes, &a, "gccb_gat_forward");
  if (rc) return rc;
  if (!pos || !feat) {
    set_last_error("gccb_gat_forward: bad argument");
    return GCCB_ERR_BADARG;
  }
  a.pos = pos;
  a.stream = stream;
  switch (a.d.H) {
    case 32: return gat_run_forward<32>(a, feat);
    case 64: return gat_run_forward<64>(a, feat);
    case 128: return gat_run_forward<128>(a, feat);
    default: return gat_run_forward<256>(a, feat);
  }
}

extern "C" int gccb_gat_backward(const gccb_gat_cfg_t* cfg, const gccb_batch_t* batch, int32_t view,
                                 const float* params, const void* acts, const float* dfeat, float* grads,
                                 void* workspace, size_t workspace_bytes, gccb_stream_t stream) {
  GatArgs a;
  int rc = gat_prepare(cfg, batch, view, params, acts, (size_t)-1, &a, "gccb_gat_backward");
  if (rc) return rc;
  if (!dfeat || !grads || !workspace) {
    set_last_error("gccb_gat_backward: bad argument");
    return GCCB_ERR_BADARG;
  }
  const GatBwd bl = gat_bwd_layout(a.d, batch->batch, batch->node_cap);
  if (workspace_bytes < bl.total) {
    set_last_error("gccb_gat_backward: workspace too small (%zu < %zu)", workspace_bytes, bl.total);
    return GCCB_ERR_CAPACITY;
  }
  a.pos = nullptr;
  a.stream = stream;
  switch (a.d.H) {
    case 32: return gat_run_backward<32>(a, dfeat, grads, (char*)workspace, bl);
    case 64: return gat_run_backward<64>(a, dfeat, grads, (char*)workspace, bl);
    case 128: return gat_run_backward<128>(a, dfeat, grads, (char*)workspace, bl);
    default: return gat_run_backward<256>(a, dfeat, grads, (char*)workspace, bl);
  }
}
