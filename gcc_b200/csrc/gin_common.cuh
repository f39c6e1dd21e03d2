// gin_common.cuh -- layouts and tile helpers shared by the GIN forward / backward kernels.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace gccb {

#define GCCB_DINP 64          // padded width of the layer-0 input [pos | deg_emb | seed | 0..]
#define GCCB_TILE_ROWS 64
#define GCCB_KC 64            // K-chunk of the weight operand staged in shared memory
#define GCCB_MAX_L 8

struct GinDims {
  int L, H, P, D, maxdeg, din;   // din = P + D + 1 (49)
  int norm;
  int tc;                        // 1: Linear layers / their gradients on wgmma tensor cores (bf16 operands)
  float bn_eps, bn_mom, norm_eps, drop_p;
};

__host__ __device__ __forceinline__ int gin_in_features(const GinDims& d, int l) { return l == 0 ? d.din : d.H; }
__host__ __device__ __forceinline__ int gin_in_width(const GinDims& d, int l) { return l == 0 ? GCCB_DINP : d.H; }

// byte offsets inside the activation stash of ONE view
struct ActsLayout {
  size_t x0;                                   // float [node_cap][64]
  size_t a[GCCB_MAX_L], z1[GCCB_MAX_L], z2[GCCB_MAX_L], h[GCCB_MAX_L];
  size_t stats;                                // double [L-1][3][2][H]  column sums / sums of squares
  size_t pool_acc;                             // double [L][B][PW] sum-pooling accumulators (follow stats: one memset)
  size_t pooled;                               // float [L][B][PW]
  size_t score;                                // float [B][H]  (pre-normalisation)
  size_t feat;                                 // float [B][H]
  // tensor-core path only (d.tc): bf16 operands of the current layer's GEMMs and the bf16 weight copies
  size_t a16;                                  // bf16 [node_cap][max(H, 64)]   a = h + sum_nbr h
  size_t x16;                                  // bf16 [node_cap][H]            x1 = relu(bn1(z1))
  size_t w16[GCCB_MAX_L];                      // bf16 per layer: W1 [H][KW] | W2 [H][H] | W1^T [KW][H] | W2^T [H][H]
  size_t total;
  int PW;
};
// padded input width of layer l's first Linear on the tensor-core path (K of the GEMM, multiple of 64)
__host__ __device__ __forceinline__ int gin_kw(const GinDims& d, int l) { return l == 0 ? GCCB_DINP : d.H; }
inline size_t gin_w16_elems(const GinDims& d, int l) { return (size_t)2 * d.H * gin_kw(d, l) + (size_t)2 * d.H * d.H; }

inline ActsLayout make_acts_layout(const GinDims& d, int B, int node_cap) {
  ActsLayout a;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  a.x0 = take((size_t)node_cap * GCCB_DINP * 4);
  for (int l = 0; l < GCCB_MAX_L; ++l) a.a[l] = a.z1[l] = a.z2[l] = a.h[l] = 0;
  for (int l = 0; l < d.L - 1; ++l) {
    a.a[l] = take((size_t)node_cap * gin_in_width(d, l) * 4);
    a.z1[l] = take((size_t)node_cap * d.H * 4);
    a.z2[l] = take((size_t)node_cap * d.H * 4);
    a.h[l] = take((size_t)node_cap * d.H * 4);
  }
  a.stats = take((size_t)(d.L - 1) * 3 * 2 * d.H * 8);
  a.PW = d.H > GCCB_DINP ? d.H : GCCB_DINP;
  a.pool_acc = take((size_t)d.L * B * a.PW * 8);
  a.pooled = take((size_t)d.L * B * a.PW * 4);
  a.score = take((size_t)B * d.H * 4);
  a.feat = take((size_t)B * d.H * 4);
  a.a16 = a.x16 = 0;
  for (int l = 0; l < GCCB_MAX_L; ++l) a.w16[l] = 0;
  if (d.tc) {
    a.a16 = take((size_t)node_cap * (d.H > GCCB_DINP ? d.H : GCCB_DINP) * 2);
    a.x16 = take((size_t)node_cap * d.H * 2);
    for (int l = 0; l < d.L - 1; ++l) a.w16[l] = take(gin_w16_elems(d, l) * 2);
  }
  a.total = off;
  return a;
}

#define GCCB_WG_CHUNKS GCCB_NUM_SMS    // row chunks of the weight-gradient split-K (SIMT backward)

struct BwdLayout {            // byte offsets in the backward workspace
  size_t dh, g1[2], dz2[2], da, red, dS, dpool, part, part1, total;   // g1/dz2 alternate between layers
  // tensor-core path: bf16 operand of the input-gradient GEMMs, two transposed bf16 operands of the weight-
  // gradient GEMMs ([W][cap_pad]), per-layer BatchNorm-1 coefficients (sc | sh) and the split-K partials
  size_t dz16, tA, tB, coef1, splitk;
  int DW;                     // width of dh / da rows = max(H, 64)
  int cap_pad, splits;
};

inline BwdLayout make_bwd_layout(const GinDims& d, int B, int node_cap) {
  BwdLayout b;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  b.DW = d.H > GCCB_DINP ? d.H : GCCB_DINP;
  b.dh = take((size_t)node_cap * b.DW * 4);
  for (int i = 0; i < 2; ++i) {
    b.g1[i] = take((size_t)node_cap * d.H * 4);
    b.dz2[i] = take((size_t)node_cap * d.H * 4);
  }
  b.da = take((size_t)node_cap * b.DW * 4);
  b.red = take((size_t)(d.L - 1) * 3 * 2 * d.H * 8);
  b.dS = take((size_t)d.L * B * d.H * 4);
  b.dpool = take((size_t)d.L * B * b.DW * 4);
  b.part = take((size_t)GCCB_WG_CHUNKS * ((size_t)d.H * b.DW + d.H) * 4);
  b.dz16 = b.tA = b.tB = b.coef1 = b.splitk = b.part1 = 0;
  b.cap_pad = (node_cap + 63) & ~63;
  b.splits = 0;
  if (!d.tc) b.part1 = take((size_t)GCCB_WG_CHUNKS * ((size_t)d.H * b.DW + d.H) * 4);   // dW1's own stream (SIMT)
#ifndef GCCB_EMU
  if (d.tc) {
    b.dz16 = take((size_t)node_cap * d.H * 2);
    b.tA = take((size_t)d.H * b.cap_pad * 2);
    b.tB = take((size_t)b.DW * b.cap_pad * 2);
    b.coef1 = take((size_t)(d.L - 1) * 2 * d.H * 4);
    const int tiles = (d.H / 128) * 1;                      // 128-row output tiles of a [H x <=256] weight gradient
    b.splits = GCCB_NUM_SMS / tiles;
    if (b.splits > b.cap_pad / 64) b.splits = b.cap_pad / 64;
    if (b.splits < 1) b.splits = 1;
    b.splitk = take((size_t)b.splits * d.H * b.DW * 4);
  }
#endif
  b.total = off;
  return b;
}

// flat parameter layout (floats); mirrors gccb_gin_layout_t
inline void make_param_layout(const GinDims& d, gccb_gin_layout_t* o) {
  int64_t off = 0;
  auto take = [&](int64_t n) { int64_t r = off; off += n; return r; };
  for (int l = 0; l < 8; ++l)
    o->w1[l] = o->b1[l] = o->bn1_w[l] = o->bn1_b[l] = o->w2[l] = o->b2[l] = o->bna_w[l] = o->bna_b[l] =
        o->bnb_w[l] = o->bnb_b[l] = o->wp[l] = o->bp[l] = -1;
  for (int l = 0; l < d.L - 1; ++l) {
    o->w1[l] = take((int64_t)d.H * gin_in_features(d, l));
    o->b1[l] = take(d.H);
    o->bn1_w[l] = take(d.H);
    o->bn1_b[l] = take(d.H);
    o->w2[l] = take((int64_t)d.H * d.H);
    o->b2[l] = take(d.H);
    o->bna_w[l] = take(d.H);
    o->bna_b[l] = take(d.H);
    o->bnb_w[l] = take(d.H);
    o->bnb_b[l] = take(d.H);
  }
  for (int l = 0; l < d.L; ++l) {
    o->wp[l] = take((int64_t)d.H * gin_in_features(d, l));
    o->bp[l] = take(d.H);
  }
  o->emb = take((int64_t)(d.maxdeg + 1) * d.D);
  o->total = off;
  o->run_total = (int64_t)(d.L - 1) * 3 * 2 * d.H;
}

inline int dims_from_cfg(const gccb_gin_cfg_t* c, GinDims* d) {
  if (!c) return GCCB_ERR_BADARG;
  d->L = c->num_layers; d->H = c->hidden; d->P = c->pos_dim; d->D = c->deg_dim;
  d->maxdeg = c->max_degree; d->din = c->pos_dim + c->deg_dim + 1; d->norm = c->norm;
  d->bn_eps = c->bn_eps; d->bn_mom = c->bn_momentum; d->norm_eps = c->norm_eps; d->drop_p = c->dropout_p;
#ifdef GCCB_EMU
  d->tc = 0;                                              // the CPU emulator has no tensor cores
#else
  d->tc = (c->tensor_cores && c->hidden >= 128) ? 1 : 0;  // tensor-core tiles are 128 x {128, 256}: hidden 32 / 64 stay SIMT fp32
#endif
  if (d->L < 2 || d->L > GCCB_MAX_L || (d->H != 32 && d->H != 64 && d->H != 128 && d->H != 256) ||
      d->din > GCCB_DINP || d->P < 2 || d->P > 32 || d->D < 1 || d->maxdeg < 1) {
    set_last_error("gin: unsupported configuration (L=%d H=%d pos=%d deg=%d): need 2<=L<=8, "
                   "H in {32,64,128,256}, pos+deg+1<=64, pos<=32", d->L, d->H, d->P, d->D);
    return GCCB_ERR_BADARG;
  }
  return GCCB_OK;
}

// ---------------------------------------------------------------------------------------
// BatchNorm coefficients from accumulated column sums (train mode) or running stats.
//   sums: double [2][H] (sum, sum of squares) over N rows.
//   out (shared memory): mean[H], invstd[H], sc[H] = gamma*invstd, sh[H] = beta - mean*sc
// Block 0 optionally applies the running-statistics update (momentum, unbiased variance).
__device__ __forceinline__ void bn_prepare(const double* __restrict__ sums, int N, int H,
                                           const float* __restrict__ gamma,
                                           const float* __restrict__ beta, float eps,
                                           float* mean_s, float* invstd_s, float* sc_s, float* sh_s,
                                           float* __restrict__ running /* [2][H] or null */,
                                           bool use_running, bool update_running, float momentum) {
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    double mean, var;
    if (use_running) {
      mean = running[c];
      var = running[H + c];
    } else {
      double n = N > 0 ? (double)N : 1.0;
      mean = sums[c] / n;
      var = sums[H + c] / n - mean * mean;
      if (var < 0.0) var = 0.0;
      if (update_running && running && blockIdx.x == 0 && N > 0) {   // an empty (overflowed) view leaves them alone
        double unb = N > 1 ? var * n / (n - 1.0) : var;
        running[c] = (float)((1.0 - momentum) * running[c] + momentum * mean);
        running[H + c] = (float)((1.0 - momentum) * running[H + c] + momentum * unb);
      }
    }
    // only the cancellation-prone E[x^2]-E[x]^2 is done in float64 (fp64 runs at a small
    // fraction of the fp32 rate on this part); the square root is float like torch's batch_norm
    float invstd = 1.0f / sqrtf((float)var + eps);
    float g = gamma[c];
    mean_s[c] = (float)mean;
    invstd_s[c] = invstd;
    sc_s[c] = g * invstd;
    sh_s[c] = beta[c] - (float)mean * g * invstd;
  }
}

// ---------------------------------------------------------------------------------------
// acc[j] += sum over edges e in [beg, end) of src[indices[e]][lane + 32 j]: one warp, lanes across
// the feature dimension (one coalesced row read per neighbour), eight neighbour rows in flight.
#ifndef GCCB_HUB_DEG
#define GCCB_HUB_DEG 256      // rows with more neighbours are split across the warps of the CTA
#endif
#define GCCB_GPB 8            // graphs per CTA of the pooled prediction heads (one warp per graph at the end)
#define GCCB_HUB_QUEUE 64     // hub rows a CTA of the barrier-free gather kernels defers to its cooperative pass

// Transform applied to every element a scalar gather reads: xf(x, j) for the column lane + 32 j of the lane.
struct GatherIdentity {
  __device__ __forceinline__ float operator()(float x, int) const { return x; }
};

// h = relu(bn_b(relu(bn_a(z2)))): the tail of a GIN layer (gin.py:55-57, :219-220) from its two BatchNorms'
// scale / shift, in the order gin_bn_tail_kernel applies it
__device__ __forceinline__ float bn_tail_h(float z, float sca, float sha, float scb, float shb) {
  return fmaxf(fmaf(fmaxf(fmaf(z, sca, sha), 0.f), scb, shb), 0.f);
}

// bn_tail_h with the coefficients of the lane's columns lane + 32 j held in registers
template <int PER>
struct BnTailXf {
  float sca[PER], sha[PER], scb[PER], shb[PER];
  __device__ __forceinline__ float operator()(float z, int j) const { return bn_tail_h(z, sca[j], sha[j], scb[j], shb[j]); }
};

template <int W, class Xf = GatherIdentity>
__device__ __forceinline__ void gather_range(const float* __restrict__ src, const int32_t* __restrict__ indices,
                                             int beg, int end, int lane, float (&acc)[(W + 31) / 32],
                                             const Xf& xf = Xf()) {
  constexpr int PER = (W + 31) / 32;
  int e = beg;
  for (; e + 7 < end; e += 8) {
    int u[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] = indices[e + k];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int c = lane + 32 * j;
      if (c < W) {
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = xf(src[(size_t)u[k] * W + c], j);
        acc[j] += ((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7]));
      }
    }
  }
  for (; e < end; ++e) {
    const int u = indices[e];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int c = lane + 32 * j;
      if (c < W) acc[j] += xf(src[(size_t)u * W + c], j);
    }
  }
}

// 128-bit variant for the barrier-free gather kernels: lane owns the float4 slots v = lane + 32 j of a row of W
// floats (a warp reads 512 contiguous bytes per instruction); four neighbour rows in flight.
template <int W>
__device__ __forceinline__ void gather_range4(const float* __restrict__ src, const int32_t* __restrict__ indices,
                                              int beg, int end, int lane, float4 (&acc)[(W / 4 + 31) / 32]) {
  constexpr int V4 = W / 4, PERV = (V4 + 31) / 32;
  int e = beg;
  for (; e + 3 < end; e += 4) {
    const int u0 = indices[e], u1 = indices[e + 1], u2 = indices[e + 2], u3 = indices[e + 3];
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = lane + 32 * j;
      if (v < V4) {
        const float4 x0 = *reinterpret_cast<const float4*>(src + (size_t)u0 * W + 4 * v);
        const float4 x1 = *reinterpret_cast<const float4*>(src + (size_t)u1 * W + 4 * v);
        const float4 x2 = *reinterpret_cast<const float4*>(src + (size_t)u2 * W + 4 * v);
        const float4 x3 = *reinterpret_cast<const float4*>(src + (size_t)u3 * W + 4 * v);
        acc[j].x += (x0.x + x1.x) + (x2.x + x3.x);
        acc[j].y += (x0.y + x1.y) + (x2.y + x3.y);
        acc[j].z += (x0.z + x1.z) + (x2.z + x3.z);
        acc[j].w += (x0.w + x1.w) + (x2.w + x3.w);
      }
    }
  }
  for (; e < end; ++e) {
    const int u = indices[e];
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = lane + 32 * j;
      if (v < V4) {
        const float4 x = *reinterpret_cast<const float4*>(src + (size_t)u * W + 4 * v);
        acc[j].x += x.x; acc[j].y += x.y; acc[j].z += x.z; acc[j].w += x.w;
      }
    }
  }
}

// Hub row: the 8 warps of a 256-thread CTA each gather a contiguous eighth of the neighbour list;
// partial sums meet in `scratch` [8][W]; on return (after the internal barriers) every thread
// c < W holds the full neighbour sum of column c in the return value.  All 256 threads must call.
template <int W, class Xf = GatherIdentity>
__device__ __forceinline__ float gather_hub(const float* __restrict__ src, const int32_t* __restrict__ indices,
                                            int beg, int end, float* scratch, const Xf& xf = Xf()) {
  constexpr int PER = (W + 31) / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int len = end - beg, per = (len + 7) / 8;
  const int b = beg + warp * per, e = min(b + per, end);
  float acc[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) acc[j] = 0.f;
  gather_range<W>(src, indices, b, e > b ? e : b, lane, acc, xf);
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int c = lane + 32 * j;
    if (c < W) scratch[warp * W + c] = acc[j];
  }
  __syncthreads();
  float s = 0.f;
  if ((int)threadIdx.x < W) {
#pragma unroll
    for (int w = 0; w < 8; ++w) s += scratch[w * W + threadIdx.x];
  }
  __syncthreads();
  return s;
}

// ---------------------------------------------------------------------------------------
// 64-row tile GEMM: acc[4][CPT] += As[row][k] * Ws[k][col], K a multiple of 32.
// 256 threads: ty = tid/16 owns rows ty*4..+3, tx = tid%16 owns NOUT/16 columns.
template <int NOUT> struct TileCols {
  static constexpr int CPT = NOUT / 16;
  static constexpr int VEC = CPT < 4 ? CPT : 4;
  __device__ static __forceinline__ int col(int tx, int c) { return (c / VEC) * (16 * VEC) + tx * VEC + (c % VEC); }
};

// Stage a K-chunk of the weight operand: Ws[kk][c] = getw(k0 + kk, c), kk < KC, c < NOUT.
template <int NOUT, class GetW>
__device__ __forceinline__ void stage_weights(float* Ws, int k0, int kc, GetW getw) {
  constexpr int LDW = NOUT + 4;
#pragma unroll 8
  for (int idx = threadIdx.x; idx < kc * NOUT; idx += blockDim.x) {
    int kk = idx % kc, c = idx / kc;                 // consecutive threads -> consecutive k (coalesced in W rows)
    Ws[kk * LDW + c] = getw(k0 + kk, c);
  }
}

template <int NOUT>
__device__ __forceinline__ void tile_mma(const float* As, int lda, int k0, int kc, const float* Ws,
                                         float (&acc)[4][TileCols<NOUT>::CPT]) {
  using TC = TileCols<NOUT>;
  constexpr int LDW = NOUT + 4;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int kk = 0; kk < kc; ++kk) {
    float a[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = As[(ty * 4 + i) * lda + k0 + kk];
    float w[TC::CPT];
#pragma unroll
    for (int c = 0; c < TC::CPT; ++c) w[c] = Ws[kk * LDW + TC::col(tx, c)];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) acc[i][c] = fmaf(a[i], w[c], acc[i][c]);
  }
}

// Full tile GEMM over K with the weight operand streamed through shared memory in KC chunks.
// Callers must __syncthreads() after filling As and may not touch Ws concurrently.
template <int NOUT, class GetW>
__device__ __forceinline__ void tile_gemm(const float* As, int lda, int K, float* Ws, GetW getw,
                                          float (&acc)[4][TileCols<NOUT>::CPT]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < TileCols<NOUT>::CPT; ++c) acc[i][c] = 0.f;
  for (int k0 = 0; k0 < K; k0 += GCCB_KC) {
    int kc = K - k0 < GCCB_KC ? K - k0 : GCCB_KC;
    __syncthreads();                                   // previous chunk fully consumed
    stage_weights<NOUT>(Ws, k0, kc, getw);
    __syncthreads();
    tile_mma<NOUT>(As, lda, k0, kc, Ws, acc);
  }
}

// Column sums of a per-thread [4][CPT] tile fragment -> shared red[2][NOUT] (sum, sum sq),
// then double atomics into `sums` [2][NOUT].  vals outside the valid rows must be zero.
template <int NOUT>
__device__ __forceinline__ void tile_colstats(const float (&v)[4][TileCols<NOUT>::CPT], float* red /*[2][16][NOUT]*/,
                                              double* __restrict__ sums) {
  using TC = TileCols<NOUT>;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int c = 0; c < TC::CPT; ++c) {
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { s += v[i][c]; q = fmaf(v[i][c], v[i][c], q); }
    red[(0 * 16 + ty) * NOUT + TC::col(tx, c)] = s;
    red[(1 * 16 + ty) * NOUT + TC::col(tx, c)] = q;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 2 * NOUT; idx += blockDim.x) {
    int which = idx / NOUT, c = idx - which * NOUT;
    float s = 0.f;
#pragma unroll
    for (int t = 0; t < 16; ++t) s += red[(which * 16 + t) * NOUT + c];
    atomicAdd(&sums[which * NOUT + c], (double)s);
  }
  __syncthreads();
}

// Kernels of the GIN path that the GAT encoder (gat.cu) launches as they are: the input assembly, the split-K
// weight gradient with its reduce, and the degree-embedding scatter.
__global__ void __launch_bounds__(256)
gin_build_x0_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ pos,
                    const int32_t* __restrict__ sub_deg, const int32_t* __restrict__ graph_id,
                    const float* __restrict__ emb, float* __restrict__ x0, double* __restrict__ zero,
                    int64_t n_zero);
__global__ void __launch_bounds__(256)
gin_wgrad_kernel(const int32_t* __restrict__ node_off_v, int B, int H, int KQ, const float* __restrict__ P,
                 const float* __restrict__ Q, const double* __restrict__ q_sums, const float* __restrict__ q_gamma,
                 const float* __restrict__ q_beta, float bn_eps, float* __restrict__ part);
__global__ void __launch_bounds__(256)
gin_wgrad_reduce_kernel(int H, int KQ, int in_features, const float* __restrict__ part, float* __restrict__ gw,
                        float* __restrict__ gb);
__global__ void __launch_bounds__(256)
gin_bwd_emb_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ sub_deg,
                   const float* __restrict__ dx0, float* __restrict__ gemb);

}  // namespace gccb
