// gin_bwd.cu -- hand-written backward of the GIN encoder (one view).
//
// Replaces autograd's loss.backward() (train.py:408) through GraphEncoder.forward /
// UnsupervisedGIN.forward (gcc/models/graph_encoder.py:152-196, gcc/models/gin.py:213-232):
// normalize -> dropout/prediction heads -> SumPooling broadcast -> per GIN layer
// [BN_b, ReLU, BN_a, ReLU, Linear2, ReLU, BN_1, Linear1, (1+eps)h + sum_nbr h] -> degree
// embedding.  Train-mode BatchNorm backward needs two column reductions per BN over all
// N rows, so each layer is a chain of reduce / apply kernels; elementwise intermediates
// are recomputed from the stashed pre-activations (z1, z2) instead of being stored.
// Adjacency is assumed symmetric (the reference's input contract, gcc/utils/x2dgl.py:40-62),
// so the transpose aggregation is the same gather as the forward.
#include "gin_common.cuh"
#include "tc_gemm.cuh"
#ifndef GCCB_EMU
#include <cuda_bf16.h>
#endif

namespace gccb {

// ---- prediction heads + normalisation backward (one CTA per graph) ------------------------
template <int H>
__global__ void __launch_bounds__(256)
gin_pool_predict_bwd_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B,
                            const float* __restrict__ params, gccb_gin_layout_t lay,
                            const float* __restrict__ score, const float* __restrict__ dfeat,
                            uint64_t drop_key, uint64_t drop_step, int drop_layer_base,
                            uint32_t keep_thresh, int DW, float* __restrict__ dS,
                            float* __restrict__ dpool, double* __restrict__ zero, int n_zero) {
  // GCCB_GPB graphs per CTA, like the forward heads: every head weight is read once for all of them
  constexpr int G = GCCB_GPB;
  __shared__ float ds[G][H];
  __shared__ float dsl[G][H];
  const int g0 = blockIdx.x * G, tid = threadIdx.x, lane = tid & 31;
  const int ng = min(G, B - g0);
  pdl_wait();
  // the BatchNorm-backward reductions of this call (SIMT path; the tensor-core path passes none): first written by
  // gin_bwd_dh_kernel, last read on the side stream of the previous call, which the caller joined before this one
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_zero; i += gridDim.x * blockDim.x) zero[i] = 0.0;
  if (node_off_v[B] < 0) return;
  // F.normalize backward: y = x / max(||x||, eps) -- one warp per graph
  for (int gi = tid >> 5; gi < G; gi += 8) {
    if (gi >= ng) {
      for (int o = lane; o < H; o += 32) ds[gi][o] = 0.f;
      continue;
    }
    const int g = g0 + gi;
    float ss = 0.f, dot = 0.f;
    for (int o = lane; o < H; o += 32) {
      const float x = score[(size_t)g * H + o];
      ss = fmaf(x, x, ss);
      dot = fmaf(x, dfeat[(size_t)g * H + o], dot);
    }
    ss = warp_sum(ss);
    dot = warp_sum(dot);
    const float nrm = sqrtf(ss);
    for (int o = lane; o < H; o += 32) {
      const float x = score[(size_t)g * H + o], gy = dfeat[(size_t)g * H + o];
      float dx;
      if (!d.norm) dx = gy;
      else if (nrm > d.norm_eps) dx = (gy - x * (dot / (nrm * nrm))) / nrm;   // d/dx [x/||x||]
      else dx = gy / d.norm_eps;                                              // clamped branch
      ds[gi][o] = dx;
    }
  }
  __syncthreads();
  for (int l = 0; l < d.L; ++l) {
    const int inf = l == 0 ? d.din : H;
    for (int i = tid; i < G * H; i += 256) {
      const int gi = i / H, o = i - gi * H;
      float v = ds[gi][o];
      if (gi < ng) {
        if (drop_layer_base >= 0) {
          const uint32_t e = (uint32_t)((g0 + gi) * H + o);
          u32x4 w = philox_at(drop_key, drop_step, e >> 2, 0, (uint32_t)(drop_layer_base + l), GCCB_TAG_DROPOUT);
          const uint32_t word = (e & 3u) == 0 ? w.x : (e & 3u) == 1 ? w.y : (e & 3u) == 2 ? w.z : w.w;
          v = word < keep_thresh ? v / (1.0f - d.drop_p) : 0.f;
        }
        dS[((size_t)l * B + g0 + gi) * H + o] = v;
      }
      dsl[gi][o] = v;
    }
    __syncthreads();
    const float* Wp = params + lay.wp[l];
    for (int k = tid; k < DW; k += 256) {
      float sg[G];
#pragma unroll
      for (int gi = 0; gi < G; ++gi) sg[gi] = 0.f;
      if (k < inf) {
#pragma unroll 4
        for (int o = 0; o < H; ++o) {
          const float w = Wp[(size_t)o * inf + k];
#pragma unroll
          for (int gi = 0; gi < G; ++gi) sg[gi] = fmaf(dsl[gi][o], w, sg[gi]);
        }
      }
#pragma unroll
      for (int gi = 0; gi < G; ++gi)
        if (gi < ng) dpool[((size_t)l * B + g0 + gi) * DW + k] = sg[gi];
    }
    __syncthreads();
  }
}

// dWp_l[o][k] += sum_g dS[l][g][o] * pooled_l[g][k] ;  dbp_l[o] += sum_g dS[l][g][o]
__global__ void __launch_bounds__(256)
gin_pred_wgrad_kernel(GinDims d, int B, gccb_gin_layout_t lay, const float* __restrict__ dS,
                      const float* __restrict__ pooled, int PW, float* __restrict__ grads) {
  const int l = blockIdx.y, H = d.H;
  const int inf = l == 0 ? d.din : H;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();
  if (idx < H * inf) {
    const int o = idx / inf, k = idx - o * inf;
    float s = 0.f;
    for (int g = 0; g < B; ++g)
      s = fmaf(dS[((size_t)l * B + g) * H + o], pooled[((size_t)l * B + g) * PW + k], s);
    grads[lay.wp[l] + idx] += s;
  } else if (idx < H * inf + H) {
    const int o = idx - H * inf;
    float s = 0.f;
    for (int g = 0; g < B; ++g) s += dS[((size_t)l * B + g) * H + o];
    grads[lay.bp[l] + o] += s;
  }
}

// BN coefficient bundle in shared memory: mean | invstd | sc | sh   (4*H floats)
struct BnC { const float *mean, *invstd, *sc, *sh; };
__device__ __forceinline__ BnC bnc(const float* p, int H) { BnC b; b.mean = p; b.invstd = p + H; b.sc = p + 2 * H; b.sh = p + 3 * H; return b; }

// Recompute the elementwise chain at (r, c) from z2 and dh:
//   ya = bn_a(z2), y = relu(ya), yhat = (y - mean_b) invstd_b, hb = bn_b(y); g4 = hb > 0 ? dh : 0
__device__ __forceinline__ void chain_g4(float z2v, float dhv, const BnC& A, const BnC& Bc, int c,
                                         float* ya, float* yhat, float* g4) {
  float yap = fmaf(z2v, A.sc[c], A.sh[c]);
  float y = fmaxf(yap, 0.f);
  float hb = fmaf(y, Bc.sc[c], Bc.sh[c]);
  *ya = yap;
  *yhat = (y - Bc.mean[c]) * Bc.invstd[c];
  *g4 = hb > 0.f ? dhv : 0.f;
}

// dh_j[i] = dpool_j[gid[i]] + (has_da ? da[i] + sum_nbr da[nbr] : 0)      (width W)
// BNB: also BN_b's backward reduction of the layer (sum g4, sum g4*yhat per column, chain_g4 from z2 and the
// finished dh row) into redB_out, the quantities gin_bwd_reduce_kernel's BN_a pass and GEMM2 consume.
template <int W, bool BNB>
__global__ void __launch_bounds__(256)
gin_bwd_dh_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
                  const int32_t* __restrict__ indices, const int32_t* __restrict__ graph_id,
                  const float* __restrict__ dpool_j, int DW, const float* __restrict__ da, int has_da,
                  float* __restrict__ dh, const float* __restrict__ z2, const double* __restrict__ sums_a,
                  const float* __restrict__ ga, const float* __restrict__ bea, const double* __restrict__ sums_b,
                  const float* __restrict__ gb, const float* __restrict__ beb, float bn_eps,
                  double* __restrict__ redB_out) {
  __shared__ float scratch[8 * W];
  __shared__ float coef[BNB ? 8 * W : 1];            // bn_a | bn_b bundles
  __shared__ float red[BNB ? 9 * 2 * W : 1];         // [8 warps + hub rows][sum g4 | sum g4*yhat][W]
  __shared__ int hub_rows[GCCB_HUB_QUEUE];
  __shared__ int n_hub;
  pdl_wait();
  const int N = node_off_v[B];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int V4 = W / 4, PERV = (V4 + 31) / 32;
  // A warp pass finishes RPW rows, LW lanes per row (W = 64: two half-warps, W = 32: four quarter-warps, wider rows:
  // one warp), rows dealt round-robin over the grid's warps, no barrier in the loop; hub rows are queued per CTA and
  // gathered by its 8 warps together afterwards (see gin_agg_cast_kernel).  A lane owns the same columns in every
  // row it finishes, so its BN_b partial sums stay in registers until one combine per CTA.
  constexpr int LW = V4 < 32 ? V4 : 32, RPW = 32 / LW;
  const int sub = lane / LW, vl = lane - sub * LW;
  if (tid == 0) n_hub = 0;
  if constexpr (BNB) {
    bn_prepare(sums_a, N, W, ga, bea, bn_eps, coef, coef + W, coef + 2 * W, coef + 3 * W, nullptr, false, false, 0.f);
    bn_prepare(sums_b, N, W, gb, beb, bn_eps, coef + 4 * W, coef + 5 * W, coef + 6 * W, coef + 7 * W, nullptr, false,
               false, 0.f);
  }
  __syncthreads();
  const BnC A = bnc(coef, W), Bc = bnc(coef + 4 * W, W);
  float bs[PERV][4], bq[PERV][4];
#pragma unroll
  for (int j = 0; j < PERV; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) bs[j][k] = bq[j][k] = 0.f;
  for (int r0 = (blockIdx.x * 8 + warp) * RPW; r0 < N; r0 += gridDim.x * 8 * RPW) {
    const int r = r0 + sub;
    const bool live = r < N;
    int beg = 0, end = 0;
    if (live) { beg = indptr[r]; end = indptr[r + 1]; }
    bool queued = false;
    if (has_da) {                                    // every lane reaches the shuffle, whatever its row
      const bool hub = live && end - beg > GCCB_HUB_DEG;
      int slot = GCCB_HUB_QUEUE;
      if (hub && vl == 0) slot = atomicAdd(&n_hub, 1);
      slot = __shfl_sync(0xffffffffu, slot, sub * LW);
      if (hub && slot < GCCB_HUB_QUEUE) {            // queue full: the lanes of the row gather it alone
        if (vl == 0) hub_rows[slot] = r;
        queued = true;
      }
    }
    if (!live || queued) continue;
    float4 zv[PERV];                                 // BN_b's input, loaded before the gather so that it overlaps it
    if constexpr (BNB) {
#pragma unroll
      for (int j = 0; j < PERV; ++j) {
        const int v = vl + 32 * j;
        if (v < V4) zv[j] = *reinterpret_cast<const float4*>(z2 + (size_t)r * W + 4 * v);
      }
    }
    const int g = graph_id[r];
    float4 acc[PERV];
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = vl + 32 * j;
      acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v < V4) {
        acc[j] = *reinterpret_cast<const float4*>(dpool_j + (size_t)g * DW + 4 * v);
        if (has_da) {
          const float4 x = *reinterpret_cast<const float4*>(da + (size_t)r * W + 4 * v);
          acc[j].x += x.x; acc[j].y += x.y; acc[j].z += x.z; acc[j].w += x.w;
        }
      }
    }
    if (has_da) gather_range4<W>(da, indices, beg, end, vl, acc);
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = vl + 32 * j;
      if (v < V4) {
        *reinterpret_cast<float4*>(dh + (size_t)r * W + 4 * v) = acc[j];
        if constexpr (BNB) {
          const float zz[4] = {zv[j].x, zv[j].y, zv[j].z, zv[j].w}, dd[4] = {acc[j].x, acc[j].y, acc[j].z, acc[j].w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float ya, yhat, g4;
            chain_g4(zz[k], dd[k], A, Bc, 4 * v + k, &ya, &yhat, &g4);
            bs[j][k] += g4;
            bq[j][k] = fmaf(g4, yhat, bq[j][k]);
          }
        }
      }
    }
  }
  __syncthreads();
  float hs = 0.f, hq = 0.f;                          // hub rows: thread tid < W owns column tid
  const int nh = min(n_hub, GCCB_HUB_QUEUE);
  for (int hi = 0; hi < nh; ++hi) {
    const int rh = hub_rows[hi];
    const float s = gather_hub<W>(da, indices, indptr[rh], indptr[rh + 1], scratch);
    if (tid < W) {
      const float dv = dpool_j[(size_t)graph_id[rh] * DW + tid] + da[(size_t)rh * W + tid] + s;
      dh[(size_t)rh * W + tid] = dv;
      if constexpr (BNB) {
        float ya, yhat, g4;
        chain_g4(z2[(size_t)rh * W + tid], dv, A, Bc, tid, &ya, &yhat, &g4);
        hs += g4;
        hq = fmaf(g4, yhat, hq);
      }
    }
  }
  if constexpr (BNB) {
#pragma unroll
    for (int o = LW; o < 32; o <<= 1)                // the RPW rows of a warp pass share their columns
#pragma unroll
      for (int j = 0; j < PERV; ++j)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          bs[j][k] += __shfl_xor_sync(0xffffffffu, bs[j][k], o);
          bq[j][k] += __shfl_xor_sync(0xffffffffu, bq[j][k], o);
        }
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = vl + 32 * j;
      if (sub == 0 && v < V4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          red[(warp * 2 + 0) * W + 4 * v + k] = bs[j][k];
          red[(warp * 2 + 1) * W + 4 * v + k] = bq[j][k];
        }
      }
    }
    if (tid < W) {
      red[16 * W + tid] = hs;
      red[17 * W + tid] = hq;
    }
    __syncthreads();
    for (int idx = tid; idx < 2 * W; idx += 256) {
      const int which = idx / W, c = idx - which * W;
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 9; ++w) t += red[(w * 2 + which) * W + c];
      atomicAdd(&redB_out[which * W + c], (double)t);
    }
  }
}

// Column reductions for BN_a (sum g3, sum g3*z2hat); BN_b's (sum g4, sum g4*yhat) come from gin_bwd_dh_kernel
// thread -> 4 consecutive columns of every RP-th row, two rows (4 x 16-byte loads) in flight per thread
template <int H>
__global__ void __launch_bounds__(256)
gin_bwd_reduce_kernel(const int32_t* __restrict__ node_off_v, int B,
                      const float* __restrict__ z2, const float* __restrict__ dh,
                      const double* __restrict__ sums_a, const float* __restrict__ ga,
                      const float* __restrict__ bea, const double* __restrict__ sums_b,
                      const float* __restrict__ gb, const float* __restrict__ beb, float bn_eps,
                      const double* __restrict__ redB_in, double* __restrict__ red_out) {
  __shared__ float coef_a[4 * H];
  __shared__ float coef_b[4 * H];
  __shared__ float red[2 * 1024];
  pdl_wait();
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  bn_prepare(sums_a, N, H, ga, bea, bn_eps, coef_a, coef_a + H, coef_a + 2 * H, coef_a + 3 * H, nullptr, false, false, 0.f);
  bn_prepare(sums_b, N, H, gb, beb, bn_eps, coef_b, coef_b + H, coef_b + 2 * H, coef_b + 3 * H, nullptr, false, false, 0.f);
  __syncthreads();
  const BnC A = bnc(coef_a, H), Bc = bnc(coef_b, H);
  constexpr int TPR = H / 4, RP = 256 / TPR;
  const int c4 = (tid % TPR) * 4, rsub = tid / TPR;
  const float invN = N > 0 ? 1.0f / (float)N : 0.f;
  float m_g4[4], m_g4y[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { m_g4[k] = (float)(redB_in[c4 + k] * invN); m_g4y[k] = (float)(redB_in[H + c4 + k] * invN); }
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  const int stride = gridDim.x * RP;
  for (int r = blockIdx.x * RP + rsub; r < N; r += 2 * stride) {
    float4 zv[2], dv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int rr = r + u * stride;
      const bool ok = rr < N;
      zv[u] = ok ? *reinterpret_cast<const float4*>(z2 + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      dv[u] = ok ? *reinterpret_cast<const float4*>(dh + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (r + u * stride < N) {
        const float zz[4] = {zv[u].x, zv[u].y, zv[u].z, zv[u].w}, dd[4] = {dv[u].x, dv[u].y, dv[u].z, dv[u].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = c4 + k;
          float ya, yhat, g4;
          chain_g4(zz[k], dd[k], A, Bc, c, &ya, &yhat, &g4);
          const float dy = Bc.sc[c] * (g4 - m_g4[k] - yhat * m_g4y[k]);
          const float g3 = ya > 0.f ? dy : 0.f;
          const float z2hat = (zz[k] - A.mean[c]) * A.invstd[c];
          s[k] += g3;
          q[k] = fmaf(g3, z2hat, q[k]);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    red[(0 * RP + rsub) * H + c4 + k] = s[k];
    red[(RP + rsub) * H + c4 + k] = q[k];
  }
  __syncthreads();
  for (int idx = tid; idx < 2 * H; idx += 256) {
    int which = idx / H, cc = idx - which * H;
    float t = 0.f;
    for (int j = 0; j < RP; ++j) t += red[(which * RP + j) * H + cc];
    atomicAdd(&red_out[which * H + cc], (double)t);
  }
}

// two-quantity column statistics of tile fragments (sum of s, sum of q) -> double atomics
template <int NOUT>
__device__ __forceinline__ void tile_colstats2(const float (&sv)[4][TileCols<NOUT>::CPT],
                                               const float (&qv)[4][TileCols<NOUT>::CPT], float* red,
                                               double* __restrict__ sums) {
  using TC = TileCols<NOUT>;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int c = 0; c < TC::CPT; ++c) {
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { s += sv[i][c]; q += qv[i][c]; }
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

// dz2 = BN_a backward of g3 (written out); dx1 = dz2 W2; g1 = [bn1(z1) > 0] dx1 (written out);
// column sums of g1 and g1 * z1hat.
// At hidden 64 at most 64 registers per thread (63, no spills; 80 unbounded, same instructions otherwise): a CTA
// then takes 16,384 registers and fits on an SM whose eigensolver CTAs leave a quarter of the register file free
// (three dense n <= 96 CTAs, or a 512-thread ChFSI CTA and a dense one), where an 80-register CTA has to wait.
template <int H>
__global__ void __launch_bounds__(256, H == 64 ? 4 : 0)
gin_bwd_gemm2_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                     const float* __restrict__ z2, const float* __restrict__ dh,
                     const double* __restrict__ sums_1, const float* __restrict__ g1w,
                     const float* __restrict__ be1, const double* __restrict__ sums_a,
                     const float* __restrict__ ga, const float* __restrict__ bea,
                     const double* __restrict__ sums_b, const float* __restrict__ gb,
                     const float* __restrict__ beb, float bn_eps, const double* __restrict__ redB,
                     const double* __restrict__ redA, const float* __restrict__ W2,
                     float* __restrict__ dz2_out, float* __restrict__ g1_out,
                     double* __restrict__ red1_out) {
  GCCB_DYN_SMEM(float, smem);
  constexpr int LDA = H + 1;
  float* As = smem;
  float* Ws = As + GCCB_TILE_ROWS * LDA;
  float* red = Ws + GCCB_KC * (H + 4);
  float* coef = red + 2 * 16 * H;            // 3 bundles of 4H: bn1 | bn_a | bn_b
  float* rmean = coef + 12 * H;              // m_g4 | m_g4y | m_g3 | m_g3z   (4H)
  pdl_wait();
  const int N = node_off_v[B];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  using TC = TileCols<H>;
  bn_prepare(sums_1, N, H, g1w, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, nullptr, false, false, 0.f);
  bn_prepare(sums_a, N, H, ga, bea, bn_eps, coef + 4 * H, coef + 5 * H, coef + 6 * H, coef + 7 * H, nullptr, false, false, 0.f);
  bn_prepare(sums_b, N, H, gb, beb, bn_eps, coef + 8 * H, coef + 9 * H, coef + 10 * H, coef + 11 * H, nullptr, false, false, 0.f);
  const double invN = N > 0 ? 1.0 / (double)N : 0.0;
  for (int c = tid; c < H; c += 256) {
    rmean[c] = (float)(redB[c] * invN);
    rmean[H + c] = (float)(redB[H + c] * invN);
    rmean[2 * H + c] = (float)(redA[c] * invN);
    rmean[3 * H + c] = (float)(redA[H + c] * invN);
  }
  __syncthreads();
  const BnC C1 = bnc(coef, H), A = bnc(coef + 4 * H, H), Bc = bnc(coef + 8 * H, H);
  for (int tile = blockIdx.x; tile * GCCB_TILE_ROWS < N; tile += gridDim.x) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();
#pragma unroll 8
    for (int idx = tid; idx < GCCB_TILE_ROWS * H; idx += 256) {   // 8 independent L2 loads in flight
      int rr = idx / H, c = idx - rr * H;
      int r = row0 + rr;
      float dz = 0.f;
      if (r < N) {
        float ya, yhat, g4;
        float zv = z2[(size_t)r * H + c];
        chain_g4(zv, dh[(size_t)r * H + c], A, Bc, c, &ya, &yhat, &g4);
        float dy = Bc.sc[c] * (g4 - rmean[c] - yhat * rmean[H + c]);
        float g3 = ya > 0.f ? dy : 0.f;
        float z2hat = (zv - A.mean[c]) * A.invstd[c];
        dz = A.sc[c] * (g3 - rmean[2 * H + c] - z2hat * rmean[3 * H + c]);
        dz2_out[(size_t)r * H + c] = dz;
      }
      As[rr * LDA + c] = dz;
    }
    __syncthreads();
    float acc[4][TC::CPT];
    // dx1[r][k] = sum_o dz2[r][o] W2[o][k]  -> operand row index = o, column = k
    tile_gemm<H>(As, LDA, H, Ws, [&](int o, int k) { return W2[(size_t)o * H + k]; }, acc);
    float sv[4][TC::CPT], qv[4][TC::CPT];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + ty * 4 + i;
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) {
        const int col = TC::col(tx, c);
        float g = 0.f, gz = 0.f;
        if (r < N) {
          float zv = z1[(size_t)r * H + col];
          float pre = fmaf(zv, C1.sc[col], C1.sh[col]);
          g = pre > 0.f ? acc[i][c] : 0.f;
          gz = g * ((zv - C1.mean[col]) * C1.invstd[col]);
          g1_out[(size_t)r * H + col] = g;
        }
        sv[i][c] = g;
        qv[i][c] = gz;
      }
    }
    tile_colstats2<H>(sv, qv, red, red1_out);
  }
}

// dz1 = BN_1 backward of g1 (in place over g1); da = dz1 W1 (width KIN, zero beyond in_features)
template <int KIN, int H>
__global__ void __launch_bounds__(256)
gin_bwd_gemm1_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                     float* __restrict__ g1_dz1, const double* __restrict__ sums_1,
                     const float* __restrict__ g1w, const float* __restrict__ be1, float bn_eps,
                     const double* __restrict__ red1, const float* __restrict__ W1, int in_features,
                     float* __restrict__ da_out) {
  GCCB_DYN_SMEM(float, smem);
  constexpr int LDA = H + 1;
  float* As = smem;
  float* Ws = As + GCCB_TILE_ROWS * LDA;
  float* coef = Ws + GCCB_KC * (KIN + 4);
  float* rmean = coef + 4 * H;
  pdl_wait();
  const int N = node_off_v[B];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  using TC = TileCols<KIN>;
  bn_prepare(sums_1, N, H, g1w, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, nullptr, false, false, 0.f);
  const double invN = N > 0 ? 1.0 / (double)N : 0.0;
  for (int c = tid; c < H; c += 256) {
    rmean[c] = (float)(red1[c] * invN);
    rmean[H + c] = (float)(red1[H + c] * invN);
  }
  __syncthreads();
  const BnC C1 = bnc(coef, H);
  for (int tile = blockIdx.x; tile * GCCB_TILE_ROWS < N; tile += gridDim.x) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();
#pragma unroll 8
    for (int idx = tid; idx < GCCB_TILE_ROWS * H; idx += 256) {   // 8 independent L2 loads in flight
      int rr = idx / H, c = idx - rr * H;
      int r = row0 + rr;
      float dz = 0.f;
      if (r < N) {
        float zhat = (z1[(size_t)r * H + c] - C1.mean[c]) * C1.invstd[c];
        dz = C1.sc[c] * (g1_dz1[(size_t)r * H + c] - rmean[c] - zhat * rmean[H + c]);
        g1_dz1[(size_t)r * H + c] = dz;
      }
      As[rr * LDA + c] = dz;
    }
    __syncthreads();
    float acc[4][TC::CPT];
    tile_gemm<KIN>(As, LDA, H, Ws,
                   [&](int o, int k) { return k < in_features ? W1[(size_t)o * in_features + k] : 0.f; }, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + ty * 4 + i;
      if (r < N) {
#pragma unroll
        for (int c = 0; c < TC::CPT; ++c) da_out[(size_t)r * KIN + TC::col(tx, c)] = acc[i][c];
      }
    }
  }
}

// Weight gradient split over row chunks: part[chunk][o][k] = sum_{r in chunk} P[r][o] * Q'[r][k],
// bias part[chunk][H*KQ + o] = sum_r P[r][o].  Q' = relu(Q*sc + sh) when sc != null (x1 from z1).
// grid = (CHUNKS, ceil(H/64) * ceil(KQ/64)), block 256: thread (ty, tx) owns a 4x4 output patch.
__global__ void __launch_bounds__(256)
gin_wgrad_kernel(const int32_t* __restrict__ node_off_v, int B, int H, int KQ,
                 const float* __restrict__ P, const float* __restrict__ Q,
                 const double* __restrict__ q_sums, const float* __restrict__ q_gamma,
                 const float* __restrict__ q_beta, float bn_eps, float* __restrict__ part) {
  __shared__ float Ps[GCCB_TILE_ROWS][65];
  __shared__ float Qs[GCCB_TILE_ROWS][65];
  __shared__ float qsc[64], qsh[64];
  pdl_wait();
  const int N = node_off_v[B];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int kblocks = (KQ + 63) / 64;
  const int ob = blockIdx.y / kblocks, kb = blockIdx.y - ob * kblocks;
  const int o0 = ob * 64, k0 = kb * 64;
  const bool xform = q_sums != nullptr;
  if (xform) {
    for (int c = tid; c < 64; c += 256) {
      int k = k0 + c;
      float sc = 0.f, sh = 0.f;
      if (k < KQ) {
        double n = N > 0 ? (double)N : 1.0;
        double mean = q_sums[k] / n, var = q_sums[KQ + k] / n - mean * mean;
        if (var < 0.0) var = 0.0;
        float invstd = 1.0f / sqrtf((float)var + bn_eps);
        sc = q_gamma[k] * invstd;
        sh = q_beta[k] - (float)mean * sc;
      }
      qsc[c] = sc; qsh[c] = sh;
    }
  }
  __syncthreads();
  float acc[4][4];
  float bacc = 0.f;                                   // bias partial: thread (tid < 64) owns column o0+tid
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int tiles = (N + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  const int per = (tiles + GCCB_WG_CHUNKS - 1) / GCCB_WG_CHUNKS;
  const int t_beg = blockIdx.x * per, t_end = min(tiles, t_beg + per);
  for (int tile = t_beg; tile < t_end; ++tile) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();
#pragma unroll 8
    for (int idx = tid; idx < GCCB_TILE_ROWS * 64; idx += 256) {
      int rr = idx >> 6, c = idx & 63;
      int r = row0 + rr;
      float pv = 0.f, qv = 0.f;
      if (r < N) {
        if (o0 + c < H) pv = P[(size_t)r * H + o0 + c];
        if (k0 + c < KQ) {
          qv = Q[(size_t)r * KQ + k0 + c];
          if (xform) qv = fmaxf(fmaf(qv, qsc[c], qsh[c]), 0.f);
        }
      }
      Ps[rr][c] = pv;
      Qs[rr][c] = qv;
    }
    __syncthreads();
    for (int rr = 0; rr < GCCB_TILE_ROWS; ++rr) {
      float p[4], q[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) p[i] = Ps[rr][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) q[j] = Qs[rr][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(p[i], q[j], acc[i][j]);
    }
    if (kb == 0 && tid < 64)
      for (int rr = 0; rr < GCCB_TILE_ROWS; ++rr) bacc += Ps[rr][tid];
  }
  float* mypart = part + (size_t)blockIdx.x * ((size_t)H * KQ + H);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int o = o0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = k0 + tx * 4 + j;
      if (o < H && k < KQ) mypart[(size_t)o * KQ + k] = acc[i][j];
    }
  }
  if (kb == 0 && tid < 64 && o0 + tid < H) mypart[(size_t)H * KQ + o0 + tid] = bacc;
}

// grads[w_off + o*in_features + k] += sum_chunks part[.][o][k] (k < in_features);  bias likewise
__global__ void __launch_bounds__(256)
gin_wgrad_reduce_kernel(int H, int KQ, int in_features, const float* __restrict__ part,
                        float* __restrict__ gw, float* __restrict__ gb) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)H * KQ + H;
  pdl_wait();
  if (idx < H * KQ) {
    const int o = idx / KQ, k = idx - o * KQ;
    if (k < in_features) {
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;          // fixed order, 4 loads in flight
      for (int ch = 0; ch < GCCB_WG_CHUNKS; ch += 4) {
        s0 += part[(ch + 0) * stride + idx]; s1 += part[(ch + 1) * stride + idx];
        s2 += part[(ch + 2) * stride + idx]; s3 += part[(ch + 3) * stride + idx];
      }
      gw[(size_t)o * in_features + k] += (s0 + s1) + (s2 + s3);
    }
  } else if (idx < H * KQ + H) {
    float s = 0.f;
    for (int ch = 0; ch < GCCB_WG_CHUNKS; ++ch) s += part[ch * stride + idx];
    gb[idx - H * KQ] += s;
  }
}

// BN affine gradients: d gamma = sum g*xhat (red[1]), d beta = sum g (red[0])
__global__ void gin_bn_grads_kernel(int H, const double* __restrict__ red, float* __restrict__ gw,
                                    float* __restrict__ gb) {
  pdl_wait();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < H) { gb[c] += (float)red[c]; gw[c] += (float)red[H + c]; }
}

// degree-embedding gradient: demb[clamp(deg_i)][c] += dX0[i][P + c]  (shared-memory histogram
// per CTA, then one global atomic per touched entry)
__global__ void __launch_bounds__(256)
gin_bwd_emb_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B,
                   const int32_t* __restrict__ sub_deg, const float* __restrict__ dx0,
                   float* __restrict__ gemb) {
  GCCB_DYN_SMEM(float, hist);                // [(maxdeg+1)][D]
  pdl_wait();
  const int N = node_off_v[B];
  const int cells = (d.maxdeg + 1) * d.D;
  for (int i = threadIdx.x; i < cells; i += blockDim.x) hist[i] = 0.f;
  __syncthreads();
  const int total = N * d.D;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int r = idx / d.D, c = idx - r * d.D;
    int dg = sub_deg[r];
    dg = dg < 0 ? 0 : (dg > d.maxdeg ? d.maxdeg : dg);
    atomicAdd(&hist[dg * d.D + c], dx0[(size_t)r * GCCB_DINP + d.P + c]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cells; i += blockDim.x) {
    float v = hist[i];
    if (v != 0.f) atomicAdd(&gemb[i], v);
  }
}

struct BwdArgs {
  GinDims d;
  const gccb_batch_t* batch;
  int view;
  const float* params;
  gccb_gin_layout_t lay;
  const char* acts;
  ActsLayout al;
  const float* dfeat;
  float* grads;
  char* ws;
  BwdLayout bl;
  uint64_t drop_key, drop_step;
  int drop_base;
  gccb_stream_t stream;
};

template <int H>
static int run_backward(const BwdArgs& a) {
  const GinDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const int32_t* graph_id = a.batch->graph_id + (size_t)a.view * cap;
  const double* stats = (const double*)(a.acts + a.al.stats);
  float* dh = (float*)(a.ws + a.bl.dh);
  float* da = (float*)(a.ws + a.bl.da);
  double* red = (double*)(a.ws + a.bl.red);
  float* dS = (float*)(a.ws + a.bl.dS);
  float* dpool = (float*)(a.ws + a.bl.dpool);
  float* part = (float*)(a.ws + a.bl.part);
  float* part1 = (float*)(a.ws + a.bl.part1);
  const float* P = a.params;
  float* G = a.grads;
  const int DW = a.bl.DW;
  const int tiles = (cap + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  const int grid = tiles < 4 * GCCB_NUM_SMS ? tiles : 4 * GCCB_NUM_SMS;
  const uint32_t keep = (uint32_t)fmin((1.0 - (double)d.drop_p) * 4294967296.0, 4294967295.0);
  // The input-gradient chain (dh -> BN reductions -> GEMM2 -> GEMM1 -> next layer) is the critical
  // path; weight / BatchNorm / head gradients only consume its by-products, so they run on a side
  // stream (two event forks per layer, after GEMM2 and after GEMM1, one join at the end).  g1/dz2
  // alternate between two buffers so that layer l-1 may overwrite nothing the side stream still reads
  // from layer l; layer l-2 waits for the side work of layer l before reusing its buffers.
  // dW1 runs on a second side stream with its own split-K partials: behind dW2 and the BatchNorm gradients on
  // one stream it started late, and the last layer's dW1 held the final join (before the optimiser).  The
  // second stream follows the first (ev_dw2) before it signals a layer done (ev_side) and before the join.
#ifndef GCCB_EMU
  // The side stream runs one step above the caller's priority: its kernels are short (one wave of CTAs), and
  // at equal priority they queued behind the next chain kernel's CTAs, so the side stream fell behind and the
  // final join (before the optimiser) waited for the last layers' weight gradients.
  StreamKit* kit = stream_kit((cudaStream_t)a.stream, 2, SidePriority::kAboveCaller);
  cudaStream_t main_s = (cudaStream_t)a.stream;
  gccb_stream_t side = kit->side[0], side1 = kit->side[1];
  cudaEvent_t* ev_main = kit->ev;                          // [0..7]  main -> side, per layer
  cudaEvent_t* ev_side = kit->ev + 8;                      // [8..15] side -> main, per layer
  cudaEvent_t ev_head = kit->ev[16], ev_join = kit->ev[17];
  cudaEvent_t ev_gemm2 = kit->ev[18];                      // main -> side after GEMM2, re-recorded per layer
  cudaEvent_t ev_dw2 = kit->ev[19];                        // side -> side1 after a layer's side work, likewise
#else
  gccb_stream_t side = a.stream, side1 = a.stream;
#endif
  // Every kernel here is a programmatic dependent of the one before it on its stream (common.cuh); the heads'
  // backward zeroes the BatchNorm-backward reductions, so that no memset node breaks the chain.
  auto kpb = gin_pool_predict_bwd_kernel<H>;
  GCCB_LAUNCH_PDL(kpb, (B + GCCB_GPB - 1) / GCCB_GPB, 256, 0, a.stream, d, node_off_v, B, P, a.lay, (const float*)(a.acts + a.al.score),
              a.dfeat, a.drop_key, a.drop_step, a.drop_base, keep, DW, dS, dpool, red, (d.L - 1) * 3 * 2 * H);
#ifndef GCCB_EMU
  cudaEventRecord(ev_head, main_s);
  cudaStreamWaitEvent((cudaStream_t)side, ev_head, 0);
#endif
  {
    int maxout = H * (d.din > H ? d.din : H) + H;
    dim3 gr((maxout + 255) / 256, d.L);
    GCCB_LAUNCH_PDL(gin_pred_wgrad_kernel, gr, 256, 0, side, d, B, a.lay, (const float*)dS,
                (const float*)(a.acts + a.al.pooled), a.al.PW, G);
  }
  for (int l = d.L - 2; l >= 0; --l) {
    float* g1 = (float*)(a.ws + a.bl.g1[l & 1]);
    float* dz2 = (float*)(a.ws + a.bl.dz2[l & 1]);
    const int j = l + 1;                                  // hidden_rep index of this layer's output
    const float* z1 = (const float*)(a.acts + a.al.z1[l]);
    const float* z2 = (const float*)(a.acts + a.al.z2[l]);
    const float* a_l = (const float*)(a.acts + a.al.a[l]);
    const double* s1 = stats + (size_t)(l * 3 + 0) * 2 * H;
    const double* sa = stats + (size_t)(l * 3 + 1) * 2 * H;
    const double* sb = stats + (size_t)(l * 3 + 2) * 2 * H;
    double* r1 = red + (size_t)(l * 3 + 0) * 2 * H;
    double* rA = red + (size_t)(l * 3 + 1) * 2 * H;
    double* rB = red + (size_t)(l * 3 + 2) * 2 * H;
    // dh_j = dpool_j broadcast + (I + A) da_{j}   (da of the layer above; none for the top)
    // and BN_b's backward reduction (rB) of this layer
    auto kdh = gin_bwd_dh_kernel<H, true>;
    GCCB_LAUNCH_PDL(kdh, (tiles < 1184 ? tiles : 1184), 256, 0, a.stream, node_off_v, B, indptr, indices, graph_id,
                (const float*)(dpool + (size_t)j * B * DW), DW, (const float*)da, j < d.L - 1 ? 1 : 0, dh, z2, sa,
                P + a.lay.bna_w[l], P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], d.bn_eps, rB);
    auto kred = gin_bwd_reduce_kernel<H>;
    GCCB_LAUNCH_PDL(kred, grid, 256, 0, a.stream, node_off_v, B, z2, (const float*)dh, sa, P + a.lay.bna_w[l],
                P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], d.bn_eps,
                (const double*)rB, rA);
#ifndef GCCB_EMU
    if (l + 2 <= d.L - 2) cudaStreamWaitEvent(main_s, ev_side[l + 2], 0);   // g1/dz2[l&1] free again
#endif
    {
      auto k = gin_bwd_gemm2_kernel<H>;
      size_t sm = ((size_t)GCCB_TILE_ROWS * (H + 1) + (size_t)GCCB_KC * (H + 4) + 2 * 16 * H + 16 * H) * 4;
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH_PDL(k, grid, 256, sm, a.stream, node_off_v, B, z1, z2, (const float*)dh, s1, P + a.lay.bn1_w[l],
                  P + a.lay.bn1_b[l], sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l],
                  P + a.lay.bnb_b[l], d.bn_eps, (const double*)rB, (const double*)rA, P + a.lay.w2[l], dz2,
                  g1, r1);
    }
#ifndef GCCB_EMU
    cudaEventRecord(ev_gemm2, main_s);
    cudaStreamWaitEvent((cudaStream_t)side, ev_gemm2, 0);
#endif
    // side stream, as soon as GEMM2 has left dz2 and the last BatchNorm reduction (r1): dW2 = dz2^T x1
    // (x1 = relu(bn1(z1))) and the three BatchNorm affine gradients
    {
      dim3 gr(GCCB_WG_CHUNKS, ((H + 63) / 64) * ((H + 63) / 64));
      GCCB_LAUNCH_PDL(gin_wgrad_kernel, gr, 256, 0, side, node_off_v, B, H, H, (const float*)dz2, z1, s1,
                  P + a.lay.bn1_w[l], P + a.lay.bn1_b[l], d.bn_eps, part);
      GCCB_LAUNCH_PDL(gin_wgrad_reduce_kernel, (H * H + H + 255) / 256, 256, 0, side, H, H, H,
                  (const float*)part, G + a.lay.w2[l], G + a.lay.b2[l]);
    }
    GCCB_LAUNCH_PDL(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)rB,
                G + a.lay.bnb_w[l], G + a.lay.bnb_b[l]);
    GCCB_LAUNCH_PDL(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)rA,
                G + a.lay.bna_w[l], G + a.lay.bna_b[l]);
    GCCB_LAUNCH_PDL(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)r1,
                G + a.lay.bn1_w[l], G + a.lay.bn1_b[l]);
    const int KQ1 = gin_in_width(d, l), inf = gin_in_features(d, l);
    if (l == 0) {
      auto k = gin_bwd_gemm1_kernel<GCCB_DINP, H>;
      size_t sm = ((size_t)GCCB_TILE_ROWS * (H + 1) + (size_t)GCCB_KC * (GCCB_DINP + 4) + 6 * H) * 4;
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH_PDL(k, grid, 256, sm, a.stream, node_off_v, B, z1, g1, s1, P + a.lay.bn1_w[l], P + a.lay.bn1_b[l],
                  d.bn_eps, (const double*)r1, P + a.lay.w1[l], inf, da);
    } else {
      auto k = gin_bwd_gemm1_kernel<H, H>;
      size_t sm = ((size_t)GCCB_TILE_ROWS * (H + 1) + (size_t)GCCB_KC * (H + 4) + 6 * H) * 4;
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH_PDL(k, grid, 256, sm, a.stream, node_off_v, B, z1, g1, s1, P + a.lay.bn1_w[l], P + a.lay.bn1_b[l],
                  d.bn_eps, (const double*)r1, P + a.lay.w1[l], inf, da);
    }
#ifndef GCCB_EMU
    cudaEventRecord(ev_main[l], main_s);
    cudaStreamWaitEvent((cudaStream_t)side1, ev_main[l], 0);
#endif
    // second side stream, once GEMM1 has turned g1 into dz1: dW1 = dz1^T a
    {
      dim3 gr1(GCCB_WG_CHUNKS, ((H + 63) / 64) * ((KQ1 + 63) / 64));
      GCCB_LAUNCH_PDL(gin_wgrad_kernel, gr1, 256, 0, side1, node_off_v, B, H, KQ1, (const float*)g1, a_l,
                  (const double*)nullptr, (const float*)nullptr, (const float*)nullptr, d.bn_eps, part1);
      GCCB_LAUNCH_PDL(gin_wgrad_reduce_kernel, (H * KQ1 + H + 255) / 256, 256, 0, side1, H, KQ1, inf,
                  (const float*)part1, G + a.lay.w1[l], G + a.lay.b1[l]);
    }
#ifndef GCCB_EMU
    cudaEventRecord(ev_dw2, (cudaStream_t)side);
    cudaStreamWaitEvent((cudaStream_t)side1, ev_dw2, 0);
    cudaEventRecord(ev_side[l], (cudaStream_t)side1);
#endif
  }
  // layer-0 input gradient -> degree embedding
  auto kdh0 = gin_bwd_dh_kernel<GCCB_DINP, false>;
  GCCB_LAUNCH_PDL(kdh0, (tiles < 1184 ? tiles : 1184), 256, 0, a.stream, node_off_v, B, indptr, indices, graph_id, (const float*)dpool, DW,
              (const float*)da, 1, dh, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f, nullptr);
  {
    size_t sm = (size_t)(d.maxdeg + 1) * d.D * sizeof(float);
    auto k = gin_bwd_emb_kernel;
    gccb::ensure_dyn_smem(k, sm);
    GCCB_LAUNCH_PDL(k, 64, 256, sm, a.stream, d, node_off_v, B, sub_deg, (const float*)dh, G + a.lay.emb);
  }
#ifndef GCCB_EMU
  cudaEventRecord(ev_join, (cudaStream_t)side1);
  cudaStreamWaitEvent(main_s, ev_join, 0);
#endif
  return check_launch("gccb_gin_backward");
}


#ifndef GCCB_EMU
// ================================================================================================
// Tensor-core backward (cfg.tensor_cores, hidden >= 128): the four GEMMs of a layer -- dx1 = dz2 W2,
// da = dz1 W1, dW2 = dz2^T x1, dW1 = dz1^T a -- run on wgmma (csrc/tc_gemm.cu); the BatchNorm-backward
// chains between them are the same arithmetic as the SIMT kernels above, as elementwise passes that also
// emit the bf16 operand of the next GEMM.  The biases of the two Linear layers feed train-mode BatchNorms:
// their true gradient is exactly zero (the SIMT path computes rounding noise ~1e-9 there); this path adds
// nothing to them.

// dz2 = BN_a backward of g3 (fp32 stash for the weight gradient + bf16 GEMM operand); block 0 also leaves the
// BatchNorm-1 coefficients (sc | sh) of this layer for the transposed cast of x1 = relu(bn1(z1)).
template <int H>
__global__ void __launch_bounds__(256)
gin_bwd_dz2_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z2,
                   const float* __restrict__ dh, const double* __restrict__ sums_1, const float* __restrict__ g1w,
                   const float* __restrict__ be1, const double* __restrict__ sums_a, const float* __restrict__ ga,
                   const float* __restrict__ bea, const double* __restrict__ sums_b, const float* __restrict__ gb,
                   const float* __restrict__ beb, float bn_eps, const double* __restrict__ redB,
                   const double* __restrict__ redA, float* __restrict__ dz2_out, __nv_bfloat16* __restrict__ dz16,
                   float* __restrict__ coef1_out) {
  __shared__ float coef[12 * H];
  __shared__ float rmean[4 * H];
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  bn_prepare(sums_1, N, H, g1w, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, nullptr, false, false, 0.f);
  bn_prepare(sums_a, N, H, ga, bea, bn_eps, coef + 4 * H, coef + 5 * H, coef + 6 * H, coef + 7 * H, nullptr, false, false, 0.f);
  bn_prepare(sums_b, N, H, gb, beb, bn_eps, coef + 8 * H, coef + 9 * H, coef + 10 * H, coef + 11 * H, nullptr, false, false, 0.f);
  const double invN = N > 0 ? 1.0 / (double)N : 0.0;
  for (int c = tid; c < H; c += 256) {
    rmean[c] = (float)(redB[c] * invN);
    rmean[H + c] = (float)(redB[H + c] * invN);
    rmean[2 * H + c] = (float)(redA[c] * invN);
    rmean[3 * H + c] = (float)(redA[H + c] * invN);
  }
  __syncthreads();
  if (blockIdx.x == 0)
    for (int c = tid; c < H; c += 256) { coef1_out[c] = coef[2 * H + c]; coef1_out[H + c] = coef[3 * H + c]; }
  const BnC A = bnc(coef + 4 * H, H), Bc = bnc(coef + 8 * H, H);
  // 4 consecutive columns per thread (16-byte accesses), two element groups in flight
  const size_t total4 = (size_t)(N > 0 ? N : 0) * (H / 4);
  const size_t gstride = (size_t)gridDim.x * blockDim.x;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x + tid; i0 < total4; i0 += 2 * gstride) {
    float4 zv[2], dv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t i = i0 + u * gstride;
      const bool ok = i < total4;
      zv[u] = ok ? reinterpret_cast<const float4*>(z2)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      dv[u] = ok ? reinterpret_cast<const float4*>(dh)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t i = i0 + u * gstride;
      if (i < total4) {
        const int c0 = (int)(i % (H / 4)) * 4;
        const float zz[4] = {zv[u].x, zv[u].y, zv[u].z, zv[u].w}, dd[4] = {dv[u].x, dv[u].y, dv[u].z, dv[u].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = c0 + k;
          float ya, yhat, g4;
          chain_g4(zz[k], dd[k], A, Bc, c, &ya, &yhat, &g4);
          const float dy = Bc.sc[c] * (g4 - rmean[c] - yhat * rmean[H + c]);
          const float g3 = ya > 0.f ? dy : 0.f;
          const float z2hat = (zz[k] - A.mean[c]) * A.invstd[c];
          o[k] = A.sc[c] * (g3 - rmean[2 * H + c] - z2hat * rmean[3 * H + c]);
        }
        reinterpret_cast<float4*>(dz2_out)[i] = make_float4(o[0], o[1], o[2], o[3]);
        const __nv_bfloat162 p0 = __floats2bfloat162_rn(o[0], o[1]), p1 = __floats2bfloat162_rn(o[2], o[3]);
        uint2 w;
        w.x = *reinterpret_cast<const uint32_t*>(&p0);
        w.y = *reinterpret_cast<const uint32_t*>(&p1);
        reinterpret_cast<uint2*>(dz16)[i] = w;
      }
    }
  }
}

// g1 = [bn1(z1) > 0] dx1 in place; column sums of g1 and g1 * z1hat (BatchNorm-1 backward reductions)
template <int H>
__global__ void __launch_bounds__(256)
gin_bwd_g1_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                  float* __restrict__ dx1_g1, const double* __restrict__ sums_1, const float* __restrict__ g1w,
                  const float* __restrict__ be1, float bn_eps, double* __restrict__ red1_out) {
  __shared__ float coef[4 * H];
  __shared__ float red[2 * 1024];
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  bn_prepare(sums_1, N, H, g1w, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, nullptr, false, false, 0.f);
  __syncthreads();
  const BnC C1 = bnc(coef, H);
  constexpr int TPR = H / 4, RP = 256 / TPR;
  const int c4 = (tid % TPR) * 4, rsub = tid / TPR;
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  const int stride = gridDim.x * RP;
  for (int r = blockIdx.x * RP + rsub; r < N; r += 2 * stride) {
    float4 zv[2], dv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int rr = r + u * stride;
      const bool ok = rr < N;
      zv[u] = ok ? *reinterpret_cast<const float4*>(z1 + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      dv[u] = ok ? *reinterpret_cast<const float4*>(dx1_g1 + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int rr = r + u * stride;
      if (rr < N) {
        const float zz[4] = {zv[u].x, zv[u].y, zv[u].z, zv[u].w}, dd[4] = {dv[u].x, dv[u].y, dv[u].z, dv[u].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = c4 + k;
          const float pre = fmaf(zz[k], C1.sc[c], C1.sh[c]);
          o[k] = pre > 0.f ? dd[k] : 0.f;
          s[k] += o[k];
          q[k] = fmaf(o[k], (zz[k] - C1.mean[c]) * C1.invstd[c], q[k]);
        }
        *reinterpret_cast<float4*>(dx1_g1 + (size_t)rr * H + c4) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    red[(0 * RP + rsub) * H + c4 + k] = s[k];
    red[(RP + rsub) * H + c4 + k] = q[k];
  }
  __syncthreads();
  for (int idx = tid; idx < 2 * H; idx += 256) {
    const int which = idx / H, cc = idx - which * H;
    float t = 0.f;
    for (int j = 0; j < RP; ++j) t += red[(which * RP + j) * H + cc];
    atomicAdd(&red1_out[which * H + cc], (double)t);
  }
}

// dz1 = BN_1 backward of g1 (in place, fp32) + bf16 GEMM operand
template <int H>
__global__ void __launch_bounds__(256)
gin_bwd_dz1_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                   float* __restrict__ g1_dz1, const double* __restrict__ sums_1, const float* __restrict__ g1w,
                   const float* __restrict__ be1, float bn_eps, const double* __restrict__ red1,
                   __nv_bfloat16* __restrict__ dz16) {
  __shared__ float coef[4 * H];
  __shared__ float rmean[2 * H];
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  bn_prepare(sums_1, N, H, g1w, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, nullptr, false, false, 0.f);
  const double invN = N > 0 ? 1.0 / (double)N : 0.0;
  for (int c = tid; c < H; c += 256) {
    rmean[c] = (float)(red1[c] * invN);
    rmean[H + c] = (float)(red1[H + c] * invN);
  }
  __syncthreads();
  const BnC C1 = bnc(coef, H);
  const size_t total4 = (size_t)(N > 0 ? N : 0) * (H / 4);
  const size_t gstride = (size_t)gridDim.x * blockDim.x;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x + tid; i0 < total4; i0 += 2 * gstride) {
    float4 zv[2], gv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t i = i0 + u * gstride;
      const bool ok = i < total4;
      zv[u] = ok ? reinterpret_cast<const float4*>(z1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      gv[u] = ok ? reinterpret_cast<const float4*>(g1_dz1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t i = i0 + u * gstride;
      if (i < total4) {
        const int c0 = (int)(i % (H / 4)) * 4;
        const float zz[4] = {zv[u].x, zv[u].y, zv[u].z, zv[u].w}, gg[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = c0 + k;
          const float zhat = (zz[k] - C1.mean[c]) * C1.invstd[c];
          o[k] = C1.sc[c] * (gg[k] - rmean[c] - zhat * rmean[H + c]);
        }
        reinterpret_cast<float4*>(g1_dz1)[i] = make_float4(o[0], o[1], o[2], o[3]);
        const __nv_bfloat162 p0 = __floats2bfloat162_rn(o[0], o[1]), p1 = __floats2bfloat162_rn(o[2], o[3]);
        uint2 w;
        w.x = *reinterpret_cast<const uint32_t*>(&p0);
        w.y = *reinterpret_cast<const uint32_t*>(&p1);
        reinterpret_cast<uint2*>(dz16)[i] = w;
      }
    }
  }
}

template <int H>
static int run_backward_tc(const BwdArgs& a) {
  const GinDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* n_dev = node_off_v + B;
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const int32_t* graph_id = a.batch->graph_id + (size_t)a.view * cap;
  const double* stats = (const double*)(a.acts + a.al.stats);
  float* dh = (float*)(a.ws + a.bl.dh);
  float* da = (float*)(a.ws + a.bl.da);
  double* red = (double*)(a.ws + a.bl.red);
  float* dS = (float*)(a.ws + a.bl.dS);
  float* dpool = (float*)(a.ws + a.bl.dpool);
  __nv_bfloat16* dz16 = (__nv_bfloat16*)(a.ws + a.bl.dz16);
  __nv_bfloat16* tA = (__nv_bfloat16*)(a.ws + a.bl.tA);
  __nv_bfloat16* tB = (__nv_bfloat16*)(a.ws + a.bl.tB);
  float* coef1 = (float*)(a.ws + a.bl.coef1);
  float* splitk = (float*)(a.ws + a.bl.splitk);
  const float* P = a.params;
  float* G = a.grads;
  const int DW = a.bl.DW, capP = a.bl.cap_pad;
  const int tiles = (cap + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  const int grid = tiles < 4 * GCCB_NUM_SMS ? tiles : 4 * GCCB_NUM_SMS;
  const uint32_t keep = (uint32_t)fmin((1.0 - (double)d.drop_p) * 4294967296.0, 4294967295.0);
  StreamKit* kit = stream_kit((cudaStream_t)a.stream, 1);
  cudaStream_t main_s = (cudaStream_t)a.stream;
  cudaStream_t side = kit->side[0];
  cudaEvent_t* ev_main = kit->ev;
  cudaEvent_t* ev_side = kit->ev + 8;
  cudaEvent_t ev_head = kit->ev[16], ev_join = kit->ev[17];
  cudaMemsetAsync(red, 0, (size_t)(d.L - 1) * 3 * 2 * H * sizeof(double), main_s);
  auto kpb = gin_pool_predict_bwd_kernel<H>;
  GCCB_LAUNCH(kpb, (B + GCCB_GPB - 1) / GCCB_GPB, 256, 0, a.stream, d, node_off_v, B, P, a.lay, (const float*)(a.acts + a.al.score),
              a.dfeat, a.drop_key, a.drop_step, a.drop_base, keep, DW, dS, dpool, (double*)nullptr, 0);
  cudaEventRecord(ev_head, main_s);
  cudaStreamWaitEvent(side, ev_head, 0);
  {
    int maxout = H * (d.din > H ? d.din : H) + H;
    dim3 gr((maxout + 255) / 256, d.L);
    GCCB_LAUNCH(gin_pred_wgrad_kernel, gr, 256, 0, side, d, B, a.lay, (const float*)dS,
                (const float*)(a.acts + a.al.pooled), a.al.PW, G);
  }
  for (int l = d.L - 2; l >= 0; --l) {
    float* g1 = (float*)(a.ws + a.bl.g1[l & 1]);
    float* dz2 = (float*)(a.ws + a.bl.dz2[l & 1]);
    const int j = l + 1;
    const float* z1 = (const float*)(a.acts + a.al.z1[l]);
    const float* z2 = (const float*)(a.acts + a.al.z2[l]);
    const float* a_l = (const float*)(a.acts + a.al.a[l]);
    const double* s1 = stats + (size_t)(l * 3 + 0) * 2 * H;
    const double* sa = stats + (size_t)(l * 3 + 1) * 2 * H;
    const double* sb = stats + (size_t)(l * 3 + 2) * 2 * H;
    double* r1 = red + (size_t)(l * 3 + 0) * 2 * H;
    double* rA = red + (size_t)(l * 3 + 1) * 2 * H;
    double* rB = red + (size_t)(l * 3 + 2) * 2 * H;
    const int KW = gin_kw(d, l), inf = gin_in_features(d, l);
    const __nv_bfloat16* w1b = (const __nv_bfloat16*)(a.acts + a.al.w16[l]);
    const __nv_bfloat16* w1t = w1b + (size_t)H * KW + (size_t)H * H;
    const __nv_bfloat16* w2t = w1t + (size_t)KW * H;
    float* c1 = coef1 + (size_t)l * 2 * H;
    auto kdh = gin_bwd_dh_kernel<H, true>;                // dh and BN_b's backward reduction (rB)
    GCCB_LAUNCH(kdh, (tiles < 1184 ? tiles : 1184), 256, 0, a.stream, node_off_v, B, indptr, indices, graph_id,
                (const float*)(dpool + (size_t)j * B * DW), DW, (const float*)da, j < d.L - 1 ? 1 : 0, dh, z2, sa,
                P + a.lay.bna_w[l], P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], d.bn_eps, rB);
    auto kred = gin_bwd_reduce_kernel<H>;
    GCCB_LAUNCH(kred, grid, 256, 0, a.stream, node_off_v, B, z2, (const float*)dh, sa, P + a.lay.bna_w[l],
                P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], d.bn_eps, (const double*)rB, rA);
    if (l + 2 <= d.L - 2) cudaStreamWaitEvent(main_s, ev_side[l + 2], 0);   // g1 / dz2 [l&1] free again
    // the side stream of the layer above still reads dz16's transposed copies, not dz16 itself: no wait needed
    auto kz2 = gin_bwd_dz2_kernel<H>;
    GCCB_LAUNCH(kz2, grid, 256, 0, a.stream, node_off_v, B, z2, (const float*)dh, s1, P + a.lay.bn1_w[l],
                P + a.lay.bn1_b[l], sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l], sb, P + a.lay.bnb_w[l],
                P + a.lay.bnb_b[l], d.bn_eps, (const double*)rB, (const double*)rA, dz2, dz16, c1);
    int rc = tc::gemm_bf16(dz16, w2t, cap, H, H, n_dev, nullptr, 1.0f, g1, nullptr, H, nullptr, 1, nullptr, main_s);
    if (rc) return rc;
    auto kg1 = gin_bwd_g1_kernel<H>;
    GCCB_LAUNCH(kg1, grid, 256, 0, a.stream, node_off_v, B, z1, g1, s1, P + a.lay.bn1_w[l], P + a.lay.bn1_b[l],
                d.bn_eps, r1);
    auto kz1 = gin_bwd_dz1_kernel<H>;
    GCCB_LAUNCH(kz1, grid, 256, 0, a.stream, node_off_v, B, z1, g1, s1, P + a.lay.bn1_w[l], P + a.lay.bn1_b[l],
                d.bn_eps, (const double*)r1, dz16);
    rc = tc::gemm_bf16(dz16, w1t, cap, KW, H, n_dev, nullptr, 1.0f, da, nullptr, KW, nullptr, 1, nullptr, main_s);
    if (rc) return rc;
    cudaEventRecord(ev_main[l], main_s);
    cudaStreamWaitEvent(side, ev_main[l], 0);
    // weight gradients on the side stream: transposed bf16 operands, split-K over the rows, fixed-order reduce
    rc = tc::cast_bf16(dz2, cap, H, H, tA, capP, H, 1, n_dev, side);
    if (!rc) rc = tc::cast_bf16(z1, cap, H, H, tB, capP, H, 1, n_dev, side, c1, c1 + H, 1);      // x1^T
    if (!rc) rc = tc::gemm_bf16(tA, tB, H, H, capP, nullptr, nullptr, 1.0f, G + a.lay.w2[l], nullptr, H, nullptr,
                                a.bl.splits, splitk, side, 1.0f, H);
    if (!rc) rc = tc::cast_bf16(g1, cap, H, H, tA, capP, H, 1, n_dev, side);                       // dz1^T
    if (!rc) rc = tc::cast_bf16(a_l, cap, KW, KW, tB, capP, KW, 1, n_dev, side);                   // a^T
    if (!rc) rc = tc::gemm_bf16(tA, tB, H, KW, capP, nullptr, nullptr, 1.0f, G + a.lay.w1[l], nullptr, inf, nullptr,
                                a.bl.splits, splitk, side, 1.0f, inf);
    if (rc) return rc;
    GCCB_LAUNCH(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)rB,
                G + a.lay.bnb_w[l], G + a.lay.bnb_b[l]);
    GCCB_LAUNCH(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)rA,
                G + a.lay.bna_w[l], G + a.lay.bna_b[l]);
    GCCB_LAUNCH(gin_bn_grads_kernel, (H + 127) / 128, 128, 0, side, H, (const double*)r1,
                G + a.lay.bn1_w[l], G + a.lay.bn1_b[l]);
    cudaEventRecord(ev_side[l], side);
  }
  auto kdh0 = gin_bwd_dh_kernel<GCCB_DINP, false>;
  GCCB_LAUNCH(kdh0, (tiles < 1184 ? tiles : 1184), 256, 0, a.stream, node_off_v, B, indptr, indices, graph_id, (const float*)dpool, DW,
              (const float*)da, 1, dh, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f, nullptr);
  {
    size_t sm = (size_t)(d.maxdeg + 1) * d.D * sizeof(float);
    auto k = gin_bwd_emb_kernel;
    gccb::ensure_dyn_smem(k, sm);
    GCCB_LAUNCH(k, 64, 256, sm, a.stream, d, node_off_v, B, sub_deg, (const float*)dh, G + a.lay.emb);
  }
  cudaEventRecord(ev_join, side);
  cudaStreamWaitEvent(main_s, ev_join, 0);
  return check_launch("gccb_gin_backward (tensor cores)");
}
#endif  // !GCCB_EMU

}  // namespace gccb

using namespace gccb;

extern "C" size_t gccb_gin_backward_workspace(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap) {
  GinDims d;
  if (dims_from_cfg(cfg, &d)) return 0;
  return make_bwd_layout(d, batch, node_cap).total;
}

extern "C" int gccb_gin_stash_layout(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap,
                                     gccb_gin_stash_t* out) {
  GinDims d;
  int rc = dims_from_cfg(cfg, &d);
  if (rc) return rc;
  if (!out || batch < 1 || node_cap < 1) {
    set_last_error("gccb_gin_stash_layout: bad argument");
    return GCCB_ERR_BADARG;
  }
  const ActsLayout al = make_acts_layout(d, batch, node_cap);
  const BwdLayout bl = make_bwd_layout(d, batch, node_cap);
  auto tc = [&](size_t off) { return d.tc ? (int64_t)off : (int64_t)-1; };
  out->x0 = (int64_t)al.x0;
  for (int l = 0; l < 8; ++l) {
    const bool live = l < d.L - 1;
    out->a[l] = live ? (int64_t)al.a[l] : -1;
    out->z1[l] = live ? (int64_t)al.z1[l] : -1;
    out->z2[l] = live ? (int64_t)al.z2[l] : -1;
    out->h[l] = live ? (int64_t)al.h[l] : -1;
    out->w16[l] = live ? tc(al.w16[l]) : -1;
  }
  out->stats = (int64_t)al.stats;
  out->pooled = (int64_t)al.pooled;
  out->a16 = tc(al.a16);
  out->x16 = tc(al.x16);
  out->dh = (int64_t)bl.dh;
  for (int i = 0; i < 2; ++i) {
    out->g1[i] = (int64_t)bl.g1[i];
    out->dz2[i] = (int64_t)bl.dz2[i];
  }
  out->da = (int64_t)bl.da;
  out->dpool = (int64_t)bl.dpool;
  out->coef1 = tc(bl.coef1);
  out->dz16 = tc(bl.dz16);
  out->tA = tc(bl.tA);
  out->tB = tc(bl.tB);
  out->cap_pad = d.tc ? bl.cap_pad : -1;
  out->splits = d.tc ? bl.splits : -1;
  out->DW = bl.DW;
  out->PW = al.PW;
  return GCCB_OK;
}

extern "C" int gccb_gin_backward(const gccb_gin_cfg_t* cfg, const gccb_batch_t* batch, int32_t view,
                                 const float* params, const void* acts, const float* dfeat, float* grads,
                                 uint64_t dropout_key, uint64_t dropout_step,
                                 int32_t dropout_layer_base, void* workspace, size_t workspace_bytes,
                                 gccb_stream_t stream) {
  BwdArgs a;
  int rc = dims_from_cfg(cfg, &a.d);
  if (rc) return rc;
  if (!batch || !params || !acts || !dfeat || !grads || !workspace || view < 0 || view > 1) {
    set_last_error("gccb_gin_backward: bad argument");
    return GCCB_ERR_BADARG;
  }
  a.al = make_acts_layout(a.d, batch->batch, batch->node_cap);
  a.bl = make_bwd_layout(a.d, batch->batch, batch->node_cap);
  if (workspace_bytes < a.bl.total) {
    set_last_error("gccb_gin_backward: workspace too small");
    return GCCB_ERR_CAPACITY;
  }
  make_param_layout(a.d, &a.lay);
  a.batch = batch; a.view = view; a.params = params; a.acts = (const char*)acts; a.dfeat = dfeat;
  a.grads = grads; a.ws = (char*)workspace; a.stream = stream;
  // the forward's dropout mask is re-derived from the same Philox counters
  a.drop_key = dropout_key; a.drop_step = dropout_step; a.drop_base = dropout_layer_base;
#ifndef GCCB_EMU
  if (a.d.tc) return a.d.H == 128 ? run_backward_tc<128>(a) : run_backward_tc<256>(a);
#endif
  switch (a.d.H) {
    case 32: return run_backward<32>(a);
    case 64: return run_backward<64>(a);
    case 128: return run_backward<128>(a);
    default: return run_backward<256>(a);
  }
}
