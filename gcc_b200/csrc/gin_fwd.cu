// gin_fwd.cu -- GIN encoder forward for one view of a batch of ego-nets.
//
// Replaces GraphEncoder.forward (gcc/models/graph_encoder.py:132-200, gin branch) and
// UnsupervisedGIN.forward (gcc/models/gin.py:213-232) including what DGL does inside:
//   GINConv('sum', eps buffer = 0): rst = (1+eps)*h + sum_{u in N(v)} h_u ; apply_func(rst)
//   SumPooling: per-graph segment sum.
// Per GIN layer (gin.py:54-58, :107-116, :218-220):
//   a  = h + sum_nbr h          (gather / segmented reduce, fused into GEMM1's A tile)
//   z1 = a W1^T + b1            -> train-mode BatchNorm statistics in the epilogue
//   x1 = relu(bn1(z1))          (applied on load of GEMM2's A tile)
//   z2 = x1 W2^T + b2           -> statistics
//   y  = relu(bn_a(z2))         -> statistics (needs the full-batch mean of y)
//   h' = relu(bn_b(y))
// Every "-> statistics" is a column reduction over all N rows of the view, i.e. a
// grid-wide dependency; kernel boundaries provide it.  Round 1 uses fp32 SIMT tiles
// (bit-level agreement with an fp32 reference matters more than tensor-pipe speed
// at hidden=64, where the layer is bandwidth/launch bound -- see DESIGN.md).
#include "gin_common.cuh"
#include "tc_gemm.cuh"
#ifndef GCCB_EMU
#include <cuda_bf16.h>
#endif

namespace gccb {

// X0 = [pos | degree_embedding(clamp(deg)) | seed one-hot | 0]   graph_encoder.py:152-165
__global__ void __launch_bounds__(256)
gin_build_x0_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B,
                    const float* __restrict__ pos, const int32_t* __restrict__ sub_deg,
                    const int32_t* __restrict__ graph_id, const float* __restrict__ emb,
                    float* __restrict__ x0) {
  const int N = node_off_v[B];
  const int total = N * GCCB_DINP;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int r = idx / GCCB_DINP, c = idx - r * GCCB_DINP;
    float v = 0.f;
    if (c < d.P) {
      v = pos[(size_t)r * d.P + c];
    } else if (c < d.P + d.D) {
      int dg = sub_deg[r];
      dg = dg < 0 ? 0 : (dg > d.maxdeg ? d.maxdeg : dg);
      v = emb[(size_t)dg * d.D + (c - d.P)];
    } else if (c == d.P + d.D) {
      v = (r == node_off_v[graph_id[r]]) ? 1.0f : 0.f;     // seed = first row of its graph
    }
    x0[idx] = v;
  }
}

// K1: a = h + sum_nbr h ; z1 = a W1^T + b1 ; column statistics of z1.
template <int KIN, int H>
__global__ void __launch_bounds__(256)
gin_agg_gemm1_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
                     const int32_t* __restrict__ indices, const float* __restrict__ h,
                     const float* __restrict__ W1, int in_features, const float* __restrict__ b1,
                     float eps_gin, float* __restrict__ a_out, float* __restrict__ z1,
                     double* __restrict__ sums) {
  GCCB_DYN_SMEM(float, smem);
  constexpr int LDA = KIN + 1;
  float* As = smem;                          // [64][KIN+1]
  float* Ws = As + GCCB_TILE_ROWS * LDA;     // [KC][H+4]
  float* red = Ws + GCCB_KC * (H + 4);       // [2][16][H]; also the hub-row scratch [8][KIN]
  __shared__ int hub_rows[GCCB_TILE_ROWS];
  __shared__ int n_hub;
  static_assert(8 * KIN <= 2 * 16 * H, "hub scratch must fit in the statistics scratch");
  const int N = node_off_v[B];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  using TC = TileCols<H>;
  for (int tile = blockIdx.x; tile * GCCB_TILE_ROWS < N; tile += gridDim.x) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();                                   // As free (previous tile consumed)
    // gather / segmented reduce: one warp per row, lanes across the feature dimension; hub rows
    // (a seed's row in a large ego-net has n-1 neighbours) are deferred and split across the CTA
    if (tid == 0) n_hub = 0;
    __syncthreads();
    for (int rr = warp; rr < GCCB_TILE_ROWS; rr += 8) {
      const int r = row0 + rr;
      constexpr int PER = (KIN + 31) / 32;
      float acc[PER];
#pragma unroll
      for (int j = 0; j < PER; ++j) acc[j] = 0.f;
      if (r < N) {
        const int beg = indptr[r], end = indptr[r + 1];
        if (end - beg > GCCB_HUB_DEG) {
          if (lane == 0) hub_rows[atomicAdd(&n_hub, 1)] = rr;
          continue;
        }
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          int c = lane + 32 * j;
          if (c < KIN) acc[j] = (1.0f + eps_gin) * h[(size_t)r * KIN + c];
        }
        gather_range<KIN>(h, indices, beg, end, lane, acc);
      }
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        int c = lane + 32 * j;
        if (c < KIN) {
          As[rr * LDA + c] = acc[j];
          if (r < N) a_out[(size_t)r * KIN + c] = acc[j];
        }
      }
    }
    __syncthreads();
    for (int hi = 0; hi < n_hub; ++hi) {
      const int rr = hub_rows[hi], r = row0 + rr;
      const float s = gather_hub<KIN>(h, indices, indptr[r], indptr[r + 1], red);
      if (tid < KIN) {
        const float v = (1.0f + eps_gin) * h[(size_t)r * KIN + tid] + s;
        As[rr * LDA + tid] = v;
        a_out[(size_t)r * KIN + tid] = v;
      }
    }
    __syncthreads();
    float acc[4][TC::CPT];
    tile_gemm<H>(As, LDA, KIN, Ws,
                 [&](int k, int o) { return k < in_features ? W1[(size_t)o * in_features + k] : 0.f; }, acc);
    float v[4][TC::CPT];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + ty * 4 + i;
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) {
        const int col = TC::col(tx, c);
        float z = acc[i][c] + b1[col];
        v[i][c] = r < N ? z : 0.f;
        if (r < N) z1[(size_t)r * H + col] = z;
      }
    }
    tile_colstats<H>(v, red, sums);
  }
}

// K2: x1 = relu(bn1(z1)) ; z2 = x1 W2^T + b2 ; column statistics of z2.
template <int H>
__global__ void __launch_bounds__(256)
gin_bn_gemm2_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                    const double* __restrict__ sums1, const float* __restrict__ g1,
                    const float* __restrict__ be1, float bn_eps, float* __restrict__ running1,
                    int use_running, int update_running, float momentum,
                    const float* __restrict__ W2, const float* __restrict__ b2,
                    float* __restrict__ z2, double* __restrict__ sums2) {
  GCCB_DYN_SMEM(float, smem);
  constexpr int LDA = H + 1;
  float* As = smem;
  float* Ws = As + GCCB_TILE_ROWS * LDA;
  float* red = Ws + GCCB_KC * (H + 4);
  float* coef = red + 2 * 16 * H;            // mean | invstd | sc | sh
  const int N = node_off_v[B];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  using TC = TileCols<H>;
  bn_prepare(sums1, N, H, g1, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, running1,
             use_running != 0, update_running != 0, momentum);
  __syncthreads();
  const float* sc = coef + 2 * H;
  const float* sh = coef + 3 * H;
  for (int tile = blockIdx.x; tile * GCCB_TILE_ROWS < N; tile += gridDim.x) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();
#pragma unroll 8
    for (int idx = tid; idx < GCCB_TILE_ROWS * H; idx += 256) {   // 8 independent L2 loads in flight
      int rr = idx / H, c = idx - rr * H;
      int r = row0 + rr;
      float x = 0.f;
      if (r < N) x = fmaxf(fmaf(z1[(size_t)r * H + c], sc[c], sh[c]), 0.f);
      As[rr * LDA + c] = x;
    }
    __syncthreads();
    float acc[4][TC::CPT];
    tile_gemm<H>(As, LDA, H, Ws, [&](int k, int o) { return W2[(size_t)o * H + k]; }, acc);
    float v[4][TC::CPT];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + ty * 4 + i;
#pragma unroll
      for (int c = 0; c < TC::CPT; ++c) {
        const int col = TC::col(tx, c);
        float z = acc[i][c] + b2[col];
        v[i][c] = r < N ? z : 0.f;
        if (r < N) z2[(size_t)r * H + col] = z;
      }
    }
    tile_colstats<H>(v, red, sums2);
  }
}

// K3: y = relu(bn_a(z2)); column statistics of y.   (elementwise + reduction)
// K4 (mode 1): h' = relu(bn_b(y)) written out.
// One kernel, two modes: mode 0 accumulates sums of y; mode 1 writes h'.
template <int H>
__global__ void __launch_bounds__(256)
gin_bn_tail_kernel(int mode, const int32_t* __restrict__ node_off_v, int B,
                   const float* __restrict__ z2, const double* __restrict__ sums_a,
                   const float* __restrict__ ga, const float* __restrict__ bea,
                   float* __restrict__ running_a, const double* __restrict__ sums_b_in,
                   const float* __restrict__ gb, const float* __restrict__ beb,
                   float* __restrict__ running_b, float bn_eps, int use_running, int update_running,
                   float momentum, double* __restrict__ sums_b_out, float* __restrict__ h_out) {
  __shared__ float coef_a[4 * H];
  __shared__ float coef_b[4 * H];
  __shared__ float red[2 * 1024];
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  // BN_a running stats are updated by mode 0 only, BN_b's by mode 1 only (once each)
  bn_prepare(sums_a, N, H, ga, bea, bn_eps, coef_a, coef_a + H, coef_a + 2 * H, coef_a + 3 * H,
             running_a, use_running != 0, update_running != 0 && mode == 0, momentum);
  if (mode == 1)
    bn_prepare(sums_b_in, N, H, gb, beb, bn_eps, coef_b, coef_b + H, coef_b + 2 * H, coef_b + 3 * H,
               running_b, use_running != 0, update_running != 0, momentum);
  __syncthreads();
  // thread -> 4 consecutive columns (one 16-byte access) of every RP-th row; four rows in flight per thread
  // (this pass is bandwidth bound: N x H floats in, N x H out)
  constexpr int TPR = H / 4, RP = 256 / TPR;
  const int c4 = (tid % TPR) * 4, rsub = tid / TPR;
  float sca[4], sha[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { sca[k] = coef_a[2 * H + c4 + k]; sha[k] = coef_a[3 * H + c4 + k]; }
  const int stride = gridDim.x * RP;
  if (mode == 0) {
    float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = blockIdx.x * RP + rsub; r < N; r += 4 * stride) {
      float4 z[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int rr = r + u * stride;
        z[u] = rr < N ? *reinterpret_cast<const float4*>(z2 + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + u * stride < N) {
          const float zz[4] = {z[u].x, z[u].y, z[u].z, z[u].w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float y = fmaxf(fmaf(zz[k], sca[k], sha[k]), 0.f);
            s[k] += y;
            q[k] = fmaf(y, y, q[k]);
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
      atomicAdd(&sums_b_out[which * H + cc], (double)t);
    }
  } else {
    float scb[4], shb[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { scb[k] = coef_b[2 * H + c4 + k]; shb[k] = coef_b[3 * H + c4 + k]; }
    for (int r = blockIdx.x * RP + rsub; r < N; r += 4 * stride) {
      float4 z[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int rr = r + u * stride;
        z[u] = rr < N ? *reinterpret_cast<const float4*>(z2 + (size_t)rr * H + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int rr = r + u * stride;
        if (rr < N) {
          const float zz[4] = {z[u].x, z[u].y, z[u].z, z[u].w};
          float o[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float y = fmaxf(fmaf(zz[k], sca[k], sha[k]), 0.f);
            o[k] = fmaxf(fmaf(y, scb[k], shb[k]), 0.f);
          }
          *reinterpret_cast<float4*>(h_out + (size_t)rr * H + c4) = make_float4(o[0], o[1], o[2], o[3]);
        }
      }
    }
  }
}

// Sum pooling of every layer's node features (SumPooling, gin.py:213-232), parallel over 64-row
// tiles so that a 3,000-node ego-net does not serialise on one CTA: each thread owns a column and a
// run of consecutive rows, accumulates while the graph id stays the same and flushes with a float64
// atomic (same policy as the BatchNorm statistics).  pool_acc is zeroed with the statistics.
template <int H>
__global__ void __launch_bounds__(256)
gin_pool_kernel(int L, const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ graph_id,
                const float* __restrict__ x0, const float* const* __restrict__ h_layers, int PW,
                double* __restrict__ pool_acc) {
  __shared__ int gid[GCCB_TILE_ROWS];
  const int N = node_off_v[B];
  const int tid = threadIdx.x;
  for (int tile = blockIdx.x; tile * GCCB_TILE_ROWS < N; tile += gridDim.x) {
    const int row0 = tile * GCCB_TILE_ROWS;
    __syncthreads();
    if (tid < GCCB_TILE_ROWS) gid[tid] = row0 + tid < N ? graph_id[row0 + tid] : -1;
    __syncthreads();
    for (int l = 0; l < L; ++l) {
      // thread = (row group, float4 column): 128-bit loads, GCCB_TILE_ROWS / RG rows each, all of them in flight
      // (a scalar column per thread with 64 dependent-issue loads ran this pass at 0.9 TB/s at hidden 256)
      const int W = l == 0 ? GCCB_DINP : H;
      const float* src = l == 0 ? x0 : h_layers[l - 1];
      if (W < 128) {
        // narrow rows: one column per thread, 256 / W row groups (fewer, longer runs = fewer atomics)
        const int RGs = 256 / W > 0 ? 256 / W : 1;
        const int c = tid % W, rgs = tid / W;
        if (rgs >= RGs) continue;
        const int pers = GCCB_TILE_ROWS / RGs;
        const int rbs = rgs * pers;
        int g_run = gid[rbs];
        float acc = 0.f;
#pragma unroll 8
        for (int k = 0; k < pers; ++k) {
          const int g = gid[rbs + k];
          if (g < 0) break;
          const float x = src[(size_t)(row0 + rbs + k) * W + c];
          if (g != g_run) {
            atomicAdd(&pool_acc[((size_t)l * B + g_run) * PW + c], (double)acc);
            acc = 0.f;
            g_run = g;
          }
          acc += x;
        }
        if (g_run >= 0) atomicAdd(&pool_acc[((size_t)l * B + g_run) * PW + c], (double)acc);
        continue;
      }
      const int VW = W >> 2;                                // float4 columns (W is a multiple of 4)
      const int RG = 256 / VW < GCCB_TILE_ROWS ? 256 / VW : GCCB_TILE_ROWS;
      const int v = tid % VW, rg = tid / VW;
      if (rg >= RG) continue;
      const int per = GCCB_TILE_ROWS / RG;
      const int rb = rg * per;
      int g_run = gid[rb];
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      auto flush = [&](int g) {
        double* dst = &pool_acc[((size_t)l * B + g) * PW + 4 * v];
        atomicAdd(dst, (double)acc.x);
        atomicAdd(dst + 1, (double)acc.y);
        atomicAdd(dst + 2, (double)acc.z);
        atomicAdd(dst + 3, (double)acc.w);
      };
#pragma unroll 8
      for (int k = 0; k < per; ++k) {
        const int g = gid[rb + k];
        if (g < 0) break;
        const float4 x = *reinterpret_cast<const float4*>(src + (size_t)(row0 + rb + k) * W + 4 * v);
        if (g != g_run) {
          flush(g_run);
          acc = make_float4(0.f, 0.f, 0.f, 0.f);
          g_run = g;
        }
        acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
      }
      if (g_run >= 0) flush(g_run);
    }
  }
}

// K5: SumPooling per graph for every layer's representation, the prediction heads with
// dropout, the layer sum and the final L2 normalisation (gin.py:222-232, graph_encoder.py:195-196).
// grid = B (one CTA per graph), block = 256.
template <int H>
__global__ void __launch_bounds__(256)
gin_pool_predict_kernel(GinDims d, const int32_t* __restrict__ node_off_v, int B,
                        const double* __restrict__ pool_acc,
                        const float* __restrict__ params, const int64_t* __restrict__ wp_off,
                        const int64_t* __restrict__ bp_off, int PW, uint64_t drop_key,
                        uint64_t drop_step, int drop_layer_base, uint32_t keep_thresh,
                        float* __restrict__ pooled, float* __restrict__ score_out,
                        float* __restrict__ feat_out, float* __restrict__ pooled_user) {
  // GCCB_GPB graphs per CTA: a head weight row is read once and used for all of them (one graph per CTA re-read
  // the L x H x H weights from L2 for every graph: 1.3 GB per launch at hidden 256 / batch 1024)
  constexpr int MAXW = H > GCCB_DINP ? H : GCCB_DINP;
  constexpr int G = GCCB_GPB;
  __shared__ float pl[G][MAXW];
  __shared__ float score[G][H];
  const int g0 = blockIdx.x * G, tid = threadIdx.x;
  const int ng = min(G, B - g0);
  if (node_off_v[B] < 0) {                               // view published empty: defined (zero) outputs, the
    for (int i = tid; i < ng * H; i += 256) {            // optimiser / enqueue skip the step (gccb200.h)
      score_out[(size_t)g0 * H + i] = 0.f;
      feat_out[(size_t)g0 * H + i] = 0.f;
    }
    return;
  }
  for (int i = tid; i < G * H; i += 256) (&score[0][0])[i] = 0.f;
  __syncthreads();
  for (int l = 0; l < d.L; ++l) {
    const int W = l == 0 ? GCCB_DINP : H;                 // stored width
    const int inf = l == 0 ? d.din : H;                   // in_features of the head
    const float* Wp = params + wp_off[l];
    const float* bp = params + bp_off[l];
    __syncthreads();
    for (int i = tid; i < G * W; i += 256) {
      const int gi = i / W, cc = i - gi * W;
      float s = 0.f;
      if (gi < ng) {
        const int g = g0 + gi;
        s = (float)pool_acc[((size_t)l * B + g) * PW + cc];
        pooled[((size_t)l * B + g) * PW + cc] = s;
        if (pooled_user && l > 0) pooled_user[((size_t)(l - 1) * B + g) * H + cc] = s;   // all_outputs[1:]
      }
      pl[gi][cc] = s;
    }
    __syncthreads();
    // head GEMV: four lanes share an output, lane q takes k = q, q+4, ... (the four weight reads of a step are
    // 16 contiguous bytes); every weight is used for the G graphs of the CTA
    for (int o0 = 0; o0 < H; o0 += 64) {
      const int o = o0 + (tid >> 2), kq = tid & 3;
      float sg[G];
#pragma unroll
      for (int gi = 0; gi < G; ++gi) sg[gi] = 0.f;
      const float* wrow = Wp + (size_t)(o < H ? o : 0) * inf;
      if (o < H) {
#pragma unroll 4
        for (int k = kq; k < inf; k += 4) {
          const float w = wrow[k];
#pragma unroll
          for (int gi = 0; gi < G; ++gi) sg[gi] = fmaf(pl[gi][k], w, sg[gi]);
        }
      }
#pragma unroll
      for (int gi = 0; gi < G; ++gi) {
        sg[gi] += __shfl_xor_sync(0xffffffffu, sg[gi], 1);
        sg[gi] += __shfl_xor_sync(0xffffffffu, sg[gi], 2);
      }
      if (kq != 0 || o >= H) continue;
      const float bias = bp[o];
#pragma unroll
      for (int gi = 0; gi < G; ++gi) {
        if (gi >= ng) break;
        float sv = sg[gi] + bias;
        if (drop_layer_base >= 0) {                        // Dropout(p) in train mode, Philox mask
          const uint32_t e = (uint32_t)((g0 + gi) * H + o);
          u32x4 w = philox_at(drop_key, drop_step, e >> 2, 0, (uint32_t)(drop_layer_base + l),
                              GCCB_TAG_DROPOUT);
          const uint32_t word = (e & 3u) == 0 ? w.x : (e & 3u) == 1 ? w.y : (e & 3u) == 2 ? w.z : w.w;
          sv = word < keep_thresh ? sv / (1.0f - d.drop_p) : 0.f;
        }
        score[gi][o] += sv;
      }
    }
    __syncthreads();
  }
  // F.normalize(x, p=2, dim=-1, eps): x / max(||x||, eps) -- one warp per graph
  for (int gi = tid >> 5; gi < ng; gi += 8) {
    const int lane = tid & 31;
    float ss = 0.f;
    for (int o = lane; o < H; o += 32) ss = fmaf(score[gi][o], score[gi][o], ss);
    ss = warp_sum(ss);
    const float nrm = fmaxf(sqrtf(ss), d.norm_eps);
    for (int o = lane; o < H; o += 32) {
      score_out[(size_t)(g0 + gi) * H + o] = score[gi][o];
      feat_out[(size_t)(g0 + gi) * H + o] = d.norm ? score[gi][o] / nrm : score[gi][o];
    }
  }
}

// ------------------------------------------------------------------------------------------
template <int KIN, int H>
static size_t smem_gemm() {
  return ((size_t)GCCB_TILE_ROWS * (KIN + 1) + (size_t)GCCB_KC * (H + 4) + 2 * 16 * H + 4 * H) * sizeof(float);
}

struct FwdArgs {
  GinDims d;
  const gccb_batch_t* batch;
  int view;
  const float* pos;
  const float* params;
  gccb_gin_layout_t lay;
  float* running;
  int64_t* nbt;
  int bn_train;
  uint64_t drop_key, drop_step;
  int drop_base;
  char* acts;
  ActsLayout al;
  float* feat;
  float* pooled_user;
  const float** d_hptrs;    // device array [L-1] of layer outputs (lives in acts tail)
  int64_t* d_offs;          // device array [2][8] wp/bp offsets
  gccb_stream_t stream;
};

template <int H>
static int run_forward(const FwdArgs& a) {
  const GinDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const int32_t* graph_id = a.batch->graph_id + (size_t)a.view * cap;
  const float* pos_v = a.pos + (size_t)a.view * cap * d.P;
  float* x0 = (float*)(a.acts + a.al.x0);
  double* stats = (double*)(a.acts + a.al.stats);
  const int tiles = (cap + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  const int grid = tiles < 4 * GCCB_NUM_SMS ? tiles : 4 * GCCB_NUM_SMS;   // 4 waves at most
  const int use_running = a.bn_train ? 0 : 1, upd = a.bn_train ? 1 : 0;
  // BatchNorm statistics and the pooling accumulators are adjacent: one memset
  cudaMemsetAsync(stats, 0, a.al.pool_acc + (size_t)d.L * B * a.al.PW * sizeof(double) - a.al.stats,
                  (cudaStream_t)a.stream);
  GCCB_LAUNCH(gin_build_x0_kernel, grid, 256, 0, a.stream, d, node_off_v, B, pos_v, sub_deg, graph_id,
              a.params + a.lay.emb, x0);
  const float* hin = x0;
  for (int l = 0; l < d.L - 1; ++l) {
    float* a_l = (float*)(a.acts + a.al.a[l]);
    float* z1 = (float*)(a.acts + a.al.z1[l]);
    float* z2 = (float*)(a.acts + a.al.z2[l]);
    float* hout = (float*)(a.acts + a.al.h[l]);
    double* s1 = stats + (size_t)(l * 3 + 0) * 2 * H;
    double* sa = stats + (size_t)(l * 3 + 1) * 2 * H;
    double* sb = stats + (size_t)(l * 3 + 2) * 2 * H;
    float* run1 = a.running ? a.running + (size_t)(l * 3 + 0) * 2 * H : nullptr;
    float* runa = a.running ? a.running + (size_t)(l * 3 + 1) * 2 * H : nullptr;
    float* runb = a.running ? a.running + (size_t)(l * 3 + 2) * 2 * H : nullptr;
    const float* P = a.params;
    if (l == 0) {
      auto k = gin_agg_gemm1_kernel<GCCB_DINP, H>;
      size_t sm = smem_gemm<GCCB_DINP, H>();
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH(k, grid, 256, sm, a.stream, node_off_v, B, indptr, indices, hin, P + a.lay.w1[l], d.din,
                  P + a.lay.b1[l], 0.0f, a_l, z1, s1);
    } else {
      auto k = gin_agg_gemm1_kernel<H, H>;
      size_t sm = smem_gemm<H, H>();
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH(k, grid, 256, sm, a.stream, node_off_v, B, indptr, indices, hin, P + a.lay.w1[l], H,
                  P + a.lay.b1[l], 0.0f, a_l, z1, s1);
    }
    {
      auto k = gin_bn_gemm2_kernel<H>;
      size_t sm = smem_gemm<H, H>();
      gccb::ensure_dyn_smem(k, sm);
      GCCB_LAUNCH(k, grid, 256, sm, a.stream, node_off_v, B, z1, s1, P + a.lay.bn1_w[l], P + a.lay.bn1_b[l],
                  d.bn_eps, run1, use_running, upd, d.bn_mom, P + a.lay.w2[l], P + a.lay.b2[l], z2, sa);
    }
    auto kt = gin_bn_tail_kernel<H>;
    GCCB_LAUNCH(kt, grid, 256, 0, a.stream, 0, node_off_v, B, z2, sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l],
                runa, sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], runb, d.bn_eps, use_running, upd,
                d.bn_mom, sb, hout);
    GCCB_LAUNCH(kt, grid, 256, 0, a.stream, 1, node_off_v, B, z2, sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l],
                runa, sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], runb, d.bn_eps, use_running, upd,
                d.bn_mom, sb, hout);
    hin = hout;
  }
  const uint32_t keep = (uint32_t)fmin((1.0 - (double)d.drop_p) * 4294967296.0, 4294967295.0);
  double* pool_acc = (double*)(a.acts + a.al.pool_acc);
  auto kpl = gin_pool_kernel<H>;
  GCCB_LAUNCH(kpl, grid, 256, 0, a.stream, d.L, node_off_v, B, graph_id, (const float*)x0, a.d_hptrs, a.al.PW,
              pool_acc);
  auto kp = gin_pool_predict_kernel<H>;
  GCCB_LAUNCH(kp, (B + GCCB_GPB - 1) / GCCB_GPB, 256, 0, a.stream, d, node_off_v, B, (const double*)pool_acc, a.params, a.d_offs, a.d_offs + 8,
              a.al.PW, a.drop_key, a.drop_step, a.drop_base, keep, (float*)(a.acts + a.al.pooled),
              (float*)(a.acts + a.al.score), a.feat, a.pooled_user);
  return check_launch("gccb_gin_forward");
}


#ifndef GCCB_EMU
// ================================================================================================
// Tensor-core path (cfg.tensor_cores, hidden >= 128; BASELINE config 4): the two Linear layers of every
// GIN MLP (gin.py:113-116) run as wgmma GEMMs (csrc/tc_gemm.cu) with bf16 operands staged by TMA and
// fp32 accumulation in registers; bias add and the BatchNorm column statistics are the GEMM epilogue.  The
// gather / segmented reduce and the BatchNorm + ReLU between the GEMMs are bandwidth-bound passes that
// also emit the bf16 operand of the next GEMM.  Activations stay fp32 in the stash (the backward's
// elementwise chain is unchanged).

// bf16 copies of one layer's weights: W1 [H][KW] (zero padded k >= in_features), W2 [H][H], and their
// transposes W1^T [KW][H], W2^T [H][H] (the B operands of the input-gradient GEMMs).  grid = (blocks, L-1)
__global__ void __launch_bounds__(256)
gin_cast_weights_kernel(GinDims d, gccb_gin_layout_t lay, const float* __restrict__ params, char* acts,
                        ActsLayout al) {
  const int l = blockIdx.y, H = d.H, KW = gin_kw(d, l), inf = gin_in_features(d, l);
  const float* W1 = params + lay.w1[l];
  const float* W2 = params + lay.w2[l];
  __nv_bfloat16* w1b = (__nv_bfloat16*)(acts + al.w16[l]);
  __nv_bfloat16* w2b = w1b + (size_t)H * KW;
  __nv_bfloat16* w1t = w2b + (size_t)H * H;
  __nv_bfloat16* w2t = w1t + (size_t)KW * H;
  const int n1 = H * KW, n2 = H * H;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * n1 + 2 * n2; idx += gridDim.x * blockDim.x) {
    if (idx < n1) {
      const int o = idx / KW, k = idx - o * KW;
      w1b[idx] = __float2bfloat16_rn(k < inf ? W1[(size_t)o * inf + k] : 0.f);
    } else if (idx < n1 + n2) {
      w2b[idx - n1] = __float2bfloat16_rn(W2[idx - n1]);
    } else if (idx < 2 * n1 + n2) {
      const int j = idx - n1 - n2, k = j / H, o = j - k * H;
      w1t[j] = __float2bfloat16_rn(k < inf ? W1[(size_t)o * inf + k] : 0.f);
    } else {
      const int j = idx - 2 * n1 - n2, k = j / H, o = j - k * H;
      w2t[j] = __float2bfloat16_rn(W2[(size_t)o * H + k]);
    }
  }
}

// a = (1 + eps) h + sum_nbr h  -> fp32 stash + bf16 GEMM operand.  One warp per row, 8 rows per CTA pass;
// hub rows (more than GCCB_HUB_DEG neighbours) are split across the CTA's warps.
template <int W>
__global__ void __launch_bounds__(256)
gin_agg_cast_kernel(const int32_t* __restrict__ node_off_v, int B, const int32_t* __restrict__ indptr,
                    const int32_t* __restrict__ indices, const float* __restrict__ h, float eps_gin,
                    float* __restrict__ a_out, __nv_bfloat16* __restrict__ a16) {
  __shared__ float scratch[8 * W];
  __shared__ int hub_rows[GCCB_HUB_QUEUE];
  __shared__ int n_hub;
  const int N = node_off_v[B];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int V4 = W / 4, PERV = (V4 + 31) / 32;
  // One warp per row, rows dealt round-robin over all warps of the grid, NO barrier on the way: a tile-wise version
  // with two barriers per 64 rows spent 53 % of its cycles waiting at them (ncu) and ran at 0.9 TB/s.  Hub rows
  // (> GCCB_HUB_DEG neighbours, a handful per batch) are queued per CTA and gathered by its 8 warps together after
  // the loop, in a fixed order.  128-bit loads / stores: lane owns the float4 slots lane + 32 j of a row.
  if (tid == 0) n_hub = 0;
  __syncthreads();
  for (int r = blockIdx.x * 8 + warp; r < N; r += gridDim.x * 8) {
    const int beg = indptr[r], end = indptr[r + 1];
    if (end - beg > GCCB_HUB_DEG) {
      int slot = GCCB_HUB_QUEUE;
      if (lane == 0) slot = atomicAdd(&n_hub, 1);
      slot = __shfl_sync(0xffffffffu, slot, 0);
      if (slot < GCCB_HUB_QUEUE) {
        if (lane == 0) hub_rows[slot] = r;
        continue;
      }                                                  // queue full: this warp gathers the row alone
    }
    float4 acc[PERV];
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = lane + 32 * j;
      acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v < V4) {
        const float4 x = *reinterpret_cast<const float4*>(h + (size_t)r * W + 4 * v);
        const float s1 = 1.0f + eps_gin;
        acc[j] = make_float4(s1 * x.x, s1 * x.y, s1 * x.z, s1 * x.w);
      }
    }
    gather_range4<W>(h, indices, beg, end, lane, acc);
#pragma unroll
    for (int j = 0; j < PERV; ++j) {
      const int v = lane + 32 * j;
      if (v < V4) {
        if (a_out) *reinterpret_cast<float4*>(a_out + (size_t)r * W + 4 * v) = acc[j];
        const __nv_bfloat162 p0 = __floats2bfloat162_rn(acc[j].x, acc[j].y), p1 = __floats2bfloat162_rn(acc[j].z, acc[j].w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&p0);
        pk.y = *reinterpret_cast<const uint32_t*>(&p1);
        *reinterpret_cast<uint2*>(a16 + (size_t)r * W + 4 * v) = pk;
      }
    }
  }
  __syncthreads();
  const int nh = min(n_hub, GCCB_HUB_QUEUE);
  for (int hi = 0; hi < nh; ++hi) {
    const int rh = hub_rows[hi];
    const float sacc = gather_hub<W>(h, indices, indptr[rh], indptr[rh + 1], scratch);
    if (tid < W) {
      const float v = (1.0f + eps_gin) * h[(size_t)rh * W + tid] + sacc;
      if (a_out) a_out[(size_t)rh * W + tid] = v;
      a16[(size_t)rh * W + tid] = __float2bfloat16_rn(v);
    }
  }
}

// x1 = relu(bn1(z1)) as the bf16 operand of the second GEMM (BatchNorm coefficients from the column sums the
// first GEMM's epilogue accumulated; block 0 updates the running statistics).  4 columns per thread.
template <int H>
__global__ void __launch_bounds__(256)
gin_bn_relu_cast_kernel(const int32_t* __restrict__ node_off_v, int B, const float* __restrict__ z1,
                        const double* __restrict__ sums1, const float* __restrict__ g1, const float* __restrict__ be1,
                        float bn_eps, float* __restrict__ running1, int use_running, int update_running,
                        float momentum, __nv_bfloat16* __restrict__ x16) {
  __shared__ float coef[4 * H];
  const int N = node_off_v[B];
  bn_prepare(sums1, N, H, g1, be1, bn_eps, coef, coef + H, coef + 2 * H, coef + 3 * H, running1, use_running != 0,
             update_running != 0, momentum);
  __syncthreads();
  const float* sc = coef + 2 * H;
  const float* sh = coef + 3 * H;
  const size_t total4 = (size_t)(N > 0 ? N : 0) * (H / 4);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % (H / 4)) * 4;
    const float4 z = reinterpret_cast<const float4*>(z1)[i];
    const __nv_bfloat162 p0 = __floats2bfloat162_rn(fmaxf(fmaf(z.x, sc[c], sh[c]), 0.f), fmaxf(fmaf(z.y, sc[c + 1], sh[c + 1]), 0.f));
    const __nv_bfloat162 p1 = __floats2bfloat162_rn(fmaxf(fmaf(z.z, sc[c + 2], sh[c + 2]), 0.f), fmaxf(fmaf(z.w, sc[c + 3], sh[c + 3]), 0.f));
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t*>(&p0);
    u.y = *reinterpret_cast<const uint32_t*>(&p1);
    reinterpret_cast<uint2*>(x16)[i] = u;
  }
}

template <int H>
static int run_forward_tc(const FwdArgs& a) {
  const GinDims& d = a.d;
  const int B = a.batch->batch, cap = a.batch->node_cap;
  const int32_t* node_off_v = a.batch->node_off + (size_t)a.view * (B + 1);
  const int32_t* n_dev = node_off_v + B;
  const int32_t* indptr = a.batch->indptr + (size_t)a.view * (cap + 1);
  const int32_t* indices = a.batch->indices + (size_t)a.view * a.batch->edge_cap;
  const int32_t* sub_deg = a.batch->sub_deg + (size_t)a.view * cap;
  const int32_t* graph_id = a.batch->graph_id + (size_t)a.view * cap;
  const float* pos_v = a.pos + (size_t)a.view * cap * d.P;
  cudaStream_t st = (cudaStream_t)a.stream;
  float* x0 = (float*)(a.acts + a.al.x0);
  double* stats = (double*)(a.acts + a.al.stats);
  __nv_bfloat16* a16 = (__nv_bfloat16*)(a.acts + a.al.a16);
  __nv_bfloat16* x16 = (__nv_bfloat16*)(a.acts + a.al.x16);
  const int tiles = (cap + GCCB_TILE_ROWS - 1) / GCCB_TILE_ROWS;
  const int grid = tiles < 4 * GCCB_NUM_SMS ? tiles : 4 * GCCB_NUM_SMS;
  const int use_running = a.bn_train ? 0 : 1, upd = a.bn_train ? 1 : 0;
  cudaMemsetAsync(stats, 0, a.al.pool_acc + (size_t)d.L * B * a.al.PW * sizeof(double) - a.al.stats, st);
  GCCB_LAUNCH(gin_build_x0_kernel, grid, 256, 0, a.stream, d, node_off_v, B, pos_v, sub_deg, graph_id,
              a.params + a.lay.emb, x0);
  {
    dim3 gw(64, d.L - 1);
    GCCB_LAUNCH(gin_cast_weights_kernel, gw, 256, 0, a.stream, d, a.lay, a.params, a.acts, a.al);
  }
  const float* hin = x0;
  const float* P = a.params;
  const int agg_grid = tiles < 1184 ? tiles : 1184;
  for (int l = 0; l < d.L - 1; ++l) {
    float* a_l = (float*)(a.acts + a.al.a[l]);
    float* z1 = (float*)(a.acts + a.al.z1[l]);
    float* z2 = (float*)(a.acts + a.al.z2[l]);
    float* hout = (float*)(a.acts + a.al.h[l]);
    double* s1 = stats + (size_t)(l * 3 + 0) * 2 * H;
    double* sa = stats + (size_t)(l * 3 + 1) * 2 * H;
    double* sb = stats + (size_t)(l * 3 + 2) * 2 * H;
    float* run1 = a.running ? a.running + (size_t)(l * 3 + 0) * 2 * H : nullptr;
    float* runa = a.running ? a.running + (size_t)(l * 3 + 1) * 2 * H : nullptr;
    float* runb = a.running ? a.running + (size_t)(l * 3 + 2) * 2 * H : nullptr;
    const int KW = gin_kw(d, l);
    const __nv_bfloat16* w1b = (const __nv_bfloat16*)(a.acts + a.al.w16[l]);
    const __nv_bfloat16* w2b = w1b + (size_t)H * KW;
    if (l == 0) {
      auto k = gin_agg_cast_kernel<GCCB_DINP>;
      GCCB_LAUNCH(k, agg_grid, 256, 0, a.stream, node_off_v, B, indptr, indices, hin, 0.0f, a_l, a16);
    } else {
      auto k = gin_agg_cast_kernel<H>;
      GCCB_LAUNCH(k, agg_grid, 256, 0, a.stream, node_off_v, B, indptr, indices, hin, 0.0f, a_l, a16);
    }
    int rc = tc::gemm_bf16(a16, w1b, cap, H, KW, n_dev, P + a.lay.b1[l], 1.0f, z1, nullptr, H, s1, 1, nullptr, st);
    if (rc) return rc;
    auto kb = gin_bn_relu_cast_kernel<H>;
    GCCB_LAUNCH(kb, grid, 256, 0, a.stream, node_off_v, B, (const float*)z1, (const double*)s1, P + a.lay.bn1_w[l],
                P + a.lay.bn1_b[l], d.bn_eps, run1, use_running, upd, d.bn_mom, x16);
    rc = tc::gemm_bf16(x16, w2b, cap, H, H, n_dev, P + a.lay.b2[l], 1.0f, z2, nullptr, H, sa, 1, nullptr, st);
    if (rc) return rc;
    auto kt = gin_bn_tail_kernel<H>;
    GCCB_LAUNCH(kt, grid, 256, 0, a.stream, 0, node_off_v, B, z2, sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l],
                runa, sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], runb, d.bn_eps, use_running, upd,
                d.bn_mom, sb, hout);
    GCCB_LAUNCH(kt, grid, 256, 0, a.stream, 1, node_off_v, B, z2, sa, P + a.lay.bna_w[l], P + a.lay.bna_b[l],
                runa, sb, P + a.lay.bnb_w[l], P + a.lay.bnb_b[l], runb, d.bn_eps, use_running, upd,
                d.bn_mom, sb, hout);
    hin = hout;
  }
  const uint32_t keep = (uint32_t)fmin((1.0 - (double)d.drop_p) * 4294967296.0, 4294967295.0);
  double* pool_acc = (double*)(a.acts + a.al.pool_acc);
  auto kpl = gin_pool_kernel<H>;
  GCCB_LAUNCH(kpl, grid, 256, 0, a.stream, d.L, node_off_v, B, graph_id, (const float*)x0, a.d_hptrs, a.al.PW,
              pool_acc);
  auto kp = gin_pool_predict_kernel<H>;
  GCCB_LAUNCH(kp, (B + GCCB_GPB - 1) / GCCB_GPB, 256, 0, a.stream, d, node_off_v, B, (const double*)pool_acc, a.params, a.d_offs, a.d_offs + 8,
              a.al.PW, a.drop_key, a.drop_step, a.drop_base, keep, (float*)(a.acts + a.al.pooled),
              (float*)(a.acts + a.al.score), a.feat, a.pooled_user);
  return check_launch("gccb_gin_forward (tensor cores)");
}
#endif  // !GCCB_EMU

}  // namespace gccb

using namespace gccb;

extern "C" int gccb_gin_param_layout(const gccb_gin_cfg_t* cfg, gccb_gin_layout_t* out) {
  GinDims d;
  int rc = dims_from_cfg(cfg, &d);
  if (rc) return rc;
  if (!out) return GCCB_ERR_BADARG;
  make_param_layout(d, out);
  return GCCB_OK;
}

// the stash tail also holds two small device tables the pooling kernel reads
static size_t acts_tables_bytes() { return 256 + 8 * sizeof(void*) + 16 * sizeof(int64_t); }

extern "C" size_t gccb_gin_acts_bytes(const gccb_gin_cfg_t* cfg, int32_t batch, int32_t node_cap) {
  GinDims d;
  if (dims_from_cfg(cfg, &d)) return 0;
  return make_acts_layout(d, batch, node_cap).total + acts_tables_bytes();
}

namespace gccb {
// fills the device tables (layer-output pointers, head offsets) with a tiny kernel so that no
// host->device copy (and no pinned staging) is needed and the call stays graph-capturable
__global__ void gin_fill_tables_kernel(char* acts, ActsLayout al, gccb_gin_layout_t lay, int L,
                                       const float** hptrs, int64_t* offs, int64_t* nbt,
                                       const int32_t* n_valid) {
  int t = threadIdx.x;
  if (t < L - 1) hptrs[t] = (const float*)(acts + al.h[t]);
  if (t < 8) { offs[t] = lay.wp[t]; offs[8 + t] = lay.bp[t]; }
  if (nbt && *n_valid >= 0 && t < 3 * (L - 1)) nbt[t] += 1;      // BatchNorm.num_batches_tracked (train mode)
}
}  // namespace gccb

extern "C" int gccb_gin_forward(const gccb_gin_cfg_t* cfg, const gccb_batch_t* batch, int32_t view,
                                const float* pos, const float* params, float* bn_running,
                                int64_t* num_batches_tracked, int32_t bn_train, uint64_t dropout_key,
                                uint64_t dropout_step, int32_t dropout_layer_base, void* acts,
                                size_t acts_bytes, float* feat, float* pooled_out,
                                gccb_stream_t stream) {
  FwdArgs a;
  int rc = dims_from_cfg(cfg, &a.d);
  if (rc) return rc;
  if (!batch || !pos || !params || !acts || !feat || view < 0 || view > 1 || (!bn_train && !bn_running)) {
    set_last_error("gccb_gin_forward: bad argument");
    return GCCB_ERR_BADARG;
  }
  a.al = make_acts_layout(a.d, batch->batch, batch->node_cap);
  if (acts_bytes < a.al.total + acts_tables_bytes()) {
    set_last_error("gccb_gin_forward: activation stash too small (%zu < %zu)", acts_bytes,
                   a.al.total + acts_tables_bytes());
    return GCCB_ERR_CAPACITY;
  }
  make_param_layout(a.d, &a.lay);
  a.batch = batch; a.view = view; a.pos = pos; a.params = params; a.running = bn_running;
  a.nbt = num_batches_tracked; a.bn_train = bn_train; a.drop_key = dropout_key; a.drop_step = dropout_step;
  a.drop_base = dropout_layer_base; a.acts = (char*)acts; a.feat = feat; a.pooled_user = pooled_out;
  a.stream = stream;
  char* tail = (char*)acts + a.al.total;
  a.d_hptrs = (const float**)tail;
  a.d_offs = (int64_t*)(tail + 8 * sizeof(void*));
  GCCB_LAUNCH(gin_fill_tables_kernel, 1, 32, 0, stream, (char*)acts, a.al, a.lay, a.d.L, a.d_hptrs, a.d_offs,
              bn_train ? num_batches_tracked : (int64_t*)nullptr,
              (const int32_t*)(batch->node_off + (size_t)view * (batch->batch + 1) + batch->batch));
#ifndef GCCB_EMU
  if (a.d.tc) return a.d.H == 128 ? run_forward_tc<128>(a) : run_forward_tc<256>(a);
#endif
  switch (a.d.H) {
    case 32: return run_forward<32>(a);
    case 64: return run_forward<64>(a);
    case 128: return run_forward<128>(a);
    default: return run_forward<256>(a);
  }
}
