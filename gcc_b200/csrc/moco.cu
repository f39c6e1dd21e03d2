// moco.cu -- contrastive head: MoCo queue logits, InfoNCE loss (separate and fused), enqueue,
// and the E2E (in-batch negatives) head.
//
// Replaces (reference file:line):
//   MemoryMoCo.forward logits [q.k | q.queue^T]/T           gcc/contrastive/memory_moco.py:33-44
//   FIFO enqueue via index_copy_                            gcc/contrastive/memory_moco.py:55-61
//   NCESoftmaxLoss / NCESoftmaxLossNS (CrossEntropy)        gcc/contrastive/criterions.py:12-17,27-33
//   E2E logits feat_k @ feat_q^T / T                        train.py:397-401
// The reference materialises the B x (K+1) logits (16 MiB at K=16384), clones the 4 MiB queue
// every step (:36) and syncs the host (:30).  The fused kernel streams the queue once,
// keeps an online softmax per row (running max / sum / sum_j p_j key_j, the attention
// recurrence with V = K) and never writes logits; the unfused entry points exist so the
// reference's module API (MemoryMoCo.forward returning `out`) stays drop-in.
#include "common.cuh"
#include "tc_gemm.cuh"
#ifndef GCCB_EMU
#include <cuda_bf16.h>
#endif

namespace gccb {

#define GCCB_NCE_RB 8          // query rows per CTA

// out[i][0] = q_i.k_i/T ; out[i][1+j] = q_i.mem_j/T.   grid = (ceil(K/256), ceil(B/RB)), block 256
__global__ void __launch_bounds__(256)
moco_logits_kernel(const float* __restrict__ q, const float* __restrict__ k,
                   const float* __restrict__ mem, int B, int d, int K, float invT,
                   float* __restrict__ out) {
  GCCB_DYN_SMEM(float, qs);               // [RB][d]
  const int tid = threadIdx.x;
  const int i0 = blockIdx.y * GCCB_NCE_RB;
  for (int idx = tid; idx < GCCB_NCE_RB * d; idx += 256) {
    int i = i0 + idx / d;
    qs[idx] = i < B ? q[(size_t)i * d + idx % d] : 0.f;
  }
  __syncthreads();
  const int j = blockIdx.x * 256 + tid;
  float acc[GCCB_NCE_RB];
#pragma unroll
  for (int r = 0; r < GCCB_NCE_RB; ++r) acc[r] = 0.f;
  if (j < K) {
    const float* mj = mem + (size_t)j * d;
    for (int c = 0; c < d; ++c) {
      const float m = mj[c];
#pragma unroll
      for (int r = 0; r < GCCB_NCE_RB; ++r) acc[r] = fmaf(qs[r * d + c], m, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < GCCB_NCE_RB; ++r)
      if (i0 + r < B) out[(size_t)(i0 + r) * (K + 1) + 1 + j] = acc[r] * invT;
  }
  if (blockIdx.x == 0 && tid < GCCB_NCE_RB && i0 + tid < B) {      // positive logit
    const int i = i0 + tid;
    float s = 0.f;
    for (int c = 0; c < d; ++c) s = fmaf(qs[tid * d + c], k[(size_t)i * d + c], s);
    out[(size_t)i * (K + 1)] = s * invT;
  }
}

// dq_i = (1/T) (dout[i][0] k_i + sum_j dout[i][1+j] mem_j).   grid = B, block 256
__global__ void __launch_bounds__(256)
moco_logits_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ k,
                       const float* __restrict__ mem, int B, int d, int K, float invT,
                       float* __restrict__ dq) {
  GCCB_DYN_SMEM(float, part);             // [groups][d]
  const int i = blockIdx.x, tid = threadIdx.x;
  const int groups = 256 / d > 0 ? 256 / d : 1;
  const int c = tid % d, gidx = tid / d;
  const float* drow = dout + (size_t)i * (K + 1);
  float s = 0.f;
  if (gidx < groups)
    for (int j = gidx; j < K; j += groups) s = fmaf(drow[1 + j], mem[(size_t)j * d + c], s);
  if (gidx < groups) part[gidx * d + c] = s;
  __syncthreads();
  for (int cc = tid; cc < d; cc += 256) {
    float t = drow[0] * k[(size_t)i * d + cc];
    for (int gi = 0; gi < groups; ++gi) t += part[gi * d + cc];
    dq[(size_t)i * d + cc] = t * invT;
  }
}

// Cross entropy of out[B][C] against label 0 (mode 0) or i (mode 1); optional dout.
// grid = B, block 256.  loss accumulated with one atomic per row (caller zeroes).
__global__ void __launch_bounds__(256)
nce_loss_kernel(const float* __restrict__ out, int B, int C, int label_mode,
                float* __restrict__ loss, float* __restrict__ dout) {
  __shared__ float red_s[8];
  __shared__ float bc[2];
  const int i = blockIdx.x, tid = threadIdx.x;
  const float* row = out + (size_t)i * C;
  float mx = -3.0e38f;
  for (int j = tid; j < C; j += 256) mx = fmaxf(mx, row[j]);
  mx = warp_max(mx);
  if ((tid & 31) == 0) red_s[tid >> 5] = mx;
  __syncthreads();
  if (tid == 0) { float m = red_s[0]; for (int w = 1; w < 8; ++w) m = fmaxf(m, red_s[w]); bc[0] = m; }
  __syncthreads();
  mx = bc[0];
  float s = 0.f;
  for (int j = tid; j < C; j += 256) s += expf(row[j] - mx);
  s = warp_sum(s);
  __syncthreads();
  if ((tid & 31) == 0) red_s[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red_s[w]; bc[1] = t; }
  __syncthreads();
  const float sum = bc[1];
  const int label = label_mode == 0 ? 0 : i;
  if (tid == 0) atomicAdd(loss, (logf(sum) + mx - row[label]) / (float)B);
  if (dout) {
    float* drow = dout + (size_t)i * C;
    const float invB = 1.0f / (float)B;
    for (int j = tid; j < C; j += 256) {
      float p = expf(row[j] - mx) / sum;
      drow[j] = (p - (j == label ? 1.0f : 0.f)) * invB;
    }
  }
}

// ---- fused InfoNCE -------------------------------------------------------------------------
// partial record per (chunk, row): m, s, acc[d]  ->  stride d + 2 floats
// d in {32, 64, 128, 256}: 32 query rows x CK = 32*KPT keys per CTA, register tiles for both products.
// Warp w owns rows 4w..4w+3; lane owns keys lane + 32t (logits) and columns lane + 32u (accumulator).
// grid = (nchunks, ceil(B/32)), block 256; dyn smem: qs[32][d] | ms[CK][d+1] | ps[32][CK]
#define GCCB_NCE_RB2 32
template <int KPT, int DU>
__global__ void __launch_bounds__(256)
infonce_partial_tiled_kernel(const float* __restrict__ q, const float* __restrict__ mem, int B, int K,
                             float invT, float* __restrict__ part, float* __restrict__ stats) {
  constexpr int CK = 32 * KPT, d = 32 * DU, RB = GCCB_NCE_RB2;
  GCCB_DYN_SMEM(float, smem);
  float* qs = smem;
  float* ms = qs + RB * d;
  float* ps = ms + (size_t)CK * (d + 1);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_wait();
  if (blockIdx.x == 0 && blockIdx.y == 0 && tid < 2) stats[tid] = 0.f;   // infonce_merge_kernel accumulates them
  const int i0 = blockIdx.y * RB, j0 = blockIdx.x * CK;
  const int nk = min(CK, K - j0);
  for (int idx = tid; idx < RB * d; idx += 256) {
    const int i = i0 + idx / d;
    qs[idx] = i < B ? q[(size_t)i * d + idx % d] : 0.f;
  }
  for (int idx = tid; idx < CK * d; idx += 256) {
    const int j = idx / d, c = idx - j * d;
    ms[j * (d + 1) + c] = j < nk ? mem[(size_t)(j0 + j) * d + c] : 0.f;
  }
  __syncthreads();
  float lg[4][KPT];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int t = 0; t < KPT; ++t) lg[i][t] = 0.f;
#pragma unroll 4
  for (int c = 0; c < d; ++c) {
    float qv[4], kv[KPT];
#pragma unroll
    for (int i = 0; i < 4; ++i) qv[i] = qs[(warp * 4 + i) * d + c];
#pragma unroll
    for (int t = 0; t < KPT; ++t) kv[t] = ms[(lane + 32 * t) * (d + 1) + c];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int t = 0; t < KPT; ++t) lg[i][t] = fmaf(qv[i], kv[t], lg[i][t]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = warp * 4 + i;
    float mx = -3.0e38f;
#pragma unroll
    for (int t = 0; t < KPT; ++t) {
      lg[i][t] = lane + 32 * t < nk ? lg[i][t] * invT : -3.0e38f;
      mx = fmaxf(mx, lg[i][t]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < KPT; ++t) {
      const float p = lane + 32 * t < nk ? expf(lg[i][t] - mx) : 0.f;
      ps[r * CK + lane + 32 * t] = p;
      sum += p;
    }
    sum = warp_sum(sum);
    if (lane == 0 && i0 + r < B) {
      float* rec = part + ((size_t)blockIdx.x * B + i0 + r) * (d + 2);
      rec[0] = mx;
      rec[1] = sum;
    }
  }
  __syncwarp();                                        // ps rows of this warp are read by this warp only
  float ac[4][DU];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int u = 0; u < DU; ++u) ac[i][u] = 0.f;
#pragma unroll 4
  for (int j = 0; j < nk; ++j) {
    float pv[4], mv[DU];
#pragma unroll
    for (int i = 0; i < 4; ++i) pv[i] = ps[(warp * 4 + i) * CK + j];
#pragma unroll
    for (int u = 0; u < DU; ++u) mv[u] = ms[j * (d + 1) + lane + 32 * u];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int u = 0; u < DU; ++u) ac[i][u] = fmaf(pv[i], mv[u], ac[i][u]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = warp * 4 + i;
    if (i0 + r >= B) continue;
    float* rec = part + ((size_t)blockIdx.x * B + i0 + r) * (d + 2) + 2;
#pragma unroll
    for (int u = 0; u < DU; ++u) rec[lane + 32 * u] = ac[i][u];
  }
}

// merge partials with the positive logit; loss_i, dq_i; stats[0] += loss_i/B, stats[1] += l_pos/B
// grid = B, block 128 (threads over d)
__global__ void __launch_bounds__(128)
infonce_merge_kernel(const float* __restrict__ q, const float* __restrict__ k,
                     const float* __restrict__ part, int B, int d, int nchunks, float invT,
                     float* __restrict__ stats, float* __restrict__ dq) {
  __shared__ float red_s[4];
  __shared__ float bc[3];
  const int i = blockIdx.x, tid = threadIdx.x;
  pdl_wait();
  float s = 0.f;
  for (int c = tid; c < d; c += 128) s = fmaf(q[(size_t)i * d + c], k[(size_t)i * d + c], s);
  s = warp_sum(s);
  if ((tid & 31) == 0) red_s[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    const float lpos = (red_s[0] + red_s[1] + red_s[2] + red_s[3]) * invT;
    float M = lpos;
    for (int ch = 0; ch < nchunks; ++ch) M = fmaxf(M, part[((size_t)ch * B + i) * (d + 2)]);
    float S = expf(lpos - M);
    for (int ch = 0; ch < nchunks; ++ch) {
      const float* rec = part + ((size_t)ch * B + i) * (d + 2);
      S += rec[1] * expf(rec[0] - M);
    }
    bc[0] = M; bc[1] = S; bc[2] = lpos;
    atomicAdd(&stats[0], (logf(S) + M - lpos) / (float)B);
    atomicAdd(&stats[1], lpos / (float)B);
  }
  __syncthreads();
  const float M = bc[0], S = bc[1], lpos = bc[2];
  const float scale = invT / (float)B;
  for (int c = tid; c < d; c += 128) {
    float a = (expf(lpos - M) / S - 1.0f) * k[(size_t)i * d + c];
    for (int ch = 0; ch < nchunks; ++ch) {
      const float* rec = part + ((size_t)ch * B + i) * (d + 2);
      a = fmaf(expf(rec[0] - M) / S, rec[2 + c], a);
    }
    dq[(size_t)i * d + c] = a * scale;
  }
}

// `parts` blocks of B keys each, part r at k + r * part_stride (one rank's keys inside the gathered
// exchange buffer): all ranks' keys go in with one launch, in rank order (identical queues).
__global__ void moco_enqueue_kernel(float* __restrict__ mem, const float* __restrict__ k, int B, int d,
                                    int K, const int64_t* __restrict__ index_dev, int parts, int64_t part_stride,
                                    const int32_t* __restrict__ skip_word, int32_t skip_mask) {
  pdl_wait();
  if (skip_word && (*skip_word & skip_mask)) return;   // step skipped (empty view): the queue keeps its keys
  const int64_t base = *index_dev;
  const int per = B * d, total = parts * per;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int r = idx / per, w = idx - r * per;
    const int i = w / d, c = w - i * d;
    int64_t row = (base + (int64_t)r * B + i) % K;      // torch.fmod(arange(B) + index, K)
    mem[(size_t)row * d + c] = k[(size_t)r * part_stride + w];
  }
}
__global__ void moco_advance_kernel(int64_t* index_dev, int B, int K, const int32_t* __restrict__ skip_word,
                                    int32_t skip_mask) {
  pdl_wait();
  if (skip_word && (*skip_word & skip_mask)) return;
  if (threadIdx.x == 0 && blockIdx.x == 0) *index_dev = (*index_dev + B) % K;
}

// ---- E2E head: out[i][j] = k_i . q_j / T, label i ------------------------------------------
// pass 1 (grid B, block 256): logits row, softmax, dout row into workspace, loss / prob stats
__global__ void __launch_bounds__(256)
e2e_rows_kernel(const float* __restrict__ q, const float* __restrict__ k, int B, int d, float invT,
                float* __restrict__ stats, float* __restrict__ dout) {
  GCCB_DYN_SMEM(float, smem);            // ks[d] | row[B]
  __shared__ float red_s[8];
  __shared__ float bc[2];
  float* ks = smem;
  float* row = smem + d;
  const int i = blockIdx.x, tid = threadIdx.x;
  for (int c = tid; c < d; c += 256) ks[c] = k[(size_t)i * d + c];
  __syncthreads();
  float mx = -3.0e38f;
  for (int j = tid; j < B; j += 256) {
    float s = 0.f;
    for (int c = 0; c < d; ++c) s = fmaf(ks[c], q[(size_t)j * d + c], s);
    s *= invT;
    row[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) red_s[tid >> 5] = mx;
  __syncthreads();
  if (tid == 0) { float m = red_s[0]; for (int w = 1; w < 8; ++w) m = fmaxf(m, red_s[w]); bc[0] = m; }
  __syncthreads();
  mx = bc[0];
  float s = 0.f;
  for (int j = tid; j < B; j += 256) s += expf(row[j] - mx);
  s = warp_sum(s);
  __syncthreads();
  if ((tid & 31) == 0) red_s[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red_s[w];
    bc[1] = t;
    atomicAdd(&stats[0], (logf(t) + mx - row[i]) / (float)B);
    atomicAdd(&stats[1], row[i] / (float)B);
  }
  __syncthreads();
  const float sum = bc[1], invB = 1.0f / (float)B;
  for (int j = tid; j < B; j += 256)
    dout[(size_t)i * B + j] = (expf(row[j] - mx) / sum - (j == i ? 1.0f : 0.f)) * invB;
}
// pass 2 (grid (B, 2), block 128): y=0: dk_i = invT sum_j dout[i][j] q_j ; y=1: dq_j = invT sum_i dout[i][j] k_i
__global__ void __launch_bounds__(128)
e2e_grads_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ dout,
                 int B, int d, float invT, float* __restrict__ dq, float* __restrict__ dk) {
  const int x = blockIdx.x, tid = threadIdx.x;
  for (int c = tid; c < d; c += 128) {
    float a = 0.f;
    if (blockIdx.y == 0) {
      for (int j = 0; j < B; ++j) a = fmaf(dout[(size_t)x * B + j], q[(size_t)j * d + c], a);
      dk[(size_t)x * d + c] = a * invT;
    } else {
      for (int i = 0; i < B; ++i) a = fmaf(dout[(size_t)i * B + x], k[(size_t)i * d + c], a);
      dq[(size_t)x * d + c] = a * invT;
    }
  }
}

#ifndef GCCB_EMU
// ---- tensor-core InfoNCE (d >= 128: BASELINE config 4, K = 65536, B = 1024, d = 256) ------------------------
// logits = (q . queue^T) / T and dq = P . queue are the two big products of memory_moco.py:33-44 and its
// backward; both run on wgmma (csrc/tc_gemm.cu) with bf16 operands: the queue is cast once per step into a
// [K][d] copy (B operand of the logits GEMM) and a transposed [d][K] copy (B operand of the dq GEMM, split-K
// over the keys).  Between them one CTA per query row does the softmax in fp32 on the fp32 logits: loss,
// probabilities (bf16 operand of the second GEMM) and the positive-pair terms.
struct NceTcLayout { size_t q16, m16, mt16, logits, p16, ppos, dqn, splitk, total; int splits; };
static NceTcLayout nce_tc_layout(int B, int d, int K) {
  NceTcLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  L.q16 = take((size_t)B * d * 2);
  L.m16 = take((size_t)K * d * 2);
  L.mt16 = take((size_t)d * K * 2);
  L.logits = take((size_t)B * K * 4);
  L.p16 = take((size_t)B * K * 2);
  L.ppos = take((size_t)B * 4);
  L.dqn = take((size_t)B * d * 4);
  const int tiles = ((B + 127) / 128) * 1;
  L.splits = GCCB_NUM_SMS / tiles < 1 ? 1 : GCCB_NUM_SMS / tiles;
  if (L.splits > K / 64) L.splits = K / 64;
  L.splitk = take((size_t)L.splits * B * d * 4);
  L.total = off;
  return L;
}
static bool nce_use_tc(int B, int d, int K) {
  return d >= 128 && K % 64 == 0 && B >= 128;       // d is 128 or 256 here
}

// one CTA per query row: positive logit (fp32 q.k), row max / sum over [lpos | logits], loss and statistics,
// probabilities as the bf16 A operand of the dq GEMM, p_pos for the finalisation
__global__ void __launch_bounds__(256)
nce_tc_softmax_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ logits,
                      int B, int d, int K, float invT, float* __restrict__ stats, __nv_bfloat16* __restrict__ p16,
                      float* __restrict__ ppos) {
  __shared__ float red_s[8];
  __shared__ float bc[3];
  const int i = blockIdx.x, tid = threadIdx.x;
  const float* row = logits + (size_t)i * K;
  float s = 0.f;
  for (int c = tid; c < d; c += 256) s = fmaf(q[(size_t)i * d + c], k[(size_t)i * d + c], s);
  s = warp_sum(s);
  if ((tid & 31) == 0) red_s[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red_s[w]; bc[2] = t * invT; }
  __syncthreads();
  const float lpos = bc[2];
  float mx = lpos;
  for (int j = tid * 4; j < K; j += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + j);
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  mx = warp_max(mx);
  __syncthreads();
  if ((tid & 31) == 0) red_s[tid >> 5] = mx;
  __syncthreads();
  if (tid == 0) { float m = red_s[0]; for (int w = 1; w < 8; ++w) m = fmaxf(m, red_s[w]); bc[0] = m; }
  __syncthreads();
  mx = bc[0];
  float sum = 0.f;
  for (int j = tid * 4; j < K; j += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + j);
    sum += (expf(v.x - mx) + expf(v.y - mx)) + (expf(v.z - mx) + expf(v.w - mx));
  }
  sum = warp_sum(sum);
  __syncthreads();
  if ((tid & 31) == 0) red_s[tid >> 5] = sum;
  __syncthreads();
  if (tid == 0) {
    float t = expf(lpos - mx);
    for (int w = 0; w < 8; ++w) t += red_s[w];
    bc[1] = t;
    atomicAdd(&stats[0], (logf(t) + mx - lpos) / (float)B);
    atomicAdd(&stats[1], lpos / (float)B);
    ppos[i] = expf(lpos - mx) / t;
  }
  __syncthreads();
  const float inv = 1.0f / bc[1];
  __nv_bfloat16* prow = p16 + (size_t)i * K;
  for (int j = tid * 4; j < K; j += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + j);
    const __nv_bfloat162 a = __floats2bfloat162_rn(expf(v.x - mx) * inv, expf(v.y - mx) * inv);
    const __nv_bfloat162 b = __floats2bfloat162_rn(expf(v.z - mx) * inv, expf(v.w - mx) * inv);
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t*>(&a);
    u.y = *reinterpret_cast<const uint32_t*>(&b);
    *reinterpret_cast<uint2*>(prow + j) = u;
  }
}
// dq_i = ((p_pos - 1) k_i + sum_j p_ij queue_j) / (T B)
__global__ void __launch_bounds__(256)
nce_tc_finish_kernel(const float* __restrict__ k, const float* __restrict__ dqn, const float* __restrict__ ppos,
                     int B, int d, float scale, float* __restrict__ dq) {
  const int total = B * d;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int i = idx / d;
    dq[idx] = fmaf(ppos[i] - 1.0f, k[idx], dqn[idx]) * scale;
  }
}

static int infonce_tc(const float* q, const float* k, const float* memory, int B, int d, int K, float T, float* stats,
                      float* dq, char* ws, cudaStream_t st) {
  const NceTcLayout L = nce_tc_layout(B, d, K);
  __nv_bfloat16* q16 = (__nv_bfloat16*)(ws + L.q16);
  __nv_bfloat16* m16 = (__nv_bfloat16*)(ws + L.m16);
  __nv_bfloat16* mt16 = (__nv_bfloat16*)(ws + L.mt16);
  float* logits = (float*)(ws + L.logits);
  __nv_bfloat16* p16 = (__nv_bfloat16*)(ws + L.p16);
  float* ppos = (float*)(ws + L.ppos);
  float* dqn = (float*)(ws + L.dqn);
  float* splitk = (float*)(ws + L.splitk);
  int rc = tc::cast_bf16(q, B, d, d, q16, B, d, 0, nullptr, st);
  if (!rc) rc = tc::cast_bf16(memory, K, d, d, m16, K, d, 0, nullptr, st);
  if (!rc) rc = tc::cast_bf16(memory, K, d, d, mt16, K, d, 1, nullptr, st);
  if (!rc) rc = tc::gemm_bf16(q16, m16, B, K, d, nullptr, nullptr, 1.0f / T, logits, nullptr, K, nullptr, 1, nullptr, st);
  if (rc) return rc;
  GCCB_LAUNCH(nce_tc_softmax_kernel, B, 256, 0, st, q, k, (const float*)logits, B, d, K, 1.0f / T, stats, p16, ppos);
  rc = tc::gemm_bf16(p16, mt16, B, d, K, nullptr, nullptr, 1.0f, dqn, nullptr, d, nullptr, L.splits, splitk, st);
  if (rc) return rc;
  int blocks = (B * d + 255) / 256;
  if (blocks > 1184) blocks = 1184;
  GCCB_LAUNCH(nce_tc_finish_kernel, blocks, 256, 0, st, k, (const float*)dqn, (const float*)ppos, B, d,
              1.0f / (T * (float)B), dq);
  return check_launch("gccb_infonce_fused (tensor cores)");
}
#endif  // !GCCB_EMU

// the encoder widths; the fused head has a tiled kernel for each
static bool infonce_width(int d) { return d == 32 || d == 64 || d == 128 || d == 256; }
static int infonce_ck(int d) { return d <= 128 ? 128 : 64; }   // keys per CTA of infonce_partial_tiled_kernel

}  // namespace gccb

using namespace gccb;

static int bad_head_args(const char* who, const void* a, const void* b, int B, int d, int K) {
  if (!a || !b || B <= 0 || d <= 0 || d > 256 || K <= 0) {
    set_last_error("%s: bad argument (need 0 < d <= 256)", who);
    return 1;
  }
  return 0;
}

extern "C" int gccb_moco_logits(const float* q, const float* k, const float* memory, int32_t B,
                                int32_t d, int32_t K, float T, float* out, gccb_stream_t stream) {
  if (bad_head_args("gccb_moco_logits", q, k, B, d, K) || !memory || !out) return GCCB_ERR_BADARG;
  dim3 grid((K + 255) / 256, (B + GCCB_NCE_RB - 1) / GCCB_NCE_RB);
  GCCB_LAUNCH(moco_logits_kernel, grid, 256, (size_t)GCCB_NCE_RB * d * 4, stream, q, k, memory, B, d, K,
              1.0f / T, out);
  return check_launch("gccb_moco_logits");
}

extern "C" int gccb_moco_logits_backward(const float* dout, const float* k, const float* memory,
                                         int32_t B, int32_t d, int32_t K, float T, float* dq,
                                         gccb_stream_t stream) {
  if (bad_head_args("gccb_moco_logits_backward", dout, k, B, d, K) || !memory || !dq) return GCCB_ERR_BADARG;
  GCCB_LAUNCH(moco_logits_bwd_kernel, B, 256, (size_t)256 * 4 + (size_t)d * 4, stream, dout, k, memory, B, d, K,
              1.0f / T, dq);
  return check_launch("gccb_moco_logits_backward");
}

extern "C" int gccb_nce_loss(const float* out, int32_t B, int32_t C, int32_t label_mode, float* loss,
                             float* dout, gccb_stream_t stream) {
  if (!out || !loss || B <= 0 || C <= 0 || (label_mode == 1 && C < B)) {
    set_last_error("gccb_nce_loss: bad argument");
    return GCCB_ERR_BADARG;
  }
  cudaMemsetAsync(loss, 0, sizeof(float), (cudaStream_t)stream);
  GCCB_LAUNCH(nce_loss_kernel, B, 256, 0, stream, out, B, C, label_mode, loss, dout);
  return check_launch("gccb_nce_loss");
}

extern "C" size_t gccb_infonce_workspace(int32_t B, int32_t d, int32_t K) {
  if (!infonce_width(d)) return 0;
  int ck = infonce_ck(d);
  size_t nch = (size_t)(K + ck - 1) / ck;
  size_t simt = nch * (size_t)B * (d + 2) * sizeof(float);
#ifndef GCCB_EMU
  if (nce_use_tc(B, d, K)) { size_t t = nce_tc_layout(B, d, K).total; return t > simt ? t : simt; }
#endif
  return simt;
}

extern "C" int gccb_infonce_fused(const float* q, const float* k, const float* memory, int32_t B,
                                  int32_t d, int32_t K, float T, float* stats, float* dq, void* workspace,
                                  size_t workspace_bytes, gccb_stream_t stream) {
  if (bad_head_args("gccb_infonce_fused", q, k, B, d, K) || !memory || !stats || !dq || !workspace)
    return GCCB_ERR_BADARG;
  if (!infonce_width(d)) {
    set_last_error("gccb_infonce_fused: d = %d (need d in {32, 64, 128, 256})", d);
    return GCCB_ERR_BADARG;
  }
  if (workspace_bytes < gccb_infonce_workspace(B, d, K)) {
    set_last_error("gccb_infonce_fused: workspace too small");
    return GCCB_ERR_CAPACITY;
  }
  const int ck = infonce_ck(d);
  const int nch = (K + ck - 1) / ck;
#ifndef GCCB_EMU
  if (nce_use_tc(B, d, K)) {
    cudaMemsetAsync(stats, 0, 2 * sizeof(float), (cudaStream_t)stream);
    return infonce_tc(q, k, memory, B, d, K, T, stats, dq, (char*)workspace, (cudaStream_t)stream);
  }
#endif
  // both kernels are programmatic dependents of the kernel before them (common.cuh); the partial pass zeroes the
  // statistics the merge accumulates, so that no memset node breaks the chain
  const size_t smem = ((size_t)GCCB_NCE_RB2 * d + (size_t)ck * (d + 1) + (size_t)GCCB_NCE_RB2 * ck) * 4;
  dim3 grid(nch, (B + GCCB_NCE_RB2 - 1) / GCCB_NCE_RB2);
#define GCCB_NCE_TILED(KPT, DU)                                                              \
  do {                                                                                       \
    auto kt = infonce_partial_tiled_kernel<KPT, DU>;                                         \
    gccb::ensure_dyn_smem(kt, smem);                                                         \
    GCCB_LAUNCH_PDL(kt, grid, 256, smem, stream, q, memory, B, K, 1.0f / T, (float*)workspace, stats); \
  } while (0)
  if (d == 32) GCCB_NCE_TILED(4, 1);
  else if (d == 64) GCCB_NCE_TILED(4, 2);
  else if (d == 128) GCCB_NCE_TILED(4, 4);
  else GCCB_NCE_TILED(2, 8);
#undef GCCB_NCE_TILED
  GCCB_LAUNCH_PDL(infonce_merge_kernel, B, 128, 0, stream, q, k, (const float*)workspace, B, d, nch, 1.0f / T,
                  stats, dq);
  return check_launch("gccb_infonce_fused");
}

extern "C" int gccb_moco_enqueue(float* memory, const float* k, int32_t B, int32_t d, int32_t K,
                                 int64_t* index_dev, int32_t parts, int64_t part_stride,
                                 const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream) {
  if (!memory || !k || !index_dev || B <= 0 || d <= 0 || K <= 0 || parts < 1 || (parts > 1 && part_stride < (int64_t)B * d)) {
    set_last_error("gccb_moco_enqueue: bad argument");
    return GCCB_ERR_BADARG;
  }
  int blocks = (parts * B * d + 255) / 256;
  if (blocks > 1184) blocks = 1184;
  GCCB_LAUNCH_PDL(moco_enqueue_kernel, blocks, 256, 0, stream, memory, k, B, d, K, (const int64_t*)index_dev, parts,
                  part_stride, skip_word, skip_mask);
  GCCB_LAUNCH_PDL(moco_advance_kernel, 1, 32, 0, stream, index_dev, parts * B, K, skip_word, skip_mask);
  return check_launch("gccb_moco_enqueue");
}

extern "C" int gccb_e2e_nce(const float* q, const float* k, int32_t B, int32_t d, float T, float* stats,
                            float* dq, float* dk, void* workspace, size_t workspace_bytes,
                            gccb_stream_t stream) {
  if (bad_head_args("gccb_e2e_nce", q, k, B, d, 1) || !stats || !dq || !dk || !workspace) return GCCB_ERR_BADARG;
  if (workspace_bytes < (size_t)B * B * sizeof(float)) {
    set_last_error("gccb_e2e_nce: workspace needs B*B floats");
    return GCCB_ERR_CAPACITY;
  }
  cudaMemsetAsync(stats, 0, 2 * sizeof(float), (cudaStream_t)stream);
  const size_t smem = ((size_t)d + B) * 4;
  auto k1 = e2e_rows_kernel;
  gccb::ensure_dyn_smem(k1, smem);
  GCCB_LAUNCH(k1, B, 256, smem, stream, q, k, B, d, 1.0f / T, stats, (float*)workspace);
  dim3 grid(B, 2);
  GCCB_LAUNCH(e2e_grads_kernel, grid, 128, 0, stream, q, k, (const float*)workspace, B, d, 1.0f / T, dq, dk);
  return check_launch("gccb_e2e_nce");
}
