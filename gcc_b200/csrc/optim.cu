// optim.cu -- gradient clipping, Adam and the momentum-encoder update on flat buffers.
//
// Replaces (reference file:line):
//   clip_grad_norm -> torch.nn.utils.clip_grad_norm_(params, 1.0)     train.py:340-347,409
//   torch.optim.Adam(lr, betas, weight_decay = L2 added to the grad)  train.py:417,667-672
//   moment_update: p_ema = m p_ema + (1-m) p over model.parameters()  train.py:169-172,430-431
// The reference launches 51 + 2*67 tiny per-tensor kernels; here all live parameters are one
// flat buffer (gccb_gin_layout_t), so a step is one reduction and one elementwise kernel.
#include "common.cuh"

namespace gccb {

__global__ void __launch_bounds__(256)
gradnorm_kernel(const float* __restrict__ g, int64_t n, float scale, double* __restrict__ acc) {
  __shared__ double red_s[8];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double v = (double)g[i] * (double)scale;
    s += v * v;
  }
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red_s[w];
    atomicAdd(acc, t);
  }
}

// hyper: [0] lr, [1] 1 - beta1^t, [2] sqrt(1 - beta2^t)
__global__ void __launch_bounds__(256)
adam_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                float* __restrict__ v, float* __restrict__ p_ema, int64_t n_live, int64_t n_all,
                const float* __restrict__ hyper, float beta1, float beta2, float eps, float wd,
                float clip_norm, float alpha, float grad_scale, const double* __restrict__ sumsq,
                float* __restrict__ grad_norm_out, const int32_t* __restrict__ skip_word, int32_t skip_mask) {
  // a batch whose view was published empty (capacity overflow) must not move the weights: the whole
  // update (Adam moments, parameters, momentum encoder) is a no-op for that step
  if (skip_word && (*skip_word & skip_mask)) return;
  const float total = (float)sqrt(*sumsq);
  float coef = 1.0f;
  if (clip_norm > 0.f) {                                  // clip_grad_norm_: coef = max_norm/(norm+1e-6), clamped to 1
    coef = clip_norm / (total + 1e-6f);
    if (coef > 1.0f) coef = 1.0f;
  }
  const float lr = hyper[0], bc1 = hyper[1], sbc2 = hyper[2];
  if (blockIdx.x == 0 && threadIdx.x == 0 && grad_norm_out) *grad_norm_out = total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (int64_t)gridDim.x * blockDim.x) {
    float pv = p[i];
    if (i < n_live) {
      float gv = g[i] * grad_scale * coef;
      gv = fmaf(wd, pv, gv);                              // L2 weight decay folded into the gradient
      float mv = beta1 * m[i] + (1.0f - beta1) * gv;
      float vv = beta2 * v[i] + (1.0f - beta2) * gv * gv;
      m[i] = mv;
      v[i] = vv;
      float denom = sqrtf(vv) / sbc2 + eps;
      pv = pv - (lr / bc1) * (mv / denom);
      p[i] = pv;
    }
    if (alpha >= 0.f && p_ema) p_ema[i] = p_ema[i] * alpha + (1.0f - alpha) * pv;
  }
}

__global__ void __launch_bounds__(256)
sum_ranks_kernel(const float* __restrict__ gathered, int world, int64_t stride, int64_t n,
                 float* __restrict__ out, int64_t flag_index, int32_t* __restrict__ any_flag_out) {
  if (any_flag_out && blockIdx.x == 0 && threadIdx.x == 0) {
    int f = 0;
    for (int r = 0; r < world; ++r) f |= gathered[(size_t)r * stride + flag_index] != 0.f;
    *any_flag_out = f;
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < world; ++r) s += gathered[(size_t)r * stride + i];   // fixed rank order
    out[i] = s;
  }
}

}  // namespace gccb

using namespace gccb;

extern "C" int gccb_clip_adam_ema(float* p, float* g, float* m, float* v, float* p_ema, int64_t n_live,
                                  int64_t n_all, const float* hyper, float beta1, float beta2, float eps,
                                  float weight_decay, float clip_norm, float alpha, float grad_scale,
                                  float* grad_norm_out, double* workspace, const int32_t* skip_word,
                                  int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || !m || !v || !hyper || !workspace || n_live <= 0 || n_all < n_live) {
    set_last_error("gccb_clip_adam_ema: bad argument");
    return GCCB_ERR_BADARG;
  }
  cudaMemsetAsync(workspace, 0, sizeof(double), (cudaStream_t)stream);
  int blocks = (int)((n_live + 255) / 256);
  if (blocks > 4 * GCCB_NUM_SMS) blocks = 4 * GCCB_NUM_SMS;
  GCCB_LAUNCH(gradnorm_kernel, blocks, 256, 0, stream, (const float*)g, n_live, grad_scale, workspace);
  int blocks2 = (int)((n_all + 255) / 256);
  if (blocks2 > 1184) blocks2 = 1184;
  GCCB_LAUNCH(adam_ema_kernel, blocks2, 256, 0, stream, p, (const float*)g, m, v, p_ema, n_live, n_all, hyper,
              beta1, beta2, eps, weight_decay, clip_norm, alpha, grad_scale, (const double*)workspace,
              grad_norm_out, skip_word, skip_mask);
  return check_launch("gccb_clip_adam_ema");
}

extern "C" int gccb_sum_ranks(const float* gathered, int32_t world, int64_t stride, int64_t n, float* out,
                              int64_t flag_index, int32_t* any_flag_out, gccb_stream_t stream) {
  if (!gathered || !out || world <= 0 || n <= 0 || stride < n) {
    set_last_error("gccb_sum_ranks: bad argument");
    return GCCB_ERR_BADARG;
  }
  int blocks = (int)((n + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  GCCB_LAUNCH(sum_ranks_kernel, blocks, 256, 0, stream, gathered, world, stride, n, out, flag_index, any_flag_out);
  return check_launch("gccb_sum_ranks");
}
