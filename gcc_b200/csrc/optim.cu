// optim.cu -- gradient clipping, the optimiser step and the momentum-encoder update on flat buffers.
//
// Replaces (reference file:line):
//   clip_grad_norm -> torch.nn.utils.clip_grad_norm_(params, 1.0)     train.py:340-347,409
//   torch.optim.{SGD,Adam,Adagrad}(lr, ..., weight_decay = L2 added to the grad)  train.py:417,659-678
//   moment_update: p_ema = m p_ema + (1-m) p over model.parameters()  train.py:169-172,430-431
// The reference launches 51 + 2*67 tiny per-tensor kernels; here all live parameters are one
// flat buffer (gccb_gin_layout_t), so a step is one reduction and one elementwise kernel.
#include "optim_rules.cuh"

namespace gccb {

__global__ void __launch_bounds__(256)
gradnorm_kernel(const float* __restrict__ g, int64_t n, float scale, double* __restrict__ acc) {
  __shared__ double red_s[8];
  pdl_wait();
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

// The update rules (AdamRule, SgdRule, AdagradRule) are in optim_rules.cuh, shared with finetune.cu.

template <class Rule>
__global__ void __launch_bounds__(256)
clip_update_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s0,
                       float* __restrict__ s1, float* __restrict__ p_ema, int64_t n_live, int64_t n_all,
                       const float* __restrict__ hyper, Rule rule, float wd, float clip_norm, float alpha,
                       float grad_scale, const double* __restrict__ sumsq, float* __restrict__ grad_norm_out,
                       const int32_t* __restrict__ skip_word, int32_t skip_mask) {
  // a batch whose view was published empty (capacity overflow) must not move the weights: the whole
  // update (optimiser state, parameters, momentum encoder) is a no-op for that step
  pdl_wait();
  if (skip_word && (*skip_word & skip_mask)) return;
  const float total = (float)sqrt(*sumsq);
  float coef = 1.0f;
  if (clip_norm > 0.f) {                                  // clip_grad_norm_: coef = max_norm/(norm+1e-6), clamped to 1
    coef = clip_norm / (total + 1e-6f);
    if (coef > 1.0f) coef = 1.0f;
  }
  rule.load(hyper);
  if (blockIdx.x == 0 && threadIdx.x == 0 && grad_norm_out) *grad_norm_out = total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (int64_t)gridDim.x * blockDim.x) {
    float pv = p[i];
    if (i < n_live) {
      float gv = g[i] * grad_scale * coef;
      pv = decay_and_update(rule, i, pv, gv, wd, s0, s1);
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

namespace {

// The clip norm (gradnorm_kernel) then the update of every live entry and the EMA of all n_all entries
// (clip_update_ema_kernel<Rule>), on `stream`, both programmatic dependents of the kernel before them
// (common.cuh).  The norm's accumulator stays a memset: every block of gradnorm_kernel adds to it, so no block of
// it could zero it first, and the call has no earlier kernel.
template <class Rule>
int clip_update_ema(const char* name, float* p, const float* g, float* s0, float* s1, float* p_ema, int64_t n_live,
                    int64_t n_all, const float* hyper, Rule rule, float weight_decay, float clip_norm, float alpha,
                    float grad_scale, float* grad_norm_out, double* workspace, const int32_t* skip_word,
                    int32_t skip_mask, gccb_stream_t stream) {
  cudaMemsetAsync(workspace, 0, sizeof(double), (cudaStream_t)stream);
  int blocks = (int)((n_live + 255) / 256);
  if (blocks > 4 * GCCB_NUM_SMS) blocks = 4 * GCCB_NUM_SMS;
  GCCB_LAUNCH_PDL(gradnorm_kernel, blocks, 256, 0, stream, g, n_live, grad_scale, workspace);
  int blocks2 = (int)((n_all + 255) / 256);
  if (blocks2 > 1184) blocks2 = 1184;
  GCCB_LAUNCH_PDL(clip_update_ema_kernel<Rule>, blocks2, 256, 0, stream, p, g, s0, s1, p_ema, n_live, n_all, hyper,
                  rule, weight_decay, clip_norm, alpha, grad_scale, (const double*)workspace, grad_norm_out, skip_word,
                  skip_mask);
  return check_launch(name);
}

}  // namespace

extern "C" int gccb_clip_adam_ema(float* p, float* g, float* m, float* v, float* p_ema, int64_t n_live,
                                  int64_t n_all, const float* hyper, float beta1, float beta2, float eps,
                                  float weight_decay, float clip_norm, float alpha, float grad_scale,
                                  float* grad_norm_out, double* workspace, const int32_t* skip_word,
                                  int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || !m || !v || !hyper || !workspace || n_live <= 0 || n_all < n_live) {
    set_last_error("gccb_clip_adam_ema: bad argument");
    return GCCB_ERR_BADARG;
  }
  AdamRule rule{beta1, beta2, eps, 0.f, 0.f, 0.f};
  return clip_update_ema("gccb_clip_adam_ema", p, g, m, v, p_ema, n_live, n_all, hyper, rule, weight_decay,
                         clip_norm, alpha, grad_scale, grad_norm_out, workspace, skip_word, skip_mask, stream);
}

extern "C" int gccb_clip_sgd_ema(float* p, float* g, float* buf, float* p_ema, int64_t n_live, int64_t n_all,
                                 const float* hyper, float momentum, float weight_decay, float clip_norm, float alpha,
                                 float grad_scale, float* grad_norm_out, double* workspace, const int32_t* skip_word,
                                 int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || (momentum != 0.f && !buf) || !hyper || !workspace || n_live <= 0 || n_all < n_live) {
    set_last_error("gccb_clip_sgd_ema: bad argument");
    return GCCB_ERR_BADARG;
  }
  SgdRule rule{momentum, 0.f};
  return clip_update_ema("gccb_clip_sgd_ema", p, g, buf, nullptr, p_ema, n_live, n_all, hyper, rule, weight_decay,
                         clip_norm, alpha, grad_scale, grad_norm_out, workspace, skip_word, skip_mask, stream);
}

extern "C" int gccb_clip_adagrad_ema(float* p, float* g, float* sum, float* p_ema, int64_t n_live, int64_t n_all,
                                     const float* hyper, float eps, float weight_decay, float clip_norm, float alpha,
                                     float grad_scale, float* grad_norm_out, double* workspace,
                                     const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || !sum || !hyper || !workspace || n_live <= 0 || n_all < n_live) {
    set_last_error("gccb_clip_adagrad_ema: bad argument");
    return GCCB_ERR_BADARG;
  }
  AdagradRule rule{eps, 0.f};
  return clip_update_ema("gccb_clip_adagrad_ema", p, g, sum, nullptr, p_ema, n_live, n_all, hyper, rule,
                         weight_decay, clip_norm, alpha, grad_scale, grad_norm_out, workspace, skip_word, skip_mask,
                         stream);
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
