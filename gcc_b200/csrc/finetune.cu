// finetune.cu -- the supervised finetune step's own kernels: the classification head, the clip-by-value optimiser
// steps and the whole-graph feature gather from a cache.
//
// Replaces (reference file:line):
//   output_layer(feat_q), CrossEntropyLoss, the head's autograd      train.py:219-226
//   torch.nn.utils.clip_grad_value_(params, 1) + optimizer.step()    train.py:227-238
//   out.argmax(dim=1) + f1_score(average="micro")                    train.py:239-241,321-325
//   the per-item positional features of GraphClassificationDatasetLabeled (self.dict, graph_dataset.py:362)
//
// Every reduction over rows runs in a fixed order (no float atomics), so each call is bit-identical from run to run.
#include <math.h>

#include "optim_rules.cuh"

namespace gccb {

constexpr int kHeadMaxC = 128;       // classes: one thread of head_row_kernel per class
constexpr int kHeadMaxH = 256;       // the widest encoder
constexpr int kHeadMaxB = 4096;
constexpr int kHeadReduceThreads = 256;

// (value, index) of the first maximum: a larger value wins, an equal value goes to the smaller index (torch.argmax)
__device__ __forceinline__ void first_max(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}

// One batch row per CTA, one thread per class.  logits = feat W^T + bias (fixed-order h loop), max-subtracted
// log-sum-exp, the row's loss and whether its first maximum is the label; with train != 0 also
// dlogits = (softmax - onehot(y)) / b and dfeat = dlogits W.  block = kHeadMaxC.
__global__ void __launch_bounds__(kHeadMaxC)
head_row_kernel(const float* __restrict__ feat, int H, int C, const float* __restrict__ W,
                const float* __restrict__ bias, const int64_t* __restrict__ item_ids,
                const int64_t* __restrict__ labels, int64_t n_items, float inv_b, int train,
                float* __restrict__ dlogits, float* __restrict__ row_loss, int* __restrict__ row_correct,
                float* __restrict__ dfeat) {
  __shared__ float x_s[kHeadMaxH];
  __shared__ float d_s[kHeadMaxC];
  __shared__ float rv_s[kHeadMaxC / 32];
  __shared__ int ri_s[kHeadMaxC / 32];
  __shared__ float rs_s[kHeadMaxC / 32];
  const int i = blockIdx.x, c = threadIdx.x, lane = c & 31, w = c >> 5;
  for (int h = c; h < H; h += blockDim.x) x_s[h] = feat[(size_t)i * H + h];
  __syncthreads();
  float logit = -INFINITY;
  if (c < C) {
    float acc = 0.f;
    const float* wr = W + (size_t)c * H;
    for (int h = 0; h < H; ++h) acc = fmaf(x_s[h], wr[h], acc);
    logit = acc + bias[c];
  }
  // max and first argmax over the CTA: butterfly within each warp, then the warps in order
  float mv = logit;
  int mi = c < C ? c : 0x7fffffff;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, mv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
    first_max(mv, mi, ov, oi);
  }
  if (lane == 0) {
    rv_s[w] = mv;
    ri_s[w] = mi;
  }
  __syncthreads();
  mv = rv_s[0];
  mi = ri_s[0];
  for (int k = 1; k < (int)(blockDim.x >> 5); ++k) first_max(mv, mi, rv_s[k], ri_s[k]);
  const float e = c < C ? expf(logit - mv) : 0.f;
  float s = warp_sum(e);
  if (lane == 0) rs_s[w] = s;
  __syncthreads();
  s = 0.f;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += rs_s[k];
  int64_t item = item_ids[i];
  item = item < 0 ? 0 : (item >= n_items ? n_items - 1 : item);
  int64_t y = labels[item];
  y = y < 0 ? 0 : (y >= C ? C - 1 : y);
  if (c == (int)y) {
    row_loss[i] = (mv + logf(s)) - logit;               // log-sum-exp - logit_y
    row_correct[i] = mi == c;
  }
  if (!train) return;
  const float dl = c < C ? (e / s - (c == (int)y ? 1.f : 0.f)) * inv_b : 0.f;
  if (c < C) {
    d_s[c] = dl;
    dlogits[(size_t)i * C + c] = dl;
  }
  __syncthreads();
  for (int h = c; h < H; h += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < C; ++k) acc = fmaf(d_s[k], W[(size_t)k * H + h], acc);
    dfeat[(size_t)i * H + h] = acc;
  }
}

// Fixed-order sum of one value per thread over the CTA (kHeadReduceThreads threads): butterflies, then warps in order.
template <class T>
__device__ __forceinline__ T block_sum_fixed(T v, T* red_s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red_s[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = 0;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red_s[k];
  return t;
}

// Blocks 0 .. n_dw-1: dW[c][h] = sum_i dlogits[i][c] feat[i][h] (rows in order) and db[c].  Block n_dw: the batch
// statistics loss = mean row loss (double), correct = sum, b.  block = kHeadReduceThreads.
__global__ void __launch_bounds__(kHeadReduceThreads)
head_reduce_kernel(const float* __restrict__ feat, int b, int H, int C, int n_dw,
                   const float* __restrict__ dlogits, const float* __restrict__ row_loss,
                   const int* __restrict__ row_correct, float* __restrict__ dW, float* __restrict__ db,
                   float* __restrict__ stats) {
  __shared__ double rd_s[kHeadReduceThreads / 32];
  __shared__ float rf_s[kHeadReduceThreads / 32];
  __shared__ int ri_s[kHeadReduceThreads / 32];
  const int tid = threadIdx.x;
  if ((int)blockIdx.x == n_dw) {
    double l = 0.0;
    int k = 0;
    for (int i = tid; i < b; i += blockDim.x) {
      l += (double)row_loss[i];
      k += row_correct[i];
    }
    const double lt = block_sum_fixed(l, rd_s);
    const int kt = block_sum_fixed(k, ri_s);
    if (tid == 0) {
      stats[0] = (float)(lt / b);
      stats[1] = (float)kt;
      stats[2] = (float)b;
    }
    return;
  }
  const int c = blockIdx.x;
  for (int h = tid; h < H; h += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < b; ++i) acc = fmaf(dlogits[(size_t)i * C + c], feat[(size_t)i * H + h], acc);
    dW[(size_t)c * H + h] = acc;
  }
  float s = 0.f;
  for (int i = tid; i < b; i += blockDim.x) s += dlogits[(size_t)i * C + c];
  s = block_sum_fixed(s, rf_s);
  if (tid == 0) db[c] = s;
}

// clip_grad_value_(params, clip) then the rule's step: g <- clamp(g, -clip, clip), then the same update as the
// clip-by-norm kernels apply after their clip (optim_rules.cuh).  The gradient buffer is not written.
template <class Rule>
__global__ void __launch_bounds__(256)
clip_value_update_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s0,
                         float* __restrict__ s1, int64_t n, const float* __restrict__ hyper, Rule rule, float wd,
                         float clip_value, const int32_t* __restrict__ skip_word, int32_t skip_mask) {
  if (skip_word && (*skip_word & skip_mask)) return;        // a batch published empty does not train
  rule.load(hyper);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gv = fminf(fmaxf(g[i], -clip_value), clip_value);
    p[i] = decay_and_update(rule, i, p[i], gv, wd, s0, s1);
  }
}

// Row r of batch graph g (view `view`) <- cache row set.node_off[ids[g]] + (r - batch.node_off[g]).
// grid = B, block = 256.
__global__ void __launch_bounds__(256)
gather_features_kernel(const int64_t* __restrict__ g_node_off, int64_t n_graphs, const int64_t* __restrict__ graph_ids,
                       int B, int node_cap, const int32_t* __restrict__ node_off, int view,
                       const float* __restrict__ cache, int P, float* __restrict__ pos) {
  const int32_t* no = node_off + view * (B + 1);
  if (no[B] < 0) return;                                    // view overflowed: published empty
  const int g = blockIdx.x;
  const int64_t id = clamp_graph(graph_ids[g], n_graphs);
  const int r0 = no[g];
  const int64_t n = (int64_t)(no[g + 1] - r0) * P;
  const float* src = cache + g_node_off[id] * P;
  float* dst = pos + ((size_t)view * node_cap + r0) * P;
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
}

}  // namespace gccb

using namespace gccb;

namespace {

size_t head_ws_floats(int32_t B, int32_t C) { return (size_t)B * C + 2 * (size_t)B; }

template <class Rule>
int clip_value_update(const char* name, float* p, const float* g, float* s0, float* s1, int64_t n, const float* hyper,
                      Rule rule, float weight_decay, float clip_value, const int32_t* skip_word, int32_t skip_mask,
                      gccb_stream_t stream) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  GCCB_LAUNCH(clip_value_update_kernel<Rule>, blocks, 256, 0, stream, p, g, s0, s1, n, hyper, rule, weight_decay,
              clip_value, skip_word, skip_mask);
  return check_launch(name);
}

}  // namespace

extern "C" size_t gccb_ft_head_workspace(int32_t B, int32_t C) {
  if (B <= 0 || C <= 0) return 0;
  return head_ws_floats(B, C) * sizeof(float);
}

extern "C" int gccb_ft_head(const float* feat, int32_t B, int32_t b, int32_t H, int32_t C, const float* W,
                            const float* bias, const int64_t* item_ids, const int64_t* labels, int64_t n_items,
                            int32_t eval, float* dfeat, float* dW, float* db, float* stats, void* workspace,
                            size_t workspace_bytes, gccb_stream_t stream) {
  if (!(H == 32 || H == 64 || H == 128 || H == 256) || C < 2 || C > kHeadMaxC || B <= 0 || B > kHeadMaxB ||
      b <= 0 || b > B || n_items <= 0) {
    set_last_error("gccb_ft_head: unsupported sizes B=%d b=%d H=%d C=%d (H in {32,64,128,256}, 2 <= C <= %d, "
                   "0 < b <= B <= %d)", B, b, H, C, kHeadMaxC, kHeadMaxB);
    return GCCB_ERR_BADARG;
  }
  if (!feat || !W || !bias || !item_ids || !labels || !stats || !workspace ||
      workspace_bytes < gccb_ft_head_workspace(B, C) || (!eval && (!dfeat || !dW || !db))) {
    set_last_error("gccb_ft_head: bad argument");
    return GCCB_ERR_BADARG;
  }
  float* dlogits = (float*)workspace;
  float* row_loss = dlogits + (size_t)B * C;
  int* row_correct = (int*)(row_loss + B);
  const int train = eval ? 0 : 1;
  GCCB_LAUNCH(head_row_kernel, b, kHeadMaxC, 0, stream, feat, H, C, W, bias, item_ids, labels, n_items,
              1.0f / (float)b, train, dlogits, row_loss, row_correct, dfeat);
  const int n_dw = train ? C : 0;
  GCCB_LAUNCH(head_reduce_kernel, n_dw + 1, kHeadReduceThreads, 0, stream, feat, b, H, C, n_dw, dlogits, row_loss,
              row_correct, dW, db, stats);
  return check_launch("gccb_ft_head");
}

extern "C" int gccb_clip_value_adam(float* p, const float* g, float* m, float* v, int64_t n, const float* hyper,
                                    float beta1, float beta2, float eps, float weight_decay, float clip_value,
                                    const int32_t* skip_word, int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || !m || !v || !hyper || n <= 0 || !(clip_value > 0.f)) {
    set_last_error("gccb_clip_value_adam: bad argument");
    return GCCB_ERR_BADARG;
  }
  AdamRule rule{beta1, beta2, eps, 0.f, 0.f, 0.f};
  return clip_value_update("gccb_clip_value_adam", p, g, m, v, n, hyper, rule, weight_decay, clip_value, skip_word,
                           skip_mask, stream);
}

extern "C" int gccb_clip_value_sgd(float* p, const float* g, float* buf, int64_t n, const float* hyper,
                                   float momentum, float weight_decay, float clip_value, const int32_t* skip_word,
                                   int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || (momentum != 0.f && !buf) || !hyper || n <= 0 || !(clip_value > 0.f)) {
    set_last_error("gccb_clip_value_sgd: bad argument");
    return GCCB_ERR_BADARG;
  }
  SgdRule rule{momentum, 0.f};
  return clip_value_update("gccb_clip_value_sgd", p, g, buf, nullptr, n, hyper, rule, weight_decay, clip_value,
                           skip_word, skip_mask, stream);
}

extern "C" int gccb_clip_value_adagrad(float* p, const float* g, float* sum, int64_t n, const float* hyper, float eps,
                                       float weight_decay, float clip_value, const int32_t* skip_word,
                                       int32_t skip_mask, gccb_stream_t stream) {
  if (!p || !g || !sum || !hyper || n <= 0 || !(clip_value > 0.f)) {
    set_last_error("gccb_clip_value_adagrad: bad argument");
    return GCCB_ERR_BADARG;
  }
  AdagradRule rule{eps, 0.f};
  return clip_value_update("gccb_clip_value_adagrad", p, g, sum, nullptr, n, hyper, rule, weight_decay, clip_value,
                           skip_word, skip_mask, stream);
}

extern "C" int gccb_gather_features(const gccb_graph_set_t* set, const int64_t* graph_ids, const gccb_batch_t* batch,
                                    int32_t view, const float* cache, int32_t pos_dim, float* pos,
                                    gccb_stream_t stream) {
  if (!set || !batch || !graph_ids || !cache || !pos || batch->batch <= 0 || set->n_graphs <= 0 || !set->node_off ||
      (view != 0 && view != 1) || pos_dim <= 0) {
    set_last_error("gccb_gather_features: bad argument");
    return GCCB_ERR_BADARG;
  }
  GCCB_LAUNCH(gather_features_kernel, batch->batch, 256, 0, stream, set->node_off, set->n_graphs, graph_ids,
              batch->batch, batch->node_cap, batch->node_off, view, cache, pos_dim, pos);
  return check_launch("gccb_gather_features");
}
