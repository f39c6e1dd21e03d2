// knn.cu -- exact, deterministic cosine top-k between two sets of fp32 rows (structural similarity search).
//
// Definition (include/gccb200.h, DESIGN.md 4f):
//   rows are zero-padded to d4 = d rounded up to 4 and normalised once: s = the sequential __fmaf_rn chain of x_j x_j
//   over j = 0 .. d4-1, x^_j = x_j / sqrtf(s) (IEEE division and square root); s = 0 leaves the row all zeros, and a
//   row holding a NaN or Inf raises GCCB_FLAG_NONFINITE.  score(q, c) = the sequential __fmaf_rn chain of q^_j c^_j over
//   j = 0 .. d4-1 from +0.  The result of a query is the first k candidates under (score descending, index ascending),
//   -0 == +0 (a score of -0 is reported as +0), its excluded id left out.  Every score's bits depend on its two rows
//   alone and the order is strict, so the output does not depend on tiles, splits, query chunks or devices.
//
// Kernels:
//   knn_normalize_kernel  one warp per row: lanes load the row into shared memory, every lane runs the sequential
//                         chain over it (broadcast reads), lanes write the normalised row, zero-padded to ds = d4
//                         rounded up to KNN_KC, so that every dimension chunk of the score kernel is a whole 16-byte
//                         copy.
//   knn_score_kernel      grid (query tiles of KNN_TQ, candidate splits).  A CTA streams the KNN_TC-row candidate tiles
//                         of its split through a two-stage cp.async pipeline, KNN_KC dimensions at a time together with
//                         the matching chunk of its query tile.  Each thread holds a 4 x 8 register micro-tile of
//                         scores, each a full in-order chain (the FMAs are written out: nothing is left to
//                         contraction).  Selection per query: a sorted top list and a queue of kp = max(32, pow2 >= k)
//                         keys each in shared memory, and a threshold = the current k-th key.  A score below the
//                         threshold's score is dropped with one float compare; a survivor is keyed and, if below the
//                         threshold key, appended to the queue.  A full queue is merged into the top list by one warp
//                         (bitonic sort of the 2 kp keys), which raises the threshold; insertions that found their queue
//                         full retry after the merge.  At the end each (query, split) writes its k smallest keys.
//   knn_merge_kernel      one warp per query: a k-step merge of the splits' sorted lists (warp minimum of the heads).
// Key of (score, candidate) = (~ord(score) << 32) | candidate, ord the order-preserving map of the fp32 bits: ascending
// keys = descending scores, ascending candidates.
#include "common.cuh"

#include <math.h>

namespace gccb {

#define KNN_TQ 64                      // queries per CTA
#define KNN_TC 128                     // candidates per tile
#define KNN_KC 32                      // dimensions per pipeline stage
#define KNN_LD (KNN_KC + 4)            // shared row pitch (floats): 16-byte rows, conflict-free float4 reads
#define KNN_STAGE ((KNN_TQ + KNN_TC) * KNN_LD)
#define KNN_NT 256
#define KNN_MAXDIM 512
#define KNN_MAXK 128
#define KNN_MAX_SPLITS 128             // four per lane of the merge warp
#define KNN_SENT 0xFFFFFFFFFFFFFFFFull // empty slot: larger than every key

typedef unsigned long long knn_key_t;

#ifdef GCCB_EMU
static inline float knn_fma(float a, float b, float c) { return fmaf(a, b, c); }
static inline float knn_sqrt(float x) { return sqrtf(x); }
static inline float knn_div(float a, float b) { return a / b; }
static inline void knn_cp16(void* dst, const void* src, bool valid) {
  if (valid) memcpy(dst, src, 16);
  else memset(dst, 0, 16);
}
static inline void knn_cp_commit() {}
static inline void knn_cp_wait1() {}
static inline void knn_cp_wait0() {}
#else
__device__ __forceinline__ float knn_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float knn_sqrt(float x) { return __fsqrt_rn(x); }
__device__ __forceinline__ float knn_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ void knn_cp16(void* dst, const void* src, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void knn_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void knn_cp_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
__device__ __forceinline__ void knn_cp_wait0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
#endif

__device__ __forceinline__ knn_key_t knn_key(float s, uint32_t cand) {
  uint32_t u = __float_as_uint(s);
  if ((u << 1) == 0) u = 0;                                        // -0 == +0
  const uint32_t ord = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((knn_key_t)(~ord) << 32) | cand;
}
__device__ __forceinline__ float knn_key_score(knn_key_t key) {
  const uint32_t ord = ~(uint32_t)(key >> 32);
  return __uint_as_float((ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord);
}

// grid ceil(n / 8), block 256: warp w of block b normalises row 8b + w of x [n][dim] into out [n][ds]
__global__ void __launch_bounds__(256)
knn_normalize_kernel(const float* __restrict__ x, int64_t n, int dim, int d4, int ds, float* __restrict__ out,
                     int32_t* __restrict__ flags) {
  __shared__ float rows[8][KNN_MAXDIM];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * 8 + w;
  if (r >= n) return;                                              // whole warps; no block barrier below
  float* row = rows[w];
  bool bad = false;
  for (int j = lane; j < d4; j += 32) {
    const float v = j < dim ? x[r * dim + j] : 0.f;
    bad |= (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u;
    row[j] = v;
  }
  __syncwarp();
  float s = 0.f;
  for (int j = 0; j < d4; ++j) s = knn_fma(row[j], row[j], s);    // the defined sequential chain
  const float den = knn_sqrt(s);
  float* o = out + r * ds;
  for (int j = lane; j < ds; j += 32) o[j] = (j < dim && s != 0.f) ? knn_div(row[j], den) : 0.f;
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(flags, GCCB_FLAG_NONFINITE);
}

// One warp merges query ql's queue into its top list: b[0, kp) sorted top keys, b[kp, kp + cnt) the queue.  After the
// sort b[0, kp) holds the kp smallest keys; the threshold becomes the k-th.
__device__ __forceinline__ void knn_merge_queue(knn_key_t* __restrict__ b, int kp, int k, int* cnt,
                                                knn_key_t* thr, float* thr_s, int lane) {
  const int m = min(*cnt, kp);
  for (int j = kp + m + lane; j < 2 * kp; j += 32) b[j] = KNN_SENT;
  __syncwarp();
  const int n = 2 * kp;
  for (int size = 2; size <= n; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < n / 2; t += 32) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const knn_key_t a = b[i], c = b[j];
        if ((a > c) == ((i & size) == 0)) { b[i] = c; b[j] = a; }
      }
      __syncwarp();
    }
  if (lane == 0) {
    const knn_key_t t = b[k - 1];
    *thr = t;
    *thr_s = t == KNN_SENT ? -INFINITY : knn_key_score(t);
    *cnt = 0;
  }
  __syncwarp();
}

// grid (ceil(nq / KNN_TQ), splits), block KNN_NT, dynamic shared memory knn_smem_bytes(kp).  qn [nq][ds], cn [nc][ds]:
// normalised rows.  partial [nq][splits][k]: each (query, split)'s k smallest keys, ascending (KNN_SENT pads a split
// with fewer admissible candidates).
__global__ void __launch_bounds__(KNN_NT, 2)
knn_score_kernel(const float* __restrict__ qn, int64_t nq, const float* __restrict__ cn, int64_t nc, int d4, int ds,
                 int k, int kp, const int64_t* __restrict__ exclude, int splits, knn_key_t* __restrict__ partial) {
  GCCB_DYN_SMEM(float, smem);
  float* tiles = smem;
  knn_key_t* buf = reinterpret_cast<knn_key_t*>(smem + 2 * KNN_STAGE);
  knn_key_t* thr = buf + KNN_TQ * 2 * kp;
  float* thr_s = reinterpret_cast<float*>(thr + KNN_TQ);
  int* cnt = reinterpret_cast<int*>(thr_s + KNN_TQ);
  int64_t* excl = reinterpret_cast<int64_t*>(cnt + KNN_TQ);           // per query: the excluded candidate or -1
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lane = tid & 31, warp = tid >> 5;
  const int64_t q0 = (int64_t)blockIdx.x * KNN_TQ;
  const int split = blockIdx.y;
  const int64_t ctiles = (nc + KNN_TC - 1) / KNN_TC;
  const int64_t t_lo = ctiles * split / splits, t_hi = ctiles * (split + 1) / splits;
  const int nch = ds / KNN_KC;
  const int64_t steps = (t_hi - t_lo) * nch;

  for (int i = tid; i < KNN_TQ * 2 * kp; i += KNN_NT) buf[i] = KNN_SENT;
  if (tid < KNN_TQ) {
    thr[tid] = KNN_SENT;
    thr_s[tid] = -INFINITY;
    cnt[tid] = 0;
    excl[tid] = (exclude != nullptr && q0 + tid < nq) ? exclude[q0 + tid] : -1;
  }

  // step t: dimension chunk t % nch of candidate tile t_lo + t / nch, with the same chunk of the query tile
  auto issue = [&](int64_t t) {
    const int64_t tile = t_lo + t / nch;
    const int ch = (int)(t % nch);
    float* st = tiles + (t & 1) * KNN_STAGE;
    for (int e = tid; e < (KNN_TQ + KNN_TC) * (KNN_KC / 4); e += KNN_NT) {
      const int row = e / (KNN_KC / 4), part = e % (KNN_KC / 4);
      const float* src;
      bool valid;
      if (row < KNN_TQ) {
        const int64_t q = q0 + row;
        valid = q < nq;
        src = valid ? qn + q * ds + ch * KNN_KC + part * 4 : qn;
      } else {
        const int64_t c = tile * KNN_TC + (row - KNN_TQ);
        valid = c < nc;
        src = valid ? cn + c * ds + ch * KNN_KC + part * 4 : cn;
      }
      knn_cp16(st + row * KNN_LD + part * 4, src, valid);
    }
  };

  float acc[4][8];
  if (steps > 0) {
    issue(0);
    knn_cp_commit();
  }
  __syncthreads();
  for (int64_t t = 0; t < steps; ++t) {
    if (t + 1 < steps) {
      issue(t + 1);
      knn_cp_commit();
      knn_cp_wait1();
    } else {
      knn_cp_wait0();
    }
    __syncthreads();
    const int ch = (int)(t % nch);
    if (ch == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) acc[i][jj] = 0.f;
    }
    const float* Qs = tiles + (t & 1) * KNN_STAGE;
    const float* Cs = Qs + KNN_TQ * KNN_LD;
    // 4 dimensions of the chain for each of the 32 scores, in order x, y, z, w
    auto step4 = [&](int j4) {
      float4 a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(Qs + (ty * 4 + i) * KNN_LD + j4 * 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {                                   // candidates in two halves: fewer live registers
        float4 b[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          b[jj] = *reinterpret_cast<const float4*>(Cs + (tx + 16 * (4 * h + jj)) * KNN_LD + j4 * 4);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            float v = acc[i][4 * h + jj];
            v = knn_fma(a[i].x, b[jj].x, v);
            v = knn_fma(a[i].y, b[jj].y, v);
            v = knn_fma(a[i].z, b[jj].z, v);
            v = knn_fma(a[i].w, b[jj].w, v);
            acc[i][4 * h + jj] = v;
          }
      }
    };
    const int nd = min(KNN_KC, d4 - ch * KNN_KC);   // the chain stops at d4: the zero padding beyond is not summed
    if (nd == KNN_KC) {
#pragma unroll
      for (int j4 = 0; j4 < KNN_KC / 4; ++j4) step4(j4);
    } else {
      for (int j4 = 0; j4 < nd / 4; ++j4) step4(j4);
    }

    if (ch == nch - 1) {
      const int64_t c_base = (t_lo + t / nch) * KNN_TC;
      uint32_t pend = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ql = ty * 4 + i;
        const float ts = thr_s[ql];
        const knn_key_t tk = thr[ql];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int64_t c = c_base + tx + 16 * jj;
          if (q0 + ql < nq && c < nc && c != excl[ql] && !(acc[i][jj] < ts) && knn_key(acc[i][jj], (uint32_t)c) < tk)
            pend |= 1u << (i * 8 + jj);
        }
      }
      while (__syncthreads_or(pend != 0)) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ql = ty * 4 + i;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t bit = 1u << (i * 8 + jj);
            if (pend & bit) {
              const knn_key_t key = knn_key(acc[i][jj], (uint32_t)(c_base + tx + 16 * jj));
              if (key >= thr[ql]) {
                pend &= ~bit;                                       // the threshold rose past it
              } else {
                const int pos = atomicAdd(&cnt[ql], 1);
                if (pos < kp) {
                  buf[(size_t)ql * 2 * kp + kp + pos] = key;
                  pend &= ~bit;
                }                                                   // else: queue full, retry after its merge
              }
            }
          }
        }
        __syncthreads();
        for (int ql = warp; ql < KNN_TQ; ql += KNN_NT / 32)
          if (cnt[ql] >= kp) knn_merge_queue(buf + (size_t)ql * 2 * kp, kp, k, &cnt[ql], &thr[ql], &thr_s[ql], lane);
      }
    }
    __syncthreads();                                                // stage t & 1 is refilled by step t + 2
  }

  for (int ql = warp; ql < KNN_TQ; ql += KNN_NT / 32)
    if (cnt[ql] > 0) knn_merge_queue(buf + (size_t)ql * 2 * kp, kp, k, &cnt[ql], &thr[ql], &thr_s[ql], lane);
  __syncthreads();
  for (int e = tid; e < KNN_TQ * k; e += KNN_NT) {
    const int ql = e / k, i = e % k;
    const int64_t q = q0 + ql;
    if (q < nq) partial[((size_t)q * splits + split) * k + i] = buf[(size_t)ql * 2 * kp + i];
  }
}

__device__ __forceinline__ knn_key_t knn_warp_min(knn_key_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const knn_key_t u = __shfl_xor_sync(0xffffffffu, v, o);
    v = u < v ? u : v;
  }
  return v;
}

// grid ceil(nq / 8), block 256: warp w of block b merges the split lists of query 8b + w into out_ids / out_scores
__global__ void __launch_bounds__(256)
knn_merge_kernel(const knn_key_t* __restrict__ partial, int64_t nq, int k, int splits, int64_t* __restrict__ out_ids,
                 float* __restrict__ out_scores) {
  const int lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q >= nq) return;
  const knn_key_t* p = partial + (size_t)q * splits * k;
  int pos[4];
  knn_key_t head[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int s = lane + 32 * r;
    pos[r] = 0;
    head[r] = s < splits ? p[(size_t)s * k] : KNN_SENT;
  }
  for (int o = 0; o < k; ++o) {
    knn_key_t best = head[0];
#pragma unroll
    for (int r = 1; r < 4; ++r) best = head[r] < best ? head[r] : best;
    const knn_key_t m = knn_warp_min(best);
    if (m == KNN_SENT) {                                            // fewer admissible candidates than k: excluded
      if (lane == 0) {                                              // by the caller's check, never reached
        out_ids[q * k + o] = -1;
        out_scores[q * k + o] = NAN;
      }
      continue;
    }
    if (best == m) {                                                // keys are unique: one lane owns the minimum
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (head[r] == m) {
          ++pos[r];
          head[r] = pos[r] < k ? p[(size_t)(lane + 32 * r) * k + pos[r]] : KNN_SENT;
        }
      out_ids[q * k + o] = (int64_t)(uint32_t)m;
      out_scores[q * k + o] = knn_key_score(m);
    }
  }
}

static int knn_splits(int64_t nq, int64_t nc, int32_t splits) {
  if (splits > 0) return splits;
  const int64_t qt = (nq + KNN_TQ - 1) / KNN_TQ, ct = (nc + KNN_TC - 1) / KNN_TC;
  int64_t s = (2 * GCCB_NUM_SMS + qt - 1) / qt;                     // two waves of CTAs over the SMs
  if (s > ct) s = ct;
  if (s > KNN_MAX_SPLITS) s = KNN_MAX_SPLITS;
  return s < 1 ? 1 : (int)s;
}
static int knn_row_pitch(int dim) { return (((dim + 3) & ~3) + KNN_KC - 1) / KNN_KC * KNN_KC; }
static int knn_kp(int k) {
  int kp = 32;
  while (kp < k) kp <<= 1;
  return kp;
}
static size_t knn_align(size_t b) { return (b + 255) & ~(size_t)255; }
static size_t knn_smem_bytes(int kp) {
  return (size_t)2 * KNN_STAGE * 4 + (size_t)KNN_TQ * 2 * kp * 8 + (size_t)KNN_TQ * (8 + 4 + 4 + 8);
}
static bool knn_shape_ok(int64_t nq, int64_t nc, int32_t dim, int32_t k, int32_t splits) {
  return nq >= 1 && nc >= 1 && nc <= 0x7fffffffll && dim >= 1 && dim <= KNN_MAXDIM && k >= 1 && k <= KNN_MAXK &&
         splits >= 0 && splits <= KNN_MAX_SPLITS;
}

}  // namespace gccb

using namespace gccb;

extern "C" size_t gccb_knn_workspace(int64_t nq, int64_t nc, int32_t dim, int32_t k, int32_t splits) {
  if (!knn_shape_ok(nq, nc, dim, k, splits)) return 0;
  const size_t ds = (size_t)knn_row_pitch(dim);
  return knn_align((size_t)nc * ds * 4) + knn_align((size_t)nq * ds * 4) +
         (size_t)nq * knn_splits(nq, nc, splits) * k * 8;
}

extern "C" int gccb_knn(const float* queries, int64_t nq, const float* cands, int64_t nc, int32_t dim, int32_t k,
                        const int64_t* exclude, int32_t splits, int64_t* out_ids, float* out_scores, int32_t* flags,
                        void* ws, size_t ws_bytes, gccb_stream_t stream) {
  if (!knn_shape_ok(nq, nc, dim, k, splits)) {
    set_last_error("gccb_knn: need nq >= 1, 1 <= nc < 2^31, 1 <= dim <= %d, 1 <= k <= %d, 0 <= splits <= %d "
                   "(got nq=%lld nc=%lld dim=%d k=%d splits=%d)", KNN_MAXDIM, KNN_MAXK, KNN_MAX_SPLITS,
                   (long long)nq, (long long)nc, dim, k, splits);
    return GCCB_ERR_BADARG;
  }
  const int64_t admissible = nc - (exclude != nullptr ? 1 : 0);
  if (k > admissible) {
    set_last_error("gccb_knn: k = %d exceeds the %lld admissible candidates (%lld candidates%s)", k,
                   (long long)admissible, (long long)nc, exclude != nullptr ? ", one excluded per query" : "");
    return GCCB_ERR_BADARG;
  }
  if (!queries || !out_ids || !out_scores || !flags || !ws || ((uintptr_t)ws & 15) != 0) {
    set_last_error("gccb_knn: queries, out_ids, out_scores, flags and a 16-byte aligned workspace are required");
    return GCCB_ERR_BADARG;
  }
  const size_t need = gccb_knn_workspace(nq, nc, dim, k, splits);
  if (ws_bytes < need) {
    set_last_error("gccb_knn: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return GCCB_ERR_CAPACITY;
  }
  const int S = knn_splits(nq, nc, splits);
  const int d4 = (dim + 3) & ~3, ds = knn_row_pitch(dim), kp = knn_kp(k);
  float* cn = reinterpret_cast<float*>(ws);
  float* qn = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + knn_align((size_t)nc * ds * 4));
  knn_key_t* partial = reinterpret_cast<knn_key_t*>(reinterpret_cast<char*>(qn) + knn_align((size_t)nq * ds * 4));
  if (cands)
    GCCB_LAUNCH(knn_normalize_kernel, (unsigned)((nc + 7) / 8), 256, 0, stream, cands, nc, dim, d4, ds, cn, flags);
  GCCB_LAUNCH(knn_normalize_kernel, (unsigned)((nq + 7) / 8), 256, 0, stream, queries, nq, dim, d4, ds, qn, flags);
  const size_t smem = knn_smem_bytes(kp);
  ensure_dyn_smem(knn_score_kernel, smem);
  GCCB_LAUNCH(knn_score_kernel, dim3((unsigned)((nq + KNN_TQ - 1) / KNN_TQ), (unsigned)S), KNN_NT, smem, stream,
              (const float*)qn, nq, (const float*)cn, nc, d4, ds, k, kp, exclude, S, partial);
  GCCB_LAUNCH(knn_merge_kernel, (unsigned)((nq + 7) / 8), 256, 0, stream, (const knn_key_t*)partial, nq, k, S,
              out_ids, out_scores);
  return check_launch("gccb_knn");
}
