// baselines.cu -- the reference's two embedding baselines, GraphWave and ProNE, in float64.
//
// Replaces (reference file:line):
//   heat_diffusion_ind (Chebyshev heat wavelets)       gcc/models/emb/_graphwave/graphwave.py:48-91
//   charac_function(_multiscale)                       gcc/models/emb/_graphwave/characteristic_functions.py:63-86
//   ProNE._pre_factorization (F on A's pattern)        gcc/models/emb/prone.py:56-76
//   ProNE._chebyshev_gaussian (spectral propagation)   gcc/models/emb/prone.py:78-108
//
// Everything is one building block, a CSR x dense-block product with an epilogue (spmm_kernel):
//   Y = alpha * dr * ((A + sigma I) (dc X)) + beta X + gamma Z + delta W,   acc_h += h_h * Y  (h = 0, 1)
// X, Y, Z, W are n x k row-major with row stride ld.  A row is gathered by one warp, each lane owning column pairs
// (128-bit loads when ld is even and every block starts on 16 bytes, single columns otherwise); a row's entries are
// summed in CSR order with explicit fma, so the arithmetic of a column does not depend on k, ld or which path (pair
// or single column) computed it.  That is what makes GraphWave's output bit-identical for every column-block size.  Y may alias Z or W (each element is read by the
// thread that writes it), never X.
#include <math.h>

#include "common.cuh"

namespace gccb {

struct SpmmArgs {
  const int64_t* indptr;
  const int32_t* indices;
  const double* vals;      // NULL: every entry weighs 1 (a repeated column is a parallel edge)
  int64_t n;
  int32_t k;
  int64_t ld;
  double alpha, sigma;
  const double* dr;        // NULL: 1
  const double* dc;        // NULL: 1
  double beta;
  const double* X;
  double gamma;
  const double* Z;         // NULL: term dropped
  double delta;
  const double* W;         // NULL: term dropped
  double* Y;
  double h0;
  double* acc0;            // NULL: no accumulation
  double h1;
  double* acc1;
  int pairs;               // set by launch_spmm: every row of every block starts on 16 bytes
};

template <int P>
__device__ __forceinline__ void load_cols(const double* p, double* v) {
  if (P == 2) {
    const double2 t = *reinterpret_cast<const double2*>(p);
    v[0] = t.x;
    v[1] = t.y;
  } else {
    v[0] = *p;
  }
}

template <int P>
__device__ __forceinline__ void store_cols(double* p, const double* v) {
  if (P == 2) {
    double2 t;
    t.x = v[0];
    t.y = v[1];
    *reinterpret_cast<double2*>(p) = t;
  } else {
    *p = v[0];
  }
}

// columns [c, c + P) of row i
template <int P>
__device__ __forceinline__ void spmm_cols(const SpmmArgs& s, int64_t i, int64_t e0, int64_t e1, int64_t c) {
  double acc[P];
#pragma unroll
  for (int w = 0; w < P; ++w) acc[w] = 0.0;
  for (int64_t e = e0; e < e1; ++e) {
    const int64_t j = __ldg(s.indices + e);
    double a = s.vals ? __ldg(s.vals + e) : 1.0;
    if (s.dc) a *= __ldg(s.dc + j);
    double x[P];
    load_cols<P>(s.X + j * s.ld + c, x);
#pragma unroll
    for (int w = 0; w < P; ++w) acc[w] = fma(a, x[w], acc[w]);
  }
  double xi[P], z[P], wv[P], y[P];
  load_cols<P>(s.X + i * s.ld + c, xi);
  if (s.sigma != 0.0) {
    const double a = s.dc ? s.sigma * s.dc[i] : s.sigma;
#pragma unroll
    for (int w = 0; w < P; ++w) acc[w] = fma(a, xi[w], acc[w]);
  }
  const double scale = s.dr ? s.alpha * s.dr[i] : s.alpha;
  if (s.Z) load_cols<P>(s.Z + i * s.ld + c, z);
  if (s.W) load_cols<P>(s.W + i * s.ld + c, wv);
#pragma unroll
  for (int w = 0; w < P; ++w) {
    double v = fma(s.beta, xi[w], scale * acc[w]);
    if (s.Z) v = fma(s.gamma, z[w], v);
    if (s.W) v = fma(s.delta, wv[w], v);
    y[w] = v;
  }
  store_cols<P>(s.Y + i * s.ld + c, y);
  if (s.acc0) {
    double h[P];
    load_cols<P>(s.acc0 + i * s.ld + c, h);
#pragma unroll
    for (int w = 0; w < P; ++w) h[w] = fma(s.h0, y[w], h[w]);
    store_cols<P>(s.acc0 + i * s.ld + c, h);
  }
  if (s.acc1) {
    double h[P];
    load_cols<P>(s.acc1 + i * s.ld + c, h);
#pragma unroll
    for (int w = 0; w < P; ++w) h[w] = fma(s.h1, y[w], h[w]);
    store_cols<P>(s.acc1 + i * s.ld + c, h);
  }
}

// one warp per row, 8 rows per CTA
__global__ void __launch_bounds__(256) spmm_kernel(SpmmArgs s) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= s.n) return;
  const int64_t e0 = s.indptr[i], e1 = s.indptr[i + 1];
  const int64_t pairs = s.pairs ? s.k / 2 : 0;
  for (int64_t p = lane; p < pairs; p += 32) spmm_cols<2>(s, i, e0, e1, 2 * p);
  for (int64_t c = 2 * pairs + lane; c < s.k; c += 32) spmm_cols<1>(s, i, e0, e1, c);
}

static int launch_spmm(SpmmArgs s, gccb_stream_t stream) {
  if (s.n <= 0 || s.k <= 0) return GCCB_OK;
  const uintptr_t bases = (uintptr_t)s.X | (uintptr_t)s.Y | (uintptr_t)s.Z | (uintptr_t)s.W | (uintptr_t)s.acc0 |
                          (uintptr_t)s.acc1;
  s.pairs = (s.ld % 2 == 0) && (bases % 16 == 0);
  GCCB_LAUNCH(spmm_kernel, (unsigned)((s.n + 7) / 8), 256, 0, stream, s);
  return GCCB_OK;
}

// out[i] = f(sum of row i's weights): mode 0 the sum, 1 its inverse square root (0 for a sum <= 1e-10, as the
// reference's laplacian), 2 the inverse of sum + 1 (the l1 row normaliser of I + A)
__global__ void __launch_bounds__(256)
rowsum_kernel(const int64_t* __restrict__ indptr, const double* __restrict__ vals, int64_t n, int mode,
              double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  double d = 0.0;
  for (int64_t e = indptr[i] + lane; e < indptr[i + 1]; e += 32) d += vals ? vals[e] : 1.0;
  d = warp_sum_d(d);
  if (lane == 0) out[i] = mode == 0 ? d : mode == 1 ? (d > 1e-10 ? 1.0 / sqrt(d) : 0.0) : 1.0 / (d + 1.0);
}

static void launch_rowsum(const int64_t* indptr, const double* vals, int64_t n, int mode, double* out,
                          gccb_stream_t stream) {
  GCCB_LAUNCH(rowsum_kernel, (unsigned)((n + 7) / 8), 256, 0, stream, indptr, vals, n, mode, out);
}

// ---------------------------------------------------------------------------------------------------------------
// GraphWave

#define GW_MAX_TIMES 64
#define GW_MAX_ORDER 64
#define GW_TCHUNK 8

struct GwTimes {
  double t[GW_MAX_TIMES];
};

// T0 = the identity columns c0 .. c0 + bc of the block, H_s = c_s0 * T0
__global__ void __launch_bounds__(256)
gw_init_kernel(int64_t n, int64_t c0, int bc, int64_t ld, double c00, double c10, double* __restrict__ t0,
               double* __restrict__ h0, double* __restrict__ h1) {
  const int64_t total = n * ld;
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = x / ld, j = x - i * ld;
    const double v = (j < bc && i == c0 + j) ? 1.0 : 0.0;
    t0[x] = v;
    h0[x] = c00 * v;
    h1[x] = c10 * v;
  }
}

// chi[c0 + j, s * 2T + 2t + {0, 1}] = (1/n) sum_i {cos, sin}(times[t] * thr(H_s[i, j])).
// grid = (ceil(bc / 32), 2 scales, ceil(T / 8)), block = (32 columns, 8 row phases).  Row phase w sums rows
// i = w (mod 8) in ascending order and the phases are added 0..7: the same order for every column whatever bc.
__global__ void __launch_bounds__(256)
gw_chi_kernel(int64_t n, int64_t c0, int bc, int64_t ld, const double* __restrict__ h0,
              const double* __restrict__ h1, GwTimes times, int n_times, double thr, double* __restrict__ chi) {
  __shared__ double part[8][GW_TCHUNK * 2][32];
  const int lane = threadIdx.x, w = threadIdx.y;
  const int j = blockIdx.x * 32 + lane;
  const int scale = blockIdx.y;
  const int t0 = blockIdx.z * GW_TCHUNK;
  const int nt = min(GW_TCHUNK, n_times - t0);
  const double* h = scale ? h1 : h0;
  double cs[GW_TCHUNK], sn[GW_TCHUNK];
#pragma unroll
  for (int t = 0; t < GW_TCHUNK; ++t) cs[t] = sn[t] = 0.0;
  if (j < bc) {
    for (int64_t i = w; i < n; i += 8) {
      double v = h[i * ld + j];
      if (!(v > thr)) {                                   // thresholded to 0: cos 0 = 1, sin 0 = 0
#pragma unroll
        for (int t = 0; t < GW_TCHUNK; ++t) cs[t] += 1.0;
        continue;
      }
#pragma unroll
      for (int t = 0; t < GW_TCHUNK; ++t) {
        if (t < nt) {
          double sv, cv;
          sincos(times.t[t0 + t] * v, &sv, &cv);
          cs[t] += cv;
          sn[t] += sv;
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < GW_TCHUNK; ++t) {
    part[w][2 * t][lane] = cs[t];
    part[w][2 * t + 1][lane] = sn[t];
  }
  __syncthreads();
  if (j < bc) {
    const int q = w;                                     // 8 phases reduce 16 (t, cos/sin) slots: two each
    for (int slot = q; slot < 2 * nt; slot += 8) {
      double acc = 0.0;
      for (int p = 0; p < 8; ++p) acc += part[p][slot][lane];
      const int t = t0 + slot / 2;
      chi[(c0 + j) * (int64_t)(4 * n_times) + scale * 2 * n_times + 2 * t + (slot & 1)] = acc / (double)n;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ProNE

// p[j] = (sum_i A_ij / d_i)^0.75 for a symmetric A: column j's sum gathered from row j
__global__ void __launch_bounds__(256)
prone_colpow_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const double* __restrict__ vals, int64_t n, const double* __restrict__ d,
                    double* __restrict__ p) {
  const int lane = threadIdx.x & 31;
  const int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= n) return;
  double s = 0.0;
  for (int64_t e = indptr[j] + lane; e < indptr[j + 1]; e += 32) s += (vals ? vals[e] : 1.0) / d[indices[e]];
  s = warp_sum_d(s);
  if (lane == 0) p[j] = pow(s, 0.75);
}

// out[0] = sum of x (one CTA, fixed order)
__global__ void __launch_bounds__(1024) sum_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ out) {
  __shared__ double part[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += x[i];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.0;
    s = warp_sum_d(s);
    if (threadIdx.x == 0) out[0] = s;
  }
}

// F_ij = log(A_ij / d_i) - log(A_ij * neg_j) and FT_ij = F_ji on A's (symmetric) pattern, neg = p / sum(p)
__global__ void __launch_bounds__(256)
prone_values_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const double* __restrict__ vals, int64_t n, const double* __restrict__ d,
                    const double* __restrict__ p, const double* __restrict__ psum, double* __restrict__ F,
                    double* __restrict__ FT) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const double total = psum[0];
  const double negi = p[i] / total;
  for (int64_t e = indptr[i] + lane; e < indptr[i + 1]; e += 32) {
    const int64_t j = indices[e];
    const double a = vals ? vals[e] : 1.0;
    F[e] = log(a / d[i]) - log(a * (p[j] / total));
    FT[e] = log(a / d[j]) - log(a * negi);
  }
}

// out[i, j] = a standard normal from Philox (key, counter (i, j, 0, tag)) by Box-Muller
__global__ void __launch_bounds__(256)
gaussian_kernel(double* __restrict__ out, int64_t rows, int cols, uint64_t key) {
  const int64_t total = rows * cols;
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = x / cols;
    const uint32_t j = (uint32_t)(x - i * cols);
    const u32x4 r = philox_at(key, (uint64_t)i, j, 0, 0, GCCB_TAG_PRONE);
    const double u1 = (double)(((((uint64_t)r.x) << 32) | r.y) >> 11) * 0x1.0p-53 + 0x1.0p-53;   // (0, 1]
    const double u2 = (double)(((((uint64_t)r.z) << 32) | r.w) >> 11) * 0x1.0p-53;               // [0, 1)
    out[x] = sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
  }
}

// Y = p X + q Z (Z may be NULL)
__global__ void __launch_bounds__(256)
axpby_kernel(int64_t total, double p, const double* __restrict__ X, double q, const double* __restrict__ Z,
             double* __restrict__ Y) {
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x)
    Y[x] = Z ? fma(q, Z[x], p * X[x]) : p * X[x];
}

static unsigned grid_for(int64_t total) {
  const int64_t g = (total + 255) / 256;
  return (unsigned)(g < 4 * GCCB_NUM_SMS ? (g < 1 ? 1 : g) : 4 * GCCB_NUM_SMS);
}

static bool bad_csr(const int64_t* indptr, const int32_t* indices, int64_t n) {
  return !indptr || !indices || n <= 0;
}

static int64_t even(int64_t x) { return (x + 1) & ~(int64_t)1; }

}  // namespace gccb

using namespace gccb;

extern "C" int gccb_spmm_f64(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                             int32_t k, int64_t ld, double alpha, double sigma, const double* dr, const double* dc,
                             double beta, const double* X, double gamma, const double* Z, double* Y,
                             gccb_stream_t stream) {
  if (bad_csr(indptr, indices, n) || k <= 0 || ld < k || !X || !Y || X == Y) {
    set_last_error("gccb_spmm_f64: bad argument");
    return GCCB_ERR_BADARG;
  }
  SpmmArgs s = {indptr, indices, vals, n, k, ld, alpha, sigma, dr, dc, beta, X, gamma, Z, 0.0, nullptr, Y,
                0.0, nullptr, 0.0, nullptr};
  launch_spmm(s, stream);
  return check_launch("gccb_spmm_f64");
}

extern "C" size_t gccb_graphwave_workspace(int64_t n, int32_t bc) {
  if (n <= 0 || bc <= 0) return 0;
  return (size_t)(4 * n * even(bc) + n) * sizeof(double);
}

extern "C" int gccb_graphwave(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                              const double* cheb, int32_t order, const double* times, int32_t n_times, int32_t bc,
                              void* workspace, size_t workspace_bytes, double* chi, gccb_stream_t stream) {
  if (bad_csr(indptr, indices, n) || !cheb || order < 1 || order > GW_MAX_ORDER || !times || n_times < 1 ||
      n_times > GW_MAX_TIMES || bc < 1 || !workspace || !chi) {
    set_last_error("gccb_graphwave: bad argument");
    return GCCB_ERR_BADARG;
  }
  if (bc > n) bc = (int32_t)n;
  if (workspace_bytes < gccb_graphwave_workspace(n, bc)) {
    set_last_error("gccb_graphwave: workspace of %zu bytes, %zu needed", workspace_bytes,
                   gccb_graphwave_workspace(n, bc));
    return GCCB_ERR_CAPACITY;
  }
  const int64_t ld = even(bc);
  double* ta = static_cast<double*>(workspace);
  double* tb = ta + n * ld;
  double* h0 = tb + n * ld;
  double* h1 = h0 + n * ld;
  double* dinv = h1 + n * ld;
  GwTimes tt;
  for (int t = 0; t < GW_MAX_TIMES; ++t) tt.t[t] = t < n_times ? times[t] : 0.0;
  const double thr = 1e-4 * 1.0 / (double)n;
  const double* c_s0 = cheb;                 // scale 0: cheb[0 .. order], scale 1: cheb[order + 1 ..]
  const double* c_s1 = cheb + order + 1;
  launch_rowsum(indptr, vals, n, 1, dinv, stream);
  for (int64_t c0 = 0; c0 < n; c0 += bc) {
    const int cols = (int)(n - c0 < bc ? n - c0 : bc);
    GCCB_LAUNCH(gw_init_kernel, grid_for(n * ld), 256, 0, stream, n, c0, cols, ld, c_s0[0], c_s1[0], ta, h0, h1);
    // T_1 = (L - I) T_0 = -D^-1/2 A D^-1/2 T_0;  T_k = 2 (L - I) T_{k-1} - T_{k-2}, written over T_{k-2}
    SpmmArgs s = {indptr, indices, vals, n, cols, ld, -1.0, 0.0, dinv, dinv, 0.0, ta, 0.0, nullptr, 0.0, nullptr,
                  tb, c_s0[1], h0, c_s1[1], h1};
    launch_spmm(s, stream);
    double* prev = ta;
    double* cur = tb;
    for (int k = 2; k <= order; ++k) {
      s.alpha = -2.0;
      s.X = cur;
      s.gamma = -1.0;
      s.Z = prev;
      s.Y = prev;
      s.h0 = c_s0[k];
      s.h1 = c_s1[k];
      launch_spmm(s, stream);
      double* t = prev;
      prev = cur;
      cur = t;
    }
    dim3 grid((unsigned)((cols + 31) / 32), 2, (unsigned)((n_times + GW_TCHUNK - 1) / GW_TCHUNK));
    GCCB_LAUNCH(gw_chi_kernel, grid, dim3(32, 8), 0, stream, n, c0, cols, ld, h0, h1, tt, n_times, thr, chi);
  }
  return check_launch("gccb_graphwave");
}

extern "C" size_t gccb_prone_factor_workspace(int64_t n) {
  return n <= 0 ? 0 : (size_t)(2 * n + 1) * sizeof(double);
}

extern "C" int gccb_prone_factor(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                                 void* workspace, size_t workspace_bytes, double* F, double* FT,
                                 gccb_stream_t stream) {
  if (bad_csr(indptr, indices, n) || !workspace || !F || !FT) {
    set_last_error("gccb_prone_factor: bad argument");
    return GCCB_ERR_BADARG;
  }
  if (workspace_bytes < gccb_prone_factor_workspace(n)) {
    set_last_error("gccb_prone_factor: workspace of %zu bytes, %zu needed", workspace_bytes,
                   gccb_prone_factor_workspace(n));
    return GCCB_ERR_CAPACITY;
  }
  double* d = static_cast<double*>(workspace);
  double* p = d + n;
  double* psum = p + n;
  launch_rowsum(indptr, vals, n, 0, d, stream);
  GCCB_LAUNCH(prone_colpow_kernel, (unsigned)((n + 7) / 8), 256, 0, stream, indptr, indices, vals, n, d, p);
  GCCB_LAUNCH(sum_kernel, 1, 1024, 0, stream, p, n, psum);
  GCCB_LAUNCH(prone_values_kernel, (unsigned)((n + 7) / 8), 256, 0, stream, indptr, indices, vals, n, d, p, psum,
              F, FT);
  return check_launch("gccb_prone_factor");
}

extern "C" int gccb_gaussian_f64(double* out, int64_t rows, int32_t cols, uint64_t key, gccb_stream_t stream) {
  if (!out || rows <= 0 || cols <= 0) {
    set_last_error("gccb_gaussian_f64: bad argument");
    return GCCB_ERR_BADARG;
  }
  GCCB_LAUNCH(gaussian_kernel, grid_for(rows * cols), 256, 0, stream, out, rows, cols, key);
  return check_launch("gccb_gaussian_f64");
}

extern "C" size_t gccb_prone_propagate_workspace(int64_t n, int32_t k) {
  if (n <= 0 || k <= 0) return 0;
  return (size_t)(4 * n * (int64_t)k + n) * sizeof(double);
}

extern "C" int gccb_prone_propagate(const int64_t* indptr, const int32_t* indices, const double* vals, int64_t n,
                                    const double* a, int32_t k, double mu, const double* bessel, int32_t order,
                                    void* workspace, size_t workspace_bytes, double* mm, gccb_stream_t stream) {
  if (bad_csr(indptr, indices, n) || !a || k <= 0 || !bessel || order < 2 || !workspace || !mm || mm == a) {
    set_last_error("gccb_prone_propagate: bad argument");
    return GCCB_ERR_BADARG;
  }
  if (workspace_bytes < gccb_prone_propagate_workspace(n, k)) {
    set_last_error("gccb_prone_propagate: workspace of %zu bytes, %zu needed", workspace_bytes,
                   gccb_prone_propagate_workspace(n, k));
    return GCCB_ERR_CAPACITY;
  }
  const int64_t nk = n * (int64_t)k;
  double* t = static_cast<double*>(workspace);
  double* b0 = t + nk;
  double* b1 = b0 + nk;
  double* conv = b1 + nk;
  double* dr = conv + nk;
  launch_rowsum(indptr, vals, n, 2, dr, stream);                  // DA = (I + A) / rowsum
  GCCB_LAUNCH(axpby_kernel, grid_for(nk), 256, 0, stream, nk, bessel[0], a, 0.0, (const double*)nullptr, conv);
  // M x = (1 - mu) x - DA x,  with DA x = dr * (A x + x)
  SpmmArgs s = {indptr, indices, vals, n, k, k, -1.0, 1.0, dr, nullptr, 1.0 - mu, a, 0.0, nullptr, 0.0, nullptr,
                t, 0.0, nullptr, 0.0, nullptr};
  launch_spmm(s, stream);                                          // t = M a
  s.alpha = -0.5;
  s.beta = 0.5 * (1.0 - mu);
  s.X = t;
  s.gamma = -1.0;
  s.Z = a;
  s.Y = b1;
  s.h0 = -2.0 * bessel[1];
  s.acc0 = conv;
  launch_spmm(s, stream);                                          // Lx1 = 0.5 M t - a;  conv -= 2 I_1 Lx1
  const double* lx0 = a;
  double* lx1 = b1;
  for (int i = 2; i < order; ++i) {
    s.alpha = -1.0;
    s.beta = 1.0 - mu;
    s.X = lx1;
    s.gamma = 0.0;
    s.Z = nullptr;
    s.Y = t;
    s.acc0 = nullptr;
    launch_spmm(s, stream);                                        // t = M Lx1
    double* lx2 = lx1 == b1 ? b0 : b1;                             // overwrites Lx0 unless Lx0 is the input
    s.X = t;
    s.gamma = -2.0;
    s.Z = lx1;
    s.delta = -1.0;
    s.W = lx0;
    s.Y = lx2;
    s.h0 = (i % 2 == 0 ? 2.0 : -2.0) * bessel[i];
    s.acc0 = conv;
    launch_spmm(s, stream);                                        // Lx2 = M t - 2 Lx1 - Lx0;  conv +-= 2 I_i Lx2
    s.delta = 0.0;
    s.W = nullptr;
    lx0 = lx1;
    lx1 = lx2;
  }
  GCCB_LAUNCH(axpby_kernel, grid_for(nk), 256, 0, stream, nk, 1.0, a, -1.0, (const double*)conv, t);
  SpmmArgs f = {indptr, indices, vals, n, k, k, 1.0, 1.0, nullptr, nullptr, 0.0, t, 0.0, nullptr, 0.0, nullptr,
                mm, 0.0, nullptr, 0.0, nullptr};
  launch_spmm(f, stream);                                          // mm = (I + A)(a - conv)
  return check_launch("gccb_prone_propagate");
}
