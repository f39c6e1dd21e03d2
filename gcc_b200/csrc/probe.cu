// probe.cu -- linear-probe classification: exact one-vs-rest logistic regression over embedding rows, in float64.
//
// Definition (include/gccb200.h, DESIGN.md 4g).  Rows x_i (float32, used exactly in float64), labels Y [n][c] (0/1),
// one fold id per row.  Problem p = f * c + j (fold f, class j) is the binary problem on the training rows of f (the
// rows whose fold id is not f), targets t_i = Y[i][j]:
//   minimise  1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w.x_i + b))),  s_i = 2 t_i - 1, the intercept b not penalised.
// A problem whose training rows all have the same target is a constant predictor (decision value +inf or -inf).
// Every other problem is solved by damped Newton from w = 0, b = 0: the exact gradient and Hessian
// [X 1]^T diag(C p(1-p)) [X 1] + diag(I_d, 0), a Cholesky solve, and backtracking over alpha = 2^-m, m = 0..15, on
// the Armijo condition.  It stops when |grad|_inf <= 1e-10 max(1, |grad at 0|_inf).
//
// z_i = the sequential fma chain of w_j x_ij over j = 0 .. d-1 from +0, plus b: the same chain in every kernel.
//
// Kernels (per Newton iteration, over the active problems of one launch chunk):
//   probe_gram_kernel    grid (Gram column chunks, problem groups of PROBE_PB, row splits).  A CTA stages PROBE_R
//                        rows of [X 1] in shared memory as float64, computes z and the row terms of its PROBE_PB
//                        problems, and accumulates the upper-triangle 8 x 8 blocks of sum_i s_i [x_i 1][x_i 1]^T on
//                        the float64 tensor cores (mma.sync m8n8k4): each warp owns a "quad", four blocks of one
//                        block row, and reuses one A fragment across them.  Chunk 0 also accumulates the gradient
//                        sums sum_i r_i [x_i 1] and the loss.  Partials go to [split][problem].  A Newton
//                        iteration runs chunk 0 first; the problems its gradient shows converged skip the other chunks.
//   probe_solve_kernel   one CTA per problem: merges the splits in split order; tests convergence (after chunk 0);
//                        factors the Hessian (Cholesky, in shared memory for d <= 128, in global memory for d = 256)
//                        and writes the Newton step.
//   probe_ls_kernel      grid (problem groups, row splits): the loss at a window of PROBE_LS_W consecutive step
//                        lengths, partials per split.
//   probe_update_kernel  one thread per problem: the first step length of the window meeting the Armijo condition.
//                        If none does, the next pass evaluates the next window along the same Newton step (the
//                        problem skips the Gram and solve kernels), so the accepted length is the first of all 16,
//                        while a pass usually evaluates only four.
// and once per call: probe_init_kernel (the non-finite check, fold and class counts), probe_setup_kernel (constant
// predictors), probe_active_kernel (the ordered list of active problems) and probe_score_kernel (decision values,
// top-k per test row, tp/fp/fn per fold).
// Every sum has a fixed order that depends on n, d and the problem alone: the row splits are chosen from n, rows are
// taken in order within a split, splits are merged in order, and no problem's arithmetic depends on which others share
// its launch.
#include "common.cuh"

#include <math.h>

namespace gccb {

#define PROBE_MAXDIM 256
#define PROBE_MAXC 1024
#define PROBE_MAXFOLDS 64
#define PROBE_R 32                   // rows per Gram tile (8 k-steps of the m8n8k4 mma)
#define PROBE_PB 4                   // problems per CTA
#define PROBE_NT 256
#define PROBE_QUADS (PROBE_NT / 32)  // Gram quads per CTA: one per warp
#define PROBE_LS_R 64                // rows per line-search tile: PROBE_LS_R * PROBE_PB = PROBE_NT row terms
#define PROBE_NA 16                  // step lengths 2^-m, m = 0 .. PROBE_NA-1
#define PROBE_LS_W 4                 // step lengths evaluated per pass
#define PROBE_LS_LD (PROBE_PB * PROBE_LS_W + 1)   // odd pitch (in doubles) of the line-search loss tile
#define PROBE_SPLIT_ROWS 65536       // rows per split: S = ceil(n / PROBE_SPLIT_ROWS), at most PROBE_MAX_SPLITS
#define PROBE_MAX_SPLITS 64
#define PROBE_SMEM_MAXDIM 128        // the Cholesky runs in shared memory up to this width
#define PROBE_TOL 1e-10
#define PROBE_ARMIJO 1e-4
#define PROBE_ARMIJO_SLACK 1e-12     // relative: absorbs the rounding of the loss itself near the optimum

// ---- per-row terms -------------------------------------------------------------------------------------------------
template <class T>
__device__ __forceinline__ double probe_z(const double* __restrict__ w, const T* __restrict__ x, int d) {
  double z = 0.0;
  for (int j = 0; j < d; ++j) z = fma(w[j], (double)x[j], z);
  return z + w[d];
}

// log(1 + exp(-m)) for margin m = s z
__device__ __forceinline__ double probe_softplus_neg(double m) {
  return m > 0.0 ? log1p(exp(-m)) : -m + log1p(exp(m));
}

// curvature q = sigmoid(z) (1 - sigmoid(z))
__device__ __forceinline__ double probe_curv(double z) {
  const double e = exp(-fabs(z));
  return e / ((1.0 + e) * (1.0 + e));
}

// residual r = sigmoid(z) - t, curvature q = sigmoid(z) (1 - sigmoid(z)), loss log(1 + exp(-s z))
__device__ __forceinline__ void probe_terms(double z, int t, double* r, double* q, double* loss) {
  *r = t ? -1.0 / (1.0 + exp(z)) : 1.0 / (1.0 + exp(-z));
  *q = probe_curv(z);
  *loss = probe_softplus_neg(t ? z : -z);
}

// ---- the float64 tensor-core mma: d[0..1] += A (8x4, row) * B (4x8, col) ---------------------------------------------
#ifdef GCCB_EMU
static inline void probe_dmma(double* d, double a, double b) {
  static double buf[32][2][32];
  const int w = emu::warp(), lane = emu::lane(), gid = lane >> 2, tig = lane & 3;
  buf[w][0][lane] = a;
  buf[w][1][lane] = b;
  __syncwarp();
  for (int i = 0; i < 2; ++i)
    for (int k = 0; k < 4; ++k) d[i] = fma(buf[w][0][gid * 4 + k], buf[w][1][(tig * 2 + i) * 4 + k], d[i]);
  __syncwarp();
}
#else
__device__ __forceinline__ void probe_dmma(double* d, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}
#endif

// ---- shapes --------------------------------------------------------------------------------------------------------
struct ProbeShape {
  int d1, D, Dp, NB, T, quads, chunks, S;
};

// an odd pitch (in 4-byte words) for tiles read one row per lane: the lanes of a warp hit 32 distinct banks
__host__ __device__ inline int probe_odd_pitch(int d) { return d | 1; }

__host__ __device__ inline int probe_quads(int NB) {
  int q = 0;
  for (int bi = 0; bi < NB; ++bi) q += (NB - bi + 3) / 4;
  return q;
}
// index of block (bi, bj), bi <= bj, in the row-major upper triangle of NB x NB blocks
__host__ __device__ inline int probe_block_id(int bi, int bj, int NB) { return bi * NB - bi * (bi - 1) / 2 + (bj - bi); }

static ProbeShape probe_shape(int64_t n, int d) {
  ProbeShape s;
  s.d1 = d + 1;
  s.D = (s.d1 + 7) & ~7;
  s.Dp = s.D + 4;                                                  // fragment reads of 4 rows x 8 columns hit distinct banks
  s.NB = s.D / 8;
  s.T = s.NB * (s.NB + 1) / 2;
  s.quads = probe_quads(s.NB);
  s.chunks = (s.quads + PROBE_QUADS - 1) / PROBE_QUADS;
  int64_t S = (n + PROBE_SPLIT_ROWS - 1) / PROBE_SPLIT_ROWS;
  s.S = (int)(S < 1 ? 1 : (S > PROBE_MAX_SPLITS ? PROBE_MAX_SPLITS : S));
  return s;
}

enum { PROBE_ACTIVE = GCCB_PROBE_ACTIVE, PROBE_CONVERGED = GCCB_PROBE_CONVERGED, PROBE_CONST_POS = GCCB_PROBE_CONST_POS,
       PROBE_CONST_NEG = GCCB_PROBE_CONST_NEG, PROBE_NOCONV = GCCB_PROBE_NOCONV, PROBE_LS_FAIL = GCCB_PROBE_LS_FAIL,
       PROBE_NOT_PD = GCCB_PROBE_NOT_PD };

// ---- once per call ---------------------------------------------------------------------------------------------------
// one thread per row: the non-finite check, test rows per fold, positives per (fold, class) and per class
__global__ void __launch_bounds__(256)
probe_init_kernel(const float* __restrict__ x, int64_t n, int d, const uint8_t* __restrict__ y, int c,
                  const int32_t* __restrict__ fold, int folds, int32_t* __restrict__ flags,
                  unsigned long long* __restrict__ pos, unsigned long long* __restrict__ cnt,
                  unsigned long long* __restrict__ tot) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool bad = false;
  for (int j = 0; j < d; ++j) bad |= (__float_as_uint(x[i * d + j]) & 0x7f800000u) == 0x7f800000u;
  if (bad) atomicOr(flags, GCCB_FLAG_NONFINITE);
  const int f = fold[i];
  const bool in_fold = f >= 0 && f < folds;
  if (in_fold) atomicAdd(&cnt[f], 1ull);
  for (int j = 0; j < c; ++j)
    if (y[i * c + j]) {
      atomicAdd(&tot[j], 1ull);
      if (in_fold) atomicAdd(&pos[(size_t)f * c + j], 1ull);
    }
}

// one thread per problem: constant predictors, w = 0
__global__ void __launch_bounds__(256)
probe_setup_kernel(int P, int c, int64_t n, int d1, const unsigned long long* __restrict__ pos,
                   const unsigned long long* __restrict__ cnt, const unsigned long long* __restrict__ tot,
                   int32_t* __restrict__ status, int32_t* __restrict__ iters, double* __restrict__ w,
                   double* __restrict__ gnorm, int32_t* __restrict__ lsm) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int f = p / c, j = p % c;
  const unsigned long long ntrain = (unsigned long long)n - cnt[f], npos = tot[j] - pos[p];
  status[p] = npos == 0 ? PROBE_CONST_NEG : (npos == ntrain ? PROBE_CONST_POS : PROBE_ACTIVE);
  iters[p] = 0;
  lsm[p] = 0;
  gnorm[p] = 0.0;
  for (int k = 0; k < d1; ++k) w[(size_t)p * d1 + k] = 0.0;
}

// one CTA of 1024 threads: active[0 .. counts[0]) = the active problems, ascending; newton[0 .. counts[1]) = those
// of them that start a Newton iteration (not in the middle of a line search).  mark_noconv: the iteration limit was
// reached, so the active problems become PROBE_NOCONV and raise GCCB_FLAG_PROBE_NOCONV instead.
__global__ void __launch_bounds__(1024)
probe_active_kernel(int P, int32_t* __restrict__ status, const int32_t* __restrict__ lsm, int32_t* __restrict__ active,
                    int32_t* __restrict__ newton, int32_t* __restrict__ counts, int mark_noconv,
                    int32_t* __restrict__ flags) {
  __shared__ int scratch[33];
  int base = 0, nbase = 0;
  for (int lo = 0; lo < P; lo += 1024) {
    const int p = lo + threadIdx.x;
    int a = p < P && status[p] == PROBE_ACTIVE;
    if (a && mark_noconv) {
      status[p] = PROBE_NOCONV;
      atomicOr(flags, GCCB_FLAG_PROBE_NOCONV);
      a = 0;
    }
    const int nw = a && lsm[p] == 0;
    int total, ntotal;
    const int at = block_scan_excl(a, scratch, &total);
    if (a) active[base + at] = p;
    base += total;
    const int nat = block_scan_excl(nw, scratch, &ntotal);
    if (nw) newton[nbase + nat] = p;
    nbase += ntotal;
  }
  if (threadIdx.x == 0) {
    counts[0] = base;
    counts[1] = nbase;
  }
}

// ---- per Newton iteration --------------------------------------------------------------------------------------------
// grid (chunks - chunk0, ceil(nb / PROBE_PB), S), block PROBE_NT: Gram column chunks chunk0 .. chunks-1.  plist [nb]:
// the problems of this launch; those whose status is no longer PROBE_ACTIVE are skipped (a CTA left with none returns).
// hpart [S][nb][T][64], gpart [S][nb][d1], lpart [S][nb].
__global__ void __launch_bounds__(PROBE_NT, 2)
probe_gram_kernel(const float* __restrict__ x, int64_t n, int d, const uint8_t* __restrict__ y, int c,
                  const int32_t* __restrict__ fold, const double* __restrict__ w, const int32_t* __restrict__ plist,
                  int nb, const int32_t* __restrict__ status, int chunk0, int D, int Dp, int NB, int T, int S,
                  double* __restrict__ hpart, double* __restrict__ gpart, double* __restrict__ lpart) {
  GCCB_DYN_SMEM(double, smem);
  const int d1 = d + 1;
  double* xs = smem;                                  // [PROBE_R][Dp]
  double* wsm = xs + PROBE_R * Dp;                    // [PB][D]
  double* ss = wsm + PROBE_PB * D;                    // [PB][R] curvature weights
  double* rr = ss + PROBE_PB * PROBE_R;               // [PB][R] residuals
  double* ll = rr + PROBE_PB * PROBE_R;               // [PB][R] losses
  double* gacc = ll + PROBE_PB * PROBE_R;             // [PB][D] gradient sums (chunk 0)
  double* lacc = gacc + PROBE_PB * D;                 // [PB] loss sums (chunk 0)
  const int dz = probe_odd_pitch(d);
  float* xz = reinterpret_cast<float*>(lacc + PROBE_PB);  // [PROBE_R][dz] the tile's x again, for the z chains
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
  const int chunk = chunk0 + blockIdx.x, q0 = blockIdx.y * PROBE_PB, split = blockIdx.z;
  const bool grad = chunk == 0;
  const int64_t lo = n * split / S, hi = n * (split + 1) / S;

  int prob[PROBE_PB];
  bool any = false;
#pragma unroll
  for (int qq = 0; qq < PROBE_PB; ++qq) {
    const int p = q0 + qq < nb ? plist[q0 + qq] : -1;
    prob[qq] = (p >= 0 && status[p] == PROBE_ACTIVE) ? p : -1;
    any |= prob[qq] >= 0;
  }
  if (!any) return;                                   // uniform over the CTA, before any barrier
  for (int e = tid; e < PROBE_PB * D; e += PROBE_NT) {
    const int qq = e / D, j = e % D;
    wsm[e] = (prob[qq] >= 0 && j < d1) ? w[(size_t)prob[qq] * d1 + j] : 0.0;
    gacc[e] = 0.0;
  }
  if (tid < PROBE_PB) lacc[tid] = 0.0;

  // this warp's quad: blocks (bi, bj0 .. bj0 + 3) of the upper triangle
  int bi = -1, bj0 = 0;
  {
    int qd = chunk * PROBE_QUADS + warp;
    for (int b = 0; b < NB && bi < 0; ++b) {
      const int nq = (NB - b + 3) / 4;
      if (qd < nq) {
        bi = b;
        bj0 = b + 4 * qd;
      } else {
        qd -= nq;
      }
    }
  }
  double acc[PROBE_PB][4][2];
#pragma unroll
  for (int qq = 0; qq < PROBE_PB; ++qq)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[qq][b][0] = acc[qq][b][1] = 0.0;

  for (int64_t r0 = lo; r0 < hi; r0 += PROBE_R) {
    __syncthreads();                                  // the previous tile is consumed
    for (int e = tid; e < PROBE_R * D; e += PROBE_NT) {
      const int r = e / D, j = e % D;
      const int64_t i = r0 + r;
      double v = 0.0;
      if (i < hi) v = j < d ? (double)x[i * d + j] : (j == d ? 1.0 : 0.0);
      xs[r * Dp + j] = v;
      if (j < d) xz[r * dz + j] = (float)v;           // exact: v is a float
    }
    __syncthreads();
    if (tid < PROBE_R * PROBE_PB) {
      const int qq = tid / PROBE_R, r = tid % PROBE_R;
      const int64_t i = r0 + r;
      double sv = 0.0, rv = 0.0, lv = 0.0;
      const int p = prob[qq];
      if (p >= 0 && i < hi && fold[i] != p / c) {
        const double z = probe_z(wsm + qq * D, xz + r * dz, d);
        if (grad) probe_terms(z, y[i * c + p % c] != 0, &rv, &sv, &lv);
        else sv = probe_curv(z);                      // the other chunks need the curvature alone
      }
      ss[tid] = sv;
      rr[tid] = rv;
      ll[tid] = lv;
    }
    __syncthreads();
    if (bi >= 0) {
#pragma unroll
      for (int kk = 0; kk < PROBE_R / 4; ++kk) {
        const double* xr = xs + (kk * 4 + tig) * Dp;
        const double xa = xr[bi * 8 + gid];
        double bf[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) bf[b] = bj0 + b < NB ? xr[(bj0 + b) * 8 + gid] : 0.0;
#pragma unroll
        for (int qq = 0; qq < PROBE_PB; ++qq) {
          const double a = ss[qq * PROBE_R + kk * 4 + tig] * xa;
#pragma unroll
          for (int b = 0; b < 4; ++b)
            if (bj0 + b < NB) probe_dmma(acc[qq][b], a, bf[b]);
        }
      }
    }
    if (grad) {
      for (int e = tid; e < PROBE_PB * d1; e += PROBE_NT) {
        const int qq = e / d1, j = e % d1;
        double g = gacc[qq * D + j];
        for (int r = 0; r < PROBE_R; ++r) g = fma(rr[qq * PROBE_R + r], xs[r * Dp + j], g);
        gacc[qq * D + j] = g;
      }
      if (tid < PROBE_PB) {
        double l = lacc[tid];
        for (int r = 0; r < PROBE_R; ++r) l += ll[tid * PROBE_R + r];
        lacc[tid] = l;
      }
    }
  }

  if (bi >= 0) {
#pragma unroll
    for (int qq = 0; qq < PROBE_PB; ++qq) {
      if (prob[qq] < 0) continue;
      double* hp = hpart + ((size_t)split * nb + q0 + qq) * T * 64;
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (bj0 + b < NB) {
          double* blk = hp + (size_t)probe_block_id(bi, bj0 + b, NB) * 64 + gid * 8 + tig * 2;
          blk[0] = acc[qq][b][0];
          blk[1] = acc[qq][b][1];
        }
    }
  }
  if (grad) {
    __syncthreads();
    for (int e = tid; e < PROBE_PB * d1; e += PROBE_NT) {
      const int qq = e / d1, j = e % d1;
      if (prob[qq] >= 0) gpart[((size_t)split * nb + q0 + qq) * d1 + j] = gacc[qq * D + j];
    }
    if (tid < PROBE_PB && prob[tid] >= 0) lpart[(size_t)split * nb + q0 + tid] = lacc[tid];
  }
}

// grid nb, block PROBE_NT; dynamic shared memory probe_solve_smem(d): the matrix in shared memory when
// d <= PROBE_SMEM_MAXDIM, else at hglob + q * d1 * d1.  mode 2: the convergence test alone, from the gradient sums of
// Gram chunk 0 (a problem that has converged then skips the other chunks).  mode 0: the Newton step, f and slope of
// the problems still active.  mode 1: the system at the given weights, written out: g_out [P][d1], h_out [P][d1][d1]
// (before factorisation), step.  A non-positive pivot sets PROBE_NOT_PD and, given flags, GCCB_FLAG_PROBE_NOCONV.
__global__ void __launch_bounds__(PROBE_NT)
probe_solve_kernel(const int32_t* __restrict__ plist, int nb, int d, int D, int NB, int T, int S, double C,
                   const double* __restrict__ w, const double* __restrict__ gpart, const double* __restrict__ lpart,
                   const double* __restrict__ hpart, double* __restrict__ hglob, double* __restrict__ step,
                   int32_t* __restrict__ status, double* __restrict__ g0, double* __restrict__ gnorm,
                   double* __restrict__ fval, double* __restrict__ slope, int iter, int mode,
                   double* __restrict__ g_out, double* __restrict__ h_out, int32_t* __restrict__ flags) {
  GCCB_DYN_SMEM(double, smem);
  const int d1 = d + 1, tid = threadIdx.x, q = blockIdx.x, p = plist[q];
  if (mode == 0 && status[p] != PROBE_ACTIVE) return;   // converged at the test: uniform, before any barrier
  double* G = smem;                                   // [D] full gradient
  double* red = G + D;                                // [max(D, PROBE_NT)] reduction scratch, then the solution
  double* M = d <= PROBE_SMEM_MAXDIM ? red + (D > PROBE_NT ? D : PROBE_NT) : hglob + (size_t)q * d1 * d1;
  __shared__ int s_stop;
  const double* wp = w + (size_t)p * d1;

  for (int j = tid; j < d1; j += PROBE_NT) {
    double g = 0.0;
    for (int s = 0; s < S; ++s) g += gpart[((size_t)s * nb + q) * d1 + j];
    G[j] = j < d ? fma(C, g, wp[j]) : C * g;
  }
  if (tid == 0) {
    double l = 0.0, nrm = 0.0;
    for (int s = 0; s < S; ++s) l += lpart[(size_t)s * nb + q];
    for (int j = 0; j < d; ++j) nrm = fma(wp[j], wp[j], nrm);
    red[0] = 0.5 * nrm + C * l;
  }
  __syncthreads();
  const double f = red[0];
  __syncthreads();
  double m = 0.0;
  for (int j = tid; j < d1; j += PROBE_NT) m = fmax(m, fabs(G[j]));
  red[tid] = m;
  __syncthreads();
  if (tid == 0) {
    double mx = 0.0;
    for (int t = 0; t < PROBE_NT; ++t) mx = fmax(mx, red[t]);
    if (mode == 2) {
      if (iter == 0) g0[p] = mx;
      gnorm[p] = mx;
      if (mx <= PROBE_TOL * fmax(1.0, g0[p])) status[p] = PROBE_CONVERGED;
    }
    fval[p] = f;
  }
  if (mode == 2) return;

  // the Hessian: C * (merged upper-triangle blocks) + diag(I_d, 0), both triangles
  for (int e = tid; e < d1 * d1; e += PROBE_NT) {
    const int a = e / d1, b = e % d1;
    if (a > b) continue;
    const int blk = probe_block_id(a >> 3, b >> 3, NB), off = (a & 7) * 8 + (b & 7);
    double h = 0.0;
    for (int s = 0; s < S; ++s) h += hpart[(((size_t)s * nb + q) * T + blk) * 64 + off];
    h *= C;
    if (a == b && a < d) h += 1.0;
    M[a * d1 + b] = h;
    M[b * d1 + a] = h;
  }
  __syncthreads();
  if (mode == 1) {
    for (int e = tid; e < d1 * d1; e += PROBE_NT) h_out[(size_t)p * d1 * d1 + e] = M[e];
    for (int j = tid; j < d1; j += PROBE_NT) g_out[(size_t)p * d1 + j] = G[j];
  }
  // right-looking Cholesky, lower triangle in place: M = L L^T
  for (int k = 0; k < d1; ++k) {
    if (tid == 0) {
      const double piv = M[k * d1 + k];
      s_stop = !(piv > 0.0);
      M[k * d1 + k] = s_stop ? 1.0 : sqrt(piv);
    }
    __syncthreads();
    if (s_stop) {
      if (tid == 0) {
        status[p] = PROBE_NOT_PD;
        if (flags) atomicOr(flags, GCCB_FLAG_PROBE_NOCONV);
      }
      return;
    }
    const double lkk = M[k * d1 + k];
    for (int i = k + 1 + tid; i < d1; i += PROBE_NT) M[i * d1 + k] /= lkk;
    __syncthreads();
    const int rem = d1 - k - 1;
    for (int e = tid; e < rem * rem; e += PROBE_NT) {
      const int i = k + 1 + e / rem, j = k + 1 + e % rem;
      if (j <= i) M[i * d1 + j] = fma(-M[i * d1 + k], M[j * d1 + k], M[i * d1 + j]);
    }
    __syncthreads();
  }
  // L y = -G, then L^T delta = y, column by column, in red
  for (int j = tid; j < d1; j += PROBE_NT) red[j] = -G[j];
  __syncthreads();
  for (int k = 0; k < d1; ++k) {
    if (tid == 0) red[k] /= M[k * d1 + k];
    __syncthreads();
    for (int i = k + 1 + tid; i < d1; i += PROBE_NT) red[i] = fma(-M[i * d1 + k], red[k], red[i]);
    __syncthreads();
  }
  for (int k = d1 - 1; k >= 0; --k) {
    if (tid == 0) red[k] /= M[k * d1 + k];
    __syncthreads();
    for (int i = tid; i < k; i += PROBE_NT) red[i] = fma(-M[k * d1 + i], red[k], red[i]);
    __syncthreads();
  }
  for (int j = tid; j < d1; j += PROBE_NT) step[(size_t)p * d1 + j] = red[j];
  if (tid == 0) {
    double sl = 0.0;
    for (int j = 0; j < d1; ++j) sl = fma(G[j], red[j], sl);
    slope[p] = sl;
  }
}

// grid (ceil(nb / PROBE_PB), S), block PROBE_NT, dynamic shared memory probe_ls_smem(d).  lspart [S][nb][PROBE_LS_W]:
// the loss sums at w + 2^-m step, m = lsm[p] + 0 .. PROBE_LS_W-1, over the split's training rows.
__global__ void __launch_bounds__(PROBE_NT)
probe_ls_kernel(const float* __restrict__ x, int64_t n, int d, const uint8_t* __restrict__ y, int c,
                const int32_t* __restrict__ fold, const double* __restrict__ w, const double* __restrict__ step,
                const int32_t* __restrict__ plist, int nb, const int32_t* __restrict__ status,
                const int32_t* __restrict__ lsm, int S, double* __restrict__ lspart) {
  GCCB_DYN_SMEM(double, smem);
  const int d1 = d + 1, tid = threadIdx.x;
  double* wsm = smem;                                    // [PB][d1]
  double* dsm = wsm + PROBE_PB * d1;                     // [PB][d1]
  double* lv = dsm + PROBE_PB * d1;                      // [LS_R][LS_LD]: row r's losses at (problem, length)
  float* xs = reinterpret_cast<float*>(lv + PROBE_LS_R * PROBE_LS_LD);   // [LS_R][xp]
  const int xp = probe_odd_pitch(d);
  const int q0 = blockIdx.x * PROBE_PB, split = blockIdx.y;
  const int64_t lo = n * split / S, hi = n * (split + 1) / S;
  int prob[PROBE_PB], m0[PROBE_PB];
#pragma unroll
  for (int qq = 0; qq < PROBE_PB; ++qq) {
    const int p = q0 + qq < nb ? plist[q0 + qq] : -1;
    prob[qq] = (p >= 0 && status[p] == PROBE_ACTIVE) ? p : -1;
    m0[qq] = prob[qq] >= 0 ? lsm[prob[qq]] : 0;
  }
  for (int e = tid; e < PROBE_PB * d1; e += PROBE_NT) {
    const int qq = e / d1, j = e % d1;
    wsm[e] = prob[qq] >= 0 ? w[(size_t)prob[qq] * d1 + j] : 0.0;
    dsm[e] = prob[qq] >= 0 ? step[(size_t)prob[qq] * d1 + j] : 0.0;
  }
  const int mq = tid / PROBE_LS_W, mm = tid % PROBE_LS_W;   // the (problem, step length) sum this thread owns
  double sum = 0.0;
  for (int64_t r0 = lo; r0 < hi; r0 += PROBE_LS_R) {
    __syncthreads();
    for (int e = tid; e < PROBE_LS_R * d; e += PROBE_NT) {
      const int64_t i = r0 + e / d;
      xs[(e / d) * xp + e % d] = i < hi ? x[i * d + e % d] : 0.f;
    }
    __syncthreads();
    {
      const int qq = tid / PROBE_LS_R, r = tid % PROBE_LS_R;
      const int64_t i = r0 + r;
      const int p = prob[qq];
      const bool on = p >= 0 && i < hi && fold[i] != p / c;
      double z = 0.0, dz = 0.0;
      int t = 0;
      if (on) {
        z = probe_z(wsm + qq * d1, xs + r * xp, d);
        dz = probe_z(dsm + qq * d1, xs + r * xp, d);
        t = y[i * c + p % c] != 0;
      }
      double a = 1.0;
      for (int m = 0; m < m0[qq]; ++m) a *= 0.5;                 // 2^-m0, exactly
      for (int m = 0; m < PROBE_LS_W; ++m, a *= 0.5) {
        const double zm = fma(a, dz, z);
        lv[r * PROBE_LS_LD + qq * PROBE_LS_W + m] = on ? probe_softplus_neg(t ? zm : -zm) : 0.0;
      }
    }
    __syncthreads();
    if (mq < PROBE_PB)
      for (int r = 0; r < PROBE_LS_R; ++r) sum += lv[r * PROBE_LS_LD + tid];
  }
  if (mq < PROBE_PB && q0 + mq < nb) lspart[((size_t)split * nb + q0 + mq) * PROBE_LS_W + mm] = sum;
}

// one thread per problem of the launch
__global__ void __launch_bounds__(128)
probe_update_kernel(const int32_t* __restrict__ plist, int nb, int d, int S, double C, double* __restrict__ w,
                    const double* __restrict__ step, const double* __restrict__ lspart, int32_t* __restrict__ status,
                    const double* __restrict__ fval, const double* __restrict__ slope, int32_t* __restrict__ iters,
                    int32_t* __restrict__ lsm, int32_t* __restrict__ flags) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nb) return;
  const int p = plist[q], d1 = d + 1;
  if (status[p] != PROBE_ACTIVE) return;
  double* wp = w + (size_t)p * d1;
  const double* dp = step + (size_t)p * d1;
  const double f = fval[p], sl = slope[p];
  const int m0 = lsm[p];
  double a = 1.0;
  for (int m = 0; m < m0; ++m) a *= 0.5;
  for (int m = 0; m < PROBE_LS_W; ++m, a *= 0.5) {
    double l = 0.0, nrm = 0.0;
    for (int s = 0; s < S; ++s) l += lspart[((size_t)s * nb + q) * PROBE_LS_W + m];
    for (int j = 0; j < d; ++j) {
      const double v = fma(a, dp[j], wp[j]);
      nrm = fma(v, v, nrm);
    }
    const double fm = 0.5 * nrm + C * l;
    if (fm <= f + PROBE_ARMIJO * a * sl + PROBE_ARMIJO_SLACK * fabs(f)) {
      for (int j = 0; j < d1; ++j) wp[j] = fma(a, dp[j], wp[j]);
      iters[p] += 1;
      lsm[p] = 0;
      return;
    }
  }
  if (m0 + PROBE_LS_W < PROBE_NA) lsm[p] = m0 + PROBE_LS_W;      // the next window, along the same step
  else {
    status[p] = PROBE_LS_FAIL;
    atomicOr(flags, GCCB_FLAG_PROBE_NOCONV);
  }
}

// one thread per row: decision values of its fold's problems, the top-k (k = its label count) by (z descending,
// class ascending), and tp / fp / fn into counts [folds][3]
__global__ void __launch_bounds__(256)
probe_score_kernel(const float* __restrict__ x, int64_t n, int d, const uint8_t* __restrict__ y, int c,
                   const int32_t* __restrict__ fold, int folds, const double* __restrict__ w,
                   const int32_t* __restrict__ status, double* __restrict__ z, unsigned long long* __restrict__ counts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = fold[i], d1 = d + 1;
  double* zi = z + i * c;
  if (f < 0 || f >= folds) {
    for (int j = 0; j < c; ++j) zi[j] = NAN;
    return;
  }
  int k = 0;
  for (int j = 0; j < c; ++j) {
    const int p = f * c + j, st = status[p];
    zi[j] = st == PROBE_CONST_POS ? INFINITY
          : st == PROBE_CONST_NEG ? -INFINITY : probe_z(w + (size_t)p * d1, x + i * d, d);
    k += y[i * c + j] != 0;
  }
  int prev = -1, tp = 0;
  for (int m = 0; m < k; ++m) {
    int best = -1;
    for (int j = 0; j < c; ++j) {
      const bool after = prev < 0 || zi[j] < zi[prev] || (zi[j] == zi[prev] && j > prev);
      if (after && (best < 0 || zi[j] > zi[best])) best = j;    // ties keep the lower class
    }
    tp += y[i * c + best] != 0;
    prev = best;
  }
  atomicAdd(&counts[f * 3 + 0], (unsigned long long)tp);
  atomicAdd(&counts[f * 3 + 1], (unsigned long long)(k - tp));
  atomicAdd(&counts[f * 3 + 2], (unsigned long long)(k - tp));
}

// ---- host side -------------------------------------------------------------------------------------------------------
static size_t probe_align(size_t b) { return (b + 255) & ~(size_t)255; }

struct ProbeWs {
  int32_t *active, *newton, *counts, *lsm;
  unsigned long long *pos, *cnt, *tot;
  double *g0, *fval, *slope, *step, *gpart, *lpart, *lspart, *hpart, *hglob;
  size_t bytes;
};

static int probe_batch(int P, int batch) { return batch <= 0 || batch > P ? P : batch; }

static ProbeWs probe_layout(char* base, int64_t n, int d, int c, int folds, int batch) {
  const ProbeShape sh = probe_shape(n, d);
  const int P = folds * c, B = probe_batch(P, batch), d1 = sh.d1;
  ProbeWs L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += probe_align(bytes);
    return p;
  };
  L.active = (int32_t*)take((size_t)P * 4);
  L.newton = (int32_t*)take((size_t)P * 4);
  L.lsm = (int32_t*)take((size_t)P * 4);
  L.counts = (int32_t*)take(8);
  L.pos = (unsigned long long*)take((size_t)P * 8);
  L.cnt = (unsigned long long*)take((size_t)folds * 8);
  L.tot = (unsigned long long*)take((size_t)c * 8);
  L.g0 = (double*)take((size_t)P * 8);
  L.fval = (double*)take((size_t)P * 8);
  L.slope = (double*)take((size_t)P * 8);
  L.step = (double*)take((size_t)P * d1 * 8);
  L.gpart = (double*)take((size_t)sh.S * B * d1 * 8);
  L.lpart = (double*)take((size_t)sh.S * B * 8);
  L.lspart = (double*)take((size_t)sh.S * B * PROBE_LS_W * 8);
  L.hpart = (double*)take((size_t)sh.S * B * sh.T * 64 * 8);
  L.hglob = d > PROBE_SMEM_MAXDIM ? (double*)take((size_t)B * d1 * d1 * 8) : nullptr;
  L.bytes = off;
  return L;
}

static bool probe_shape_ok(int64_t n, int d, int c, int folds) {
  return n >= 1 && n <= 0x7fffffffll && d >= 1 && d <= PROBE_MAXDIM && c >= 1 && c <= PROBE_MAXC && folds >= 1 &&
         folds <= PROBE_MAXFOLDS;
}

static size_t probe_gram_smem(const ProbeShape& sh) {
  return ((size_t)PROBE_R * sh.Dp + 2 * PROBE_PB * sh.D + 3 * PROBE_PB * PROBE_R + PROBE_PB) * 8 +
         (size_t)PROBE_R * probe_odd_pitch(sh.d1 - 1) * 4;
}
static size_t probe_solve_smem(int d) {
  const size_t D = (size_t)((d + 1 + 7) & ~7);
  const size_t red = D > PROBE_NT ? D : PROBE_NT;
  return (D + red + (d <= PROBE_SMEM_MAXDIM ? (size_t)(d + 1) * (d + 1) : 0)) * 8;
}
static size_t probe_ls_smem(int d) {
  return ((size_t)2 * PROBE_PB * (d + 1) + PROBE_LS_R * PROBE_LS_LD) * 8 + (size_t)PROBE_LS_R * probe_odd_pitch(d) * 4;
}

// k (<= 2) int32 from the device, after the work queued on `stream`: one copy and one synchronisation
static void probe_read_i32(const int32_t* dev, int k, int32_t* out, gccb_stream_t stream) {
#ifdef GCCB_EMU
  (void)stream;
  for (int i = 0; i < k; ++i) out[i] = dev[i];
#else
  cudaMemcpyAsync(out, dev, (size_t)k * 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);
#endif
}

// The Gram and solve kernels over plist[0 .. nb).  newton: a Newton iteration -- Gram chunk 0 (the gradient), the
// convergence test, the other Gram chunks for the problems still active, their steps.  Otherwise the system export of
// gccb_probe_system: every chunk, then the solve in mode 1.
static void probe_system(const ProbeShape& sh, const float* x, int64_t n, int d, const uint8_t* y, int c,
                         const int32_t* fold, double C, const double* w, const int32_t* plist, int nb,
                         const ProbeWs& L, int32_t* status, double* gnorm, int iter, bool newton, double* g_out,
                         double* h_out, int32_t* flags, gccb_stream_t stream) {
  const size_t gsm = probe_gram_smem(sh), ssm = probe_solve_smem(d);
  ensure_dyn_smem(probe_gram_kernel, gsm);
  ensure_dyn_smem(probe_solve_kernel, ssm);
  const unsigned groups = (unsigned)((nb + PROBE_PB - 1) / PROBE_PB);
  auto gram = [&](int chunk0, int chunks) {
    GCCB_LAUNCH(probe_gram_kernel, dim3((unsigned)chunks, groups, (unsigned)sh.S), PROBE_NT, gsm, stream, x, n, d, y,
                c, fold, w, plist, nb, (const int32_t*)status, chunk0, sh.D, sh.Dp, sh.NB, sh.T, sh.S, L.hpart,
                L.gpart, L.lpart);
  };
  auto solve = [&](int mode) {
    GCCB_LAUNCH(probe_solve_kernel, (unsigned)nb, PROBE_NT, ssm, stream, plist, nb, d, sh.D, sh.NB, sh.T, sh.S, C, w,
                (const double*)L.gpart, (const double*)L.lpart, (const double*)L.hpart, L.hglob, L.step, status,
                L.g0, gnorm, L.fval, L.slope, iter, mode, g_out, h_out, flags);
  };
  if (!newton) {
    gram(0, sh.chunks);
    solve(1);
    return;
  }
  gram(0, 1);
  solve(2);
  if (sh.chunks > 1) gram(1, sh.chunks - 1);
  solve(0);
}

static bool probe_args_ok(const char* what, const float* x, int64_t n, int d, const uint8_t* y, int c,
                          const int32_t* fold, int folds, double C, void* ws, size_t ws_bytes, size_t need) {
  if (!probe_shape_ok(n, d, c, folds) || !(C > 0.0)) {
    set_last_error("%s: need 1 <= n < 2^31, 1 <= d <= %d, 1 <= c <= %d, 1 <= folds <= %d, C > 0 (got n=%lld d=%d c=%d "
                   "folds=%d C=%g)", what, PROBE_MAXDIM, PROBE_MAXC, PROBE_MAXFOLDS, (long long)n, d, c, folds, C);
    return false;
  }
  if (!x || !y || !fold || !ws || ((uintptr_t)ws & 15) != 0) {
    set_last_error("%s: x, y, fold and a 16-byte aligned workspace are required", what);
    return false;
  }
  if (ws_bytes < need) {
    set_last_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
    return false;
  }
  return true;
}

}  // namespace gccb

using namespace gccb;

extern "C" size_t gccb_probe_workspace(int64_t n, int32_t d, int32_t c, int32_t folds, int32_t batch) {
  if (!probe_shape_ok(n, d, c, folds)) return 0;
  return probe_layout(nullptr, n, d, c, folds, batch).bytes;
}

extern "C" int gccb_probe_fit(const float* x, int64_t n, int32_t d, const uint8_t* y, int32_t c, const int32_t* fold,
                              int32_t folds, double C, int32_t max_iter, int32_t batch, double* w, double* z,
                              int64_t* counts, int32_t* status, double* gnorm, int32_t* iters, int32_t* flags,
                              void* ws, size_t ws_bytes, gccb_stream_t stream) {
  const size_t need = gccb_probe_workspace(n, d, c, folds, batch);
  if (!probe_args_ok("gccb_probe_fit", x, n, d, y, c, fold, folds, C, ws, ws_bytes, need)) {
    return ws_bytes < need && probe_shape_ok(n, d, c, folds) && C > 0.0 ? GCCB_ERR_CAPACITY : GCCB_ERR_BADARG;
  }
  if (!w || !z || !counts || !status || !gnorm || !iters || !flags || max_iter < 0) {
    set_last_error("gccb_probe_fit: w, z, counts, status, gnorm, iters and flags are required, max_iter >= 0");
    return GCCB_ERR_BADARG;
  }
  const ProbeShape sh = probe_shape(n, d);
  const int P = folds * c, B = probe_batch(P, batch);
  const ProbeWs L = probe_layout((char*)ws, n, d, c, folds, batch);
  cudaMemsetAsync(L.pos, 0, (size_t)P * 8, (cudaStream_t)stream);
  cudaMemsetAsync(L.cnt, 0, (size_t)folds * 8, (cudaStream_t)stream);
  cudaMemsetAsync(L.tot, 0, (size_t)c * 8, (cudaStream_t)stream);
  cudaMemsetAsync(counts, 0, (size_t)folds * 3 * 8, (cudaStream_t)stream);
  GCCB_LAUNCH(probe_init_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, x, n, d, y, c, fold, folds, flags, L.pos,
              L.cnt, L.tot);
  GCCB_LAUNCH(probe_setup_kernel, (unsigned)((P + 255) / 256), 256, 0, stream, P, c, n, sh.d1,
              (const unsigned long long*)L.pos, (const unsigned long long*)L.cnt, (const unsigned long long*)L.tot,
              status, iters, w, gnorm, L.lsm);
  int32_t fl;
  probe_read_i32(flags, 1, &fl, stream);
  if (fl & GCCB_FLAG_NONFINITE) return check_launch("gccb_probe_fit");
  const size_t lsmem = probe_ls_smem(d);
  ensure_dyn_smem(probe_ls_kernel, lsmem);
  for (int it = 0;; ++it) {
    GCCB_LAUNCH(probe_active_kernel, 1, 1024, 0, stream, P, status, (const int32_t*)L.lsm, L.active, L.newton,
                L.counts, it >= max_iter ? 1 : 0, flags);
    int32_t cnt[2];
    probe_read_i32(L.counts, 2, cnt, stream);             // the one host sync of a pass
    const int na = cnt[0], nn = cnt[1];
    if (na == 0) break;
    for (int lo = 0; lo < nn; lo += B)                    // a Newton system for the problems not in a line search
      probe_system(sh, x, n, d, y, c, fold, C, w, L.newton + lo, nn - lo < B ? nn - lo : B, L, status, gnorm, it,
                   true, nullptr, nullptr, flags, stream);
    for (int lo = 0; lo < na; lo += B) {                  // a window of step lengths for every active problem
      const int nb = na - lo < B ? na - lo : B;
      const int32_t* pl = L.active + lo;
      GCCB_LAUNCH(probe_ls_kernel, dim3((unsigned)((nb + PROBE_PB - 1) / PROBE_PB), (unsigned)sh.S), PROBE_NT, lsmem,
                  stream, x, n, d, y, c, fold, (const double*)w, (const double*)L.step, pl, nb,
                  (const int32_t*)status, (const int32_t*)L.lsm, sh.S, L.lspart);
      GCCB_LAUNCH(probe_update_kernel, (unsigned)((nb + 127) / 128), 128, 0, stream, pl, nb, d, sh.S, C, w,
                  (const double*)L.step, (const double*)L.lspart, status, (const double*)L.fval,
                  (const double*)L.slope, iters, L.lsm, flags);
    }
    if (check_launch("gccb_probe_fit") != GCCB_OK) return GCCB_ERR_CUDA;
  }
  GCCB_LAUNCH(probe_score_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, x, n, d, y, c, fold, folds,
              (const double*)w, (const int32_t*)status, z, (unsigned long long*)counts);
  return check_launch("gccb_probe_fit");
}

extern "C" int gccb_probe_system(const float* x, int64_t n, int32_t d, const uint8_t* y, int32_t c,
                                 const int32_t* fold, int32_t folds, double C, int32_t batch, const double* w,
                                 double* g_out, double* h_out, double* step_out, double* f_out, int32_t* status,
                                 void* ws, size_t ws_bytes, gccb_stream_t stream) {
  const size_t need = gccb_probe_workspace(n, d, c, folds, batch);
  if (!probe_args_ok("gccb_probe_system", x, n, d, y, c, fold, folds, C, ws, ws_bytes, need)) {
    return ws_bytes < need && probe_shape_ok(n, d, c, folds) && C > 0.0 ? GCCB_ERR_CAPACITY : GCCB_ERR_BADARG;
  }
  if (!w || !g_out || !h_out || !step_out || !f_out || !status) {
    set_last_error("gccb_probe_system: w, g_out, h_out, step_out, f_out and status are required");
    return GCCB_ERR_BADARG;
  }
  const ProbeShape sh = probe_shape(n, d);
  const int P = folds * c, B = probe_batch(P, batch);
  const ProbeWs L = probe_layout((char*)ws, n, d, c, folds, batch);
  cudaMemsetAsync(status, 0, (size_t)P * 4, (cudaStream_t)stream);          // PROBE_ACTIVE: every problem
  cudaMemsetAsync(L.lsm, 0, (size_t)P * 4, (cudaStream_t)stream);
  GCCB_LAUNCH(probe_active_kernel, 1, 1024, 0, stream, P, status, (const int32_t*)L.lsm, L.active, L.newton, L.counts,
              0, (int32_t*)nullptr);
  for (int lo = 0; lo < P; lo += B) {
    const int nb = P - lo < B ? P - lo : B;
    probe_system(sh, x, n, d, y, c, fold, C, w, L.active + lo, nb, L, status, L.g0, 0, false, g_out, h_out, nullptr,
                 stream);
  }
  cudaMemcpyAsync(step_out, L.step, (size_t)P * sh.d1 * 8, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  cudaMemcpyAsync(f_out, L.fval, (size_t)P * 8, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  return check_launch("gccb_probe_system");
}
