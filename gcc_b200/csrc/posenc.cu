// posenc.cu -- Laplacian positional features of every ego-net in a batch, on device.
//
// Replaces _add_undirected_graph_positional_embedding + eigen_decomposision
// (gcc/datasets/data_util.py:242-281): L = D^-1/2 A D^-1/2 (D = in_deg.clip(1)),
// k = min(n-2, pos_dim) largest-algebraic eigenvectors in ascending order,
// row-L2 normalised (sklearn normalize), float32, zero-padded to pos_dim;
// k <= 0 -> zeros.  The reference runs ARPACK (scipy eigsh, float64, random v0)
// per ego-net on a CPU worker: ~2.8 ms each, the dominant cost of its pipeline.
//
// Three device solvers, one CTA (or one cluster) per ego-net, chosen by size through device-built work lists:
//
//  (0) n <= 96 by default (up to 228 with GCCB200_DENSE_MAX): the dense tridiagonal solver -- Householder
//      tridiagonalisation of the whole matrix in shared memory, multisection on Sturm counts, inverse iteration
//      with one common shift per multiple eigenvalue, Gram-Schmidt inside clusters, back-transformation in
//      registers.  A direct method: eigenvalues / residuals / orthonormality to 1e-6.  See its own comment below.
//
//  (1) n <= 64, only with solver (0) off: dense one-sided (Hestenes) Jacobi.  G = L + 2I (SPD, spectrum in [1,3]) lives in
//      shared memory, column-major; plane rotations applied on the right orthogonalise its
//      columns; because G is symmetric positive definite the converged columns are
//      lambda_j' v_j, so the eigenvectors are the normalised columns and no V matrix is stored.
//      A warp owns one column pair per step of a round-robin tournament; dot products by
//      shuffle reduction, rotations in registers.
//
//  (2) every larger n: Chebyshev-filtered subspace iteration (ChFSI) on a block of 48 vectors, any n.
//      Ego-nets are star-like: their spectra have one huge degenerate cluster, so a degree-4/8
//      Chebyshev filter on [-1, cut] followed by Rayleigh-Ritz converges in ~3 outer iterations
//      (measured on the C2 workload).  Per iteration: 8 sparse products with the sub-CSR (fused
//      three-term recurrence), CGS2 re-orthonormalisation, H = Q^T L Q, the 48x48 Ritz problem
//      solved by solver (1) in shared memory, X = Q W, residual check.  The n x 48 blocks live in
//      an L2-resident workspace (2 blocks per ego-net), so shared memory does not bound n and
//      8 CTAs fit per SM.  Cost is O(n * 48^2) instead of the O(n^3) of a dense solve.
//
// All return an orthonormal basis of every eigenspace (degenerate clusters included), Ritz
// values as Rayleigh quotients, a deterministic sign (largest-|.| component positive) and are
// deterministic run to run (no floating-point atomics on the results).
#include "common.cuh"

#include <stdlib.h>

namespace gccb {

#define GCCB_EIG_SMALL 64          // largest n solved by the dense Jacobi kernel
#define GCCB_EIG_MAXSWEEP 14
#define GCCB_EIG_TOL 1.0e-6f
#define GCCB_CF_B 48               // ChFSI block size (>= pos_dim 32 + guard vectors)
// Chebyshev degree per outer iteration: as high as the fp32 block tolerates.  The filter on [-1, cut] gains
// T_d(x1), x1 = (3 - cut) / (1 + cut), on the top eigenvalue relative to the damped interval; directions whose
// relative gain drops below eps_fp32 vanish from the block, Gram-Schmidt then normalises noise into "Ritz vectors"
// with arbitrary Ritz values, and those collide with wanted eigenvalues near the cut (measured: an n = 66 ego-net
// diverges at a fixed degree 16).  So d = floor(acosh(G) / acosh(x1)) with G = 1e8, clamped to [4, GCCB_CF_DEG];
// the first iteration (random block) is capped at GCCB_CF_DEG0.  Hub ego-nets (cut ~ 0.6-0.7, x1 ~ 1.4) run at
// degree 16, small ones (cut ~ 0, x1 = 3) at 10.  Measured on C2 ego-nets (fp32 model of this kernel): 2.5 outer
// iterations instead of 3.0 at the round-1 schedule (4, 8), hub ego-nets 2.6 instead of 3.9, worst residual 4e-5
// instead of 3e-4 on n <= 160.
#ifndef GCCB_CF_DEG0
#define GCCB_CF_DEG0 8
#endif
#ifndef GCCB_CF_DEG
#define GCCB_CF_DEG 16
#endif
#define GCCB_CF_LOGGAIN 19.1138f    // acosh(1e8)
// When the smallest WANTED Ritz value sits at the bottom of the block (ego-nets whose top-32 reaches into the
// null space: theta_k ~ theta_48 ~ 0), a cut at the lowest Ritz value leaves the wanted null vectors on the
// boundary of the damped interval, where they are not separated from the negative spectrum; the cut then moves
// GCCB_CF_MARGIN below theta_k.  Only for theta_k < GCCB_CF_MARGIN_BELOW: the degenerate cluster of hub ego-nets
// (1/sqrt 2) is wider than any block and must not drag the cut down.
#define GCCB_CF_MARGIN 0.05f
#define GCCB_CF_MARGIN_BELOW 0.25f
// Jacobi sweeps of the FIRST Ritz solve (random block after one low-degree filter: it never converges there).
// Single-CTA kernels (n <= 384): none -- the Gram-Schmidt basis goes on as it is, ordered by its Rayleigh
// quotients diag(H); measured on C2 ego-nets: 2.50 outer iterations instead of 2.76 for n <= 96 (the half-rotated
// block of a one-sweep solve gave the second filter worse cut / degree estimates than the plain diagonal), 11 %
// fewer cycles per ego-net, same residuals.  Cluster kernels (n > 384, hub ego-nets): one sweep -- without it the
// largest ego-nets need 6-7 outer iterations instead of 3-4 and become the long pole of the batch.
#ifndef GCCB_CF_SWEEPS0
#define GCCB_CF_SWEEPS0 0
#endif
#ifndef GCCB_CF_SWEEPS0_CLUSTER
#define GCCB_CF_SWEEPS0_CLUSTER 1
#endif
#define GCCB_CF_NSM_A 96            // shared-memory block classes: n <= 96 (3 CTAs/SM) and
#define GCCB_CF_NSM 160            //   n <= 160 (2 CTAs/SM),
#define GCCB_CF_NSM_C 384          //   n <= 384 (one GCCB_BIG_NT-thread CTA; 150 KB + 30 KB static leave room
                                   //   for a 46 KB training CTA on the same SM);
#define GCCB_CF_NSM_D1 1536        //   n <= 1536: cluster of 8 CTAs (DSMEM), 192-row slabs (75 KB per CTA);
#define GCCB_CF_NSM_D 3584         //   n <= 3584: cluster of 8 CTAs, 448-row slabs; larger: L2 workspace
#define GCCB_EIG_NCLASS 7
#ifndef GCCB_CF_SMEM_PAD_A
#define GCCB_CF_SMEM_PAD_A 0       // A/B builds: extra shared memory per n <= 96 CTA (lowers its CTAs per SM)
#endif
#ifndef GCCB_CAP_MID1
#define GCCB_CAP_MID1 (GCCB_NUM_SMS * 3)     // persistent grid of the n <= 96 class (3 CTAs per SM)
#endif
#ifndef GCCB_CAP_MID2
#define GCCB_CAP_MID2 (GCCB_NUM_SMS * 2)     // persistent grid of the n <= 160 class (2 CTAs per SM)
#endif
#ifndef GCCB_CAP_DN_A
#define GCCB_CAP_DN_A (GCCB_NUM_SMS * 4)     // persistent grids of the dense classes
#endif
#ifndef GCCB_CAP_DN_B
#define GCCB_CAP_DN_B (GCCB_NUM_SMS * 2)
#endif
#ifndef GCCB_CAP_DN_C
#define GCCB_CAP_DN_C GCCB_NUM_SMS
#endif
#ifndef GCCB_BIG_NT
#define GCCB_BIG_NT 512            // threads of the large-ego-net CTAs: 512 x 64 registers leave half of
#endif                             // the SM's register file to concurrent kernels (these CTAs live for ms)
#define GCCB_CF_MAXIT 8
#define GCCB_GS_PANEL 4            // columns orthogonalised per Gram-Schmidt step (single-CTA kernels)
#define GCCB_CF_TOL 4.0e-5f        // max residual ||L x - theta x|| over the wanted pairs
#define GCCB_CF_STAG 2.0e-3f       // accepted when the residual stops halving below this: ego-nets whose
                                   // near-degenerate cluster is wider than the block stall at its spread

// phase cycle counters (diagnostics; thread 0 only, negligible cost): 0 filter, 1 gram-schmidt, 2 projected
// matrix, 3 Ritz solve, 4 X = QW, 5 residual
#ifdef GCCB_EMU
#define GCCB_CLK() 0ll
#else
#define GCCB_CLK() clock64()
#endif
#define GCCB_TICK(k) do { if (threadIdx.x == 0) { long long t_ = GCCB_CLK(); ph[k] += t_ - t_last; t_last = t_; } } while (0)

// class 0: n <= 64 (dense Jacobi); 1, 2, 3: ChFSI with shared-memory blocks; 4, 5: ChFSI on a cluster;
// 6: ChFSI with L2 blocks
__device__ __forceinline__ int eig_class(int n) {
  return n <= GCCB_EIG_SMALL ? 0 : n <= GCCB_CF_NSM_A ? 1 : n <= GCCB_CF_NSM ? 2 : n <= GCCB_CF_NSM_C ? 3 :
         n <= GCCB_CF_NSM_D1 ? 4 : n <= GCCB_CF_NSM_D ? 5 : 6;
}

// Work lists: worklist[c][i] = slot.  One CTA, deterministic order.  grid = 1, block = 256.
// Ego-nets up to `dense_max` vertices go to the dense tridiagonal solver instead (lists dense_list[3][2B], classes
// n <= dn_a / dn_b / larger; dense_max = 0: none).
__global__ void __launch_bounds__(256)
posenc_classify_kernel(const int64_t* __restrict__ counters, const int32_t* __restrict__ node_off,
                       int B, int32_t* __restrict__ worklist, int32_t* __restrict__ counts,
                       int dense_max, int dn_a, int dn_b, int32_t* __restrict__ dense_list,
                       int32_t* __restrict__ dense_counts) {
  __shared__ int scan_scratch[33];
  const int tid = threadIdx.x;
  constexpr int NC = GCCB_EIG_NCLASS + 3;
  int base[NC] = {0};
  for (int s0 = 0; s0 < 2 * B; s0 += 256) {
    int slot = s0 + tid;
    int cls = -1;
    if (slot < 2 * B) {
      int view = slot / B;
      if (node_off[view * (B + 1) + B] >= 0) {
        const int n = (int)counters[(size_t)slot * 4];
        cls = n <= dense_max ? GCCB_EIG_NCLASS + (n <= dn_a ? 0 : n <= dn_b ? 1 : 2) : eig_class(n);
      }
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      int tot;
      int ex = block_scan_excl(cls == c ? 1 : 0, scan_scratch, &tot);
      if (cls == c) {
        if (c < GCCB_EIG_NCLASS) worklist[(size_t)c * 2 * B + base[c] + ex] = slot;
        else dense_list[(size_t)(c - GCCB_EIG_NCLASS) * 2 * B + base[c] + ex] = slot;
      }
      base[c] += tot;
    }
  }
  if (tid < GCCB_EIG_NCLASS) counts[tid] = base[tid];
  if (tid < 3) dense_counts[tid] = base[GCCB_EIG_NCLASS + tid];
}

// ------------------------------------------------------------------------------------------------
// One-sided Jacobi on the n x n column-major matrix G (leading dimension ld) in shared memory:
// orthogonalises the columns in place; on return nrm[j] = ||g_j||.  Returns the number of
// sweeps used (== GCCB_EIG_MAXSWEEP means not converged).  NR = ceil(nmax/32) rows per lane.
template <int NR, int THREADS>
__device__ __forceinline__ int jacobi_onesided(float* G, float* nrm, int n, int ld) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = THREADS / 32;
  const int m = n + (n & 1);                            // tournament size (even)
  int sweep = 0;
  for (; sweep < GCCB_EIG_MAXSWEEP; ++sweep) {
    for (int p = warp; p < n; p += NW) {                // exact column norms once per sweep
      float s = 0.f;
#pragma unroll
      for (int jj = 0; jj < NR; ++jj) {
        int r = lane + 32 * jj;
        float x = r < n ? G[(size_t)p * ld + r] : 0.f;
        s = fmaf(x, x, s);
      }
      s = warp_sum(s);
      if (lane == 0) nrm[p] = s;
    }
    __syncthreads();
    int rotated = 0;
    for (int r = 0; r < m - 1; ++r) {
      for (int pi = warp; pi < m / 2; pi += NW) {
        int p, q;
        if (pi == 0) { p = m - 1; q = r; }
        else { p = (r + pi) % (m - 1); q = (r + m - 1 - pi) % (m - 1); }
        if (p >= n || q >= n) continue;                 // bye (odd n)
        if (p > q) { int t = p; p = q; q = t; }
        float gp[NR], gq[NR];
        float gam = 0.f;
#pragma unroll
        for (int jj = 0; jj < NR; ++jj) {
          int rr = lane + 32 * jj;
          gp[jj] = rr < n ? G[(size_t)p * ld + rr] : 0.f;
          gq[jj] = rr < n ? G[(size_t)q * ld + rr] : 0.f;
          gam = fmaf(gp[jj], gq[jj], gam);
        }
        // read the cached norms BEFORE the shuffle reduction: the shuffles are the
        // convergence point that orders these reads against lane 0's update below
        const float alpha = nrm[p], beta = nrm[q];
        gam = warp_sum(gam);
        if (fabsf(gam) > GCCB_EIG_TOL * sqrtf(alpha * beta)) {      // warp-uniform
          const float zeta = (beta - alpha) / (2.0f * gam);
          const float t = (zeta >= 0.f ? 1.0f : -1.0f) / (fabsf(zeta) + sqrtf(1.0f + zeta * zeta));
          const float c = 1.0f / sqrtf(1.0f + t * t);
          const float s = c * t;
#pragma unroll
          for (int jj = 0; jj < NR; ++jj) {
            int rr = lane + 32 * jj;
            if (rr < n) {
              G[(size_t)p * ld + rr] = c * gp[jj] - s * gq[jj];
              G[(size_t)q * ld + rr] = s * gp[jj] + c * gq[jj];
            }
          }
          if (lane == 0) { nrm[p] = alpha - t * gam; nrm[q] = beta + t * gam; }
          rotated = 1;
        }
      }
      __syncthreads();
    }
    if (!__syncthreads_or(rotated)) break;
  }
  for (int p = warp; p < n; p += NW) {                  // final norms: nrm[j] = ||g_j||
    float s = 0.f;
#pragma unroll
    for (int jj = 0; jj < NR; ++jj) {
      int r = lane + 32 * jj;
      float x = r < n ? G[(size_t)p * ld + r] : 0.f;
      s = fmaf(x, x, s);
    }
    s = warp_sum(s);
    if (lane == 0) nrm[p] = sqrtf(s);
  }
  __syncthreads();
  return sweep;
}



// Two-sided Jacobi specialised for the even-order Ritz problem (m = 48): per round ONE thread per pair
// derives (c, s); then every thread applies BOTH sides of the similarity transform to whole 2 x 2
// blocks (rows of pair a, columns of pair b) -- no barrier between the row and the column update --
// and rotates V.  Two barriers per round instead of three, independent items unrolled for ILP.
// `tol`: relative skip threshold (adaptive: the Ritz vectors need no more accuracy than the
// current outer residual).
template <int NT>
__device__ __forceinline__ int jacobi_ritz48(float* A, float* V, float* cs /*[64]*/, int* pq /*[32]*/, int LD,
                                              float tol, int max_sweeps, long long* n_work = nullptr,
                                              long long* n_idle = nullptr) {
  constexpr int M = GCCB_CF_B, HALF = M / 2;
  const int tid = threadIdx.x;
  // One 16-byte record per pair and round: (p | q << 16, c, s, -), written in COMPACTED order: slots
  // [0, nr) hold the pairs that rotate this round, the others fill the array from the top.  A block / column
  // update then costs one 128-bit shared-memory load per pair instead of five scalar ones (the rounds are
  // bound by shared-memory instruction throughput: three CTAs share an SM).  Two copies alternate between
  // rounds, so an idle round (nr == 0) costs ONE barrier: the next round's writer never touches the copy a
  // slow reader may still be looking at.  (cs / pq of the caller are no longer used.)
  __shared__ float4 rec2[2][HALF];
  __shared__ int nrot2[2];
  (void)cs; (void)pq;
  for (int idx = tid; idx < M * M; idx += NT) {
    const int j = idx / M, i = idx - j * M;
    V[j * LD + i] = i == j ? 1.0f : 0.f;
  }
  __syncthreads();
  int sweep = 0;
  for (; sweep < max_sweeps; ++sweep) {
    // One look at the whole triangle decides whether another sweep is needed (the same test the rounds
    // apply): a converged matrix costs one barrier instead of M - 1 idle rounds.
    if (max_sweeps > 1) {
      int any = 0;
      for (int idx = tid; idx < M * M; idx += NT) {
        const int q = idx / M, p = idx - q * M;
        if (p < q && fabsf(A[q * LD + p]) > tol * 0.5f * (fabsf(A[p * LD + p]) + fabsf(A[q * LD + q]))) any = 1;
      }
      if (!__syncthreads_or(any)) break;
    }
    for (int r = 0; r < M - 1; ++r) {
      float4* rec = rec2[r & 1];
      if (tid < 32) {                                      // warp 0: one lane per pair
        bool rot = false;
        int p = 0, q = 0;
        float c = 1.0f, sn = 0.f;
        if (tid < HALF) {
          if (tid == 0) { p = M - 1; q = r; }
          else { p = (r + tid) % (M - 1); q = (r + M - 1 - tid) % (M - 1); }
          if (p > q) { int t = p; p = q; q = t; }
          const float app = A[p * LD + p], aqq = A[q * LD + q], apq = A[q * LD + p];
          // (diagonal of G = H + 2I lies in [1, 3]: the arithmetic mean is as good a scale as the geometric one)
          if (fabsf(apq) > tol * 0.5f * (fabsf(app) + fabsf(aqq))) {
            // t = sgn(zeta) / (|zeta| + sqrt(1 + zeta^2)), zeta = d / (2 apq), without dividing by apq;
            // fast division / reciprocal square root: this dependent chain is on the critical path of
            // every round, and a 2-ulp rotation error is far below the Ritz tolerance
            const float d = aqq - app;
            const float two_apq = 2.0f * apq;
            const float den = fabsf(d) + __fsqrt_rn(fmaf(d, d, two_apq * two_apq));
            const float t = __fdividef(d >= 0.f ? two_apq : -two_apq, den);
            c = rsqrtf(fmaf(t, t, 1.0f));
            sn = c * t;
            rot = true;
          }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, rot);
        if (tid < HALF) {
          const int below = __popc(mask & ((1u << tid) - 1u));
          const int slot = rot ? below : HALF - 1 - (tid - below);
          rec[slot] = make_float4(__int_as_float(p | (q << 16)), c, sn, 0.f);
        }
        if (tid == 0) nrot2[r & 1] = __popc(mask);
      }
      __syncthreads();
      const int nr = nrot2[r & 1];
      if (nr == 0) { if (n_idle) ++*n_idle; continue; }
      if (n_work) ++*n_work;
      // A <- J^T A J on 2x2 blocks (rows of pair a, columns of pair b).  A is symmetric and only its canonical
      // triangle T(x, y) = A[max(x, y) * LD + min(x, y)] is kept up to date (the rotation test above and the
      // caller read nothing else), so each UNORDERED pair of slots {a, b} is one work item instead of two;
      // only blocks with a rotating slot change: a in [0, nr), b in [a, HALF).  Row a has HALF - a blocks:
      // rows f and nr - 1 - f are folded into one line of constant width W = 2 HALF - nr + 1, which makes the
      // item -> (a, b) map a single division (an odd nr leaves its middle row half used).
      const int W = 2 * HALF - nr + 1, n_items = ((nr + 1) >> 1) * W;
      for (int item = tid; item < n_items; item += NT) {
        const int f = item / W, j = item - f * W;
        int sa, sb;
        if (j < HALF - f) { sa = f; sb = f + j; }
        else { sa = nr - 1 - f; sb = sa + (j - (HALF - f)); if (sa == f) continue; }
        const float4 ra = rec[sa];
        const int ca = __float_as_int(ra.x);
        const int p1 = ca & 0xffff, q1 = ca >> 16;
        const float c1 = ra.y, s1 = ra.z;
        if (sa == sb) {                                    // the pair's own 2 x 2 block: app, aqq change, apq -> 0
          const float app = A[p1 * LD + p1], aqq = A[q1 * LD + q1], apq = A[q1 * LD + p1];
          const float cc = c1 * c1, ss = s1 * s1, x2 = 2.0f * c1 * s1 * apq;
          A[p1 * LD + p1] = cc * app - x2 + ss * aqq;
          A[q1 * LD + q1] = ss * app + x2 + cc * aqq;
          A[q1 * LD + p1] = 0.f;
          continue;
        }
        const float4 rb = rec[sb];
        const int cb = __float_as_int(rb.x);
        const int p2 = cb & 0xffff, q2 = cb >> 16;
        const float c2 = rb.y, s2 = rb.z;
        const int i_a = max(p1, p2) * LD + min(p1, p2), i_b = max(p1, q2) * LD + min(p1, q2);
        const int i_c = max(q1, p2) * LD + min(q1, p2), i_d = max(q1, q2) * LD + min(q1, q2);
        float a = A[i_a], b = A[i_b], c_ = A[i_c], d = A[i_d];
        // index 2 (pair b): [x y] -> [c2 x - s2 y, s2 x + c2 y]
        float a2 = c2 * a - s2 * b, b2 = s2 * a + c2 * b, c3 = c2 * c_ - s2 * d, d2 = s2 * c_ + c2 * d;
        // index 1 (pair a): [x; y] -> [c1 x - s1 y; s1 x + c1 y]
        A[i_a] = c1 * a2 - s1 * c3;
        A[i_b] = c1 * b2 - s1 * d2;
        A[i_c] = s1 * a2 + c1 * c3;
        A[i_d] = s1 * b2 + c1 * d2;
      }
      // V <- V J: only the columns of rotating pairs
      for (int item = tid; item < nr * M; item += NT) {
        const int ir = item / M, i = item - ir * M;
        const float4 rr = rec[ir];
        const int code = __float_as_int(rr.x);
        const int p = code & 0xffff, q = code >> 16;
        const float x = V[p * LD + i], y = V[q * LD + i];
        V[p * LD + i] = rr.y * x - rr.z * y;
        V[q * LD + i] = rr.z * x + rr.y * y;
      }
      __syncthreads();
    }
  }
  return sweep;
}

// Shared epilogue: write pos rows from k unit eigenvectors.
//   vec(c, r): component r of the eigenvector for output column c (ascending eigenvalue order)
template <class VecFn>
__device__ __forceinline__ void write_features(int n, int k, int pos_dim, int normalize, float* sgn /*[32] smem*/,
                                               float* __restrict__ out, VecFn vec) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NW = blockDim.x >> 5;
  // deterministic sign: the largest-|.| component (lowest row on ties) is positive
  for (int c = warp; c < k; c += NW) {
    float best = -1.f, bval = 0.f; int brow = 0x7fffffff;
    for (int r = lane; r < n; r += 32) {
      float x = vec(c, r), a = fabsf(x);
      if (a > best) { best = a; brow = r; bval = x; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ob = __shfl_xor_sync(0xffffffffu, best, o);
      int orow = __shfl_xor_sync(0xffffffffu, brow, o);
      float ov = __shfl_xor_sync(0xffffffffu, bval, o);
      if (ob > best || (ob == best && orow < brow)) { best = ob; brow = orow; bval = ov; }
    }
    if (lane == 0) sgn[c] = bval < 0.f ? -1.0f : 1.0f;
  }
  __syncthreads();
  for (int r = warp; r < n; r += NW) {                  // lane c holds component c of node r
    float u = 0.f;
    if (lane < k) u = sgn[lane] * vec(lane, r);
    if (normalize) {                                    // sklearn normalize(norm="l2")
      float ss = warp_sum(u * u);
      if (ss > 0.f) u = u / sqrtf(ss);
    }
    if (lane < pos_dim) out[(size_t)r * pos_dim + lane] = u;
  }
}

// ---- solver (1): dense one-sided Jacobi, n <= 64 ---------------------------------------------------
// (one-sided on the SPD matrix L + 2I keeps eigenVECTOR accuracy for close eigenvalues -- paths,
// rings -- where an fp32 two-sided rotation sequence loses it as eps * rotations / gap; fp64 would
// too be accurate but runs at a small fraction of the fp32 rate on this part)
__device__ __forceinline__ void posenc_jacobi_item(const int item, const int32_t* __restrict__ worklist, const int32_t* __restrict__ counts,
                     int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                     const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                     const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                     float* __restrict__ pos, float* __restrict__ eigvals, int32_t* __restrict__ flags,
                     int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res) {
  __shared__ float G[GCCB_EIG_SMALL * GCCB_EIG_SMALL];
  __shared__ float nrm[GCCB_EIG_SMALL];
  __shared__ float dinv[GCCB_EIG_SMALL];
  __shared__ int sel[32];
  __shared__ float sgn[32];
  const int slot = worklist[item];
  const int view = slot / B, g = slot - view * B;
  const int noff = node_off[view * (B + 1) + g];
  const int n = node_off[view * (B + 1) + g + 1] - noff;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = min(n - 2, pos_dim);
  float* out = pos + ((size_t)view * node_cap + noff) * pos_dim;
  if (k <= 0) {                                        // data_util.py:243-244
    for (int i = tid; i < n * pos_dim; i += 256) out[i] = 0.f;
    if (eigvals)
      for (int i = tid; i < pos_dim; i += 256) eigvals[(size_t)slot * pos_dim + i] = 0.f;
    return;
  }
  const int ld = n;
  const int32_t* v_indptr = b_indptr + (size_t)view * (node_cap + 1);
  const int32_t* v_indices = b_indices + (size_t)view * edge_cap;
  const int32_t* v_deg = sub_deg + (size_t)view * node_cap;
  for (int i = tid; i < n * ld; i += 256) G[i] = 0.f;
  for (int i = tid; i < n; i += 256) {
    int d = v_deg[noff + i];
    dinv[i] = 1.0f / sqrtf((float)(d < 1 ? 1 : d));   // in_degrees().clip(1) ** -0.5
  }
  __syncthreads();
  for (int i = warp; i < n; i += 8) {                  // row i <- its in-neighbours j
    const int beg = v_indptr[noff + i], end = v_indptr[noff + i + 1];
    const float di = dinv[i];
    for (int e = beg + lane; e < end; e += 32) {
      int j = v_indices[e] - noff;
      atomicAdd(&G[(size_t)j * ld + i], di * dinv[j]);  // shared-memory adds of exact products
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += 256) G[(size_t)i * ld + i] += 2.0f;
  __syncthreads();
  const int sweeps = jacobi_onesided<2, 256>(G, nrm, n, ld);
  if (sweeps == GCCB_EIG_MAXSWEEP && tid == 0) atomicOr(flags, (int)GCCB_FLAG_EIG_NOCONV);
  if (tid == 0) { dbg_iters[slot] = -sweeps; dbg_res[slot] = 0.f; }
  // eigenvalue of column j = ||g_j|| - 2; rank columns, keep the k largest, ascending
  const float* mu = nrm;
  for (int j = tid; j < n; j += 256) {
    const float mj = mu[j];
    int rank = 0;
    for (int i = 0; i < n; ++i) {
      float mi = mu[i];
      rank += (mi > mj) || (mi == mj && i < j);
    }
    if (rank < k) sel[k - 1 - rank] = j;                // ascending: slot k-1 = largest
  }
  __syncthreads();
  if (eigvals) {
    // eigenvalues as Rayleigh quotients v^T L v against the ORIGINAL sparse matrix: the column
    // norms carry the accumulated rounding of ~n rotations per sweep (~1e-5)
    for (int c = warp; c < pos_dim; c += 8) {
      float acc = 0.f;
      if (c < k) {
        const float* col = G + (size_t)sel[c] * ld;
        for (int i = lane; i < n; i += 32) {
          const int beg = v_indptr[noff + i], end = v_indptr[noff + i + 1];
          float rowacc = 0.f;
          for (int e = beg; e < end; ++e) {
            int j = v_indices[e] - noff;
            rowacc = fmaf(dinv[j], col[j], rowacc);
          }
          acc = fmaf(col[i] * dinv[i], rowacc, acc);
        }
        acc = warp_sum(acc);
        const float m2 = mu[sel[c]];
        acc = acc / (m2 * m2);
      }
      if (lane == 0) eigvals[(size_t)slot * pos_dim + c] = acc;
    }
  }
  const float* Gc = G;
  const int* selc = sel;
  write_features(n, k, pos_dim, normalize, sgn, out,
                 [&](int c, int r) { const int j = selc[c]; return Gc[(size_t)j * ld + r] / mu[j]; });
}

__global__ void __launch_bounds__(256)
posenc_jacobi_kernel(const int32_t* __restrict__ worklist, const int32_t* __restrict__ counts,
                     int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                     const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                     const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                     float* __restrict__ pos, float* __restrict__ eigvals, int32_t* __restrict__ flags,
                     int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res) {
  // persistent over the work list: the grid is sized for the typical count, not for 2B
  for (int item = blockIdx.x; item < counts[0]; item += gridDim.x) {
    posenc_jacobi_item(item, worklist, counts, B, node_cap, edge_cap, node_off, b_indptr, b_indices, sub_deg, pos_dim, normalize, pos, eigvals, flags, dbg_iters, dbg_res);
    __syncthreads();
  }
}

// ---- solver (2): Chebyshev-filtered subspace iteration, any n > 64 -------------------------------
// Blocks are ROW-major n x 48 (leading dimension ld): a neighbour gather reads one contiguous row,
// so the sparse products are warp-per-row with lanes across the 48 columns (any degree, coalesced).
struct SubCsr {
  const int32_t* indptr;   // view-local, index with noff + r
  const int32_t* indices;
  const float* dinv;       // [n] for this ego-net
  int noff, n;
};

// dst[r][c] = alpha * (sum_{j in N(r)} w_rj src[j][c] - cen * src[r][c]) - beta * dst[r][c]
// (beta == 0: dst is write-only).  One warp per row; lane owns columns lane and 32 + lane.
__device__ __forceinline__ void spmm_cheb(const SubCsr& S, const float* __restrict__ src, float* __restrict__ dst,
                                          int ld, float alpha, float cen, float beta) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const bool hi = lane < GCCB_CF_B - 32;
  for (int r = warp; r < S.n; r += nw) {
    const int beg = S.indptr[S.noff + r], end = S.indptr[S.noff + r + 1];
    const float dr = S.dinv[r];
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
    int e = beg;
    for (; e + 3 < end; e += 4) {                         // four edges (gathers) in flight
      const int j0 = S.indices[e] - S.noff, j1 = S.indices[e + 1] - S.noff;
      const int j2 = S.indices[e + 2] - S.noff, j3 = S.indices[e + 3] - S.noff;
      const float x0 = src[(size_t)j0 * ld + lane], x1 = src[(size_t)j1 * ld + lane];
      const float x2 = src[(size_t)j2 * ld + lane], x3 = src[(size_t)j3 * ld + lane];
      float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;
      if (hi) {
        y0 = src[(size_t)j0 * ld + 32 + lane]; y1 = src[(size_t)j1 * ld + 32 + lane];
        y2 = src[(size_t)j2 * ld + 32 + lane]; y3 = src[(size_t)j3 * ld + 32 + lane];
      }
      const float w0 = dr * S.dinv[j0], w1 = dr * S.dinv[j1], w2 = dr * S.dinv[j2], w3 = dr * S.dinv[j3];
      a0 = fmaf(w0, x0, a0); b0 = fmaf(w1, x1, b0); a0 = fmaf(w2, x2, a0); b0 = fmaf(w3, x3, b0);
      a1 = fmaf(w0, y0, a1); b1 = fmaf(w1, y1, b1); a1 = fmaf(w2, y2, a1); b1 = fmaf(w3, y3, b1);
    }
    for (; e < end; ++e) {
      const int j0 = S.indices[e] - S.noff;
      const float w0 = dr * S.dinv[j0];
      a0 = fmaf(w0, src[(size_t)j0 * ld + lane], a0);
      if (hi) a1 = fmaf(w0, src[(size_t)j0 * ld + 32 + lane], a1);
    }
    a0 += b0; a1 += b1;
    const size_t o = (size_t)r * ld + lane;
    float v = alpha * (a0 - cen * src[o]);
    if (beta != 0.f) v -= beta * dst[o];
    dst[o] = v;
    if (hi) {
      float v1 = alpha * (a1 - cen * src[o + 32]);
      if (beta != 0.f) v1 -= beta * dst[o + 32];
      dst[o + 32] = v1;
    }
  }
}

// Per-column reduction helper: every warp accumulates (lane -> columns lane, 32+lane) over its rows,
// partial sums go through part[32][48] and end up in out[48]; rr2[0] + rr2[1] = sum_{c < jlim} out[c]^2
// (the Gram-Schmidt norm update) comes out of the same pass.  Ends with a barrier.
template <class RowFn>
__device__ __forceinline__ void column_sums(int n, float* part /*[32][48]*/, float* out /*[48]*/, float* rr2 /*[2]*/,
                                            int jlim, RowFn f) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const bool hi = lane < GCCB_CF_B - 32;
  const int nwu = nw < 8 ? nw : 8;                      // 8 accumulating warps keep the partial reduce short
  if (warp < nwu) {
    float a0 = 0.f, a1 = 0.f;
    for (int r = warp; r < n; r += nwu) {
      a0 += f(r, lane);
      if (hi) a1 += f(r, 32 + lane);
    }
    part[warp * GCCB_CF_B + lane] = a0;
    if (hi) part[warp * GCCB_CF_B + 32 + lane] = a1;
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = threadIdx.x;
    float sacc = 0.f;
    if (c < GCCB_CF_B) {
      for (int w = 0; w < nwu; ++w) sacc += part[w * GCCB_CF_B + c];
      out[c] = sacc;
    }
    float sq = c < jlim ? sacc * sacc : 0.f;
    sq = warp_sum(sq);
    if (lane == 0) rr2[warp] = sq;
  }
  __syncthreads();
}

// MODE 1: both n x 48 blocks live in dynamic shared memory (ld = 49, conflict-free); MODE 0: both in
// the L2-resident workspace (ego-nets too large even for the cluster kernel).
// cls selects the work list; blockDim.x = 256 or 1024.
template <int MODE, int NT>
__device__ __forceinline__ void posenc_chfsi_item(const int item, const int32_t* __restrict__ worklist, const int32_t* __restrict__ counts, int cls,
                    int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                    const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                    const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                    float* __restrict__ blocks /* [2][2*node_cap*48] */, float* __restrict__ dinv_g /* [2*node_cap] */,
                    float* __restrict__ pos, float* __restrict__ eigvals, int32_t* __restrict__ flags,
                    int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res, long long* __restrict__ dbg_phase) {
  constexpr int CB = GCCB_CF_B, LD = CB + 1;
  GCCB_DYN_SMEM(float, dynsm);
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t_last = GCCB_CLK();
  __shared__ float Gs[CB * LD];                   // Ritz problem
  // union: Ritz vectors Ws[CB*LD] | staging tiles [2][32][CB+1] (only when the blocks are not in shared memory)
  __shared__ float WT[MODE == 1 ? CB * LD : 32 * (CB + 1) * 2];
  float* part = Gs;                               // column-sum partials [32][CB]: the Ritz matrix is dead whenever they are live
  static_assert(32 * CB <= CB * LD, "partials must fit in the Ritz matrix");
  __shared__ float rdot[CB];
  __shared__ float rr2[2];
  __shared__ float theta[CB];
  __shared__ float resid[CB];
  __shared__ float cs[64];
  __shared__ int pq[32];
  __shared__ int perm[CB];
  __shared__ float s_bc[2];
  __shared__ float sgn[32];
  __shared__ float rd4[GCCB_GS_PANEL * CB];      // panel Gram-Schmidt: dots of the 4 panel columns with all columns
  __shared__ float pl[16];                        // inverse of the panel's 4 x 4 Cholesky factor (lower triangle)
  __shared__ int pflag;
  float* Ws = WT;
  float (*tile)[32][CB + 1] = reinterpret_cast<float (*)[32][CB + 1]>(WT);
  const int slot = worklist[(size_t)cls * 2 * B + item];
  const int view = slot / B, g = slot - view * B;
  const int noff = node_off[view * (B + 1) + g];
  const int n = node_off[view * (B + 1) + g + 1] - noff;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = NT / 32;
  const bool hi = lane < CB - 32;
  const int k = min(n - 2, pos_dim);                    // n > 64 -> k = pos_dim
  float* out = pos + ((size_t)view * node_cap + noff) * pos_dim;
  float* dinv = dinv_g + (size_t)view * node_cap + noff;
  SubCsr S;
  S.indptr = b_indptr + (size_t)view * (node_cap + 1);
  S.indices = b_indices + (size_t)view * edge_cap;
  S.dinv = dinv;
  S.noff = noff; S.n = n;
  const int32_t* v_deg = sub_deg + (size_t)view * node_cap;
  const int ld = LD;                                    // 49 everywhere (odd: conflict-free in smem)
  float* X;
  float* Y;
  if (MODE == 1) {
    X = dynsm;
    Y = dynsm + (size_t)n * LD;
  } else {
    X = blocks + ((size_t)view * node_cap + noff) * LD;                // n x 48 (ld 49), row-major
    Y = X + (size_t)2 * node_cap * LD;
  }
  for (int i = tid; i < n; i += NT) {
    int d = v_deg[noff + i];
    dinv[i] = 1.0f / sqrtf((float)(d < 1 ? 1 : d));
  }
  // start block: counter-based pseudo-random entries in (-1, 1) (deterministic)
  for (int i = tid; i < n * CB; i += NT) {
    u32x4 w = philox4x32_10((uint32_t)i, (uint32_t)n, 0x51ED270Bu, 3u, 0xC0FFEEu, 0x5EEDu);
    X[(size_t)(i / CB) * ld + (i % CB)] = (float)(int32_t)w.x * (1.0f / 2147483648.0f);
  }
  __syncthreads();
#ifndef GCCB_CF_NO_DEFLATE
  // The top eigenvector of D^-1/2 A D^-1/2 is known in closed form: v0 = sqrt(deg) (eigenvalue 1; ||v0||^2 =
  // sum of degrees).  It becomes column 0 and is projected out of the random columns: the first filter
  // amplifies the v0 component ~35x more than anything below 0.5, so without this every filtered column is
  // nearly parallel to v0 and the first Gram-Schmidt pass runs on cancellation (second passes, one-column
  // fallbacks).  Only the START block changes -- any start block is valid.
  {
    float* rdot0 = rd4;
    column_sums(n, part, rdot0, rr2, 0, [&](int r, int c) { return X[(size_t)r * ld + c] / dinv[r]; });
    const float inv_vv = 1.0f / (float)max(S.indptr[noff + n] - S.indptr[noff], 1);
    for (int i = tid; i < n * CB; i += NT) {
      const int r = i / CB, c = i - r * CB;
      const float v = 1.0f / dinv[r];
      X[(size_t)r * ld + c] = c == 0 ? v : fmaf(-rdot0[c] * inv_vv, v, X[(size_t)r * ld + c]);
    }
    __syncthreads();
  }
#endif
  float cut = 0.0f;                                     // the filter suppresses [-1, cut]
  float prev_worst = 3.0e38f;
  bool converged = false;
  int iter = 0;
  for (; iter < GCCB_CF_MAXIT && !converged; ++iter) {
    // ---- Chebyshev filter on [-1, cut] (scaled three-term recurrence) -----------------------------
    {
      const float e = (cut + 1.0f) * 0.5f, cen = (cut - 1.0f) * 0.5f;
      int deg = (int)floorf(GCCB_CF_LOGGAIN / acoshf((3.0f - cut) / (1.0f + cut)));
      deg = max(4, min(iter == 0 ? GCCB_CF_DEG0 : GCCB_CF_DEG, deg));
      float sigma = e / (1.0f - cen);
      const float sigma1 = sigma;
      spmm_cheb(S, X, Y, ld, sigma1 / e, cen, 0.f);                           // Y1
      __syncthreads();
      float* cur = Y; float* prev = X;
      for (int i = 2; i <= deg; ++i) {
        const float sigma2 = 1.0f / (2.0f / sigma1 - sigma);
        spmm_cheb(S, cur, prev, ld, 2.0f * sigma2 / e, cen, sigma * sigma2);   // overwrites prev
        __syncthreads();
        float* t = cur; cur = prev; prev = t;
        sigma = sigma2;
      }
      X = cur; Y = prev;                                 // filtered block in X, Y is scratch
    }
    GCCB_TICK(0);
    // ---- Gram-Schmidt: orthonormalise the columns of X in place, FOUR columns per step ------------------
    // One pass over the rows gives the dots of the 4 panel columns with all columns (panel included): R = Q^T Y
    // and G = Y^T Y.  The Gram matrix of the projected panel follows without a second reduction,
    // G' = G - R^T R (Pythagoras, the 4 x 4 generalisation of ||y - QQ^T y||^2 = y.y - sum r_i^2), its Cholesky
    // factor orthonormalises the panel, and one update pass applies Y <- (Y - Q R) L^-T: the barriers and
    // latency chains of one column now serve four.  Heavy cancellation (diag G' <= diag G / 2) asks for a
    // second pass as before; a small Cholesky pivot (panel nearly dependent after the projection: the random
    // block of the first iteration) sends the 4 columns through the one-column code below.
    auto gs_scalar = [&](int j) {
      // classical Gram-Schmidt with selective re-orthogonalisation (Daniel-Gragg-Kaufman test): the
      // dots of column j with all columns (itself included) come from one pass over the rows;
      // ||y - Q Q^T y||^2 = y.y - sum r_i^2, so neither the test nor the norm needs another reduction
      float nrm2 = 0.f;
      bool scaled = false;
      for (int pass = 0; pass < 2; ++pass) {
        const float* Xc = X;
        column_sums(n, part, rdot, rr2, j, [&](int r, int c) { return Xc[(size_t)r * ld + c] * Xc[(size_t)r * ld + j]; });
        const float yy = rdot[j];
        const float rr = rr2[0] + rr2[1];
        nrm2 = yy - rr;
        // little was removed: this is the last pass, so the column is normalised while it is in hand
        // (norm from the same Pythagoras identity; relative error <= 2 eps when nrm2 > yy / 2)
        scaled = nrm2 > 0.5f * yy && nrm2 > 1e-30f;
        const float sc = scaled ? 1.0f / sqrtf(nrm2) : 1.0f;
        for (int r = tid; r < n; r += NT) {
          float* row = X + (size_t)r * ld;
          float v0 = row[j], v1 = 0.f;
          int i = 0;
          for (; i + 1 < j; i += 2) {
            v0 = fmaf(-rdot[i], row[i], v0);
            v1 = fmaf(-rdot[i + 1], row[i + 1], v1);
          }
          if (i < j) v0 = fmaf(-rdot[i], row[i], v0);
          row[j] = (v0 + v1) * sc;
        }
        __syncthreads();
        if (nrm2 > 0.5f * yy) break;                     // no second pass needed
      }
      if (!scaled) {
        if (!(nrm2 > 1e-30f)) {                          // cancellation: measure the norm directly
          const float* Xc = X;
          column_sums(n, part, rdot, rr2, 0, [&](int r, int c) { return c == j ? Xc[(size_t)r * ld + j] * Xc[(size_t)r * ld + j] : 0.f; });
          nrm2 = rdot[j];
        }
        const float inv = nrm2 > 1e-30f ? 1.0f / sqrtf(nrm2) : 0.f;
        for (int r = tid; r < n; r += NT) X[(size_t)r * ld + j] *= inv;
        __syncthreads();
      }
        };
    for (int j0 = 0; j0 < CB; j0 += GCCB_GS_PANEL) {
      bool done = false;
      for (int pass = 0; pass < 2 && !done; ++pass) {
        {   // dots of columns j0..j0+3 with every column
          constexpr int nwu = NW < 8 ? NW : 8;
          if (warp < nwu) {
            float a0[GCCB_GS_PANEL], a1[GCCB_GS_PANEL];
#pragma unroll
            for (int q = 0; q < GCCB_GS_PANEL; ++q) a0[q] = a1[q] = 0.f;
            for (int r = warp; r < n; r += nwu) {
              const float* row = X + (size_t)r * ld;
              const float x0 = row[lane], x1 = hi ? row[32 + lane] : 0.f;
#pragma unroll
              for (int q = 0; q < GCCB_GS_PANEL; ++q) {
                const float y = row[j0 + q];
                a0[q] = fmaf(x0, y, a0[q]);
                a1[q] = fmaf(x1, y, a1[q]);
              }
            }
#pragma unroll
            for (int q = 0; q < GCCB_GS_PANEL; ++q) {
              part[(warp * GCCB_GS_PANEL + q) * CB + lane] = a0[q];
              if (hi) part[(warp * GCCB_GS_PANEL + q) * CB + 32 + lane] = a1[q];
            }
          }
          __syncthreads();
          for (int t = tid; t < GCCB_GS_PANEL * CB; t += NT) {
            const int q = t / CB, c = t - q * CB;
            float sacc = 0.f;
#pragma unroll
            for (int w = 0; w < nwu; ++w) sacc += part[(w * GCCB_GS_PANEL + q) * CB + c];
            rd4[t] = sacc;
          }
          __syncthreads();
        }
        if (warp == 0) {
          // lane -> (a, b), a >= b, of the lower triangle of G'
          const int a = lane < 1 ? 0 : lane < 3 ? 1 : lane < 6 ? 2 : 3;
          const int b = lane - (a * (a + 1)) / 2;
          float gp = 0.f;
          if (lane < 10) {
            float sacc = 0.f;
            for (int i = 0; i < j0; ++i) sacc = fmaf(rd4[a * CB + i], rd4[b * CB + i], sacc);
            gp = rd4[a * CB + j0 + b] - sacc;
          }
          float g[10];
#pragma unroll
          for (int q = 0; q < 10; ++q) g[q] = __shfl_sync(0xffffffffu, gp, q);
          if (lane == 0) {
            // g: 0 (0,0) | 1 (1,0) 2 (1,1) | 3 (2,0) 4 (2,1) 5 (2,2) | 6 (3,0) 7 (3,1) 8 (3,2) 9 (3,3)
            const float yy0 = rd4[0 * CB + j0], yy1 = rd4[1 * CB + j0 + 1], yy2 = rd4[2 * CB + j0 + 2], yy3 = rd4[3 * CB + j0 + 3];
            int flag = 0;
            const bool tiny = !(g[0] > 1e-30f) || !(g[2] > 1e-30f) || !(g[5] > 1e-30f) || !(g[9] > 1e-30f);
            const bool again = !(g[0] > 0.5f * yy0) || !(g[2] > 0.5f * yy1) || !(g[5] > 0.5f * yy2) || !(g[9] > 0.5f * yy3);
            float li[10] = {1.f, 0.f, 1.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};   // identity: projection only
#ifdef GCCB_GS_FORCE_SCALAR                              // A/B builds (profiles/build_variant.py)
            if (true) flag = 2;
#else
            if (tiny) flag = 2;
#endif
            else if (again) flag = pass == 0 ? 1 : 2;
            else {
              const float l00 = sqrtf(g[0]);
              const float l10 = g[1] / l00;
              const float s11 = g[2] - l10 * l10;
              const float l11 = sqrtf(fmaxf(s11, 0.f));
              const float l20 = g[3] / l00;
              const float l21 = (g[4] - l20 * l10) / fmaxf(l11, 1e-30f);
              const float s22 = g[5] - l20 * l20 - l21 * l21;
              const float l22 = sqrtf(fmaxf(s22, 0.f));
              const float l30 = g[6] / l00;
              const float l31 = (g[7] - l30 * l10) / fmaxf(l11, 1e-30f);
              const float l32 = (g[8] - l30 * l20 - l31 * l21) / fmaxf(l22, 1e-30f);
              const float s33 = g[9] - l30 * l30 - l31 * l31 - l32 * l32;
              if (!(s11 > 1e-4f * g[2]) || !(s22 > 1e-4f * g[5]) || !(s33 > 1e-4f * g[9])) flag = 2;
              else {
                const float l33 = sqrtf(s33);
                li[0] = 1.0f / l00; li[2] = 1.0f / l11; li[5] = 1.0f / l22; li[9] = 1.0f / l33;
                li[1] = -l10 * li[0] * li[2];
                li[4] = -l21 * li[2] * li[5];
                li[3] = -(l20 * li[0] + l21 * li[1]) * li[5];
                li[8] = -l32 * li[5] * li[9];
                li[7] = -(l31 * li[2] + l32 * li[4]) * li[9];
                li[6] = -(l30 * li[0] + l31 * li[1] + l32 * li[3]) * li[9];
              }
            }
#pragma unroll
            for (int q = 0; q < 10; ++q) pl[q] = li[q];
            pflag = flag;
          }
        }
        __syncthreads();
        const int flag = pflag;
        if (flag == 2) break;                              // one column at a time below
        for (int r = tid; r < n; r += NT) {
          float* row = X + (size_t)r * ld;
          float v0 = row[j0], v1 = row[j0 + 1], v2 = row[j0 + 2], v3 = row[j0 + 3];
          for (int i = 0; i < j0; ++i) {
            const float q = row[i];
            v0 = fmaf(-rd4[i], q, v0);
            v1 = fmaf(-rd4[CB + i], q, v1);
            v2 = fmaf(-rd4[2 * CB + i], q, v2);
            v3 = fmaf(-rd4[3 * CB + i], q, v3);
          }
          row[j0] = pl[0] * v0;
          row[j0 + 1] = fmaf(pl[1], v0, pl[2] * v1);
          row[j0 + 2] = fmaf(pl[3], v0, fmaf(pl[4], v1, pl[5] * v2));
          row[j0 + 3] = fmaf(pl[6], v0, fmaf(pl[7], v1, fmaf(pl[8], v2, pl[9] * v3)));
        }
        __syncthreads();
        done = flag == 0;
      }
      if (!done)
        for (int j = j0; j < j0 + GCCB_GS_PANEL; ++j) gs_scalar(j);
    }
    GCCB_TICK(1);
    // ---- Z = L Q (into Y), H = Q^T Z ----------------------------------------------------------------
    spmm_cheb(S, X, Y, ld, 1.0f, 0.f, 0.f);
    __syncthreads();
    {
      const int ti = (tid & 255) >> 4, tj = tid & 15;    // first 256 threads: 16 x 16, 3 x 3 outputs each
      float acc[3][3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b2 = 0; b2 < 3; ++b2) acc[a][b2] = 0.f;
      if (MODE == 1) {
        // both blocks are already in shared memory (ld 49: a warp reads 2 Q addresses, broadcast,
        // and 16 Z addresses 3 apart, conflict-free): no staging tiles
        if (tid < 256) {
#pragma unroll 4
          for (int r = 0; r < n; ++r) {
            float qa[3], zb[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) { qa[a] = X[(size_t)r * ld + ti * 3 + a]; zb[a] = Y[(size_t)r * ld + tj * 3 + a]; }
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
              for (int b2 = 0; b2 < 3; ++b2) acc[a][b2] = fmaf(qa[a], zb[b2], acc[a][b2]);
          }
        }
        __syncthreads();                                   // partial sums lived in Gs until the Gram-Schmidt ended
      } else {
        for (int r0 = 0; r0 < n; r0 += 32) {
          for (int idx = tid; idx < 32 * CB; idx += NT) {
            const int rr = idx / CB, c = idx - rr * CB;
            const int r = r0 + rr;
            tile[0][rr][c] = r < n ? X[(size_t)r * ld + c] : 0.f;
            tile[1][rr][c] = r < n ? Y[(size_t)r * ld + c] : 0.f;
          }
          __syncthreads();
          if (tid < 256) {
#pragma unroll 4
            for (int rr = 0; rr < 32; ++rr) {
              float qa[3], zb[3];
#pragma unroll
              for (int a = 0; a < 3; ++a) { qa[a] = tile[0][rr][ti * 3 + a]; zb[a] = tile[1][rr][tj * 3 + a]; }
#pragma unroll
              for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b2 = 0; b2 < 3; ++b2) acc[a][b2] = fmaf(qa[a], zb[b2], acc[a][b2]);
            }
          }
          __syncthreads();
        }
      }
      if (tid < 256) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b2 = 0; b2 < 3; ++b2) Gs[(tj * 3 + b2) * LD + ti * 3 + a] = acc[a][b2];
      }
      __syncthreads();
      for (int idx = tid; idx < CB * CB; idx += NT) {   // G = sym(H) + 2 I, column-major
        const int i = idx / CB, j = idx - i * CB;
        if (i < j) {
          float v = 0.5f * (Gs[j * LD + i] + Gs[i * LD + j]);
          Gs[j * LD + i] = v;
          Gs[i * LD + j] = v;
        }
      }
      __syncthreads();
      for (int i = tid; i < CB; i += NT) Gs[i * LD + i] += 2.0f;
      __syncthreads();
    }
    GCCB_TICK(2);
    // ---- 48 x 48 Ritz problem: two-sided Jacobi, eigenvectors in Ws (tiles are dead now) ----------
    const bool ritz_skipped = iter == 0 && GCCB_CF_SWEEPS0 == 0;       // W = I: only the ordering below applies
    if (!ritz_skipped)
      jacobi_ritz48<NT>(Gs, Ws, cs, pq, LD, iter == 0 ? 1e-3f : 1e-6f, iter == 0 ? GCCB_CF_SWEEPS0 : GCCB_EIG_MAXSWEEP, &ph[6], &ph[7]);
    GCCB_TICK(3);
    for (int j = tid; j < CB; j += NT) {
      const float mj = Gs[j * LD + j];
      int rank = 0;
      for (int i = 0; i < CB; ++i) {
        float mi = Gs[i * LD + i];
        rank += (mi > mj) || (mi == mj && i < j);
      }
      perm[rank] = j;                                   // descending: perm[0] = largest
    }
    __syncthreads();
    // ---- X <- Q W[:, perm]: one warp per row, lanes over output columns, in place -----------------
    for (int r = warp; r < n; r += NW) {
      const float* w0 = Ws + perm[lane] * LD;
      const float* w1 = Ws + perm[hi ? 32 + lane : 0] * LD;
      const float* row = X + (size_t)r * ld;
      float a0 = 0.f, a1 = 0.f;
      if (ritz_skipped) {                                // a column permutation
        a0 = row[perm[lane]];
        a1 = row[perm[hi ? 32 + lane : 0]];
      } else {
#pragma unroll 8
        for (int i = 0; i < CB; ++i) {
          const float q = row[i];                          // broadcast
          a0 = fmaf(q, w0[i], a0);
          a1 = fmaf(q, w1[i], a1);
        }
      }
      __syncwarp();                                      // all lanes have read row r before it is overwritten
      X[(size_t)r * ld + lane] = a0;
      if (hi) X[(size_t)r * ld + 32 + lane] = a1;
    }
    __syncthreads();
    GCCB_TICK(4);
    // ---- residuals of the wanted pairs: theta_c = x_c . L x_c ; ||L x_c - theta_c x_c|| -----------
    spmm_cheb(S, X, Y, ld, 1.0f, 0.f, 0.f);              // Y = L X
    __syncthreads();
    {
      const float* Xc = X; const float* Yc = Y;
      column_sums(n, part, theta, rr2, 0, [&](int r, int c) { return Xc[(size_t)r * ld + c] * Yc[(size_t)r * ld + c]; });
      column_sums(n, part, resid, rr2, 0, [&](int r, int c) {
        float d = Yc[(size_t)r * ld + c] - theta[c] * Xc[(size_t)r * ld + c];
        return d * d;
      });
    }
    if (tid == 0) {
      float w = 0.f, lo = theta[0], tk = theta[0];
      for (int c = 0; c < k; ++c) { w = fmaxf(w, resid[c]); tk = fminf(tk, theta[c]); }
      for (int i = 1; i < CB; ++i) lo = fminf(lo, theta[i]);
      if (tk < GCCB_CF_MARGIN_BELOW) lo = fminf(lo, tk - GCCB_CF_MARGIN);
      s_bc[0] = sqrtf(w);
      s_bc[1] = lo;
    }
    __syncthreads();
    const float w_all = s_bc[0];
    // converged, or stagnating at the fp32 noise floor of the Rayleigh-Ritz residual
    converged = (w_all < GCCB_CF_TOL) || (iter >= 2 && w_all < GCCB_CF_STAG && w_all > 0.5f * prev_worst);
    prev_worst = w_all;
    cut = fminf(fmaxf(s_bc[1], -0.9f), 0.95f);          // smallest Ritz value of the block
    __syncthreads();
    GCCB_TICK(5);
  }
  if (!converged && tid == 0) atomicOr(flags, (int)GCCB_FLAG_EIG_NOCONV);
  if (tid == 0) {
    dbg_iters[slot] = iter; dbg_res[slot] = prev_worst;
    for (int i = 0; i < 8; ++i) dbg_phase[(size_t)slot * 8 + i] = ph[i];
  }
  // columns 0..k-1 of X hold the k largest Ritz pairs in DESCENDING order; emit ascending
  // (data_util.py: eigsh(which='LA') returns ascending eigenvalues)
  if (eigvals)
    for (int c = tid; c < pos_dim; c += NT) eigvals[(size_t)slot * pos_dim + c] = c < k ? theta[k - 1 - c] : 0.f;
  const float* Xf = X;
  write_features(n, k, pos_dim, normalize, sgn, out,
                 [&](int c, int r) { return Xf[(size_t)r * ld + (k - 1 - c)]; });
}

template <int MODE, int NT>
// register cap: 64 per thread whatever the CTA size, so that 256-thread CTAs run 3 per SM and the
// long-lived large-ego-net CTAs leave half of the register file to concurrent kernels
__global__ void __launch_bounds__(NT, 65536 / 64 / NT)
posenc_chfsi_kernel(const int32_t* __restrict__ worklist, const int32_t* __restrict__ counts, int cls,
                    int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                    const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                    const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                    float* __restrict__ blocks /* [2][2*node_cap*48] */, float* __restrict__ dinv_g /* [2*node_cap] */,
                    float* __restrict__ pos, float* __restrict__ eigvals, int32_t* __restrict__ flags,
                    int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res, long long* __restrict__ dbg_phase) {
  // persistent over the work list: the grid is sized for the typical count, not for 2B
  for (int item = blockIdx.x; item < counts[cls]; item += gridDim.x) {
    posenc_chfsi_item<MODE, NT>(item, worklist, counts, cls, B, node_cap, edge_cap, node_off, b_indptr, b_indices, sub_deg, pos_dim, normalize, blocks, dinv_g, pos, eigvals, flags, dbg_iters, dbg_res, dbg_phase);
    __syncthreads();
  }
}


// ---- solver (3): ChFSI over a thread-block cluster (distributed shared memory), n > 480 ------------
// A hub ego-net (up to ~3400 vertices at the C2 walk budget) would otherwise keep ONE SM busy for
// tens of milliseconds while 147 idle.  Here a cluster of CS CTAs owns it: rows are partitioned,
// each CTA keeps its slice of both n x 48 blocks in its own shared memory, neighbour rows are
// gathered from the owning CTA through DSMEM, column reductions / the 48 x 48 projected matrix are
// all-reduced through a small exchange buffer, and every CTA solves the (identical) Ritz problem
// redundantly.  With CS = 1 the code degenerates to the single-CTA algorithm (that is what the CPU
// emulator exercises); the cluster paths are validated on the GPU by the spectral parity tests.
#ifndef GCCB_EMU
}  // namespace gccb
#include <cooperative_groups.h>
namespace gccb {
namespace cg = cooperative_groups;
#endif

template <int CS> __device__ __forceinline__ int cl_rank() {
#ifndef GCCB_EMU
  if (CS > 1) return (int)cg::this_cluster().block_rank();
#endif
  return 0;
}
template <int CS> __device__ __forceinline__ void cl_sync() {
#ifndef GCCB_EMU
  if (CS > 1) { cg::this_cluster().sync(); return; }
#endif
  __syncthreads();
}
template <int CS> __device__ __forceinline__ const float* cl_map(const float* p, int rank) {
#ifndef GCCB_EMU
  if (CS > 1) return (const float*)cg::this_cluster().map_shared_rank((void*)p, (unsigned)rank);
#endif
  return p;
}

#define GCCB_CL_HEAVY 192          // rows with more neighbours are processed by the whole CTA
#define GCCB_CL_MAXHEAVY 16

template <int NT, int CS>
struct ClCtx {
  const int32_t* indptr; const int32_t* indices; const float* dinv;
  int noff, n, R, rank, r_lo, nloc, ld;
  float* part;          // [32][48] block scratch
  float* xch;           // [2][48] cluster exchange (own shared memory)
  int xbuf;
  const int* heavy; int nheavy;
};

// row j of a row-partitioned block whose local slice starts at `base`
template <int NT, int CS>
__device__ __forceinline__ const float* cl_row(const ClCtx<NT, CS>& c, const float* base, int j) {
  const int owner = j / c.R, loc = j - owner * c.R;
  const float* p = base + (size_t)loc * c.ld;
  return owner == c.rank ? p : cl_map<CS>(p, owner);
}

// dst_loc[r][c] = alpha * (sum_j w_rj src[j][c] - cen * src[r][c]) - beta * dst_loc[r][c] over OWNED rows
template <int NT, int CS>
__device__ __forceinline__ void cl_spmm(const ClCtx<NT, CS>& C, const float* src, float* dst, float alpha,
                                        float cen, float beta) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = NT / 32;
  const bool hi = lane < GCCB_CF_B - 32;
  for (int rl = warp; rl < C.nloc; rl += NW) {
    const int r = C.r_lo + rl;
    const int beg = C.indptr[C.noff + r], end = C.indptr[C.noff + r + 1];
    if (end - beg > GCCB_CL_HEAVY && C.nheavy > 0) {
      bool listed = false;
      for (int h = 0; h < C.nheavy; ++h) listed |= C.heavy[h] == rl;
      if (listed) continue;                              // done cooperatively below
    }
    const float dr = C.dinv[r];
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
    int e = beg;
    for (; e + 3 < end; e += 4) {
      const int j0 = C.indices[e] - C.noff, j1 = C.indices[e + 1] - C.noff;
      const int j2 = C.indices[e + 2] - C.noff, j3 = C.indices[e + 3] - C.noff;
      const float* p0 = cl_row(C, src, j0); const float* p1 = cl_row(C, src, j1);
      const float* p2 = cl_row(C, src, j2); const float* p3 = cl_row(C, src, j3);
      const float x0 = p0[lane], x1 = p1[lane], x2 = p2[lane], x3 = p3[lane];
      float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;
      if (hi) { y0 = p0[32 + lane]; y1 = p1[32 + lane]; y2 = p2[32 + lane]; y3 = p3[32 + lane]; }
      const float w0 = dr * C.dinv[j0], w1 = dr * C.dinv[j1], w2 = dr * C.dinv[j2], w3 = dr * C.dinv[j3];
      a0 = fmaf(w0, x0, a0); b0 = fmaf(w1, x1, b0); a0 = fmaf(w2, x2, a0); b0 = fmaf(w3, x3, b0);
      a1 = fmaf(w0, y0, a1); b1 = fmaf(w1, y1, b1); a1 = fmaf(w2, y2, a1); b1 = fmaf(w3, y3, b1);
    }
    for (; e < end; ++e) {
      const int j0 = C.indices[e] - C.noff;
      const float* p0 = cl_row(C, src, j0);
      const float w0 = dr * C.dinv[j0];
      a0 = fmaf(w0, p0[lane], a0);
      if (hi) a1 = fmaf(w0, p0[32 + lane], a1);
    }
    a0 += b0; a1 += b1;
    const size_t o = (size_t)rl * C.ld + lane;
    float v = alpha * (a0 - cen * src[o]);
    if (beta != 0.f) v -= beta * dst[o];
    dst[o] = v;
    if (hi) {
      float v1 = alpha * (a1 - cen * src[o + 32]);
      if (beta != 0.f) v1 -= beta * dst[o + 32];
      dst[o + 32] = v1;
    }
  }
  // hub rows: every warp takes a slice of the neighbour list, partial rows meet in part[][]
  for (int h = 0; h < C.nheavy; ++h) {
    const int rl = C.heavy[h], r = C.r_lo + rl;
    const int beg = C.indptr[C.noff + r], end = C.indptr[C.noff + r + 1];
    const int per = (end - beg + NW - 1) / NW;
    const int e0 = beg + warp * per, e1 = min(end, e0 + per);
    const float dr = C.dinv[r];
    float a0 = 0.f, a1 = 0.f;
    for (int e = e0; e < e1; ++e) {
      const int j0 = C.indices[e] - C.noff;
      const float* p0 = cl_row(C, src, j0);
      const float w0 = dr * C.dinv[j0];
      a0 = fmaf(w0, p0[lane], a0);
      if (hi) a1 = fmaf(w0, p0[32 + lane], a1);
    }
    __syncthreads();                                     // part[] free
    C.part[warp * GCCB_CF_B + lane] = a0;
    if (hi) C.part[warp * GCCB_CF_B + 32 + lane] = a1;
    __syncthreads();
    for (int c = threadIdx.x; c < GCCB_CF_B; c += NT) {
      float sacc = 0.f;
      for (int w = 0; w < NW; ++w) sacc += C.part[w * GCCB_CF_B + c];
      const size_t o = (size_t)rl * C.ld + c;
      float v = alpha * (sacc - cen * src[o]);
      if (beta != 0.f) v -= beta * dst[o];
      dst[o] = v;
    }
  }
}

// cluster-wide per-column sums of f(local row, column) -> out[48] (identical on every CTA);
// rr2[0] + rr2[1] = sum_{c < jlim} out[c]^2
template <int NT, int CS, class RowFn>
__device__ __forceinline__ void cl_column_sums(ClCtx<NT, CS>& C, float* out, float* rr2, int jlim, RowFn f) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = NT / 32, NWU = NW < 8 ? NW : 8;
  const bool hi = lane < GCCB_CF_B - 32;
  if (warp < NWU) {
    float a0 = 0.f, a1 = 0.f;
    for (int rl = warp; rl < C.nloc; rl += NWU) {
      a0 += f(rl, lane);
      if (hi) a1 += f(rl, 32 + lane);
    }
    C.part[warp * GCCB_CF_B + lane] = a0;
    if (hi) C.part[warp * GCCB_CF_B + 32 + lane] = a1;
  }
  __syncthreads();
  float* mine = C.xch + C.xbuf * GCCB_CF_B;
  float sacc = 0.f;
  const int c = threadIdx.x;
  if (c < GCCB_CF_B) {
#pragma unroll
    for (int w = 0; w < NWU; ++w) sacc += C.part[w * GCCB_CF_B + c];
    if (CS > 1) mine[c] = sacc;
  }
  if (CS > 1) {
    cl_sync<CS>();
    if (c < GCCB_CF_B) {
      sacc = 0.f;
#pragma unroll
      for (int q = 0; q < CS; ++q) sacc += cl_map<CS>(mine, q)[c];     // fixed rank order: deterministic
    }
    C.xbuf ^= 1;
  }
  if (c < 64) {
    if (c < GCCB_CF_B) out[c] = sacc;
    float sq = c < jlim ? sacc * sacc : 0.f;
    sq = warp_sum(sq);
    if (lane == 0) rr2[warp] = sq;
  }
  __syncthreads();
}

template <int NT, int CS>
// register cap: 64 per thread whatever the CTA size, so that 256-thread CTAs run 3 per SM and the
// long-lived large-ego-net CTAs leave half of the register file to concurrent kernels
__global__ void __launch_bounds__(NT, 65536 / 64 / NT)
posenc_chfsi_cluster_kernel(const int32_t* __restrict__ worklist, const int32_t* __restrict__ counts, int cls,
                            int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                            const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                            const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                            float* __restrict__ dinv_g, float* __restrict__ pos, float* __restrict__ eigvals,
                            int32_t* __restrict__ flags, int32_t* __restrict__ dbg_iters,
                            float* __restrict__ dbg_res, long long* __restrict__ dbg_phase) {
  constexpr int CB = GCCB_CF_B, LD = CB + 1, NW = NT / 32;
  GCCB_DYN_SMEM(float, dynsm);
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t_last = GCCB_CLK();
  __shared__ float Gs[CB * LD];                   // Ritz problem
  __shared__ float Hp[CB * LD];                   // this CTA's partial of H (read by the others)
  __shared__ float WT[32 * (CB + 1) * 2];         // union: Ritz vectors Ws[CB*LD] | tiles [2][32][CB+1]
  __shared__ float part[32 * CB];
  __shared__ float xch[2 * CB + 8];
  __shared__ float rdot[CB];
  __shared__ float rr2[2];
  __shared__ float theta[CB];
  __shared__ float resid[CB];
  __shared__ float cs[64];
  __shared__ int pq[32];
  __shared__ int perm[CB];
  __shared__ int heavy[GCCB_CL_MAXHEAVY];
  __shared__ int s_nheavy;
  __shared__ float s_bc[2];
  __shared__ float sgn[32];
  float* Ws = WT;
  float (*tile)[32][CB + 1] = reinterpret_cast<float (*)[32][CB + 1]>(WT);
  for (int item = blockIdx.x / CS; item < counts[cls]; item += gridDim.x / CS) {   // uniform over the cluster
  const int slot = worklist[(size_t)cls * 2 * B + item];
  const int view = slot / B, g = slot - view * B;
  const int noff = node_off[view * (B + 1) + g];
  const int n = node_off[view * (B + 1) + g + 1] - noff;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool hi = lane < CB - 32;
  const int k = min(n - 2, pos_dim);
  ClCtx<NT, CS> C;
  C.indptr = b_indptr + (size_t)view * (node_cap + 1);
  C.indices = b_indices + (size_t)view * edge_cap;
  float* dinv = dinv_g + (size_t)view * node_cap + noff;
  C.dinv = dinv;
  C.noff = noff; C.n = n;
  C.R = (n + CS - 1) / CS;
  C.rank = cl_rank<CS>();
  C.r_lo = C.rank * C.R;
  C.nloc = max(0, min(n, C.r_lo + C.R) - C.r_lo);
  C.ld = LD;
  C.part = part; C.xch = xch; C.xbuf = 0; C.heavy = heavy;
  const int nloc = C.nloc, r_lo = C.r_lo, ld = LD;
  float* X = dynsm;                                     // local slices: R x 49 each
  float* Y = dynsm + (size_t)C.R * LD;
  const int32_t* v_deg = sub_deg + (size_t)view * node_cap;
  if (tid == 0) s_nheavy = 0;
  __syncthreads();
  for (int rl = tid; rl < nloc; rl += NT) {
    int d = v_deg[noff + r_lo + rl];
    if (d > GCCB_CL_HEAVY) {
      int h = atomicAdd(&s_nheavy, 1);
      if (h < GCCB_CL_MAXHEAVY) heavy[h] = rl;
    }
  }
  // every CTA needs all of dinv (neighbour weights): each writes its own rows, visible after the sync
  for (int rl = tid; rl < nloc; rl += NT) {
    int d = v_deg[noff + r_lo + rl];
    dinv[r_lo + rl] = 1.0f / sqrtf((float)(d < 1 ? 1 : d));
  }
  for (int i = tid; i < nloc * CB; i += NT) {
    const int rl = i / CB, c = i - rl * CB;
    const uint32_t gi = (uint32_t)((r_lo + rl) * CB + c);           // same stream as the single-CTA kernel
    u32x4 w = philox4x32_10(gi, (uint32_t)n, 0x51ED270Bu, 3u, 0xC0FFEEu, 0x5EEDu);
    X[(size_t)rl * ld + c] = (float)(int32_t)w.x * (1.0f / 2147483648.0f);
  }
  __threadfence();                                       // dinv[] (global) before the other CTAs read it
  cl_sync<CS>();
  C.nheavy = min(s_nheavy, GCCB_CL_MAXHEAVY);
  float cut = 0.0f, prev_worst = 3.0e38f;
  bool converged = false;
  int iter = 0;
  for (; iter < GCCB_CF_MAXIT && !converged; ++iter) {
    {   // ---- Chebyshev filter ---------------------------------------------------------------------
      const float e = (cut + 1.0f) * 0.5f, cen = (cut - 1.0f) * 0.5f;
      int deg = (int)floorf(GCCB_CF_LOGGAIN / acoshf((3.0f - cut) / (1.0f + cut)));
      deg = max(4, min(iter == 0 ? GCCB_CF_DEG0 : GCCB_CF_DEG, deg));
      float sigma = e / (1.0f - cen);
      const float sigma1 = sigma;
      cl_spmm(C, X, Y, sigma1 / e, cen, 0.f);
      cl_sync<CS>();
      float* cur = Y; float* prev = X;
      for (int i = 2; i <= deg; ++i) {
        const float sigma2 = 1.0f / (2.0f / sigma1 - sigma);
        cl_spmm(C, cur, prev, 2.0f * sigma2 / e, cen, sigma * sigma2);
        cl_sync<CS>();
        float* t = cur; cur = prev; prev = t;
        sigma = sigma2;
      }
      X = cur; Y = prev;
    }
    GCCB_TICK(0);
    // ---- CGS2 over the cluster --------------------------------------------------------------------
    for (int j = 0; j < CB; ++j) {
      float nrm2 = 0.f;
      bool scaled = false;
      for (int pass = 0; pass < 2; ++pass) {
        const float* Xc = X;
        cl_column_sums(C, rdot, rr2, j, [&](int rl, int c) { return Xc[(size_t)rl * ld + c] * Xc[(size_t)rl * ld + j]; });
        const float yy = rdot[j];
        const float rr = rr2[0] + rr2[1];
        nrm2 = yy - rr;
        scaled = nrm2 > 0.5f * yy && nrm2 > 1e-30f;      // last pass: normalise in the same sweep
        const float sc = scaled ? 1.0f / sqrtf(nrm2) : 1.0f;
        for (int rl = tid; rl < nloc; rl += NT) {
          float* row = X + (size_t)rl * ld;
          float v0 = row[j], v1 = 0.f;
          int i = 0;
          for (; i + 1 < j; i += 2) {
            v0 = fmaf(-rdot[i], row[i], v0);
            v1 = fmaf(-rdot[i + 1], row[i + 1], v1);
          }
          if (i < j) v0 = fmaf(-rdot[i], row[i], v0);
          row[j] = (v0 + v1) * sc;
        }
        __syncthreads();
        if (nrm2 > 0.5f * yy) break;                     // identical decision on every CTA (same rdot bits)
      }
      if (!scaled) {
        if (!(nrm2 > 1e-30f)) {
          const float* Xc = X;
          cl_column_sums(C, rdot, rr2, 0, [&](int rl, int c) { return c == j ? Xc[(size_t)rl * ld + j] * Xc[(size_t)rl * ld + j] : 0.f; });
          nrm2 = rdot[j];
        }
        const float inv = nrm2 > 1e-30f ? 1.0f / sqrtf(nrm2) : 0.f;
        for (int rl = tid; rl < nloc; rl += NT) X[(size_t)rl * ld + j] *= inv;
        __syncthreads();
      }
    }
    GCCB_TICK(1);
    // ---- Z = L Q, H = Q^T Z (partial per CTA, summed over the cluster) -------------------------------
    cl_sync<CS>();                                       // every slice of Q final before remote gathers
    cl_spmm(C, X, Y, 1.0f, 0.f, 0.f);
    __syncthreads();
    {
      const int ti = (tid & 255) >> 4, tj = tid & 15;
      float acc[3][3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b2 = 0; b2 < 3; ++b2) acc[a][b2] = 0.f;
      for (int r0 = 0; r0 < nloc; r0 += 32) {
        for (int idx = tid; idx < 32 * CB; idx += NT) {
          const int rr = idx / CB, c = idx - rr * CB;
          const int rl = r0 + rr;
          tile[0][rr][c] = rl < nloc ? X[(size_t)rl * ld + c] : 0.f;
          tile[1][rr][c] = rl < nloc ? Y[(size_t)rl * ld + c] : 0.f;
        }
        __syncthreads();
        if (tid < 256) {
#pragma unroll 4
          for (int rr = 0; rr < 32; ++rr) {
            float qa[3], zb[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) { qa[a] = tile[0][rr][ti * 3 + a]; zb[a] = tile[1][rr][tj * 3 + a]; }
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
              for (int b2 = 0; b2 < 3; ++b2) acc[a][b2] = fmaf(qa[a], zb[b2], acc[a][b2]);
          }
        }
        __syncthreads();
      }
      if (tid < 256) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b2 = 0; b2 < 3; ++b2) Hp[(tj * 3 + b2) * LD + ti * 3 + a] = acc[a][b2];
      }
      cl_sync<CS>();
      for (int idx = tid; idx < CB * CB; idx += NT) {   // all-reduce of the partials, fixed rank order
        const int j = idx / CB, i = idx - j * CB;
        float sacc = 0.f;
        for (int q = 0; q < CS; ++q) sacc += cl_map<CS>(Hp, q)[j * LD + i];
        Gs[j * LD + i] = sacc;
      }
      __syncthreads();
      for (int idx = tid; idx < CB * CB; idx += NT) {   // G = sym(H) + 2 I
        const int i = idx / CB, j = idx - i * CB;
        if (i < j) {
          float v = 0.5f * (Gs[j * LD + i] + Gs[i * LD + j]);
          Gs[j * LD + i] = v;
          Gs[i * LD + j] = v;
        }
      }
      __syncthreads();
      for (int i = tid; i < CB; i += NT) Gs[i * LD + i] += 2.0f;
      __syncthreads();
    }
    GCCB_TICK(2);
    jacobi_ritz48<NT>(Gs, Ws, cs, pq, LD, iter == 0 ? 1e-3f : 1e-6f, iter == 0 ? GCCB_CF_SWEEPS0_CLUSTER : GCCB_EIG_MAXSWEEP, &ph[6], &ph[7]);   // redundant per CTA, bit-identical
    GCCB_TICK(3);
    for (int j = tid; j < CB; j += NT) {
      const float mj = Gs[j * LD + j];
      int rank = 0;
      for (int i = 0; i < CB; ++i) {
        float mi = Gs[i * LD + i];
        rank += (mi > mj) || (mi == mj && i < j);
      }
      perm[rank] = j;
    }
    __syncthreads();
    for (int rl = warp; rl < nloc; rl += NW) {            // X <- Q W[:, perm] on the owned rows
      const float* w0 = Ws + perm[lane] * LD;
      const float* w1 = Ws + perm[hi ? 32 + lane : 0] * LD;
      const float* row = X + (size_t)rl * ld;
      float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
      for (int i = 0; i < CB; ++i) {
        const float q = row[i];
        a0 = fmaf(q, w0[i], a0);
        a1 = fmaf(q, w1[i], a1);
      }
      __syncwarp();
      X[(size_t)rl * ld + lane] = a0;
      if (hi) X[(size_t)rl * ld + 32 + lane] = a1;
    }
    cl_sync<CS>();                                       // also orders the Hp reads before its next write
    GCCB_TICK(4);
    cl_spmm(C, X, Y, 1.0f, 0.f, 0.f);                    // Y = L X
    __syncthreads();
    {
      const float* Xc = X; const float* Yc = Y;
      cl_column_sums(C, theta, rr2, 0, [&](int rl, int c) { return Xc[(size_t)rl * ld + c] * Yc[(size_t)rl * ld + c]; });
      cl_column_sums(C, resid, rr2, 0, [&](int rl, int c) {
        float d = Yc[(size_t)rl * ld + c] - theta[c] * Xc[(size_t)rl * ld + c];
        return d * d;
      });
    }
    if (tid == 0) {
      float w = 0.f, lo = theta[0], tk = theta[0];
      for (int c = 0; c < k; ++c) { w = fmaxf(w, resid[c]); tk = fminf(tk, theta[c]); }
      for (int i = 1; i < CB; ++i) lo = fminf(lo, theta[i]);
      if (tk < GCCB_CF_MARGIN_BELOW) lo = fminf(lo, tk - GCCB_CF_MARGIN);
      s_bc[0] = sqrtf(w);
      s_bc[1] = lo;
    }
    __syncthreads();
    const float w_all = s_bc[0];
    converged = (w_all < GCCB_CF_TOL) || (iter >= 2 && w_all < GCCB_CF_STAG && w_all > 0.5f * prev_worst);
    prev_worst = w_all;
    cut = fminf(fmaxf(s_bc[1], -0.9f), 0.95f);
    __syncthreads();
    GCCB_TICK(5);
  }
  if (C.rank == 0 && tid == 0) {
    if (!converged) atomicOr(flags, (int)GCCB_FLAG_EIG_NOCONV);
    dbg_iters[slot] = iter; dbg_res[slot] = prev_worst;
    for (int i = 0; i < 8; ++i) dbg_phase[(size_t)slot * 8 + i] = ph[i];
  }
  if (eigvals && C.rank == 0)
    for (int c = tid; c < pos_dim; c += NT) eigvals[(size_t)slot * pos_dim + c] = c < k ? theta[k - 1 - c] : 0.f;
  // deterministic sign: largest-|.| component over ALL rows (lowest row on ties) positive
  {
    float* best = part;                 // [48] value of max |x|, [48..96) row, [96..144) signed value
    for (int c = warp; c < k; c += NW) {
      float bb = -1.f, bval = 0.f; int brow = 0x7fffffff;
      for (int rl = lane; rl < nloc; rl += 32) {
        float x = X[(size_t)rl * ld + (k - 1 - c)], a = fabsf(x);
        if (a > bb) { bb = a; brow = r_lo + rl; bval = x; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float ob = __shfl_xor_sync(0xffffffffu, bb, o);
        int orow = __shfl_xor_sync(0xffffffffu, brow, o);
        float ov = __shfl_xor_sync(0xffffffffu, bval, o);
        if (ob > bb || (ob == bb && orow < brow)) { bb = ob; brow = orow; bval = ov; }
      }
      if (lane == 0) { best[c] = bb; best[48 + c] = __int_as_float(brow); best[96 + c] = bval; }
    }
    cl_sync<CS>();
    for (int c = tid; c < k; c += NT) {
      float bb = -1.f, bval = 0.f; int brow = 0x7fffffff;
      for (int q = 0; q < CS; ++q) {
        const float* rb = cl_map<CS>(best, q);
        float ob = rb[c]; int orow = __float_as_int(rb[48 + c]); float ov = rb[96 + c];
        if (ob > bb || (ob == bb && orow < brow)) { bb = ob; brow = orow; bval = ov; }
      }
      sgn[c] = bval < 0.f ? -1.0f : 1.0f;
    }
    __syncthreads();
  }
  float* out = pos + ((size_t)view * node_cap + noff) * pos_dim;
  for (int rl = warp; rl < nloc; rl += NW) {
    float u = 0.f;
    if (lane < k) u = sgn[lane] * X[(size_t)rl * ld + (k - 1 - lane)];
    if (normalize) {
      float ss = warp_sum(u * u);
      if (ss > 0.f) u = u / sqrtf(ss);
    }
    if (lane < pos_dim) out[(size_t)(r_lo + rl) * pos_dim + lane] = u;
  }
  cl_sync<CS>();                                         // nobody leaves while its shared memory is still read
  }
}

// ---- solver (0): dense tridiagonal path, n <= GCCB_DN_C ------------------------------------------------
// Ego-nets are small (C2 workload: mean 104 vertices, 97 % below 230): the whole normalised adjacency matrix fits
// in the shared memory of one CTA, and the textbook dense symmetric eigensolver is both cheaper and more accurate
// in fp32 than any subspace iteration (measured on the fp32 model of this kernel, C2 ego-nets and the degenerate
// test graphs: eigenvalues to 4e-7, residuals to 5e-6, orthonormality to 1e-6, the reference's own simple-spectrum
// goldens elementwise to 2e-6; ChFSI: 2e-5 / 4e-5 / 1e-4):
//
//   1. Householder tridiagonalisation Q^T L Q = T, unblocked, full symmetric storage (row stride = 8 mod 32, two
//      threads per row reading 128-bit words: conflict-free), TWO barriers per column: the product S v is taken
//      from the raw column x (v = scale * (x - beta e1), so S v = scale * (S x - beta S e1)) and overlaps the
//      norm of x, every warp computes the scalars redundantly, w = p - gamma v is formed on the fly inside the
//      rank-2 update, and the update hands the next column over in contiguous form;
//   2. the k <= 32 largest eigenvalues of T by multisection on Sturm counts (all threads: a first cut of the
//      Gershgorin interval into NT + 1 pieces, then NT / 32 points per eigenvalue and round; 5 / 4 rounds);
//   3. eigenvectors of T by inverse iteration, one lane per eigenvalue (Gaussian elimination with partial
//      pivoting; pivot rows that were swapped are original matrix entries, so two floats per row describe the
//      factor -- kept in the L2-resident workspace, written coalesced, read back with one block prefetched), three
//      iterations from a counter-based pseudo-random start, ONE common shift per multiple eigenvalue (see there);
//   4. modified Gram-Schmidt over the k vectors (lanes = columns: conflict-free; degenerate clusters -- the null
//      space of a near-tree reaches multiplicity 30+ -- come out as an orthonormal basis), one pass after the second
//      and one after the third inverse iteration (see the comment at the loop);
//   5. back-transformation X = Q Z: every warp applies all n - 2 reflectors to its own columns held in registers
//      (no barriers);
//   6. a residual check against the sparse matrix (reported per ego-net; NOCONV above GCCB_DN_RES_FLAG).
//
// Z (n x 32) lives in the dead upper-right corner of the matrix (rows < n - 32, columns >= n - 32) plus a 32 x 32 tail.
#define GCCB_DN_A 96
#define GCCB_DN_B 144
#define GCCB_DN_C 228
#ifndef GCCB_DN_INVIT
#define GCCB_DN_INVIT 3
#endif
#ifndef GCCB_DN_MGS
#define GCCB_DN_MGS 1              // Gram-Schmidt passes after the LAST inverse iteration (one after each earlier one)
#endif
#define GCCB_DN_PIVMIN 1.0e-30f
#define GCCB_DN_GUARD 1.0e-9f      // smallest pivot of the inverse iteration (a perturbation far below eps * ||T||)
#define GCCB_DN_TIGHT 2.0e-6f      // eigenvalues closer than this form a group with one common shift ...
#define GCCB_DN_DELTA 4.0e-6f      // ... this far outside the group
#define GCCB_DN_GAPTOL 1.0e-2f     // Gram-Schmidt links eigenvalues closer than this
#define GCCB_DN_RES_FLAG 1.0e-3f


__host__ __device__ constexpr int dn_ld(int n) { return ((n + 23) / 32) * 32 + 8; }   // >= n, = 8 mod 32

// number of eigenvalues of T below x
__device__ __forceinline__ int dn_sturm(const float* __restrict__ d, const float* __restrict__ e2, int n, float x) {
  float q = d[0] - x;
  if (fabsf(q) < GCCB_DN_PIVMIN) q = -GCCB_DN_PIVMIN;
  int c = q < 0.f ? 1 : 0;
  for (int i = 1; i < n; ++i) {
    q = (d[i] - x) - __fdividef(e2[i - 1], q);
    if (fabsf(q) < GCCB_DN_PIVMIN) q = -GCCB_DN_PIVMIN;
    c += q < 0.f ? 1 : 0;
  }
  return c;
}

template <int NMAX, int NT, bool USM>
__device__ __forceinline__ void posenc_dense_item(const int slot, int B, int node_cap, int edge_cap,
                    const int32_t* __restrict__ node_off, const int32_t* __restrict__ b_indptr,
                    const int32_t* __restrict__ b_indices, const int32_t* __restrict__ sub_deg, int pos_dim, int normalize,
                    float* __restrict__ blocks, float* __restrict__ pos, float* __restrict__ eigvals,
                    int32_t* __restrict__ flags, int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res,
                    long long* __restrict__ dbg_phase) {
  constexpr int NW = NT / 32, NP = ((NMAX + 3) & ~3) + 4, NR = (NMAX + 31) / 32, CPW = 32 / NW;
  static_assert(NT >= 2 * NMAX && NW <= 32 && 32 % NW == 0, "two threads per matrix row");
  GCCB_DYN_SMEM(float, A);                              // n x ld, row-major
  // (128-bit accesses to vbuf / pbuf / xbuf: every array gets its own aligned declaration)
  __align__(16) __shared__ float d[NP];
  __align__(16) __shared__ float e[NP];
  __align__(16) __shared__ float e2[NP];
  __align__(16) __shared__ float taus[NP];
  __align__(16) __shared__ float vbuf[NP];
  __align__(16) __shared__ float pbuf[NP];
  __align__(16) __shared__ float xbuf[NP];
  __align__(16) __shared__ float dinv[NP];
  __shared__ float ztail[32 * 32];
  __shared__ float lam[32], lamp[32], lo[32], hi[32], sgn[32];
  __shared__ int cnt[NT];
  __shared__ float part[NW * 32];
  __shared__ float ufac[USM ? 2 * 32 * NMAX : 1];        // factor rows of the inverse iteration (USM: else in L2)
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t_last = GCCB_CLK();
  const int view = slot / B, g = slot - view * B;
  const int noff = node_off[view * (B + 1) + g];
  const int n = node_off[view * (B + 1) + g + 1] - noff;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = min(n - 2, pos_dim);
  float* out = pos + ((size_t)view * node_cap + noff) * pos_dim;
  if (k <= 0) {                                         // data_util.py:243-244
    for (int i = tid; i < n * pos_dim; i += NT) out[i] = 0.f;
    if (eigvals)
      for (int i = tid; i < pos_dim; i += NT) eigvals[(size_t)slot * pos_dim + i] = 0.f;
    if (tid == 0) { dbg_iters[slot] = 0; dbg_res[slot] = 0.f; }
    return;
  }
  const int ld = dn_ld(n);
  const int zb = n > 32 ? n - 32 : 0;                   // rows below zb keep their Z row inside the matrix
  auto zrow = [&](int i) -> float* { return i < zb ? A + (size_t)i * ld + (n - 32) : ztail + (i - zb) * 32; };
  const int32_t* v_indptr = b_indptr + (size_t)view * (node_cap + 1);
  const int32_t* v_indices = b_indices + (size_t)view * edge_cap;
  const int32_t* v_deg = sub_deg + (size_t)view * node_cap;
  // factor rows of the inverse iteration: two n x 32 arrays in this ego-net's part of the L2 workspace
  float* U0 = USM ? ufac : blocks + ((size_t)view * node_cap + noff) * (GCCB_CF_B + 1);
  float* U1 = USM ? ufac + 32 * NMAX : U0 + (size_t)2 * node_cap * (GCCB_CF_B + 1);
  // ---- the matrix ---------------------------------------------------------------------------------------------
  for (int i = tid; i < NP; i += NT) { d[i] = 0.f; e[i] = 0.f; e2[i] = 0.f; taus[i] = 0.f; vbuf[i] = 0.f; pbuf[i] = 0.f; xbuf[i] = 0.f; }
  for (int i = tid; i < n; i += NT) {
    int dg = v_deg[noff + i];
    dinv[i] = 1.0f / sqrtf((float)(dg < 1 ? 1 : dg));  // in_degrees().clip(1) ** -0.5
  }
  {
    float4* A4 = reinterpret_cast<float4*>(A);
    for (int i = tid; i < n * ld / 4; i += NT) A4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  for (int i = warp; i < n; i += NW) {                  // row i <- its in-neighbours j (multi-edges add up)
    const int beg = v_indptr[noff + i], end = v_indptr[noff + i + 1];
    const float di = dinv[i];
    for (int ed = beg + lane; ed < end; ed += 32) {
      int j = v_indices[ed] - noff;
      atomicAdd(&A[(size_t)j * ld + i], di * dinv[j]);  // shared-memory adds of exact products
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += NT) xbuf[i] = i >= 1 ? A[(size_t)i * ld] : 0.f;
  __syncthreads();
  GCCB_TICK(0);
  // ---- 1. Householder tridiagonalisation -------------------------------------------------------------------------
  {
    const int r = tid >> 1, h = tid & 1;
    float* row = A + (size_t)r * ld;
    for (int kk = 0; kk + 2 < n; ++kk) {
      const int c0 = (kk + 1) & ~3;
      const bool mine = r > kk && r < n;
      if (warp * 16 + 15 <= kk || warp * 16 >= n) {        // no live row in this warp (rows 16 w .. 16 w + 15)
        __syncthreads();
        __syncthreads();
        continue;
      }
      float y = 0.f;
      if (mine) {                                       // y = (S x)_r over this thread's half of the row
        float y0 = 0.f, y1 = 0.f;
        int c = c0 + 4 * h;
        for (; c + 8 < n; c += 16) {                      // two chunks per trip: four loads in flight
          const float4 a = *reinterpret_cast<const float4*>(row + c);
          const float4 x = *reinterpret_cast<const float4*>(xbuf + c);
          const float4 a2 = *reinterpret_cast<const float4*>(row + c + 8);
          const float4 x2 = *reinterpret_cast<const float4*>(xbuf + c + 8);
          y0 = fmaf(a.x, x.x, y0);
          y1 = fmaf(a.y, x.y, y1);
          y0 = fmaf(a.z, x.z, y0);
          y1 = fmaf(a.w, x.w, y1);
          y0 = fmaf(a2.x, x2.x, y0);
          y1 = fmaf(a2.y, x2.y, y1);
          y0 = fmaf(a2.z, x2.z, y0);
          y1 = fmaf(a2.w, x2.w, y1);
        }
        if (c < n) {
          const float4 a = *reinterpret_cast<const float4*>(row + c);
          const float4 x = *reinterpret_cast<const float4*>(xbuf + c);
          y0 = fmaf(a.x, x.x, y0);
          y1 = fmaf(a.y, x.y, y1);
          y0 = fmaf(a.z, x.z, y0);
          y1 = fmaf(a.w, x.w, y1);
        }
        y = y0 + y1;
      }
      y += __shfl_xor_sync(0xffffffffu, y, 1);
      float s = 0.f;                                    // every warp: ||x(kk+2:)||^2
      for (int i = kk + 2 + lane; i < n; i += 32) { const float t = xbuf[i]; s = fmaf(t, t, s); }
      s = warp_sum(s);
      const float alpha = xbuf[kk + 1];
      float tau = 0.f, beta = alpha, scale = 0.f;
      if (s > 1.0e-30f) {
        beta = -copysignf(sqrtf(fmaf(alpha, alpha, s)), alpha);
        tau = (beta - alpha) / beta;
        scale = 1.0f / (alpha - beta);
      }
      if (mine && h == 0) {
        const float vr = r == kk + 1 ? 1.0f : xbuf[r] * scale;
        vbuf[r] = vr;
        pbuf[r] = tau * scale * (y - beta * row[kk + 1]);
        row[kk] = vr;                                   // the reflector stays in column kk for step 5
      }
      if (tid == 2 * (kk + 1)) {                          // row kk + 1 is always live
        vbuf[kk] = 0.f; pbuf[kk] = 0.f;
        d[kk] = A[(size_t)kk * ld + kk]; e[kk] = beta; taus[kk] = tau;
      }
      __syncthreads();
      if (tau != 0.f) {
        float gs = 0.f;                                 // every warp: gamma = tau/2 * p.v
        for (int i = kk + 1 + lane; i < n; i += 32) gs = fmaf(pbuf[i], vbuf[i], gs);
        const float gam = 0.5f * tau * warp_sum(gs);
        if (mine) {
          const float vr = vbuf[r], wr = fmaf(-gam, vr, pbuf[r]);
          const float nvr = -vr, nwr = -wr;
          auto upd = [&](float4& a, const float4& v4, const float4& p4) {   // S -= v w^T + w v^T, w = p - gamma v
            a.x = fmaf(nwr, v4.x, fmaf(nvr, fmaf(-gam, v4.x, p4.x), a.x));
            a.y = fmaf(nwr, v4.y, fmaf(nvr, fmaf(-gam, v4.y, p4.y), a.y));
            a.z = fmaf(nwr, v4.z, fmaf(nvr, fmaf(-gam, v4.z, p4.z), a.z));
            a.w = fmaf(nwr, v4.w, fmaf(nvr, fmaf(-gam, v4.w, p4.w), a.w));
          };
          int c = c0 + 4 * h;
          for (; c + 8 < n; c += 16) {                    // two chunks per trip: six loads in flight, then the stores
            float4 a = *reinterpret_cast<float4*>(row + c);
            const float4 v4 = *reinterpret_cast<const float4*>(vbuf + c);
            const float4 p4 = *reinterpret_cast<const float4*>(pbuf + c);
            float4 a2 = *reinterpret_cast<float4*>(row + c + 8);
            const float4 v42 = *reinterpret_cast<const float4*>(vbuf + c + 8);
            const float4 p42 = *reinterpret_cast<const float4*>(pbuf + c + 8);
            upd(a, v4, p4);
            upd(a2, v42, p42);
            *reinterpret_cast<float4*>(row + c) = a;
            *reinterpret_cast<float4*>(row + c + 8) = a2;
          }
          if (c < n) {
            float4 a = *reinterpret_cast<float4*>(row + c);
            const float4 v4 = *reinterpret_cast<const float4*>(vbuf + c);
            const float4 p4 = *reinterpret_cast<const float4*>(pbuf + c);
            upd(a, v4, p4);
            *reinterpret_cast<float4*>(row + c) = a;
          }
        }
      }
      // the next column in contiguous form, from the thread that owns that element of its row
      if (r > kk + 1 && r < n && h == 0) xbuf[r] = row[kk + 1];   // column kk+1 is in the first 4-column chunk
      if (tid == 2 * (kk + 1)) xbuf[kk + 1] = 0.f;
      __syncthreads();
    }
    if (tid == 0) {
      d[n - 2] = A[(size_t)(n - 2) * ld + n - 2];
      d[n - 1] = A[(size_t)(n - 1) * ld + n - 1];
      e[n - 2] = A[(size_t)(n - 1) * ld + n - 2];
    }
    __syncthreads();
    for (int i = tid; i + 1 < n; i += NT) e2[i] = e[i] * e[i];
    __syncthreads();
  }
  GCCB_TICK(1);
  // ---- 2. the k largest eigenvalues of T: multisection on Sturm counts -------------------------------------------
  {
    float gl = 3.0e38f, gu = -3.0e38f;                    // Gershgorin interval (every warp)
    for (int i = lane; i < n; i += 32) {
      const float rad = (i > 0 ? fabsf(e[i - 1]) : 0.f) + (i + 1 < n ? fabsf(e[i]) : 0.f);
      gl = fminf(gl, d[i] - rad);
      gu = fmaxf(gu, d[i] + rad);
    }
    gl = -warp_max(-gl); gu = warp_max(gu);
    { const float pad = 1.0e-5f * fmaxf(fabsf(gl), fabsf(gu)) + 1.0e-6f; gl -= pad; gu += pad; }
    const float w0 = (gu - gl) / (float)(NT + 1);
    cnt[tid] = dn_sturm(d, e2, n, gl + (float)(tid + 1) * w0);
    __syncthreads();
    if (tid < k) {                                        // eigenvalue number n - k + tid (ascending, 0-based)
      const int want = n - k + tid + 1;
      int a = 0, b = NT;                                  // first point whose count reaches `want`
      while (a < b) { const int mid = (a + b) >> 1; if (cnt[mid] >= want) b = mid; else a = mid + 1; }
      hi[tid] = a < NT ? gl + (float)(a + 1) * w0 : gu;
      lo[tid] = a > 0 ? gl + (float)a * w0 : gl;
    }
    __syncthreads();
    constexpr int P = NT / 32;                            // points per eigenvalue and round
    constexpr int ROUNDS = P >= 16 ? 4 : 5;               // final interval 5e-8 / 1.3e-7: the fp32 spacing of the eigenvalues
    const int j = tid / P, p = tid % P;
    const int want = n - k + j + 1;
    for (int rd = 0; rd < ROUNDS; ++rd) {
      float l = 0.f, wd = 0.f;
      int ok = 0;
      if (j < k) {
        l = lo[j];
        wd = (hi[j] - l) / (float)(P + 1);
        ok = dn_sturm(d, e2, n, l + (float)(p + 1) * wd) >= want;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, ok);
      const unsigned grp = (bal >> (lane & ~(P - 1))) & ((1u << P) - 1u);
      __syncwarp();
      if (j < k && p == 0) {
        const int first = grp ? __ffs((int)grp) - 1 : P;  // first point at or above the eigenvalue
        if (first < P) hi[j] = l + (float)(first + 1) * wd;
        if (first > 0) lo[j] = l + (float)first * wd;
      }
      __syncwarp();
    }
    __syncthreads();
    if (tid < 32) lam[tid] = tid < k ? 0.5f * (lo[tid] + hi[tid]) : 0.f;
    __syncthreads();
    if (tid == 0) {
      // Shifts of the inverse iteration.  An eigenvalue resolved from its neighbours (spacing >= GCCB_DN_TIGHT) is its
      // own shift.  A tight group (multiple eigenvalue: the members of T differ by the rounding of the reduction,
      // ~3e-7) shares ONE shift, GCCB_DN_DELTA outside the group on the side of the wider gap: every member of the
      // group's eigenspace is then amplified by the same factor (+-10 %), so the iterates stay as independent as their
      // start vectors (random: condition ~50; orthonormal after the first Gram-Schmidt pass: ~1.1) and Gram-Schmidt
      // does not amplify the out-of-group contamination of a single-precision solve.  With LAPACK's recipe (sstein:
      // members pushed 10 eps apart) the members whose shifts end up on the same side of the group converge to the
      // same eigenvector, the set degenerates (condition 1e3) and the last member that Gram-Schmidt reaches came out
      // with residuals up to 3e-4 (measured on sampled ego-nets, 15-fold and 4-fold eigenvalues).
      int c = 0;
      while (c < k) {
        int ce = c;
        while (ce + 1 < k && lam[ce + 1] - lam[ce] < GCCB_DN_TIGHT) ++ce;
        if (ce > c) {
          const float below = c > 0 ? lam[c] - lam[c - 1] : 0.f;        // the next eigenvalue below lam[0] is unknown
          const float above = ce + 1 < k ? lam[ce + 1] - lam[ce] : 1.0f;  // nothing above the largest one
          const bool up = above >= below;
          const float dl = fminf(GCCB_DN_DELTA, (up ? above : below) * (1.0f / 3.0f));
          const float sh = up ? lam[ce] + dl : lam[c] - dl;
          for (int q = c; q <= ce; ++q) lamp[q] = sh;
        } else {
          lamp[c] = lam[c];
        }
        c = ce + 1;
      }
    }
    // pseudo-random start vectors (counter-based: deterministic), columns >= k stay zero
    for (int i = tid; i < n * 32; i += NT) {
      const int r_ = i >> 5, c_ = i & 31;
      float v = 0.f;
      if (c_ < k) {
        u32x4 w = philox4x32_10((uint32_t)i, (uint32_t)n, 0x51ED270Bu, 7u, 0xC0FFEEu, 0x5EEDu);
        v = (float)(int32_t)w.x * (1.0f / 2147483648.0f);
      }
      zrow(r_)[c_] = v;
    }
    __syncthreads();
  }
  GCCB_TICK(2);
  // ---- 3. + 4. inverse iteration (lane = eigenvalue) and modified Gram-Schmidt, in two stages ------------------------
  // Two iterations from the random start, ONE Gram-Schmidt pass (the group iterates are projections of random vectors:
  // condition ~50, so the pass amplifies the out-of-group contamination of the solve, eps / gap ~ 1e-4, to ~1e-2), a
  // third iteration from the orthonormal vectors -- it damps that contamination by (shift distance / gap) ~ 1e-3 and,
  // with the common shift, leaves the group members orthonormal to ~10 % -- and the final, well-conditioned pass.
  for (int stage = 0; stage < 2; ++stage) {
  if (warp == 0 && lane < k) {
    const int j = lane;
    const float lj = lamp[j];
    float bscale = 1.0f;
    const int nit = stage == 0 ? GCCB_DN_INVIT - 1 : 1;
    for (int it = 0; it < nit; ++it) {
      // forward elimination with partial pivoting of T - lj I, applied to the right-hand side in place.  One
      // branch-free path for both pivot choices (lanes differ), and the operands of row i + 2 are loaded before
      // row i is stored: shared-memory loads cannot be moved across the store by the compiler.
      float cd = d[0] - lj, cu = e[0];
      float bi = zrow(0)[j] * bscale;
      float sub = e[0], nd_raw = d[1], nu = e[1], bn_raw = zrow(1)[j];       // n >= 3
      for (int i = 0; i + 1 < n; ++i) {
        const int i2 = i + 2 < n ? i + 2 : n - 1;
        const float d_next = d[i + 2], e_next = e[i + 2], b_next = zrow(i2)[j];   // d, e are zero-padded past n
        const float nd = nd_raw - lj, bn = bn_raw * bscale;
        const bool sw = fabsf(cd) < fabsf(sub);           // rows swapped: the pivot row is (e[i], d[i+1]-lj, e[i+1])
        const float cdg = fabsf(cd) < GCCB_DN_GUARD ? copysignf(GCCB_DN_GUARD, cd) : cd;
        const float rinv = __fdividef(1.0f, sw ? sub : cdg);
        const float m = (sw ? cd : sub) * rinv;
        const float bs = sw ? bn : bi, bo = sw ? bi : bn;
        zrow(i)[j] = bs;
        U0[(size_t)i * 32 + j] = sw ? 0.f : rinv;          // 1 / pivot, kept for the back substitution (never 0: |cd| < 4)
        U1[(size_t)i * 32 + j] = sw ? 0.f : cu;
        cd = sw ? fmaf(-m, nd, cu) : fmaf(-m, cu, nd);
        cu = sw ? -m * nu : nu;
        bi = fmaf(-m, bs, bo);
        sub = nu; nd_raw = d_next; nu = e_next; bn_raw = b_next;
      }
      if (fabsf(cd) < GCCB_DN_GUARD) cd = copysignf(GCCB_DN_GUARD, cd);
      // back substitution: factor rows (L2) prefetched two blocks of four ahead, the shared-memory operands of a
      // block loaded before its chain starts
      float x1 = bi / cd, x2 = 0.f, mx = fabsf(x1);
      zrow(n - 1)[j] = x1;
      float f0[4], f1[4], g0[4], g1[4], h0[4], h1[4];
      int ib = n - 2;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = ib - q, i4 = ib - 4 - q;
        f0[q] = i >= 0 ? U0[(size_t)i * 32 + j] : 1.f; f1[q] = i >= 0 ? U1[(size_t)i * 32 + j] : 0.f;
        g0[q] = i4 >= 0 ? U0[(size_t)i4 * 32 + j] : 1.f; g1[q] = i4 >= 0 ? U1[(size_t)i4 * 32 + j] : 0.f;
      }
      while (ib >= 0) {
        float eb[5], db[4], bb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i8 = ib - 8 - q, i = ib - q >= 0 ? ib - q : 0;
          h0[q] = i8 >= 0 ? U0[(size_t)i8 * 32 + j] : 1.f; h1[q] = i8 >= 0 ? U1[(size_t)i8 * 32 + j] : 0.f;
          eb[q + 1] = e[i]; db[q] = d[i + 1]; bb[q] = zrow(i)[j];
        }
        eb[0] = e[ib + 1];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = ib - q;
          if (i >= 0) {
            float ri = f0[q], u1 = f1[q], u2 = 0.f;
            if (ri == 0.f) { ri = __fdividef(1.0f, eb[q + 1]); u1 = db[q] - lj; u2 = eb[q]; }
            const float x = (bb[q] - u1 * x1 - u2 * x2) * ri;
            zrow(i)[j] = x;
            mx = fmaxf(mx, fabsf(x));
            x2 = x1; x1 = x;
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) { f0[q] = g0[q]; f1[q] = g1[q]; g0[q] = h0[q]; g1[q] = h1[q]; }
        ib -= 4;
      }
      if (!(mx > 0.f && mx < 3.0e38f)) {                  // overflow / breakdown: never seen; keep a valid vector
        for (int i = 0; i < n; ++i) zrow(i)[j] = i == (j % n) ? 1.f : 0.f;
        mx = 1.f;
        atomicOr(flags, (int)GCCB_FLAG_EIG_NOCONV);
      }
      bscale = 1.0f / mx;
    }
    for (int i = 0; i < n; ++i) zrow(i)[j] *= bscale;
  }
  __syncthreads();
  GCCB_TICK(3);
  // modified Gram-Schmidt (right-looking), lanes = columns.  Step j removes z_j from the columns below it; it is
  // needed only when eigenvalue j has a lower neighbour within GCCB_DN_GAPTOL (eigenvectors of T further apart come
  // out of the inverse iteration orthogonal to eps / gap < 1e-5).  Columns are normalised once, at the very end.
  for (int pass = 0; pass < (stage == 0 ? 1 : GCCB_DN_MGS); ++pass)
    for (int j = k - 1; j >= 1; --j) {
      if (!(lam[j] - lam[j - 1] < GCCB_DN_GAPTOL)) continue;
      float acc = 0.f;
      for (int i0 = warp; i0 < n; i0 += 4 * NW) {         // four rows per trip: eight loads in flight
        float zj[4], zc[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = i0 + q * NW;
          const float* zr = zrow(i < n ? i : i0);
          zj[q] = i < n ? zr[j] : 0.f;
          zc[q] = zr[lane];
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc = fmaf(zj[q], zc[q], acc);
      }
      part[warp * 32 + lane] = acc;
      __syncthreads();
      float dot = 0.f, nn = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) { dot += part[w * 32 + lane]; nn += part[w * 32 + j]; }
      const float coef = dot / fmaxf(nn, 1.0e-30f);
      if (lane < j)
        for (int i0 = warp; i0 < n; i0 += 4 * NW) {       // loads of four rows, then their stores
          float zj[4], zc[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int i = i0 + q * NW;
            const float* zr = zrow(i < n ? i : i0);
            zj[q] = zr[j];
            zc[q] = zr[lane];
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int i = i0 + q * NW;
            if (i < n) zrow(i)[lane] = fmaf(-coef, zj[q], zc[q]);
          }
        }
      __syncthreads();
    }
  if (stage == 1) {                                       // unit columns
    float acc = 0.f;
    for (int i = warp; i < n; i += NW) { const float t = zrow(i)[lane]; acc = fmaf(t, t, acc); }
    part[warp * 32 + lane] = acc;
    __syncthreads();
    float nn = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) nn += part[w * 32 + lane];
    const float inv = 1.0f / sqrtf(fmaxf(nn, 1.0e-30f));
    for (int i = warp; i < n; i += NW) zrow(i)[lane] *= inv;
    __syncthreads();
  }
  GCCB_TICK(4);
  }
  // ---- 5. X = Q Z: all reflectors on this warp's columns, in registers --------------------------------------------
  {
    float xr[CPW][NR];
#pragma unroll
    for (int t = 0; t < NR; ++t) {
      const int rr = lane + 32 * t;
#pragma unroll
      for (int q = 0; q < CPW; ++q) xr[q][t] = rr < n ? zrow(rr)[warp * CPW + q] : 0.f;
    }
    for (int kk = n - 3; kk >= 0; --kk) {
      const float tau = taus[kk];
      if (tau == 0.f) continue;
      float vv[NR];
#pragma unroll
      for (int t = 0; t < NR; ++t) {
        const int rr = lane + 32 * t;
        vv[t] = (rr > kk && rr < n) ? A[(size_t)rr * ld + kk] : 0.f;
      }
#pragma unroll
      for (int q = 0; q < CPW; ++q) {
        float dt = 0.f;
#pragma unroll
        for (int t = 0; t < NR; ++t) dt = fmaf(vv[t], xr[q][t], dt);
        dt = tau * warp_sum(dt);
#pragma unroll
        for (int t = 0; t < NR; ++t) xr[q][t] = fmaf(-dt, vv[t], xr[q][t]);
      }
    }
    __syncthreads();                                      // every warp has read its Z columns
#pragma unroll
    for (int t = 0; t < NR; ++t) {
      const int rr = lane + 32 * t;
      if (rr < n) {
#pragma unroll
        for (int q = 0; q < CPW; ++q) zrow(rr)[warp * CPW + q] = xr[q][t];
      }
    }
    __syncthreads();
  }
  GCCB_TICK(5);
  // ---- 6. residuals ||L x - lambda x|| against the sparse matrix -----------------------------------------------------
  {
    float acc = 0.f;
    const float lc = lam[lane];
    for (int i = warp; i < n; i += NW) {
      const int beg = v_indptr[noff + i], end = v_indptr[noff + i + 1];
      float yv = 0.f;
      for (int ed = beg; ed < end; ++ed) {
        const int jn = v_indices[ed] - noff;
        yv = fmaf(dinv[jn], zrow(jn)[lane], yv);
      }
      const float rs = fmaf(dinv[i], yv, -lc * zrow(i)[lane]);
      acc = fmaf(rs, rs, acc);
    }
    part[warp * 32 + lane] = acc;
    __syncthreads();
    if (warp == 0) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) tot += part[w * 32 + lane];
      tot = lane < k ? tot : 0.f;
      tot = sqrtf(warp_max(tot));
      if (lane == 0) {
        dbg_iters[slot] = 0; dbg_res[slot] = tot;
        if (!(tot < GCCB_DN_RES_FLAG)) atomicOr(flags, (int)GCCB_FLAG_EIG_NOCONV);
        for (int i = 0; i < 8; ++i) dbg_phase[(size_t)slot * 8 + i] = ph[i];
      }
    }
  }
  // eigsh(which='LA') returns ascending eigenvalues (data_util.py:251): column c <-> lam[c]
  if (eigvals)
    for (int c = tid; c < pos_dim; c += NT) eigvals[(size_t)slot * pos_dim + c] = c < k ? lam[c] : 0.f;
  write_features(n, k, pos_dim, normalize, sgn, out, [&](int c, int r_) { return zrow(r_)[c]; });
}

template <int NMAX, int NT, bool USM>
__global__ void __launch_bounds__(NT, 65536 / 64 / NT)
posenc_dense_kernel(const int32_t* __restrict__ worklist /* this class */, const int32_t* __restrict__ count,
                    int B, int node_cap, int edge_cap, const int32_t* __restrict__ node_off,
                    const int32_t* __restrict__ b_indptr, const int32_t* __restrict__ b_indices,
                    const int32_t* __restrict__ sub_deg, int pos_dim, int normalize, float* __restrict__ blocks,
                    float* __restrict__ pos, float* __restrict__ eigvals, int32_t* __restrict__ flags,
                    int32_t* __restrict__ dbg_iters, float* __restrict__ dbg_res, long long* __restrict__ dbg_phase) {
  for (int item = blockIdx.x; item < count[0]; item += gridDim.x) {
    posenc_dense_item<NMAX, NT, USM>(worklist[item], B, node_cap, edge_cap, node_off, b_indptr, b_indices, sub_deg, pos_dim,
                                normalize, blocks, pos, eigvals, flags, dbg_iters, dbg_res, dbg_phase);
    __syncthreads();
  }
}

}  // namespace gccb

using namespace gccb;

// workspace: worklist[7][2B] | counts[7] | iters[2B] (ints) | pad | res[2B] | dinv[2*node_cap] | blocks[2][2*node_cap*49] (floats)
static size_t posenc_ws_ints(int B) {
  return (((size_t)GCCB_EIG_NCLASS * 2 * B + GCCB_EIG_NCLASS + 2 * B) + 63) & ~(size_t)63;
}

extern "C" size_t gccb_posenc_workspace(int32_t batch, int32_t node_cap) {
  return posenc_ws_ints(batch) * sizeof(int32_t) +
         ((size_t)2 * batch + (size_t)2 * node_cap + (size_t)2 * 2 * node_cap * (GCCB_CF_B + 1)) * sizeof(float) +
         (size_t)2 * batch * 8 * sizeof(long long) + 64 +
         ((size_t)3 * 2 * batch + 4) * sizeof(int32_t);        // work lists + counts of the dense solver (tail)
}

// Largest ego-net handed to the dense tridiagonal solver.  Default: its first class, n <= 96 -- the larger classes
// hold 108 / 224 KB of shared memory and 512 threads x 64 registers per CTA and crowd the training kernels that run
// beside them in the pipeline out of their SMs.  GCCB200_DENSE_MAX overrides (0 = ChFSI / Jacobi for every size, 228 = direct-method accuracy
// for every ego-net up to 228 vertices); read on every call so that a test can compare the solvers in one process.
static int posenc_dense_max() {
  const char* e = getenv("GCCB200_DENSE_MAX");
  int v = GCCB_DN_A;
  if (e && e[0]) v = atoi(e);
  return v < 0 ? 0 : v > GCCB_DN_C ? GCCB_DN_C : v;
}

extern "C" int gccb_posenc(const gccb_batch_t* batch, int32_t pos_dim, int32_t normalize,
                           float* pos, float* eigvals, void* workspace, size_t workspace_bytes,
                           gccb_stream_t stream) {
  if (!batch || !pos || !workspace || batch->batch <= 0 || pos_dim < 2 || pos_dim > 32) {
    set_last_error("gccb_posenc: bad argument (pos_dim must be in [2, 32])");
    return GCCB_ERR_BADARG;
  }
  const int B = batch->batch;
  if (workspace_bytes < gccb_posenc_workspace(B, batch->node_cap)) {
    set_last_error("gccb_posenc: workspace too small");
    return GCCB_ERR_CAPACITY;
  }
  int32_t* worklist = (int32_t*)workspace;
  int32_t* counts = worklist + (size_t)GCCB_EIG_NCLASS * 2 * B;
  int32_t* dbg_iters = counts + GCCB_EIG_NCLASS;                       // per slot: ChFSI outer iterations (Jacobi: -sweeps)
  float* dbg_res = (float*)((int32_t*)workspace + posenc_ws_ints(B));      // per slot: final residual
  float* dinv = dbg_res + (size_t)2 * B;
  float* blocks = dinv + (size_t)2 * batch->node_cap;
  // diagnostics tail: per-slot phase cycle counters (8-byte aligned)
  long long* dbg_phase = (long long*)(((uintptr_t)(blocks + (size_t)2 * 2 * batch->node_cap * (GCCB_CF_B + 1)) + 15) & ~(uintptr_t)15);
  int32_t* dense_list = (int32_t*)(dbg_phase + (size_t)2 * B * 8);
  int32_t* dense_counts = dense_list + (size_t)3 * 2 * B;
  const int dense_max = posenc_dense_max();
  GCCB_LAUNCH(posenc_classify_kernel, 1, 256, 0, stream, batch->counters, batch->node_off, B, worklist, counts,
              dense_max, GCCB_DN_A, GCCB_DN_B, dense_list, dense_counts);
  auto kgiant = posenc_chfsi_kernel<0, 1024>;
#ifndef GCCB_EMU
  constexpr int CLUSTER = 8;
#else
  constexpr int CLUSTER = 1;                             // the emulator runs the same kernel with one CTA
#endif
  auto khuge = posenc_chfsi_cluster_kernel<GCCB_BIG_NT, CLUSTER>;
  auto kbig = posenc_chfsi_kernel<1, GCCB_BIG_NT>;
  auto kmid = posenc_chfsi_kernel<1, 256>;
  auto ksmall = posenc_jacobi_kernel;
  const size_t s_a = (size_t)2 * GCCB_CF_NSM_A * (GCCB_CF_B + 1) * sizeof(float) + GCCB_CF_SMEM_PAD_A;
  const size_t s_b = (size_t)2 * GCCB_CF_NSM * (GCCB_CF_B + 1) * sizeof(float);
  const size_t s_c = (size_t)2 * GCCB_CF_NSM_C * (GCCB_CF_B + 1) * sizeof(float);
  const size_t s_d = (size_t)2 * ((GCCB_CF_NSM_D + CLUSTER - 1) / CLUSTER) * (GCCB_CF_B + 1) * sizeof(float);
  const size_t s_d1 = (size_t)2 * ((GCCB_CF_NSM_D1 + CLUSTER - 1) / CLUSTER) * (GCCB_CF_B + 1) * sizeof(float);
  gccb::ensure_dyn_smem(kmid, s_b);
  gccb::ensure_dyn_smem(kbig, s_c);
  gccb::ensure_dyn_smem(khuge, s_d);
  // The size classes are independent: fork them over side streams (event fork/join, legal inside
  // CUDA-graph capture) so that the few long-running large ego-nets overlap the many small ones.
#ifndef GCCB_EMU
  // per caller stream: batches in flight do not serialise.  The size-class kernels are long-lived and go to
  // lowest-priority streams whatever the caller's priority (a caller may run its short sampler kernels high)
  StreamKit* kit = stream_kit((cudaStream_t)stream, 0, true);
  cudaStream_t* side = kit->side;
  cudaEvent_t ev_fork = kit->ev[5];
  cudaEvent_t* ev_join = kit->ev;
  cudaStream_t main_s = (cudaStream_t)stream;
  cudaEventRecord(ev_fork, main_s);
  for (int i = 0; i < 5; ++i) cudaStreamWaitEvent(side[i], ev_fork, 0);
  gccb_stream_t s_giant = side[4], s_huge = side[0], s_big = side[1], s_mid2 = side[2], s_small = side[3], s_mid1 = stream;
#else
  gccb_stream_t s_giant = stream, s_huge = stream, s_big = stream, s_mid2 = stream, s_small = stream, s_mid1 = stream;
#endif
#define GCCB_PE_ARGS(cls) worklist, counts, cls, B, batch->node_cap, batch->edge_cap, batch->node_off, batch->indptr, \
    batch->indices, batch->sub_deg, pos_dim, normalize, blocks, dinv, pos, eigvals, batch->flags, dbg_iters, dbg_res, dbg_phase
  // grids are sized for the typical population of each class (persistent loops take the rest): an
  // idle CTA of these kernels still has to win 1024 thread slots / up to 188 KB of shared memory
  // just to exit, which costs concurrent kernels dearly
  auto capped = [&](int limit) { return 2 * B < limit ? 2 * B : limit; };
  GCCB_LAUNCH(kgiant, capped(8), 1024, 0, s_giant, GCCB_PE_ARGS(6));
  // two cluster launches: 192-row slabs (class 4) and 448-row slabs (class 5, same stream as the
  // L2 fallback: both are rare); persistent over their work lists
  for (int pass = 0; pass < 2; ++pass) {
    const int cls = pass == 0 ? 4 : 5;
    const size_t smem = pass == 0 ? s_d1 : s_d;
    const int items = capped(pass == 0 ? 8 : 4);
    gccb_stream_t st = pass == 0 ? s_huge : s_giant;
#ifndef GCCB_EMU
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CLUSTER * items); cfg.blockDim = dim3(GCCB_BIG_NT); cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    ++gccb::g_launch_count;
    cudaLaunchKernelEx(&cfg, khuge, (const int32_t*)worklist, (const int32_t*)counts, cls, B, batch->node_cap,
                       batch->edge_cap, (const int32_t*)batch->node_off, (const int32_t*)batch->indptr,
                       (const int32_t*)batch->indices, (const int32_t*)batch->sub_deg, pos_dim, normalize, dinv, pos,
                       eigvals, batch->flags, dbg_iters, dbg_res, dbg_phase);
#else
    GCCB_LAUNCH(khuge, items, GCCB_BIG_NT, smem, st, worklist, counts, cls, B, batch->node_cap, batch->edge_cap,
                batch->node_off, batch->indptr, batch->indices, batch->sub_deg, pos_dim, normalize, dinv, pos,
                eigvals, batch->flags, dbg_iters, dbg_res, dbg_phase);
#endif
  }
  if (dense_max > 0) {
    // dense classes: n <= 96 (256 threads, 48 KB: four CTAs per SM), n <= 144 (512 threads, 108 KB: two per SM),
    // n <= 228 (512 threads, 224 KB: one per SM); on the streams of the ChFSI classes they replace
    // GCCB200_DN_USM=1: class A keeps the factor rows of the inverse iteration in shared memory (74 KB per CTA, three
    // per SM) instead of the L2 workspace (50 KB, four per SM): a shorter inverse iteration for a larger footprint,
    // off by default.
    const char* usm_e = getenv("GCCB200_DN_USM");
    const bool usm = usm_e && usm_e[0] == '1';
    auto kd_a = usm ? posenc_dense_kernel<GCCB_DN_A, 256, true> : posenc_dense_kernel<GCCB_DN_A, 256, false>;
    auto kd_b = posenc_dense_kernel<GCCB_DN_B, 512, false>;
    auto kd_c = posenc_dense_kernel<GCCB_DN_C, 512, false>;
    const size_t sd_a = (size_t)GCCB_DN_A * dn_ld(GCCB_DN_A) * sizeof(float);
    const size_t sd_b = (size_t)GCCB_DN_B * dn_ld(GCCB_DN_B) * sizeof(float);
    const size_t sd_c = (size_t)GCCB_DN_C * dn_ld(GCCB_DN_C) * sizeof(float);
    gccb::ensure_dyn_smem(posenc_dense_kernel<GCCB_DN_A, 256, true>, sd_a);
    gccb::ensure_dyn_smem(posenc_dense_kernel<GCCB_DN_A, 256, false>, sd_a);
    gccb::ensure_dyn_smem(kd_b, sd_b);
    gccb::ensure_dyn_smem(kd_c, sd_c);
#define GCCB_DN_ARGS(c) dense_list + (size_t)(c) * 2 * B, dense_counts + (c), B, batch->node_cap, batch->edge_cap, \
    batch->node_off, batch->indptr, batch->indices, batch->sub_deg, pos_dim, normalize, blocks, pos, eigvals, \
    batch->flags, dbg_iters, dbg_res, dbg_phase
    // (diagnostics: GCCB200_DN_CAP_A / _B / _C override the persistent grid sizes, i.e. the CTAs per SM)
    auto env_cap = [](const char* name, int dflt) { const char* e = getenv(name); const int v = e && e[0] ? atoi(e) : dflt; return v > 0 ? v : dflt; };
    // classes above dense_max have empty lists: not launched (an idle CTA of theirs must still win 108 / 224 KB of
    // shared memory to exit -- 40-170 us at the head of the streams of the ChFSI classes, CUPTI timeline)
    if (dense_max > GCCB_DN_B)
      GCCB_LAUNCH(kd_c, capped(env_cap("GCCB200_DN_CAP_C", GCCB_CAP_DN_C)), 512, sd_c, s_big, GCCB_DN_ARGS(2));
    if (dense_max > GCCB_DN_A)
      GCCB_LAUNCH(kd_b, capped(env_cap("GCCB200_DN_CAP_B", GCCB_CAP_DN_B)), 512, sd_b, s_mid2, GCCB_DN_ARGS(1));
    GCCB_LAUNCH(kd_a, capped(env_cap("GCCB200_DN_CAP_A", usm ? GCCB_NUM_SMS * 3 : GCCB_CAP_DN_A)), 256, sd_a, s_mid1, GCCB_DN_ARGS(0));
  }
  GCCB_LAUNCH(kbig, capped(GCCB_NUM_SMS), GCCB_BIG_NT, s_c, s_big, GCCB_PE_ARGS(3));
  // classes the dense solver covers completely have empty lists: not launched
  if (dense_max < GCCB_CF_NSM) GCCB_LAUNCH(kmid, capped(GCCB_CAP_MID2), 256, s_b, s_mid2, GCCB_PE_ARGS(2));
  if (dense_max < GCCB_CF_NSM_A) GCCB_LAUNCH(kmid, capped(GCCB_CAP_MID1), 256, s_a, s_mid1, GCCB_PE_ARGS(1));
  if (dense_max < GCCB_EIG_SMALL)
    GCCB_LAUNCH(ksmall, capped(GCCB_NUM_SMS), 256, 0, s_small, worklist, counts, B, batch->node_cap, batch->edge_cap,
                batch->node_off, batch->indptr, batch->indices, batch->sub_deg, pos_dim, normalize, pos, eigvals,
                batch->flags, dbg_iters, dbg_res);
#ifndef GCCB_EMU
  for (int i = 0; i < 5; ++i) {
    cudaEventRecord(ev_join[i], side[i]);
    cudaStreamWaitEvent(main_s, ev_join[i], 0);
  }
#endif
  return check_launch("gccb_posenc");
}
