// tc_gemm.cuh -- internal interface of the wgmma contraction (csrc/tc_gemm.cu) for the GIN / MoCo paths.
#pragma once
#include "common.cuh"
#ifndef GCCB_EMU
namespace gccb {
namespace tc {
// out = alpha * A[M x K] . B[N x K]^T (+ bias); A, B bf16 K-major.  See gccb_tc_gemm_bf16 (gccb200.h).
// splits > 1: partials in `scratch` (splits * M_cap * ldp floats, ldp = N), then
//   out_f32[r][c] = alpha * sum_s part + beta * out_f32[r][c]   for c < n_out, row pitch ldo.
int gemm_bf16(const void* A, const void* B, int M_cap, int N, int K, const int32_t* m_dev, const float* bias,
              float alpha, float* out_f32, void* out_bf16, int ldo, double* colstats, int splits, float* scratch,
              cudaStream_t stream, float beta = 0.f, int n_out = -1);
// fp32 [rows][lds] -> bf16, optionally transposed / with a per-column affine + ReLU applied first
//   v = src[r][c] * sc[c] + sh[c] (when sc != null), v = max(v, 0) (when relu)
// transpose = 0: dst [rows_pad][cols_pad];  1: dst [cols_pad][rows_pad].  Zero padded; rows >= *rows_dev are zeros.
int cast_bf16(const float* src, int rows, int cols, int lds, void* dst, int rows_pad, int cols_pad, int transpose,
              const int32_t* rows_dev, cudaStream_t stream, const float* sc = nullptr, const float* sh = nullptr,
              int relu = 0);
int sm_count();
}  // namespace tc
}  // namespace gccb
#endif
