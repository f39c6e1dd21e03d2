// tc_gemm.cu -- the path's dense contraction on Hopper tensor cores (wgmma + TMA + mbarrier).
//
//   D[M x N] = alpha * A[M x K] . B[N x K]^T (+ bias[N])      A, B bf16 (K-major), fp32 accumulate
//
// Every GEMM-shaped product of the hot path at hidden >= 128 goes through this kernel:
//   GIN MLP Linear1 / Linear2          (gcc/models/gin.py:107-116; z = x W^T + b, BatchNorm statistics
//                                       of z fused into the epilogue -- gin.py:115 needs the column
//                                       mean / variance over all N rows)
//   their input gradients dX = dZ . W  (B operand = W^T kept as a second bf16 copy)
//   weight gradients dW = dZ^T . X     (operands transposed once, split-K over the rows)
//   MoCo logits q . queue^T            (gcc/contrastive/memory_moco.py:33-44) and dq = P . queue
// Design (one CTA per SM, persistent over 128-row output tiles):
//   warp 8    TMA producer: cp.async.bulk.tensor 2-D boxes (128 x 64 of A, BN x 64 of B, 128-byte
//             swizzle) into a 4-stage shared-memory ring, completion on mbarriers;
//   warps 0-7 two consumer warpgroups, rows 0-63 and 64-127 of the tile: wgmma.mma_async m64 x BN x 16
//             with the fp32 accumulator in registers, one wgmma group in flight while the ring slot of
//             the previous one is released; then the epilogue straight from the registers: bias / scale,
//             fp32 and/or bf16 stores, column sums and sums of squares (float64 atomics, like the SIMT
//             kernels).  The producer keeps filling the ring during the epilogue, so the MMAs of the
//             next tile start on operands already in shared memory.
// Shared-memory operand layout = the canonical K-major SWIZZLE_128B layout (8-row groups 1024 B apart),
// which is exactly what a TMA box with CU_TENSOR_MAP_SWIZZLE_128B writes.
#include "tc_gemm.cuh"

#ifndef GCCB_EMU
#include <cuda.h>
#include <cuda_bf16.h>

namespace gccb {
namespace tc {

constexpr int BM = 128, BK = 64, STAGES = 4, MMA_K = 16;
constexpr int BIAS_SMEM = 512;                             // floats of bias staged in shared memory
// Two consumer warpgroups (rows 0-63 and 64-127 of the tile) and one TMA producer warp.  The accumulator lives in
// registers (BN / 2 floats per consumer thread: 128 at BN = 256), so one CTA of 288 threads per SM (<= 224
// registers per thread) holds a full 128 x 256 tile.
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 32, CONSUMER_WARPS = CONSUMERS / 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Spin on a phase parity.  A protocol bug would otherwise hang the GPU until the driver's watchdog:
// after ~2 s of spinning the kernel traps (the launch then fails loudly instead).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint64_t spin = 0;; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
    if (spin > (1ull << 22)) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// K-major SWIZZLE_128B wgmma matrix descriptor: start address >> 4 in bits [0,14), leading byte offset (unused for
// swizzled K-major) = 1 in [16,30), stride byte offset (8-row group pitch, 1024 B) >> 4 in [32,46), base offset 0
// (every tile is 1024-byte aligned), layout type 1 = SWIZZLE_128B in [62,64).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// d[64 x BN] (+)= A[64 x 16 at da] . B[BN x 16 at db]^T, both operands K-major in shared memory.  The fragment of
// thread t of the warpgroup: d[4 j + {0, 1, 2, 3}] = (row r, col 8 j + c), (r, c + 1), (r + 8, c), (r + 8, c + 1)
// with r = 16 (warp % 4) + lane / 4, c = 2 (lane % 4).
template <int BN>
__device__ void wgmma_bf16(float* d, uint64_t da, uint64_t db, int acc);
template <> __device__ __forceinline__ void wgmma_bf16<32>(float* d, uint64_t da, uint64_t db, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t da, uint64_t db, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float* d, uint64_t da, uint64_t db, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_bf16<256>(float* d, uint64_t da, uint64_t db, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(acc));
}

struct GemmArgs {
  int M_cap, N, K, ldo;
  const int32_t* m_dev;       // optional: number of valid rows (device)
  const float* bias;          // [N] or null
  float alpha;
  float* out_f32;             // [M_cap][ldo] (or [splits][M_cap][ldo] partials when splits > 1) or null
  __nv_bfloat16* out_bf16;    // [M_cap][ldo] or null
  double* colstats;           // [2][N] (sum, sum of squares of the stored values) or null
  int splits;
};

// BRES: the whole B operand (N == BN rows, K <= 256) stays resident in shared memory for the life of the CTA --
// the GIN MLP case (a 256 x 256 weight matrix = 128 KB of bf16): only the A tiles stream through the ring, so a
// 128-row tile costs 64 KB of L2 -> shared-memory traffic instead of 192 KB.
template <int BN, bool BRES>
struct Smem {
  static constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = BRES ? A_BYTES : A_BYTES + B_BYTES;
  static constexpr int BRES_KB = 4;                        // k-blocks of the resident operand (K <= 256)
  static constexpr size_t BRES_BYTES = BRES ? (size_t)BRES_KB * B_BYTES : 0;
  static constexpr int COLACC_F = CONSUMER_WARPS * 2 * BN; // per-warp column sums / sums of squares
  static constexpr size_t TOTAL =
      1024 + BRES_BYTES + (size_t)STAGES * STAGE_BYTES + (size_t)(COLACC_F + BIAS_SMEM) * 4 + 256;
};

// Column sums over the 64 rows of a warpgroup's fragment without shared-memory traffic: x holds, for G 8-column
// groups, (sum c, sum c + 1, sum of squares c, c + 1) of the thread's two rows.  The lanes sharing lane % 4 own the
// same columns; a transpose-reduce over lane bits 4, 3, 2 (each exchange halves what a lane keeps) leaves group
// lane >> (5 - log2 G) on the lane, fully summed over the warp's 16 rows; it is added to the warp's own row of accw.
template <int N, int OFF>
__device__ __forceinline__ void colsum_level(float* x, int lane) {
  if constexpr (OFF >= 4) {
    if constexpr (N > 4) {
      const bool upper = (lane & OFF) != 0;
#pragma unroll
      for (int i = 0; i < N / 2; ++i) {
        const float send = upper ? x[i] : x[i + N / 2], keep = upper ? x[i + N / 2] : x[i];
        x[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
      }
      colsum_level<N / 2, OFF / 2>(x, lane);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] += __shfl_xor_sync(0xffffffffu, x[i], OFF);
      colsum_level<4, OFF / 2>(x, lane);
    }
  }
}
template <int G>
__device__ __forceinline__ void colstats_chunk(float (&x)[4 * G], int lane, float* accw, int BN, int col0) {
  constexpr int LOG_G = G >= 8 ? 3 : G >= 4 ? 2 : G >= 2 ? 1 : 0;
  colsum_level<4 * G, 16>(x, lane);
  if (((lane >> 2) & ((1 << (3 - LOG_G)) - 1)) == 0) {
    const int c = col0 + 8 * (lane >> (5 - LOG_G)) + 2 * (lane & 3);
    accw[c] += x[0];
    accw[c + 1] += x[1];
    accw[BN + c] += x[2];
    accw[BN + c + 1] += x[3];
  }
}

template <int BN, bool BRES>
__global__ void __launch_bounds__(THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, GemmArgs g) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  using S = Smem<BN, BRES>;
  unsigned char* base = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* bres = base;                                        // [BRES_KB][B] (BRES only)
  unsigned char* tiles = base + S::BRES_BYTES;                       // [STAGES][A | B]  (BRES: [STAGES][A])
  float* colacc = (float*)(tiles + (size_t)STAGES * S::STAGE_BYTES); // [CONSUMER_WARPS][2][BN]
  float* bias_s = colacc + S::COLACC_F;                              // [BIAS_SMEM]
  uint64_t* bars = (uint64_t*)(bias_s + BIAS_SMEM);
  uint64_t* full = bars;                 // [STAGES]   TMA -> MMA
  uint64_t* empty = bars + STAGES;       // [STAGES]   MMA -> TMA
  uint64_t* bfull = bars + 2 * STAGES;   // [1]        resident B operand landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int M = g.m_dev ? min(max(*g.m_dev, 0), g.M_cap) : g.M_cap;
  const int m_tiles = (M + BM - 1) / BM, n_tiles = g.N / BN;
  const int kb_total = g.K / BK;
  const int split = blockIdx.y;
  const int kb_per = (kb_total + g.splits - 1) / g.splits;
  const int kb0 = split * kb_per, kb1 = min(kb_total, kb0 + kb_per);
  const int nkb = max(kb1 - kb0, 0);
  const int num_tiles = m_tiles * n_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMER_WARPS); }
    mbar_init(bfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // bias (zeros when absent) in shared memory when it fits: the epilogue then needs no global loads
  const bool bias_in_smem = g.N <= BIAS_SMEM;
  if (bias_in_smem)
    for (int i = threadIdx.x; i < g.N; i += blockDim.x) bias_s[i] = g.bias ? g.bias[i] : 0.f;
  if (g.colstats)
    for (int i = threadIdx.x; i < S::COLACC_F; i += blockDim.x) colacc[i] = 0.f;
  __syncthreads();
  if (nkb == 0) return;

  if (warp == CONSUMER_WARPS) {
    // ===== TMA producer =============================================================================
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      if (BRES && blockIdx.x < num_tiles) {              // the whole B operand, once
        mbar_expect_tx(bfull, (uint32_t)(nkb * S::B_BYTES));
        for (int kb = 0; kb < nkb; ++kb) tma_load_2d(bres + (size_t)kb * S::B_BYTES, &map_b, kb * BK, 0, bfull);
      }
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          unsigned char* sa = tiles + (size_t)stage * S::STAGE_BYTES;
          mbar_expect_tx(&full[stage], S::STAGE_BYTES);
          tma_load_2d(sa, &map_a, kb * BK, mt * BM, &full[stage]);
          if (!BRES) tma_load_2d(sa + S::A_BYTES, &map_b, kb * BK, nt * BN, &full[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups: MMA, then the epilogue from registers ==================================
  const int wg = warp >> 2;                                  // rows 64 wg .. 64 wg + 63 of the tile
  const int r_lo = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // this thread's rows: r_lo, r_lo + 8
  const int cq = 2 * (lane & 3);                             // and columns 8 j + cq, 8 j + cq + 1
  float* outf = g.out_f32 ? g.out_f32 + (size_t)split * g.M_cap * g.ldo : nullptr;
  float* accw = colacc + warp * (2 * BN);
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  if (BRES && blockIdx.x < num_tiles) mbar_wait(bfull, 0);
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t st = smem_u32(tiles + (size_t)stage * S::STAGE_BYTES);
      const uint32_t sa = st + wg * (64 * BK * 2);
      const uint32_t sb = BRES ? smem_u32(bres + (size_t)kb * S::B_BYTES) : st + S::A_BYTES;
      fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / MMA_K; ++k)
        // advancing 16 elements (32 B) along K inside the 128-byte swizzle atom = +32 B on the start address
        wgmma_bf16<BN>(acc, wgmma_desc(sa + k * MMA_K * 2), wgmma_desc(sb + k * MMA_K * 2), (kb | k) != 0);
      wgmma_commit();
      fence_acc(acc);
      if (kb > 0) {                                          // one group in flight: the previous slot is free
        wgmma_wait<1>();
        fence_acc(acc);
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (lane == 0) mbar_arrive(&empty[prev]);

    const int row0 = mt * BM + r_lo, row1 = row0 + 8;
    const bool ok0 = row0 < M, ok1 = row1 < M;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = nt * BN + 8 * j + cq;
      float2 b = make_float2(0.f, 0.f);
      if (bias_in_smem) b = *reinterpret_cast<const float2*>(bias_s + c);
      else if (g.bias) b = make_float2(g.bias[c], g.bias[c + 1]);
      float* v = acc + 4 * j;
      v[0] = ok0 ? fmaf(v[0], g.alpha, b.x) : 0.f;
      v[1] = ok0 ? fmaf(v[1], g.alpha, b.y) : 0.f;
      v[2] = ok1 ? fmaf(v[2], g.alpha, b.x) : 0.f;
      v[3] = ok1 ? fmaf(v[3], g.alpha, b.y) : 0.f;
      // 4 lanes store one 32-byte sector of a row: every store instruction fills whole sectors
      if (outf) {
        if (ok0) *reinterpret_cast<float2*>(outf + (size_t)row0 * g.ldo + c) = make_float2(v[0], v[1]);
        if (ok1) *reinterpret_cast<float2*>(outf + (size_t)row1 * g.ldo + c) = make_float2(v[2], v[3]);
      }
      if (g.out_bf16) {
        if (ok0) *reinterpret_cast<__nv_bfloat162*>(g.out_bf16 + (size_t)row0 * g.ldo + c) = __floats2bfloat162_rn(v[0], v[1]);
        if (ok1) *reinterpret_cast<__nv_bfloat162*>(g.out_bf16 + (size_t)row1 * g.ldo + c) = __floats2bfloat162_rn(v[2], v[3]);
      }
    }
    if (g.colstats) {                                        // n_tiles == 1 with statistics
      constexpr int G = BN / 8 < 8 ? BN / 8 : 8;
#pragma unroll
      for (int ch = 0; ch < BN / (8 * G); ++ch) {
        float x[4 * G];
#pragma unroll
        for (int i = 0; i < G; ++i) {
          const float* v = acc + 4 * (ch * G + i);
          x[4 * i] = v[0] + v[2];
          x[4 * i + 1] = v[1] + v[3];
          x[4 * i + 2] = v[0] * v[0] + v[2] * v[2];
          x[4 * i + 3] = v[1] * v[1] + v[3] * v[3];
        }
        colstats_chunk<G>(x, lane, accw, BN, ch * 8 * G);
      }
    }
  }
  if (g.colstats) {                                          // one float64 atomic per column and CTA
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    for (int i = threadIdx.x; i < 2 * BN; i += CONSUMERS) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < CONSUMER_WARPS; ++w) t += colacc[w * 2 * BN + i];
      const int which = i / BN, c = i - which * BN;
      if (blockIdx.x < num_tiles) atomicAdd(&g.colstats[(size_t)which * g.N + c], (double)t);
    }
  }
}

// out[r][c] = alpha * sum_s part[s][r][c] (+ bias[c]) (+ beta * out[r][c]) for c < n_out; optional bf16 copy.
// Partials have row pitch ldp, the output row pitch ldo.  Fixed summation order: deterministic.
__global__ void __launch_bounds__(256)
tc_splitk_reduce_kernel(const float* __restrict__ part, int splits, int M_cap, int n_out, int ldp, int ldo,
                        const int32_t* __restrict__ m_dev, float alpha, float beta, const float* __restrict__ bias,
                        float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16) {
  const int M = m_dev ? min(max(*m_dev, 0), M_cap) : M_cap;
  const size_t total = (size_t)M * n_out;
  const size_t stride = (size_t)M_cap * ldp;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / n_out), c = (int)(idx - (size_t)r * n_out);
    const size_t ip = (size_t)r * ldp + c, o = (size_t)r * ldo + c;
    float s = 0.f;
    for (int sp = 0; sp < splits; ++sp) s += part[(size_t)sp * stride + ip];
    s *= alpha;
    if (bias) s += bias[c];
    if (out_f32) {
      if (beta != 0.f) s = fmaf(beta, out_f32[o], s);
      out_f32[o] = s;
    }
    if (out_bf16) out_bf16[o] = __float2bfloat16_rn(s);
  }
}

// ---- host side -------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D bf16 row-major [rows][cols] -> boxes of [box_rows][64], 128-byte swizzle, zero fill out of bounds
static int make_map(CUtensorMap* map, const void* ptr, int rows, int cols, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_last_error("tc_gemm: cuTensorMapEncodeTiled is not available"); return GCCB_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("tc_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r); return GCCB_ERR_CUDA; }
  return GCCB_OK;
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = GCCB_NUM_SMS;
  }
  return n;
}

template <int BN, bool BRES = false>
static int launch(const CUtensorMap& ma, const CUtensorMap& mb, const GemmArgs& g, cudaStream_t stream) {
  auto k = tc_gemm_kernel<BN, BRES>;
  const size_t smem = Smem<BN, BRES>::TOTAL;
  gccb::ensure_dyn_smem(k, smem);
  const int m_tiles = (g.M_cap + BM - 1) / BM, tiles = m_tiles * (g.N / BN);
  int gx = sm_count() / g.splits;
  if (gx < 1) gx = 1;
  if (gx > tiles) gx = tiles;
  dim3 grid(gx, g.splits);
  ++gccb::g_launch_count;
  k<<<grid, THREADS, smem, stream>>>(ma, mb, g);
  return GCCB_OK;
}

// Internal entry used by the GIN / MoCo tensor-core paths and by gccb_tc_gemm_bf16.
// splits > 1 (or an accumulating / narrow / oddly pitched output): `scratch` must hold splits * M_cap * N floats; the partial sums are reduced in a fixed order.
int gemm_bf16(const void* A, const void* B, int M_cap, int N, int K, const int32_t* m_dev, const float* bias,
              float alpha, float* out_f32, void* out_bf16, int ldo, double* colstats, int splits, float* scratch,
              cudaStream_t stream, float beta, int n_out) {
  if (n_out < 0) n_out = N;
  if (!A || !B || M_cap <= 0 || N <= 0 || K <= 0 || (K % BK) || (N % 32) || n_out > N || ldo < n_out || splits < 1 ||
      (!out_f32 && !out_bf16)) {
    set_last_error("tc_gemm: bad argument (need K %% 64 == 0, N %% 32 == 0, ldo >= n_out)");
    return GCCB_ERR_BADARG;
  }
  const int BN = (N % 256 == 0) ? 256 : (N % 128 == 0) ? 128 : (N % 64 == 0) ? 64 : 32;
  if (splits > K / BK) splits = K / BK;
  {                                         // no empty split: every partial buffer is written
    const int kb_total = K / BK, per = (kb_total + splits - 1) / splits;
    splits = (kb_total + per - 1) / per;
  }
  // partial sums go through `scratch` and the reduce kernel when K is split, and also when the output is not
  // a plain [M][N] store (accumulate into it, narrower than N, row pitch the epilogue's 16-byte stores cannot use)
  const bool via_scratch = splits > 1 || beta != 0.f || n_out != N || (ldo % 8) != 0;
  if (colstats && N != BN) {
    set_last_error("tc_gemm: fused column statistics need N in {32, 64, 128, 256} (one tile wide)");
    return GCCB_ERR_BADARG;
  }
  if (via_scratch && (!scratch || colstats)) {
    set_last_error("tc_gemm: split-K / accumulate / narrow output need a scratch buffer and cannot fuse column statistics");
    return GCCB_ERR_BADARG;
  }
  CUtensorMap ma, mb;
  int rc = make_map(&ma, A, M_cap, K, BM);
  if (rc) return rc;
  rc = make_map(&mb, B, N, K, BN);
  if (rc) return rc;
  GemmArgs g;
  g.M_cap = M_cap; g.N = N; g.K = K; g.ldo = via_scratch ? N : ldo; g.m_dev = m_dev; g.splits = splits;
  if (via_scratch) {
    g.bias = nullptr; g.alpha = 1.0f; g.out_f32 = scratch; g.out_bf16 = nullptr; g.colstats = nullptr;
  } else {
    g.bias = bias; g.alpha = alpha; g.out_f32 = out_f32; g.out_bf16 = (__nv_bfloat16*)out_bf16; g.colstats = colstats;
  }
  // the B operand stays in shared memory when it is one tile wide, at most 256 deep and reused by several row tiles
  const bool bres = !via_scratch && N == BN && K <= 256 && (BN == 256 || BN == 128) && (M_cap + BM - 1) / BM > sm_count();
  switch (BN) {
    case 256: if (bres) launch<256, true>(ma, mb, g, stream); else launch<256>(ma, mb, g, stream); break;
    case 128: if (bres) launch<128, true>(ma, mb, g, stream); else launch<128>(ma, mb, g, stream); break;
    case 64: launch<64>(ma, mb, g, stream); break;
    default: launch<32>(ma, mb, g, stream); break;
  }
  if (via_scratch) {
    const size_t total = (size_t)M_cap * n_out;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
    GCCB_LAUNCH(tc_splitk_reduce_kernel, blocks, 256, 0, stream, (const float*)scratch, splits, M_cap, n_out, N, ldo,
                m_dev, alpha, beta, bias, out_f32, (__nv_bfloat16*)out_bf16);
  }
  return check_launch("tc_gemm");
}

// fp32 -> bf16 (optionally transposed), optional per-column affine + ReLU first; zero padded to
// [rows_pad][cols_pad] (dst [cols_pad][rows_pad] when transposed); rows >= *rows_dev are zeros.
__global__ void __launch_bounds__(256)
cast_bf16_kernel(const float* __restrict__ src, int rows, int cols, int lds, __nv_bfloat16* __restrict__ dst,
                 int rows_pad, int cols_pad, const int32_t* __restrict__ rows_dev,
                 const float* __restrict__ sc, const float* __restrict__ sh, int relu) {
  const int R = rows_dev ? min(max(*rows_dev, 0), rows) : rows;
  const size_t total = (size_t)rows_pad * cols_pad;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / cols_pad), c = (int)(idx - (size_t)r * cols_pad);
    float v = 0.f;
    if (r < R && c < cols) {
      v = src[(size_t)r * lds + c];
      if (sc) v = fmaf(v, sc[c], sh[c]);
      if (relu) v = fmaxf(v, 0.f);
    }
    dst[idx] = __float2bfloat16_rn(v);
  }
}

// transposing variant: one 64 x 64 tile per CTA through shared memory: 128-bit coalesced reads along the source
// rows, 32-bit (2 x bf16) coalesced writes along the destination rows; grid = all tiles (the weight-gradient
// operands of a config-4 batch are 100k+ rows: the pass has to run near HBM speed)
__global__ void __launch_bounds__(256)
cast_bf16_t_kernel(const float* __restrict__ src, int rows, int cols, int lds, __nv_bfloat16* __restrict__ dst,
                   int rows_pad, int cols_pad, const int32_t* __restrict__ rows_dev,
                   const float* __restrict__ sc, const float* __restrict__ sh, int relu) {
  __shared__ float tile[64][65];
  const int R = rows_dev ? min(max(*rows_dev, 0), rows) : rows;
  const int tcn = (cols_pad + 63) / 64;
  const int r0 = (blockIdx.x / tcn) * 64, c0 = (blockIdx.x % tcn) * 64;
  const int tid = threadIdx.x;
  const bool vec_ok = (lds % 4) == 0 && ((uintptr_t)src % 16) == 0;
  if (r0 >= R) {                                           // nothing valid in this row band: zeros
    for (int i = tid; i < 64 * 32; i += 256) {
      const int c = c0 + i / 32, r = r0 + (i % 32) * 2;
      if (c < cols_pad && r < rows_pad) *reinterpret_cast<uint32_t*>(dst + (size_t)c * rows_pad + r) = 0u;
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = tid + k * 256;                           // 1024 float4 slots: row = i / 16, 4 columns at (i % 16) * 4
    const int rr = i >> 4, cc = (i & 15) * 4;
    const int r = r0 + rr, c = c0 + cc;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < R) {
      if (vec_ok && c + 3 < cols) {
        const float4 t = *reinterpret_cast<const float4*>(src + (size_t)r * lds + c);
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (c + q < cols) v[q] = src[(size_t)r * lds + c + q];
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (c + q < cols) {
          if (sc) v[q] = fmaf(v[q], sc[c + q], sh[c + q]);
          if (relu) v[q] = fmaxf(v[q], 0.f);
        } else v[q] = 0.f;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) tile[rr][cc + q] = v[q];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = tid + k * 256;                           // 2048 pairs: column = i / 32, rows 2 * (i % 32), +1
    const int cc = i >> 5, rr = (i & 31) * 2;
    const int c = c0 + cc, r = r0 + rr;
    if (c < cols_pad && r < rows_pad) {                    // rows_pad is even (multiple of 64)
      const __nv_bfloat162 pr = __floats2bfloat162_rn(tile[rr][cc], tile[rr + 1][cc]);
      *reinterpret_cast<uint32_t*>(dst + (size_t)c * rows_pad + r) = *reinterpret_cast<const uint32_t*>(&pr);
    }
  }
}

int cast_bf16(const float* src, int rows, int cols, int lds, void* dst, int rows_pad, int cols_pad, int transpose,
              const int32_t* rows_dev, cudaStream_t stream, const float* sc, const float* sh, int relu) {
  if (transpose && (rows_pad % 2) == 0) {
    const int tiles = ((rows_pad + 63) / 64) * ((cols_pad + 63) / 64);
    GCCB_LAUNCH(cast_bf16_t_kernel, tiles, 256, 0, stream, src, rows, cols, lds, (__nv_bfloat16*)dst, rows_pad,
                cols_pad, rows_dev, sc, sh, relu);
    return check_launch("cast_bf16 (transposed)");
  }
  if (transpose) {
    set_last_error("cast_bf16: the transposed cast needs an even rows_pad");
    return GCCB_ERR_BADARG;
  }
  const size_t total = (size_t)rows_pad * cols_pad;
  int blocks = (int)((total + 1023) / 1024);
  if (blocks > 16 * sm_count()) blocks = 16 * sm_count();
  if (blocks < 1) blocks = 1;
  GCCB_LAUNCH(cast_bf16_kernel, blocks, 256, 0, stream, src, rows, cols, lds, (__nv_bfloat16*)dst, rows_pad, cols_pad,
              rows_dev, sc, sh, relu);
  return check_launch("cast_bf16");
}

}  // namespace tc
}  // namespace gccb

using namespace gccb;

extern "C" int gccb_tc_gemm_bf16(const void* A, const void* B, int32_t M_cap, int32_t N, int32_t K,
                                 const int32_t* m_dev, const float* bias, float alpha, float* out_f32,
                                 void* out_bf16, int32_t ldo, double* colstats, int32_t splits, float* scratch,
                                 gccb_stream_t stream) {
  return tc::gemm_bf16(A, B, M_cap, N, K, m_dev, bias, alpha, out_f32, out_bf16, ldo, colstats, splits, scratch,
                       (cudaStream_t)stream);
}

extern "C" int gccb_cast_bf16(const float* src, int32_t rows, int32_t cols, int32_t lds, void* dst, int32_t rows_pad,
                              int32_t cols_pad, int32_t transpose, const int32_t* rows_dev, gccb_stream_t stream) {
  if (!src || !dst || rows < 0 || cols <= 0 || lds < cols || rows_pad < rows || cols_pad < cols) {
    set_last_error("gccb_cast_bf16: bad argument");
    return GCCB_ERR_BADARG;
  }
  return tc::cast_bf16(src, rows, cols, lds, dst, rows_pad, cols_pad, transpose, rows_dev, (cudaStream_t)stream);
}

#else   // GCCB_EMU: the CPU emulator cannot run wgmma / TMA; the entry points report it
extern "C" int gccb_tc_gemm_bf16(const void*, const void*, int32_t, int32_t, int32_t, const int32_t*, const float*,
                                 float, float*, void*, int32_t, double*, int32_t, float*, gccb_stream_t) {
  gccb::set_last_error("tc_gemm: tensor-core path is not available under the CPU emulator");
  return GCCB_ERR_ARCH;
}
extern "C" int gccb_cast_bf16(const float*, int32_t, int32_t, int32_t, void*, int32_t, int32_t, int32_t,
                              const int32_t*, gccb_stream_t) {
  gccb::set_last_error("cast_bf16: not available under the CPU emulator");
  return GCCB_ERR_ARCH;
}
#endif
