// common.cuh -- shared device/host helpers for libgccb200 (sm_90a).
#pragma once
#include <mutex>
#include <stdint.h>

// Streaming multiprocessors of the target GPU (H100 SXM: 132): sizes persistent grids and split-K partitions.
#define GCCB_NUM_SMS 132

#ifdef GCCB_EMU
// tests/emu/cuda_emu.h: CPU emulation used ONLY by the `-m "not gpu"` kernel-logic
// tests; the product library is always built by nvcc without GCCB_EMU.
#include "cuda_emu.h"
// count kernel launches like the device build does (gccb_launch_count)
namespace gccb { extern unsigned long long g_launch_count; }
#undef GCCB_LAUNCH
#define GCCB_LAUNCH(kern, grid, block, smem, stream, ...) \
  (++gccb::g_launch_count, emu::launch(dim3(grid), dim3(block), (size_t)(smem), [=]() { kern(__VA_ARGS__); }))
#else
#include <cuda_runtime.h>
#define GCCB_DYN_SMEM(type, name)                                   \
  extern __shared__ __align__(16) unsigned char name##_raw_smem[];  \
  type* name = reinterpret_cast<type*>(name##_raw_smem)
namespace gccb { extern unsigned long long g_launch_count; }
#define GCCB_LAUNCH(kern, grid, block, smem, stream, ...) \
  (++gccb::g_launch_count, kern<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__))
#endif

#ifndef GCCB_EMU
namespace gccb {
// Side streams + events owned by the library, one kit per (caller stream, family): several
// calls may be in flight on different caller streams and must not serialise on shared side streams.
// Fork/join is by events only (legal inside CUDA-graph capture).  Family 0: gccb_posenc size
// classes; family 1: gccb_gin_backward weight-gradient stream.
struct StreamKit {
  cudaStream_t key;
  int family;
  int dev;
  cudaStream_t side[5];
  cudaEvent_t ev[24];
};
// scheduling priority of a kit's side streams: the caller stream's, the lowest, or one step above the caller's
enum class SidePriority { kCaller, kLowest, kAboveCaller };
StreamKit* stream_kit(cudaStream_t caller, int family, SidePriority priority = SidePriority::kCaller);
}  // namespace gccb
#endif

namespace gccb {
// Opt a kernel into `bytes` of dynamic shared memory.  The driver call costs microseconds, so the
// largest value already granted is remembered per kernel and the call is skipped afterwards
// (per device; guarded by a mutex).
template <class K>
inline void ensure_dyn_smem(K kern, size_t bytes) {
  // the attribute is per device: one table per (kernel pointer, device ordinal); guarded, because ctypes callers
  // run without the GIL and two host threads may make their first call together
  struct Slot { const void* fn; int dev; size_t bytes; };
  static Slot slots[256];
  static int nslots = 0;
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  const void* key = (const void*)kern;
  std::lock_guard<std::mutex> lock(mu);
  for (int i = 0; i < nslots; ++i)
    if (slots[i].fn == key && slots[i].dev == dev) {
      if (slots[i].bytes >= bytes) return;
      slots[i].bytes = bytes;
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
      return;
    }
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (nslots < 256) { slots[nslots].fn = key; slots[nslots].dev = dev; slots[nslots].bytes = bytes; ++nslots; }
}
}  // namespace gccb

#include "../../include/gccb200.h"

#define GCCB_HOPCAP 64u
#define GCCB_TAG_WALK 0u
#define GCCB_TAG_SEED 1u
#define GCCB_TAG_DROPOUT 2u
#define GCCB_TAG_PRONE 3u

// device status flag bits (gccb200.h: GCCB_FLAG_*)
namespace gccb {

void set_last_error(const char* fmt, ...);
int check_launch(const char* what);   // returns GCCB_OK or GCCB_ERR_CUDA

struct u32x4 { uint32_t x, y, z, w; };

// Philox4x32-10 (Salmon et al. SC'11).  Same integers as oracle/gccb_oracle.c.
__host__ __device__ __forceinline__ u32x4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                        uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  u32x4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
  return o;
}

// counter layout of "RWR-Philox v1" (DESIGN.md): (sample lo, sample hi, trace, hop|view<<8|tag<<16)
__host__ __device__ __forceinline__ u32x4 philox_at(uint64_t key, uint64_t sample, uint32_t trace,
                                                    uint32_t hop, uint32_t view, uint32_t tag) {
  return philox4x32_10((uint32_t)sample, (uint32_t)(sample >> 32), trace,
                       hop | (view << 8) | (tag << 16), (uint32_t)key, (uint32_t)(key >> 32));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// inclusive warp scan
__device__ __forceinline__ int warp_scan_incl(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// a graph id of a gccb_graph_set_t taken from the caller: clamped, so that it never reads out of bounds
__device__ __forceinline__ int64_t clamp_graph(int64_t id, int64_t n_graphs) {
  return id < 0 ? 0 : (id >= n_graphs ? n_graphs - 1 : id);
}

// Block-wide exclusive scan of one int per thread (blockDim.x <= 1024, multiple of 32).
// `scratch` must hold 33 ints of shared memory.  Returns exclusive prefix; *total = block sum.
__device__ __forceinline__ int block_scan_excl(int v, int* scratch, int* total) {
  int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nw = blockDim.x >> 5;
  int incl = warp_scan_incl(v, lane);
  if (lane == 31) scratch[w] = incl;
  __syncthreads();
  if (w == 0) {
    int s = lane < nw ? scratch[lane] : 0;
    int si = warp_scan_incl(s, lane);
    scratch[lane] = si - s;          // exclusive warp offsets
    if (lane == 31) scratch[32] = si;
  }
  __syncthreads();
  int res = incl - v + scratch[w];
  *total = scratch[32];
  __syncthreads();                   // scratch reusable after return
  return res;
}

}  // namespace gccb
