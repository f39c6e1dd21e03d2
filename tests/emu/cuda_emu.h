// cuda_emu.h -- TEST INFRASTRUCTURE ONLY (never part of the product library).
//
// A tiny single-OS-thread emulation of the CUDA execution model, so that the
// *logic* of the SIMT kernels in gcc_b200/csrc/*.cu (indexing, barriers,
// shuffles, atomics, capacity handling) can be exercised by the CPU test-suite
// in a container without a GPU.  Each CUDA thread of a block is a ucontext
// fiber; blocks run one after another; __syncthreads()/warp collectives yield
// to a round-robin scheduler.  It proves nothing about performance, memory
// coalescing or data races -- the `-m gpu` parity tests on a real H100 do that.
// The product build (nvcc, libgccb200.so) never includes this header, and the
// Python package cannot load the emulated library.
#pragma once
#include <ucontext.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) alignas(n)
#define __constant__ static

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
struct int2 { int x, y; };
struct int4 { int x, y, z, w; };
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
struct double2 { double x, y; };
static inline float2 make_float2(float a, float b) { return {a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return {a, b, c, d}; }
static inline int2 make_int2(int a, int b) { return {a, b}; }
static inline int4 make_int4(int a, int b, int c, int d) { return {a, b, c, d}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return {a, b}; }
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return {a, b, c, d}; }

typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97,
                      cudaDevAttrComputeCapabilityMajor = 75, cudaDevAttrComputeCapabilityMinor = 76 };
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, int attr, int) {
  *v = attr == cudaDevAttrMultiProcessorCount ? 4 : attr == cudaDevAttrMaxSharedMemoryPerBlockOptin ? 232448
       : attr == cudaDevAttrComputeCapabilityMajor ? 10 : 0;
  return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
enum cudaMemcpyKind { cudaMemcpyDeviceToDevice = 3 };
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }

namespace emu {
enum State { READY, WAIT_BLOCK, WAIT_WARP, DONE };
struct Fiber {
  ucontext_t ctx;
  State st;
  char* stack;
};
struct Ctx {
  std::vector<Fiber> fibers;
  ucontext_t main_ctx;
  int cur = -1, nthreads = 0, live = 0;
  int block_arrived = 0;
  int block_or[2] = {0, 0}, block_cnt[2] = {0, 0}, block_gen = 0;
  int warp_arrived[32];
  unsigned warp_expect[32];
  // per-warp exchange buffers for shuffles / votes (double buffered)
  uint64_t xbuf[32][2][32];
  uint64_t snap[32][2][32];      // values frozen when the warp barrier releases
  unsigned snap_valid[32][2];    // lanes that took part in that collective
  int warp_gen[32];
  std::function<void()> body;
  unsigned char* dyn = nullptr;
  dim3 grid, block;
};
inline Ctx& C() { static Ctx c; return c; }
}  // namespace emu

inline uint3 threadIdx, blockIdx;
inline dim3 blockDim, gridDim;
static const int warpSize = 32;

namespace emu {
static const size_t kStack = 192 * 1024;
inline void set_tid(int t) {
  Ctx& c = C();
  threadIdx.x = t % c.block.x;
  threadIdx.y = (t / c.block.x) % c.block.y;
  threadIdx.z = t / (c.block.x * c.block.y);
}
inline void yield_to_main() {
  Ctx& c = C();
  int me = c.cur;
  swapcontext(&c.fibers[me].ctx, &c.main_ctx);
  set_tid(me);
}
inline void trampoline() {
  Ctx& c = C();
  c.body();
  c.fibers[c.cur].st = DONE;
  c.live--;
  swapcontext(&c.fibers[c.cur].ctx, &c.main_ctx);
}
inline void release_barriers() {
  Ctx& c = C();
  if (c.live > 0 && c.block_arrived == c.live) {
    for (int t = 0; t < c.nthreads; ++t)
      if (c.fibers[t].st == WAIT_BLOCK) c.fibers[t].st = READY;
    c.block_arrived = 0;
    c.block_gen ^= 1;
    c.block_or[c.block_gen] = 0;      // buffer for the NEXT barrier generation
    c.block_cnt[c.block_gen] = 0;
  }
  int nw = (c.nthreads + 31) / 32;
  for (int w = 0; w < nw; ++w) {
    if (c.warp_arrived[w] == 0) continue;
    // expected = lanes of the mask that are still alive
    int expect = 0;
    for (int l = 0; l < 32; ++l) {
      int t = w * 32 + l;
      if (t < c.nthreads && (c.warp_expect[w] >> l & 1) && c.fibers[t].st != DONE) expect++;
    }
    if (c.warp_arrived[w] >= expect) {
      int buf = c.warp_gen[w] & 1;
      c.snap_valid[w][buf] = 0;
      for (int l = 0; l < 32; ++l) {
        int t = w * 32 + l;
        if (t < c.nthreads && c.fibers[t].st == WAIT_WARP) {
          c.fibers[t].st = READY;
          c.snap[w][buf][l] = c.xbuf[w][buf][l];
          c.snap_valid[w][buf] |= 1u << l;
        }
      }
      c.warp_arrived[w] = 0;
      c.warp_gen[w]++;
    }
  }
}
inline void run_block(std::function<void()> body) {
  Ctx& c = C();
  c.body = body;
  c.nthreads = c.block.x * c.block.y * c.block.z;
  if ((int)c.fibers.size() < c.nthreads) {
    size_t old = c.fibers.size();
    c.fibers.resize(c.nthreads);
    for (size_t i = old; i < c.fibers.size(); ++i) c.fibers[i].stack = (char*)malloc(kStack);
  }
  c.live = c.nthreads;
  c.block_arrived = 0;
  c.block_gen = 0;
  c.block_or[0] = c.block_or[1] = c.block_cnt[0] = c.block_cnt[1] = 0;
  for (int w = 0; w < 32; ++w) { c.warp_arrived[w] = 0; c.warp_gen[w] = 0; c.warp_expect[w] = 0; }
  for (int t = 0; t < c.nthreads; ++t) {
    Fiber& f = c.fibers[t];
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack;
    f.ctx.uc_stack.ss_size = kStack;
    f.ctx.uc_link = nullptr;
    makecontext(&f.ctx, (void (*)())trampoline, 0);
    f.st = READY;
  }
  int guard = 0;
  while (c.live > 0) {
    bool progressed = false;
    for (int t = 0; t < c.nthreads; ++t) {
      if (c.fibers[t].st != READY) continue;
      c.cur = t;
      set_tid(t);
      swapcontext(&c.main_ctx, &c.fibers[t].ctx);
      progressed = true;
      release_barriers();
    }
    release_barriers();
    if (!progressed) {
      bool any_ready = false;
      for (int t = 0; t < c.nthreads; ++t) any_ready |= c.fibers[t].st == READY;
      if (!any_ready && ++guard > 2) {
        fprintf(stderr, "cuda_emu: DEADLOCK in block (%u,%u,%u): divergent barrier\n", blockIdx.x, blockIdx.y, blockIdx.z);
        abort();
      }
    } else {
      guard = 0;
    }
  }
}
template <class F>
inline void launch(dim3 grid, dim3 block, size_t smem, F body) {
  Ctx& c = C();
  c.grid = grid; c.block = block;
  gridDim = grid; blockDim = block;
  std::vector<unsigned char> dyn(smem + 64);
  c.dyn = (unsigned char*)(((uintptr_t)dyn.data() + 63) & ~(uintptr_t)63);
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
        run_block(body);
      }
}
inline int lane() { return C().cur & 31; }
inline int warp() { return C().cur >> 5; }
inline void warp_sync(unsigned mask) {
  Ctx& c = C();
  int w = warp();
  c.warp_expect[w] = mask;
  c.warp_arrived[w]++;
  c.fibers[c.cur].st = WAIT_WARP;
  yield_to_main();
}
}  // namespace emu

#define GCCB_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(emu::C().dyn)

static inline void __syncthreads() {
  emu::Ctx& c = emu::C();
  c.block_arrived++;
  c.fibers[c.cur].st = emu::WAIT_BLOCK;
  emu::yield_to_main();
}
static inline int __syncthreads_or(int pred) {
  emu::Ctx& c = emu::C();
  int g = c.block_gen;
  c.block_or[g] |= (pred != 0);
  __syncthreads();
  return c.block_or[g];
}
static inline int __syncthreads_count(int pred) {
  emu::Ctx& c = emu::C();
  int g = c.block_gen;
  c.block_cnt[g] += (pred != 0);
  __syncthreads();
  return c.block_cnt[g];
}
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_sync(mask); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}

// Shuffles: double-buffered exchange slots, buffer chosen by the warp barrier generation.
namespace emu {
template <class T>
inline T shfl_generic(unsigned mask, T v, int src_lane_fn_kind, int arg, int width) {
  Ctx& c = C();
  int w = warp(), l = lane();
  int buf = c.warp_gen[w] & 1;   // bumped when the warp barrier releases
  uint64_t payload = 0;
  memcpy(&payload, &v, sizeof(T));
  c.xbuf[w][buf][l] = payload;
  warp_sync(mask);
  int src;
  int base = l & ~(width - 1);
  switch (src_lane_fn_kind) {
    case 0: src = base + (arg & (width - 1)); break;                       // idx
    case 1: src = l ^ arg; if (src >= base + width) src = l; break;        // xor
    case 2: src = l - arg; if (src < base) src = l; break;                 // up
    default: src = l + arg; if (src >= base + width) src = l; break;       // down
  }
  T out = v;
  if (c.snap_valid[w][buf] >> src & 1) memcpy(&out, &c.snap[w][buf][src], sizeof(T));
  return out;
}
}  // namespace emu
#define EMU_SHFL(T)                                                                                   \
  static inline T __shfl_sync(unsigned m, T v, int s, int w = 32) { return emu::shfl_generic<T>(m, v, 0, s, w); } \
  static inline T __shfl_xor_sync(unsigned m, T v, int s, int w = 32) { return emu::shfl_generic<T>(m, v, 1, s, w); } \
  static inline T __shfl_up_sync(unsigned m, T v, unsigned s, int w = 32) { return emu::shfl_generic<T>(m, v, 2, (int)s, w); } \
  static inline T __shfl_down_sync(unsigned m, T v, unsigned s, int w = 32) { return emu::shfl_generic<T>(m, v, 3, (int)s, w); }
EMU_SHFL(int) EMU_SHFL(unsigned) EMU_SHFL(float) EMU_SHFL(double) EMU_SHFL(long long) EMU_SHFL(unsigned long long)
static inline unsigned __ballot_sync(unsigned mask, int pred) {
  emu::Ctx& c = emu::C();
  int w = emu::warp();
  int buf = c.warp_gen[w] & 1;
  c.xbuf[w][buf][emu::lane()] = pred ? 1 : 0;
  emu::warp_sync(mask);
  unsigned r = 0;
  for (int l = 0; l < 32; ++l)
    if ((mask >> l & 1) && (c.snap_valid[w][buf] >> l & 1) && c.snap[w][buf][l]) r |= 1u << l;
  return r;
}
static inline int __any_sync(unsigned m, int p) { return __ballot_sync(m, p) != 0; }
static inline int __all_sync(unsigned m, int p) {
  emu::Ctx& c = emu::C();
  int w = emu::warp();
  int buf = c.warp_gen[w] & 1;
  unsigned b = __ballot_sync(m, p);
  return b == (c.snap_valid[w][buf] & m);
}

// atomics (single OS thread: plain RMW)
template <class T> static inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { auto o = *p; *p = o + v; return o; }
template <class T> static inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

// intrinsics
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __frcp_rn(float x) { return 1.0f / x; }
static inline float __fsqrt_rn(float x) { return sqrtf(x); }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
static inline double __longlong_as_double(long long i) { double f; memcpy(&f, &i, 8); return f; }
using std::max;
using std::min;
static inline int max(int a, unsigned b) { return a > (int)b ? a : (int)b; }

#define GCCB_LAUNCH(kern, grid, block, smem, stream, ...) \
  emu::launch(dim3(grid), dim3(block), (size_t)(smem), [=]() { kern(__VA_ARGS__); })
