// capi.cu -- status / error plumbing of the C ABI (include/gccb200.h).
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"
#include <deque>
#include <mutex>

namespace gccb {
unsigned long long g_launch_count = 0;   // kernels enqueued by this library (bench.py: gpu_launches)
static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
    return GCCB_ERR_CUDA;
  }
  return GCCB_OK;
}

#ifndef GCCB_EMU
// a library side stream with the caller stream's scheduling priority (a default-priority weight-gradient
// stream starves behind queued eigensolver CTAs, DESIGN.md 5b), the lowest priority, or one step above the
// caller's (clamped to the device's greatest; a smaller number is a higher priority)
static cudaStream_t create_stream_like(cudaStream_t like, SidePriority want) {
  int prio = 0;
  if (want == SidePriority::kLowest || cudaStreamGetPriority(like, &prio) != cudaSuccess) {
    cudaGetLastError();
    prio = 0;
  } else if (want == SidePriority::kAboveCaller) {
    int least = 0, greatest = 0;
    if (cudaDeviceGetStreamPriorityRange(&least, &greatest) != cudaSuccess) cudaGetLastError();
    else if (prio > greatest) --prio;
  }
  cudaStream_t s = nullptr;
  cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, prio);
  return s;
}

StreamKit* stream_kit(cudaStream_t caller, int family, SidePriority priority) {
  // one kit per (caller stream, family, device), never shared: the concurrent finetune folds hold three families
  // on each of ten caller streams, and a kit handed to a second caller (or re-keyed to another device while its
  // first caller still launches on it) would serialise their side work or put it on another device's streams.
  // A deque keeps the kits' addresses fixed as it grows.  Kits are never freed: the table is bounded by the distinct
  // caller-stream handles a process uses, which torch's stream pools keep to a few dozen per device.  A caller that
  // creates and destroys streams of its own adds a kit (5 streams, 24 events) per new handle, and a recycled handle
  // reuses the kit keyed by it, which is harmless: a kit holds no state between calls.
  static std::deque<StreamKit> kits;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  int dev = 0;
  cudaGetDevice(&dev);                                    // streams belong to a device: the legacy stream (0) of two
  for (StreamKit& k : kits)                               // devices must not share side streams
    if (k.key == caller && k.family == family && k.dev == dev) return &k;
  StreamKit* k = &kits.emplace_back();
  for (int i = 0; i < 5; ++i) k->side[i] = create_stream_like(caller, priority);
  for (int i = 0; i < 24; ++i) cudaEventCreateWithFlags(&k->ev[i], cudaEventDisableTiming);
  k->key = caller;
  k->family = family;
  k->dev = dev;
  return k;
}
#endif
}  // namespace gccb

extern "C" int gccb_version(void) { return GCCB_VERSION; }

extern "C" unsigned long long gccb_launch_count(void) { return gccb::g_launch_count; }

extern "C" const char* gccb_last_error(void) { return gccb::g_err; }

#ifdef GCCB_EMU
// CPU emulator build only (the fiber emulator of the kernel-logic tests): counts[0..1] = programmatic launches and
// launches in which a thread returned without pdl_wait(), both since the last call; returns the first offending
// kernel's name ("" if none) and clears the log
extern "C" const char* gccb_emu_pdl_log(unsigned long long* counts) {
  gccb::EmuPdlLog& g = gccb::emu_pdl_log;
  counts[0] = g.launches;
  counts[1] = g.unwaited;
  const char* first = g.first_bad;
  g = gccb::EmuPdlLog();
  return first;
}
#endif

extern "C" int gccb_arch(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    gccb::set_last_error("gccb_arch: no CUDA device");
    cudaGetLastError();
    return GCCB_ERR_CUDA;
  }
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return major * 10 + minor;
}
