// Shared host-side helpers of libb200raster: error reporting, launch accounting, tiling geometry.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <string>
#include <utility>

#include "../../include/b200_raster.h"

namespace b200r {

// Image tiles: one CTA of the fine / backward kernels owns a TILE x TILE block of output pixels.
constexpr int TILE = 16;
constexpr int TILE_THREADS = TILE * TILE;  // 256: 8 warps, each an 8 x 4 pixel footprint

std::string& last_error_ref();
std::atomic<int64_t>& launch_counter();

inline int fail(int code, const std::string& msg) {
  last_error_ref() = msg;
  return code;
}

inline int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return B200R_OK;
  return fail(B200R_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

#define B200R_CUDA_OK(expr)                                  \
  do {                                                       \
    int _rc = ::b200r::check_cuda((expr), #expr);            \
    if (_rc != B200R_OK) return _rc;                         \
  } while (0)

#define B200R_LAUNCHED(name)                                 \
  do {                                                       \
    ::b200r::launch_counter().fetch_add(1);                  \
    int _rc = ::b200r::check_cuda(cudaGetLastError(), name); \
    if (_rc != B200R_OK) return _rc;                         \
  } while (0)

// Optional phase timing (b200r_set_profiling): events recorded on the launching stream.
struct PhaseTimer {
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool have_fwd = false, have_bwd = false;
  void record(int i, cudaStream_t s);
};
bool profiling_enabled();
PhaseTimer& phase_timer();

// Programmatic dependent launch: the small dependent launches of one call (setup -> scan -> fill -> fine) are chained
// with cudaLaunchAttributeProgrammaticStreamSerialization, so that the next kernel's CTAs are already resident when
// the previous grid drains -- the launch latency between them (a few microseconds each, a quarter of the binning
// time) overlaps the predecessor's tail.  Every chained kernel executes pdl_wait() before it touches anything a
// predecessor wrote (it returns only when the whole preceding grid has completed and its writes are visible; a
// no-op for a normally launched kernel) and every thread of every kernel in a chain executes it, so completion is
// transitive along the chain.  pdl_trigger() lets the successor start once all CTAs of this grid have issued it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_chained(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// The current device's SM count, the launch plans' measure of a full device (132 on an H100 SXM when it cannot be read).
inline int64_t num_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      sms <= 0)
    sms = 132;
  return sms;
}

// Grid-stride kernels launch at most 32 CTAs per SM of the current device: more would only queue behind resident ones.
inline int64_t cap_grid_stride_blocks(int64_t blocks) {
  const int64_t cap = num_sms() * 32;
  return blocks < cap ? blocks : cap;
}

inline int div_up(int a, int b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Index of the mesh / cloud that owns packed element e, or -1.  `first` ascending.
__device__ __forceinline__ int find_owner(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                                          int64_t e) {
  int lo = 0, hi = N;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(first + mid) <= e)
      lo = mid;
    else
      hi = mid;
  }
  const int64_t b = __ldg(first + lo);
  return (b <= e && e < b + __ldg(num + lo)) ? lo : -1;
}

}  // namespace b200r
