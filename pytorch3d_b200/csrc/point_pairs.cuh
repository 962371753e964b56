// The point-pair arithmetic and the target-tile stream shared by the point-cloud ops: chamfer
// distance (chamfer.cu, DESIGN.md section 21) and farthest point sampling and ball query (point_ops.cu, section 22).
#pragma once

#include "bulk_copy.cuh"
#include "keyed_runs.cuh"

namespace b200r {
namespace {

constexpr int kTile = 512;  // target points per shared-memory tile

// lengths[n] clamped to [0, P]; P when there are no lengths.
__device__ __forceinline__ int64_t cloud_len(const int64_t* __restrict__ len, int64_t n, int64_t P) {
  if (len == nullptr) return P;
  const int64_t l = __ldg(len + n);
  return l < 0 ? 0 : (l > P ? P : l);
}

// The reference's pair distance (KNearestNeighborKernelV3<float, 3, 1>, SASS of nvcc -O3 for sm_90a).  Norm 2 is also
// the squared distance of FarthestPointSamplingKernel and BallQueryKernel as nvcc compiles them: three FFMA from zero.
template <int NORM>
__device__ __forceinline__ float pair_dist(float qx, float qy, float qz, float tx, float ty, float tz) {
  const float dx = __fsub_rn(qx, tx), dy = __fsub_rn(qy, ty), dz = __fsub_rn(qz, tz);
  if (NORM == 2) return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmaf_rn(dx, dx, 0.0f)));
  return __fadd_rn(__fadd_rn(__fadd_rn(0.0f, fabsf(dx)), fabsf(dy)), fabsf(dz));
}

template <int NORM>
__device__ __forceinline__ float dist_to(const float* __restrict__ t, int64_t j, float qx, float qy, float qz) {
  return pair_dist<NORM>(qx, qy, qz, __ldg(t + 3 * j), __ldg(t + 3 * j + 1), __ldg(t + 3 * j + 2));
}

__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// Targets [j, j + cnt) of cloud t into buf as (x, y, z, -) float4, one 4-byte asynchronous copy per word, by a CTA of
// kThreads threads.
__device__ __forceinline__ void load_tile(float4* buf, const float* __restrict__ t, int64_t j, int cnt) {
  const float* src = t + 3 * j;
  for (int w = threadIdx.x; w < 3 * cnt; w += kThreads) {
    const int p = w / 3, c = w - 3 * p;
    cp_async4(reinterpret_cast<float*>(buf + p) + c, src + w);
  }
}

}  // namespace
}  // namespace b200r
