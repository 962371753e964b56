// Farthest point sampling and ball query: pytorch3d.ops.sample_farthest_points and pytorch3d.ops.ball_query for
// 3-D point clouds, with a deterministic ball-query backward (DESIGN.md section 22).
//
// Farthest point sampling, one launch: one thread-block cluster of C CTAs (1 <= C <= 16) per cloud.  Each CTA loads
// its share of the cloud once: kFpsRegs points per thread in registers, then up to smem_pts points in shared memory as
// (x, y, z, running distance); points beyond what the cluster holds are re-read from L2 every iteration, their running
// distances in `scratch`.  Each iteration updates the running distances with the last selected point, takes the
// maximum of the key (float bits of the distance) << 32 | ~p per thread, across the warp (two redux.sync) and across
// the CTA through shared memory, and publishes (key, x, y, z) of the CTA's winner in its own shared memory.  After one
// cluster barrier every warp of every CTA reads the C entries over DSMEM and picks the same winner; its coordinates
// travel with the key.  A single-CTA cloud skips the cluster step: every warp reduces the 8 warp entries itself.  The
// published slots and the warp entries are double-buffered by iteration parity, so one barrier per step suffices: a
// slot is rewritten only after the barrier that every reader of its previous contents has passed.
//
// The result is FarthestPointSamplingKernel's (launched with one CTA per cloud) bit for bit: the same FFMA chain, the
// running distance starting at 1e10 and lowered by fminf (a NaN distance never lowers it), so it is never NaN and
// always >= +0, and the maximum key is the largest distance with the lowest index -- the per-thread strict > combined
// with cub::ArgMax's tie rule -- whatever the decomposition.
//
// Ball query forward: a CTA owns kThreads queries of one cloud, one per thread, and streams that cloud's targets
// through shared memory in double-buffered cp.async tiles, appending hits in ascending j until every query has K hits
// (__syncthreads_and) or the targets run out.  Hits are written as found; the padding (-1, 0, 0) of the CTA's rows is
// written afterwards in coalesced stores, so every output element is written once.
//
// Ball query backward: one thread per query sums its hits' rows 2 g (p1 - p2) in k order into grad_p1; grad_p2 is, per
// target, the sum of -2 g (p1 - p2) + g_nn over its hits in (i, k) order: sort_into_runs over the hits by target and
// segmented_sum_kernel (keyed_runs.cuh) with a row recomputed from its id, in chunks of at most kBallChunk rows, each
// chunk continuing the previous chunk's sums.  No float atomics, no (N, P2, K, 3) buffer, no host synchronisation.
#include <cooperative_groups.h>

#include "point_pairs.cuh"

namespace cg = cooperative_groups;

namespace b200r {
namespace {

// ---- farthest point sampling ----------------------------------------------------------------------------------------

constexpr int kFpsThreads = 256;
constexpr int kFpsRegs = 16;                                  // points per thread held in registers
constexpr int64_t kFpsRegPoints = (int64_t)kFpsThreads * kFpsRegs;  // points per CTA held in registers
constexpr int kFpsWarps = kFpsThreads / 32;
constexpr int kFpsMaxCluster = 16;
constexpr int64_t kFpsMinPointsPerCta = 8192;  // the launch policy does not split a cloud finer than this
constexpr float kFpsInit = 1e10f;               // the reference's initial running distance

struct FpsArgs {
  const float* points;     // (N, P, 3)
  const int64_t* lengths;  // (N,) or nullptr for "all P"
  const int64_t* K;        // (N,)
  const int64_t* start;    // (N,)
  int64_t N, P, max_K;
  int64_t smem_pts;        // points per CTA in shared memory
  float* scratch;          // (N, P): running distances of the points held in neither tier
  int64_t* idx;            // (N, max_K)
};

struct FpsSlot {
  unsigned long long key;
  float x, y, z;
};

__device__ __forceinline__ unsigned long long fps_key(float d, int64_t p) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)(~(uint32_t)p);
}

__device__ __forceinline__ void fps_take(unsigned long long k, float x, float y, float z, unsigned long long& bk,
                                         float& bx, float& by, float& bz) {
  if (k > bk) {
    bk = k;
    bx = x;
    by = y;
    bz = z;
  }
}

// The largest key of the warp and its coordinates, in every lane: the high words' maximum, then the low words'
// maximum among the lanes that hold it (keys are distinct, so one lane holds the winner).
__device__ __forceinline__ void fps_warp_max(unsigned long long& k, float& x, float& y, float& z) {
  const unsigned hi = (unsigned)(k >> 32), lo = (unsigned)k;
  const unsigned mhi = __reduce_max_sync(0xffffffffu, hi);
  const unsigned mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
  const int src = __ffs(__ballot_sync(0xffffffffu, hi == mhi && lo == mlo)) - 1;
  k = ((unsigned long long)mhi << 32) | mlo;
  x = __shfl_sync(0xffffffffu, x, src);
  y = __shfl_sync(0xffffffffu, y, src);
  z = __shfl_sync(0xffffffffu, z, src);
}

__global__ void __launch_bounds__(kFpsThreads, 1) fps_kernel(FpsArgs a) {
  extern __shared__ float4 fps_smem[];  // smem_pts points as (x, y, z, running distance)
  __shared__ FpsSlot wslot[2][kFpsWarps];  // the warps' winners of the even / odd iterations
  __shared__ FpsSlot slot[2];              // the CTA's winner of the even / odd iterations, read over DSMEM
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks(), c = (int)cluster.block_rank();
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t n = blockIdx.x / C;
  const int64_t P = a.P, len = cloud_len(a.lengths, n, P), max_K = a.max_K;
  const int64_t start = __ldg(a.start + n);
  int64_t* __restrict__ row = a.idx + n * max_K;
  const int64_t rank_t = (int64_t)c * kFpsThreads + t, stride = (int64_t)C * kFpsThreads;
  // a start index outside [0, len) of a non-empty cloud selects nothing: the whole row is -1
  if (len > 0 && (start < 0 || start >= len)) {
    for (int64_t k = rank_t; k < max_K; k += stride) row[k] = -1;
    return;
  }
  int64_t kn = __ldg(a.K + n);
  kn = kn < len ? kn : len;
  kn = kn < max_K ? kn : max_K;
  if (rank_t == 0) row[0] = start;  // written unconditionally, as the reference does
  for (int64_t k = (kn > 1 ? kn : 1) + rank_t; k < max_K; k += stride) row[k] = -1;
  if (kn < 2) return;  // uniform over the cluster: no barrier is ever reached

  const float* __restrict__ pts = a.points + n * P * 3;
  // registers: points c * kFpsRegPoints + r * kFpsThreads + t
  const int reg0 = c * (int)kFpsRegPoints + t, len32 = (int)len;  // P < 2^31
  float px[kFpsRegs], py[kFpsRegs], pz[kFpsRegs], pd[kFpsRegs];
#pragma unroll
  for (int r = 0; r < kFpsRegs; ++r) {
    const int p = reg0 + r * kFpsThreads;
    const bool ok = p < len32;
    px[r] = ok ? __ldg(pts + 3 * p) : 0.0f;
    py[r] = ok ? __ldg(pts + 3 * p + 1) : 0.0f;
    pz[r] = ok ? __ldg(pts + 3 * p + 2) : 0.0f;
    pd[r] = kFpsInit;
  }
  // shared memory: points C kFpsRegPoints + c smem_pts + s
  const int64_t sm0 = (int64_t)C * kFpsRegPoints + (int64_t)c * a.smem_pts;
  const int64_t sm_cnt = len - sm0 < 0 ? 0 : (len - sm0 < a.smem_pts ? len - sm0 : a.smem_pts);
  for (int64_t s = t; s < sm_cnt; s += kFpsThreads) {
    const int64_t p = sm0 + s;
    fps_smem[s] = make_float4(__ldg(pts + 3 * p), __ldg(pts + 3 * p + 1), __ldg(pts + 3 * p + 2), kFpsInit);
  }
  // L2: points g0 + rank_t + m stride, running distances in scratch (each touched by one thread only)
  const int64_t g0 = (int64_t)C * (kFpsRegPoints + a.smem_pts);
  float* __restrict__ sd = a.scratch != nullptr ? a.scratch + n * P : nullptr;
  for (int64_t p = g0 + rank_t; p < len; p += stride) sd[p] = kFpsInit;
  __syncthreads();

  float sx = __ldg(pts + 3 * start), sy = __ldg(pts + 3 * start + 1), sz = __ldg(pts + 3 * start + 2);
  int64_t mine = -1;  // the selection of iteration k with k % kFpsThreads == t, stored once per kFpsThreads iterations
  for (int64_t k = 1; k < kn; ++k) {
    unsigned long long bk = 0;  // below every real key (distances are >= +0 and ~p != 0)
    float bx = 0.0f, by = 0.0f, bz = 0.0f;
#pragma unroll
    for (int r = 0; r < kFpsRegs; ++r) {
      const int p = reg0 + r * kFpsThreads;
      if (p < len32) {
        pd[r] = fminf(pair_dist<2>(sx, sy, sz, px[r], py[r], pz[r]), pd[r]);
        fps_take(fps_key(pd[r], p), px[r], py[r], pz[r], bk, bx, by, bz);
      }
    }
    for (int64_t s = t; s < sm_cnt; s += kFpsThreads) {
      float4 v = fps_smem[s];
      v.w = fminf(pair_dist<2>(sx, sy, sz, v.x, v.y, v.z), v.w);
      fps_smem[s].w = v.w;
      fps_take(fps_key(v.w, sm0 + s), v.x, v.y, v.z, bk, bx, by, bz);
    }
    for (int64_t p = g0 + rank_t; p < len; p += stride) {
      const float x = __ldg(pts + 3 * p), y = __ldg(pts + 3 * p + 1), z = __ldg(pts + 3 * p + 2);
      const float d = fminf(pair_dist<2>(sx, sy, sz, x, y, z), sd[p]);
      sd[p] = d;
      fps_take(fps_key(d, p), x, y, z, bk, bx, by, bz);
    }
    fps_warp_max(bk, bx, by, bz);
    const int par = (int)(k & 1);
    if (lane == 0) wslot[par][warp] = FpsSlot{bk, bx, by, bz};
    __syncthreads();
    FpsSlot e{0ull, 0.0f, 0.0f, 0.0f};
    if (C == 1) {  // every warp reduces the CTA's entries itself
      if (lane < kFpsWarps) e = wslot[par][lane];
      fps_warp_max(e.key, e.x, e.y, e.z);
    } else {  // warp 0 publishes the CTA's winner; after the barrier every warp reduces the cluster's C entries
      if (warp == 0) {
        if (lane < kFpsWarps) e = wslot[par][lane];
        fps_warp_max(e.key, e.x, e.y, e.z);
        if (lane == 0) slot[par] = e;
      }
      cluster.sync();
      e = FpsSlot{0ull, 0.0f, 0.0f, 0.0f};
      if (lane < C) e = *cluster.map_shared_rank(&slot[par], lane);
      fps_warp_max(e.key, e.x, e.y, e.z);
    }
    sx = e.x;
    sy = e.y;
    sz = e.z;
    // every thread knows the winner: CTA 0 keeps it in the thread of its residue and stores each run of kFpsThreads
    // selections in one coalesced store
    const int rk = (int)(k & (kFpsThreads - 1));
    if (rk == t) mine = (int64_t)(~(uint32_t)(e.key & 0xffffffffu));
    if (c == 0 && (rk == kFpsThreads - 1 || k == kn - 1) && t <= rk && k - rk + t >= 1) row[k - rk + t] = mine;
  }
  if (C > 1) cluster.sync();  // no CTA leaves while another may still read its slots
}

// ---- ball query forward ---------------------------------------------------------------------------------------------

struct BallArgs {
  const float* p1;  // (N, P1, 3) queries
  const float* p2;  // (N, P2, 3) targets
  const int64_t* len1;
  const int64_t* len2;
  int64_t N, P1, P2, K, qtiles;
  float r2;
  int none;  // skip_points_outside_cube with a negative radius: no target is inside the cube
  int64_t* idx;  // (N, P1, K)
  float* dists;  // (N, P1, K)
  float* nn;     // (N, P1, K, 3) or nullptr
};

__global__ void __launch_bounds__(kThreads) ball_query_kernel(BallArgs a) {
  __shared__ float4 tile[2][kTile];
  __shared__ int hits[kThreads];
  const int t = threadIdx.x;
  const int64_t n = blockIdx.x / a.qtiles, q0 = (blockIdx.x % a.qtiles) * kThreads, i = q0 + t;
  const int64_t len1 = cloud_len(a.len1, n, a.P1), len2 = cloud_len(a.len2, n, a.P2), K = a.K;
  const bool valid = i < len1;
  const float* __restrict__ q = a.p1 + (n * a.P1 + i) * 3;
  const float qx = valid ? __ldg(q) : 0.0f, qy = valid ? __ldg(q + 1) : 0.0f, qz = valid ? __ldg(q + 2) : 0.0f;
  const float r2 = a.r2;
  const int64_t o = (n * a.P1 + i) * K;
  const float* __restrict__ tp = a.p2 + n * a.P2 * 3;
  int count = 0;
  if (!a.none && len2 > 0 && q0 < len1) {  // uniform over the CTA
    const int64_t ntiles = (len2 + kTile - 1) / kTile;
    load_tile(tile[0], tp, 0, (int)min((int64_t)kTile, len2));
    cp_async_commit();
    for (int64_t it = 0; it < ntiles; ++it) {
      const int64_t jb = it * kTile;
      if (it + 1 < ntiles) {  // the other buffer was released by the previous iteration's trailing barrier
        load_tile(tile[(it + 1) & 1], tp, jb + kTile, (int)min((int64_t)kTile, len2 - jb - kTile));
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      const float4* buf = tile[it & 1];
      const int cnt = (int)min((int64_t)kTile, len2 - jb);
      if (valid)
        for (int jj = 0; jj < cnt && count < K; ++jj) {
          const float4 v = buf[jj];
          const float d = pair_dist<2>(qx, qy, qz, v.x, v.y, v.z);
          if (d < r2) {
            const int64_t e = o + count;
            a.idx[e] = jb + jj;
            a.dists[e] = d;
            if (a.nn != nullptr) {
              a.nn[3 * e] = v.x;
              a.nn[3 * e + 1] = v.y;
              a.nn[3 * e + 2] = v.z;
            }
            ++count;
          }
        }
      if (__syncthreads_and(!valid || count >= K)) break;
    }
    cp_async_wait<0>();  // a prefetch may be in flight after an early exit
  }
  // padding of the CTA's rows [q0, q1), element by element in flat order
  hits[t] = count;
  __syncthreads();
  const int64_t q1 = q0 + kThreads < a.P1 ? q0 + kThreads : a.P1;
  const int64_t e0 = (n * a.P1 + q0) * K, e1 = (n * a.P1 + q1) * K;
  for (int64_t e = e0 + t; e < e1; e += kThreads) {
    const int64_t local = e - e0, r = local / K;
    if (local - r * K < hits[r]) continue;
    a.idx[e] = -1;
    a.dists[e] = 0.0f;
    if (a.nn != nullptr) {
      a.nn[3 * e] = 0.0f;
      a.nn[3 * e + 1] = 0.0f;
      a.nn[3 * e + 2] = 0.0f;
    }
  }
}

// ---- ball query backward --------------------------------------------------------------------------------------------

constexpr int64_t kBallChunk = (int64_t)1 << 20;  // sorted rows per chunk of the grad_p2 pass

struct BallGradArgs {
  const float* p1;
  const float* p2;
  const int64_t* len1;
  const int64_t* len2;
  int64_t N, P1, P2, K;
  const int64_t* idx;     // (N, P1, K)
  const float* gd;        // (N, P1, K) upstream of dists, or nullptr
  const float* gnn;       // (N, P1, K, 3) upstream of nn, or nullptr
};

// Target index j of row r = (n, i, k), or -1 when the row is not a hit: knn_points_backward's conditions (i < lengths1,
// k < lengths2, j != -1), lengths clamped to [0, P] and j outside [0, P2) ignored.
__device__ __forceinline__ int64_t ball_hit(const BallGradArgs& a, int64_t r, int64_t n, int64_t i, int64_t k) {
  if (i >= cloud_len(a.len1, n, a.P1) || k >= cloud_len(a.len2, n, a.P2)) return -1;
  const int64_t j = __ldg(a.idx + r);
  return (j >= 0 && j < a.P2) ? j : -1;
}

// KNearestNeighborBackwardKernel's diff for norm 2: 2.0 * grad formed in double, times the float difference, rounded
// once.
__device__ __forceinline__ float3 ball_diff(const BallGradArgs& a, int64_t r, float3 q, float3 tp) {
  if (a.gd == nullptr) return make_float3(0.0f, 0.0f, 0.0f);
  const double g2 = 2.0 * (double)__ldg(a.gd + r);
  return make_float3((float)(g2 * (double)__fsub_rn(q.x, tp.x)), (float)(g2 * (double)__fsub_rn(q.y, tp.y)),
                     (float)(g2 * (double)__fsub_rn(q.z, tp.z)));
}

// grad_p1[n, i]: the diffs of the query's hits in k order from +0.
__global__ void __launch_bounds__(kThreads) ball_grad_p1_kernel(BallGradArgs a, float* __restrict__ grad_p1) {
  const int64_t Q = a.N * a.P1, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < Q; g += stride) {
    const int64_t n = g / a.P1, i = g - n * a.P1;
    float3 acc = make_float3(0.0f, 0.0f, 0.0f);
    if (a.gd != nullptr) {
      const float3 q = load3(a.p1, g);
      for (int64_t k = 0; k < a.K; ++k) {
        const int64_t r = g * a.K + k, j = ball_hit(a, r, n, i, k);
        if (j < 0) continue;
        const float3 d = ball_diff(a, r, q, load3(a.p2, n * a.P2 + j));
        acc = make_float3(__fadd_rn(acc.x, d.x), __fadd_rn(acc.y, d.y), __fadd_rn(acc.z, d.z));
      }
    }
    store3(grad_p1, g, acc);
  }
}

// (key, id) of rows [r0, r0 + cnt): the hit's target n P2 + j, or V (sorts last, in no run) for a row without one.
__global__ void __launch_bounds__(kThreads)
    ball_keys_kernel(BallGradArgs a, int64_t r0, int64_t cnt, uint32_t* __restrict__ keys, int32_t* __restrict__ ids) {
  const int64_t V = a.N * a.P2, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cnt; s += stride) {
    const int64_t r = r0 + s, q = r / a.K, k = r - q * a.K, n = q / a.P1, i = q - n * a.P1;
    const int64_t j = ball_hit(a, r, n, i, k);
    keys[s] = (uint32_t)(j >= 0 ? n * a.P2 + j : V);
    ids[s] = (int32_t)s;
  }
}

// The grad_p2 row of hit r0 + id at target point tp: -diff + g_nn, recomputed from the row.
struct BallRow : AddedRows {
  BallGradArgs a;
  int64_t r0;
  __device__ float3 at_key(int64_t v) const { return load3(a.p2, v); }
  __device__ float3 operator()(float3 tp, int32_t id) const {
    const int64_t r = r0 + id, q = r / a.K;
    const float3 d = ball_diff(a, r, load3(a.p1, q), tp);
    float3 row = make_float3(-d.x, -d.y, -d.z);
    if (a.gnn != nullptr) {
      const float3 g = load3(a.gnn, r);
      row = make_float3(__fadd_rn(row.x, g.x), __fadd_rn(row.y, g.y), __fadd_rn(row.z, g.z));
    }
    return row;
  }
};

// ---- host side ------------------------------------------------------------------------------------------------------

int max_dynamic_smem() {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return 0;
  return v - (int)(sizeof(FpsSlot) * 2 * (kFpsWarps + 1)) - 1024;  // the static slots and the runtime's reserve
}

struct FpsPlan {
  int cluster;
  int64_t smem_pts;
};

// Cluster size: a cloud gets its share of the SMs (N C <= SMs), at least kFpsMinPointsPerCta points per CTA, at most
// kFpsMaxCluster CTAs, and no more than the device can make resident with the shared memory it needs.  Shared memory
// holds what the registers of the cluster do not, up to the device limit; the rest stays in L2.
int fps_plan(int64_t N, int64_t P, int forced, cudaLaunchConfig_t& cfg, cudaLaunchAttribute& attr, FpsPlan& plan) {
  const int64_t sms = num_sms();
  int64_t C = forced;
  if (C <= 0) {
    const int64_t fill = sms / N > 1 ? sms / N : 1;
    const int64_t split = (P + kFpsMinPointsPerCta - 1) / kFpsMinPointsPerCta;
    C = fill < split ? fill : split;
    if (C > kFpsMaxCluster) C = kFpsMaxCluster;
    if (C < 1) C = 1;
  }
  const int64_t smem_cap = max_dynamic_smem() / (int64_t)sizeof(float4);
  B200R_CUDA_OK(cudaFuncSetAttribute(fps_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  for (;; --C) {
    const int64_t share = (P + C - 1) / C - kFpsRegPoints;
    plan.cluster = (int)C;
    plan.smem_pts = share <= 0 ? 0 : (share < smem_cap ? share : smem_cap);
    const int bytes = (int)(plan.smem_pts * (int64_t)sizeof(float4));
    B200R_CUDA_OK(cudaFuncSetAttribute(fps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    cfg.gridDim = dim3((unsigned)(N * C));
    cfg.blockDim = dim3(kFpsThreads);
    cfg.dynamicSmemBytes = (size_t)bytes;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)C;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int active = 0;
    if (cudaOccupancyMaxActiveClusters(&active, fps_kernel, &cfg) != cudaSuccess) {
      cudaGetLastError();
      active = 0;
    }
    if (active > 0 || C == 1 || forced > 0) return B200R_OK;
  }
}

struct BallLayout {
  int64_t chunk;
  size_t keys_in, keys_out, ids_in, ids_out, offsets, cub, cub_bytes, total;
};

bool ball_layout(int64_t N, int64_t P1, int64_t P2, int64_t K, BallLayout& L) {
  L = BallLayout{};
  const int64_t R = N * P1 * K, V = N * P2;
  L.chunk = R < kBallChunk ? R : kBallChunk;
  const size_t c = (size_t)(L.chunk > 0 ? L.chunk : 1);
  Carver w;
  L.keys_in = w.take(sizeof(uint32_t) * c);
  L.keys_out = w.take(sizeof(uint32_t) * c);
  L.ids_in = w.take(sizeof(int32_t) * c);
  L.ids_out = w.take(sizeof(int32_t) * c);
  L.offsets = w.take(sizeof(int32_t) * (size_t)(V + 1));
  const bool sized = run_sort_bytes(V, (int64_t)c, L.cub_bytes);
  L.cub = w.take(L.cub_bytes);
  L.total = w.used;
  return sized;
}

int check_ball(const char* op, int64_t N, int64_t P1, int64_t P2, int64_t K) {
  if (N < 0 || P1 < 0 || P2 < 0 || K < 0) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": bad sizes");
  if (N * P1 * K >= ((int64_t)1 << 31) || N * P2 >= ((int64_t)1 << 31))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": takes N P1 K < 2^31 and N P2 < 2^31");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" int b200r_sample_farthest_points(const float* points, int64_t N, int64_t P, const int64_t* lengths,
                                            const int64_t* K, const int64_t* start_idxs, int64_t max_K,
                                            int32_t cluster_size, float* scratch, int64_t* idx, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (N < 0 || P < 0 || max_K < 0 || P >= ((int64_t)1 << 31) || cluster_size < 0 || cluster_size > kFpsMaxCluster)
    return fail(B200R_ERR_INVALID_ARGUMENT, "sample_farthest_points: bad sizes");
  if (N == 0 || max_K == 0) return B200R_OK;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr{};
  FpsPlan plan{};
  int rc = fps_plan(N, P, cluster_size, cfg, attr, plan);
  if (rc != B200R_OK) return rc;
  cfg.stream = stream;
  if (P > (int64_t)plan.cluster * (kFpsRegPoints + plan.smem_pts) && scratch == nullptr)
    return fail(B200R_ERR_INVALID_ARGUMENT, "sample_farthest_points: this cloud size needs the (N, P) scratch");
  FpsArgs a{points, lengths, K, start_idxs, N, P, max_K, plan.smem_pts, scratch, idx};
  B200R_CUDA_OK(cudaLaunchKernelEx(&cfg, fps_kernel, a));
  B200R_LAUNCHED("fps_kernel");
  return B200R_OK;
}

extern "C" size_t b200r_ball_query_workspace_bytes(int64_t N, int64_t P1, int64_t P2, int64_t K) {
  if (check_ball("ball_query", N, P1, P2, K) != B200R_OK) return 0;
  BallLayout L;
  const bool sized = ball_layout(N, P1, P2, K, L);
  return workspace_size(sized, L.total);
}

extern "C" int b200r_ball_query_forward(const float* p1, const float* p2, int64_t N, int64_t P1, int64_t P2,
                                        const int64_t* lengths1, const int64_t* lengths2, int64_t K, float radius,
                                        int32_t skip_points_outside_cube, int64_t* idx, float* dists, float* nn,
                                        void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_ball("ball_query_forward", N, P1, P2, K);
  if (rc != B200R_OK) return rc;
  if (N == 0 || P1 == 0 || K == 0) return B200R_OK;
  BallArgs a{};
  a.p1 = p1;
  a.p2 = p2;
  a.len1 = lengths1;
  a.len2 = lengths2;
  a.N = N;
  a.P1 = P1;
  a.P2 = P2;
  a.K = K;
  a.qtiles = (P1 + kThreads - 1) / kThreads;
  a.r2 = radius * radius;  // BallQueryCuda's float radius2
  // |p1_d - p2_d| <= radius fails for every pair when radius < 0; for radius >= 0 the cube test removes no pair that
  // dist2 < radius2 keeps (|d| > r gives rn(d^2) >= rn(r^2), and the FFMA chain never decreases)
  a.none = skip_points_outside_cube != 0 && radius < 0.0f;
  a.idx = idx;
  a.dists = dists;
  a.nn = nn;
  ball_query_kernel<<<(unsigned)(N * a.qtiles), kThreads, 0, stream>>>(a);
  B200R_LAUNCHED("ball_query_kernel");
  return B200R_OK;
}

extern "C" int b200r_ball_query_backward(const float* p1, const float* p2, int64_t N, int64_t P1, int64_t P2,
                                         const int64_t* lengths1, const int64_t* lengths2, int64_t K,
                                         const int64_t* idx, const float* grad_dists, const float* grad_nn,
                                         void* workspace, size_t workspace_bytes, float* grad_p1, float* grad_p2,
                                         void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_ball("ball_query_backward", N, P1, P2, K);
  if (rc != B200R_OK) return rc;
  BallGradArgs a{p1, p2, lengths1, lengths2, N, P1, P2, K, idx, grad_dists, grad_nn};
  if (grad_p1 != nullptr && N * P1 > 0) {
    ball_grad_p1_kernel<<<grid_for(N * P1), kThreads, 0, stream>>>(a, grad_p1);
    B200R_LAUNCHED("ball_grad_p1_kernel");
  }
  const int64_t R = N * P1 * K, V = N * P2;
  if (grad_p2 == nullptr || V == 0) return B200R_OK;
  if (R == 0 || (grad_dists == nullptr && grad_nn == nullptr)) {
    B200R_CUDA_OK(cudaMemsetAsync(grad_p2, 0, sizeof(float) * 3 * (size_t)V, stream));
    return B200R_OK;
  }
  BallLayout L;
  const bool sized = ball_layout(N, P1, P2, K, L);
  rc = check_workspace("ball_query_backward", "b200r_ball_query_workspace_bytes", sized, L.total, workspace,
                       workspace_bytes);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  uint32_t* keys_in = reinterpret_cast<uint32_t*>(ws + L.keys_in);
  uint32_t* keys_out = reinterpret_cast<uint32_t*>(ws + L.keys_out);
  int32_t* ids_in = reinterpret_cast<int32_t*>(ws + L.ids_in);
  int32_t* ids_out = reinterpret_cast<int32_t*>(ws + L.ids_out);
  int32_t* offsets = reinterpret_cast<int32_t*>(ws + L.offsets);
  for (int64_t r0 = 0; r0 < R; r0 += L.chunk) {
    const int64_t cnt = R - r0 < L.chunk ? R - r0 : L.chunk;
    ball_keys_kernel<<<grid_for(cnt), kThreads, 0, stream>>>(a, r0, cnt, keys_in, ids_in);
    B200R_LAUNCHED("ball_keys_kernel");
    rc = sort_into_runs(keys_in, keys_out, ids_in, ids_out, cnt, V, ws + L.cub, L.cub_bytes, offsets, stream);
    if (rc != B200R_OK) return rc;
    if (r0 == 0)
      segmented_sum_kernel<Mode::kSum>
          <<<grid_for(V), kThreads, 0, stream>>>(offsets, ids_out, V, BallRow{{}, a, r0}, nullptr, grad_p2);
    else
      segmented_sum_kernel<Mode::kContinue>
          <<<grid_for(V), kThreads, 0, stream>>>(offsets, ids_out, V, BallRow{{}, a, r0}, nullptr, grad_p2);
    B200R_LAUNCHED("segmented_sum_kernel");
  }
  return B200R_OK;
}
