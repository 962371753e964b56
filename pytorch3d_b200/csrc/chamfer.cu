// Chamfer distance: pytorch3d.loss.chamfer_distance for 3-D point clouds, forward and deterministic backward
// (DESIGN.md section 21).
//
// Forward, three kernels (two when the target range is not split) and no host synchronisation:
//   1. nn_search_kernel: one launch searches both directions.  A CTA owns kThreads * kQ query points of one cloud of
//      one direction, kQ per thread in registers, and streams one range of the other cloud's points through shared
//      memory in tiles of kTile points, double-buffered with cp.async.  Each pair is evaluated in the arithmetic of
//      the reference's KNearestNeighborKernelV3<float, 3, 1> as nvcc compiles it for sm_90a (norm 2: three FFMA
//      from zero; norm 1: three FADD of |delta|), in ascending target order, a target replacing the result only when
//      d < current.  When N P is too small to fill the device, the target range is split across CTAs and the splits
//      meet in a 64-bit atomicMin on (float bits of d) << 32 | j: distances are >= +0, so the minimum key is the
//      smallest distance with the lowest index, whatever order the splits arrive in.
//   2. nn_merge_kernel (split searches only): decodes the keys.  Both paths apply the reference's seeding rule
//      explicitly: a NaN distance to target 0 is never replaced, so such a query gets (d_0, 0).
//   3. cloud_reduce_kernel + batch_reduce_kernel: the masks, weights, the gathered normals' cosine term and the
//      reductions of pytorch3d/loss/chamfer.py, one CTA per (direction, cloud) in a fixed association, then one
//      thread over the batch, which also sets the status word of the data-dependent checks.
//
// Backward: one thread per query point writes a gradient row for its own coordinates and one for its neighbour's
// (and the same two for the normals), keyed by point; sort_into_runs and the segmented sum of keyed_runs.cuh add
// each point's rows in one thread, its own row first.  No float atomics, no host synchronisation.
#include <climits>

#include "point_pairs.cuh"

namespace b200r {
namespace {

constexpr int kQ = 4;        // query points per thread
constexpr float kCosEps = 1e-6f;  // F.cosine_similarity(..., eps=1e-6) in chamfer.py

struct NNArgs {
  const float* pts[2];     // x (N, P1, 3), y (N, P2, 3)
  const int64_t* len[2];   // (N,) or nullptr for "all P"
  int64_t N, P[2];
  float* dist[2];          // per query point of direction d (queries from cloud d, targets from cloud 1 - d)
  int32_t* idx[2];
  unsigned long long* key[2];  // split searches: the merge keys, initialised to all ones
  int64_t qtiles[2];       // query tiles per cloud of each direction (0: the direction is not searched)
  int64_t splits, chunk;   // the target range of split s is [s chunk, (s + 1) chunk)
};

template <int NORM>
__global__ void __launch_bounds__(kThreads) nn_search_kernel(NNArgs a) {
  __shared__ float4 tile[2][kTile];
  // decode (direction, cloud, query tile, split) from the block index
  const int64_t s = blockIdx.x % a.splits;
  int64_t r = blockIdx.x / a.splits;
  int d = 0;
  if (r >= a.N * a.qtiles[0]) {
    r -= a.N * a.qtiles[0];
    d = 1;
  }
  const int64_t n = r / a.qtiles[d], qt = r % a.qtiles[d];
  const int64_t Pq = a.P[d], Pt = a.P[1 - d];
  const float* __restrict__ q = a.pts[d] + n * Pq * 3;
  const float* __restrict__ t = a.pts[1 - d] + n * Pt * 3;
  const int64_t len_q = cloud_len(a.len[d], n, Pq), len_t = cloud_len(a.len[1 - d], n, Pt);
  const int64_t j0 = s * a.chunk, j1 = min(j0 + a.chunk, len_t);

  float qx[kQ], qy[kQ], qz[kQ], best[kQ];
  int bi[kQ];
#pragma unroll
  for (int k = 0; k < kQ; ++k) {
    const int64_t p = qt * kThreads * kQ + k * kThreads + threadIdx.x;
    const bool ok = p < len_q;
    qx[k] = ok ? __ldg(q + 3 * p) : 0.0f;
    qy[k] = ok ? __ldg(q + 3 * p + 1) : 0.0f;
    qz[k] = ok ? __ldg(q + 3 * p + 2) : 0.0f;
    best[k] = __int_as_float(0x7f800000);
    bi[k] = -1;
  }
  if (j0 < j1) {  // uniform over the CTA
    const int64_t ntiles = (j1 - j0 + kTile - 1) / kTile;
    load_tile(tile[0], t, j0, (int)min((int64_t)kTile, j1 - j0));
    cp_async_commit();
    for (int64_t it = 0; it < ntiles; ++it) {
      const int64_t jb = j0 + it * kTile;
      if (it + 1 < ntiles) {  // the other buffer was released by the previous iteration's trailing barrier
        load_tile(tile[(it + 1) & 1], t, jb + kTile, (int)min((int64_t)kTile, j1 - jb - kTile));
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      const float4* buf = tile[it & 1];
      const int cnt = (int)min((int64_t)kTile, j1 - jb);
#pragma unroll 4
      for (int jj = 0; jj < cnt; ++jj) {
        const float4 tp = buf[jj];
#pragma unroll
        for (int k = 0; k < kQ; ++k) {
          const float dd = pair_dist<NORM>(qx[k], qy[k], qz[k], tp.x, tp.y, tp.z);
          if (dd < best[k]) {
            best[k] = dd;
            bi[k] = (int)jb + jj;
          }
        }
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int k = 0; k < kQ; ++k) {
    const int64_t p = qt * kThreads * kQ + k * kThreads + threadIdx.x;
    if (p >= Pq) continue;
    const bool ok = p < len_q;
    // no distance below +inf in the range (every one inf or NaN): the first that is not NaN, as the scan keeps it
    if (ok && bi[k] < 0)
      for (int64_t j = j0; j < j1; ++j) {
        const float dd = dist_to<NORM>(t, j, qx[k], qy[k], qz[k]);
        if (!isnan(dd)) {
          best[k] = dd;
          bi[k] = (int)j;
          break;
        }
      }
    const int64_t o = n * Pq + p;
    if (a.splits > 1) {
      if (ok && bi[k] >= 0)
        atomicMin(a.key[d] + o, ((unsigned long long)__float_as_uint(best[k]) << 32) | (unsigned)bi[k]);
      continue;
    }
    float dd = 0.0f;
    int j = 0;
    if (ok && len_t > 0) {
      const float d0 = dist_to<NORM>(t, 0, qx[k], qy[k], qz[k]);
      if (isnan(d0)) {  // target 0 seeds the result and d < NaN is never true
        dd = d0;
      } else {
        dd = best[k];
        j = bi[k];
      }
    }
    a.dist[d][o] = dd;
    a.idx[d][o] = j;
  }
}

template <int NORM>
__global__ void __launch_bounds__(kThreads) nn_merge_kernel(NNArgs a) {
  const int64_t m0 = a.qtiles[0] > 0 ? a.N * a.P[0] : 0, m1 = a.qtiles[1] > 0 ? a.N * a.P[1] : 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < m0 + m1; g += stride) {
    const int d = g < m0 ? 0 : 1;
    const int64_t o = d == 0 ? g : g - m0;
    const int64_t Pq = a.P[d], Pt = a.P[1 - d];
    const int64_t n = o / Pq, p = o % Pq;
    float dd = 0.0f;
    int j = 0;
    if (p < cloud_len(a.len[d], n, Pq) && cloud_len(a.len[1 - d], n, Pt) > 0) {
      const float* q = a.pts[d] + o * 3;
      const float d0 = dist_to<NORM>(a.pts[1 - d] + n * Pt * 3, 0, __ldg(q), __ldg(q + 1), __ldg(q + 2));
      const unsigned long long key = a.key[d][o];
      if (isnan(d0) || key == ~0ull) {
        dd = d0;
      } else {
        dd = __uint_as_float((unsigned)(key >> 32));
        j = (int)(key & 0xffffffffu);
      }
    }
    a.dist[d][o] = dd;
    a.idx[d][o] = j;
  }
}

// ---- epilogue -----------------------------------------------------------------------------------------------------

struct LossArgs {
  const float* pts[2];
  const float* nrm[2];     // normals (N, P, 3) or nullptr (both or neither)
  const int64_t* len[2];
  const float* weights;    // (N,) or nullptr
  int64_t N, P[2];
  const float* dist[2];
  const int32_t* idx[2];
  int point_red, batch_red, single, abs_cos;
  float* out[2];           // point_red NONE: the distance terms (N, P_d); otherwise out[0] is the loss
  float* out_n[2];         // the same for the normal terms (nullptr without normals)
  float* cloud;            // cloud_d[2N], cloud_c[2N], div
  int32_t* argmax;         // (2N) for point_red MAX
  int32_t* status;
};

__device__ __forceinline__ float raw_len_f(const int64_t* __restrict__ len, int64_t n, int64_t P) {
  const int64_t l = len == nullptr ? P : __ldg(len + n);
  return (float)(l < 1 ? 1 : l);  // x_lengths.clamp(min=1), then the int64 -> float32 promotion of the division
}

__device__ __forceinline__ bool point_valid(const int64_t* __restrict__ len, int64_t n, int64_t p) {
  return len == nullptr || p < __ldg(len + n);  // chamfer.py's x_mask: arange(P) >= lengths
}

// F.cosine_similarity(a, b, dim, eps): (a / max(|a|, eps)) . (b / max(|b|, eps)), summed over the three components.
__device__ __forceinline__ float cosine(float3 a, float3 b) {
  const float sa = norm3(a), sb = norm3(b);
  const float ma = sa < kCosEps ? kCosEps : sa, mb = sb < kCosEps ? kCosEps : sb;  // clamp_min_: NaN stays NaN
  return __fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(a.x, ma), __fdiv_rn(b.x, mb)),
                             __fmul_rn(__fdiv_rn(a.y, ma), __fdiv_rn(b.y, mb))),
                   __fmul_rn(__fdiv_rn(a.z, ma), __fdiv_rn(b.z, mb)));
}

// The per-point terms of direction d at (n, p): the masked, weighted distance and normal terms.
__device__ __forceinline__ void point_terms(const LossArgs& a, int d, int64_t n, int64_t p, float w, bool has_w,
                                            float& vd, float& vc) {
  const int64_t o = n * a.P[d] + p;
  const bool ok = point_valid(a.len[d], n, p);
  vd = ok ? a.dist[d][o] : 0.0f;
  if (has_w) vd = __fmul_rn(vd, w);
  vc = 0.0f;
  if (a.nrm[0] != nullptr) {
    if (ok) {
      const int64_t Pt = a.P[1 - d];
      const bool has_t = cloud_len(a.len[1 - d], n, Pt) > 0;  // knn_gather's mask: zeros when lengths2 < 1
      const float3 b = has_t ? load3(a.nrm[1 - d], n * Pt + a.idx[d][o]) : make_float3(0.0f, 0.0f, 0.0f);
      const float c = cosine(load3(a.nrm[d], o), b);
      vc = __fsub_rn(1.0f, a.abs_cos ? fabsf(c) : c);
    }
    if (has_w) vc = __fmul_rn(vc, w);
  }
}

// torch's max(dim) order: NaN first, then the greater value, ties to the lower index.
__device__ __forceinline__ bool max_before(float v, int i, float u, int k) {
  if (isnan(v)) return !isnan(u) || i < k;
  if (isnan(u)) return false;
  return v == u ? i < k : v > u;
}

// One CTA per (direction, cloud): per-point terms, or their sum / max in a fixed association.
__global__ void __launch_bounds__(kThreads) cloud_reduce_kernel(LossArgs a) {
  const int d = blockIdx.y;
  const int64_t n = blockIdx.x, P = a.P[d];
  const bool has_w = a.weights != nullptr;
  const float w = has_w ? __ldg(a.weights + n) : 1.0f;
  const bool is_max = a.point_red == B200R_CHAMFER_POINT_MAX;
  float sd = is_max ? __int_as_float(0xff800000) : 0.0f, sc = 0.0f;
  int arg = P > 0 ? 0 : -1;
  bool first = true;
  for (int64_t p = threadIdx.x; p < P; p += kThreads) {
    float vd, vc;
    point_terms(a, d, n, p, w, has_w, vd, vc);
    if (a.point_red == B200R_CHAMFER_POINT_NONE) {
      a.out[d][n * P + p] = vd;
      if (a.out_n[d] != nullptr) a.out_n[d][n * P + p] = vc;
    } else if (is_max) {
      if (first || max_before(vd, (int)p, sd, arg)) {
        sd = vd;
        arg = (int)p;
      }
      first = false;
    } else {
      sd = __fadd_rn(sd, vd);
      sc = __fadd_rn(sc, vc);
    }
  }
  if (a.point_red == B200R_CHAMFER_POINT_NONE) return;
  if (is_max && first) arg = INT_MAX;  // no element: loses every comparison
  // warp tree, then the warps in order
  for (int off = 16; off > 0; off >>= 1) {
    const float od = __shfl_down_sync(0xffffffffu, sd, off), oc = __shfl_down_sync(0xffffffffu, sc, off);
    const int oa = __shfl_down_sync(0xffffffffu, arg, off);
    if (is_max) {
      if (max_before(od, oa, sd, arg)) {
        sd = od;
        arg = oa;
      }
    } else {
      sd = __fadd_rn(sd, od);
      sc = __fadd_rn(sc, oc);
    }
  }
  __shared__ float wd[kThreads / 32], wc[kThreads / 32];
  __shared__ int wa[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    wd[warp] = sd;
    wc[warp] = sc;
    wa[warp] = arg;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  sd = wd[0];
  sc = wc[0];
  arg = wa[0];
  for (int k = 1; k < kThreads / 32; ++k) {
    if (is_max) {
      if (max_before(wd[k], wa[k], sd, arg)) {
        sd = wd[k];
        arg = wa[k];
      }
    } else {
      sd = __fadd_rn(sd, wd[k]);
      sc = __fadd_rn(sc, wc[k]);
    }
  }
  if (a.point_red == B200R_CHAMFER_POINT_MEAN) {
    const float l = raw_len_f(a.len[d], n, P);
    sd = __fdiv_rn(sd, l);
    sc = __fdiv_rn(sc, l);
  }
  a.cloud[d * a.N + n] = sd;
  a.cloud[2 * a.N + d * a.N + n] = sc;
  if (is_max) a.argmax[d * a.N + n] = arg;
}

// One thread: the per-cloud losses of the two directions combined, the batch reduction, and the status word.
__global__ void batch_reduce_kernel(LossArgs a) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const int64_t N = a.N;
  int32_t st = 0;
  float wsum = 0.0f;
  for (int64_t n = 0; n < N; ++n) {
    if (a.len[0] != nullptr && __ldg(a.len[0] + n) > a.P[0]) st |= B200R_CHAMFER_X_LENGTH;
    if (a.len[1] != nullptr && __ldg(a.len[1] + n) > a.P[1]) st |= B200R_CHAMFER_Y_LENGTH;
    if (a.weights != nullptr) {
      const float w = __ldg(a.weights + n);
      if (!(w >= 0.0f)) st |= B200R_CHAMFER_W_NEGATIVE;
      wsum = __fadd_rn(wsum, w);
    }
  }
  if (a.weights != nullptr && wsum == 0.0f) st |= B200R_CHAMFER_W_ZERO_SUM;
  *a.status = st;
  const float div = a.weights != nullptr ? wsum : (float)(N > 1 ? N : 1);
  a.cloud[4 * N] = div;
  if (a.point_red == B200R_CHAMFER_POINT_NONE) return;
  const bool nrm = a.out_n[0] != nullptr;
  float acc = 0.0f, accn = 0.0f;
  for (int64_t n = 0; n < N; ++n) {
    const float cx = a.cloud[n], cy = a.cloud[N + n];
    const float cnx = a.cloud[2 * N + n], cny = a.cloud[3 * N + n];
    float l, ln = 0.0f;
    if (a.single) {
      l = cx;
      ln = cnx;
    } else if (a.point_red == B200R_CHAMFER_POINT_MAX) {
      l = (isnan(cx) || isnan(cy)) ? __int_as_float(0x7fc00000) : fmaxf(cx, cy);  // torch.maximum
    } else {
      l = __fadd_rn(cx, cy);
      ln = __fadd_rn(cnx, cny);
    }
    if (a.batch_red == B200R_CHAMFER_BATCH_NONE) {
      a.out[0][n] = l;
      if (nrm) a.out_n[0][n] = ln;
    } else {
      acc = __fadd_rn(acc, l);
      accn = __fadd_rn(accn, ln);
    }
  }
  if (a.batch_red == B200R_CHAMFER_BATCH_NONE) return;
  if (a.batch_red == B200R_CHAMFER_BATCH_MEAN) {
    acc = __fdiv_rn(acc, div);
    accn = __fdiv_rn(accn, div);
  }
  a.out[0][0] = acc;
  if (nrm) a.out_n[0][0] = accn;
}

// ---- backward -----------------------------------------------------------------------------------------------------

struct GradArgs {
  LossArgs f;              // the forward's inputs, options and per-cloud state (out / out_n unused)
  const float* g[2];       // point_red NONE: upstream of the distance terms (N, P_d); otherwise g[0] of the loss
  const float* gn[2];      // the same for the normal terms, or nullptr
  int norm;
  float* rows;             // (2V, 3) distance rows, or nullptr
  float* nrows;            // (2V, 3) normal rows, or nullptr
  uint32_t* keys;          // (2V)
  int32_t* ids;            // (2V)
};

// d cos / d a for cos = (a / max(|a|, eps)) . (b / max(|b|, eps)) as autograd forms it: F.cosine_similarity clamps
// the norms in place under no_grad, so the gradient flows through the unclamped norm (zero where |a| = 0).
__device__ __forceinline__ float3 cosine_backward(float3 a, float3 b, float g) {
  const float sa = norm3(a), sb = norm3(b);
  const float ma = sa < kCosEps ? kCosEps : sa, mb = sb < kCosEps ? kCosEps : sb;
  const float3 gu = make_float3(__fmul_rn(g, __fdiv_rn(b.x, mb)), __fmul_rn(g, __fdiv_rn(b.y, mb)),
                                __fmul_rn(g, __fdiv_rn(b.z, mb)));
  const float gm = __fadd_rn(__fadd_rn(-__fmul_rn(gu.x, __fdiv_rn(__fdiv_rn(a.x, ma), ma)),
                                       -__fmul_rn(gu.y, __fdiv_rn(__fdiv_rn(a.y, ma), ma))),
                             -__fmul_rn(gu.z, __fdiv_rn(__fdiv_rn(a.z, ma), ma)));
  const float k = sa == 0.0f ? 0.0f : __fdiv_rn(gm, sa);
  return make_float3(__fadd_rn(__fdiv_rn(gu.x, ma), __fmul_rn(a.x, k)),
                     __fadd_rn(__fdiv_rn(gu.y, ma), __fmul_rn(a.y, k)),
                     __fadd_rn(__fdiv_rn(gu.z, ma), __fmul_rn(a.z, k)));
}

// Upstream of the per-cloud value of direction d, cloud n (the loss's reductions undone).
__device__ __forceinline__ float cloud_grad(const GradArgs& a, const float* g, int d, int64_t n) {
  const LossArgs& f = a.f;
  const int64_t N = f.N;
  float gb = f.batch_red == B200R_CHAMFER_BATCH_NONE ? __ldg(g + n) : __ldg(g);
  if (f.batch_red == B200R_CHAMFER_BATCH_MEAN) gb = __fdiv_rn(gb, f.cloud[4 * N]);
  if (f.point_red == B200R_CHAMFER_POINT_MAX && !f.single) {  // torch.maximum's backward
    const float s = f.cloud[d * N + n], o = f.cloud[(1 - d) * N + n];
    if (s == o) gb = __fmul_rn(gb, 0.5f);
    if (s < o) gb = 0.0f;
  }
  return gb;
}

__global__ void __launch_bounds__(kThreads) grad_rows_kernel(GradArgs a) {
  const LossArgs& f = a.f;
  const int64_t N = f.N, m0 = N * f.P[0], V = m0 + N * f.P[1];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < V; g += stride) {
    const int d = g < m0 ? 0 : 1;
    const int64_t o = d == 0 ? g : g - m0;
    const int64_t Pq = f.P[d], Pt = f.P[1 - d];
    const int64_t n = o / Pq, p = o % Pq;
    const int64_t tbase = d == 0 ? m0 + n * Pt : n * Pt;  // the key of target point 0 of this cloud
    const bool searched = d == 0 || !f.single;
    const bool ok = searched && point_valid(f.len[d], n, p) && cloud_len(f.len[1 - d], n, Pt) > 0;
    const int64_t j = ok ? f.idx[d][o] : 0;
    float3 rd = make_float3(0.0f, 0.0f, 0.0f), rn = rd, tn = rd;
    bool has_n = false;
    if (ok) {
      float w = 1.0f;
      if (f.weights != nullptr) w = __ldg(f.weights + n);
      float gd, gc = 0.0f;
      if (f.point_red == B200R_CHAMFER_POINT_NONE) {
        gd = __ldg(a.g[d] + o);
        if (a.gn[d] != nullptr) gc = __ldg(a.gn[d] + o);
      } else {
        gd = cloud_grad(a, a.g[0], d, n);
        if (a.gn[0] != nullptr) gc = cloud_grad(a, a.gn[0], d, n);
        if (f.point_red == B200R_CHAMFER_POINT_MAX) {
          if (f.argmax[d * N + n] != (int)p) gd = 0.0f;
        } else if (f.point_red == B200R_CHAMFER_POINT_MEAN) {
          const float l = raw_len_f(f.len[d], n, Pq);
          gd = __fdiv_rn(gd, l);
          gc = __fdiv_rn(gc, l);
        }
      }
      if (f.weights != nullptr) {
        gd = __fmul_rn(gd, w);
        gc = __fmul_rn(gc, w);
      }
      if (a.rows != nullptr) {
        const float3 qp = load3(f.pts[d], o), tp = load3(f.pts[1 - d], n * Pt + j);
        const float dl[3] = {__fsub_rn(qp.x, tp.x), __fsub_rn(qp.y, tp.y), __fsub_rn(qp.z, tp.z)};
        const float qc[3] = {qp.x, qp.y, qp.z}, tc[3] = {tp.x, tp.y, tp.z};
        float r[3];
#pragma unroll
        for (int c = 0; c < 3; ++c)  // KNearestNeighborBackwardKernel: 2.0 * grad formed in double, rounded once
          r[c] = a.norm == 2 ? (float)((2.0 * (double)gd) * (double)dl[c])
                             : __fmul_rn(gd, qc[c] > tc[c] ? 1.0f : -1.0f);
        rd = make_float3(r[0], r[1], r[2]);
      }
      if (a.nrows != nullptr) {
        const float3 na = load3(f.nrm[d], o), nb = load3(f.nrm[1 - d], n * Pt + j);
        const float c = cosine(na, nb);
        // 1 - |cos| (or 1 - cos): d/dcos = -sign(cos) (or -1), torch's sign(0) = 0 and sign(NaN) = NaN
        const float sg = !f.abs_cos ? 1.0f : (isnan(c) ? c : (c > 0.0f ? 1.0f : (c < 0.0f ? -1.0f : 0.0f)));
        const float gcos = __fmul_rn(-gc, sg);
        rn = cosine_backward(na, nb, gcos);
        tn = cosine_backward(nb, na, gcos);
        has_n = true;
      }
    }
    // own row (id = key = g) and neighbour row (id V + g, keyed by the neighbour, or V for none)
    a.keys[g] = (uint32_t)g;
    a.ids[g] = (int32_t)g;
    a.keys[V + g] = (uint32_t)(ok ? tbase + j : V);
    a.ids[V + g] = (int32_t)(V + g);
    if (a.rows != nullptr) {
      store3(a.rows, g, rd);
      store3(a.rows, V + g, make_float3(-rd.x, -rd.y, -rd.z));  // -1.0f * diff
    }
    if (a.nrows != nullptr) {
      store3(a.nrows, g, rn);
      store3(a.nrows, V + g, has_n ? tn : make_float3(0.0f, 0.0f, 0.0f));
    }
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

struct Layout {
  size_t key0, key1;                                          // forward (split searches)
  size_t keys_in, keys_out, ids_out, offsets, cub, cub_bytes;  // backward (rows and ids are separate)
  size_t rows, nrows, ids_in;
  size_t total;
};

// The search's decomposition: query tiles per cloud, splits of the target range and their length.
void plan(int64_t N, int64_t P1, int64_t P2, bool single, NNArgs& a) {
  const int64_t per_cta = (int64_t)kThreads * kQ;
  a.qtiles[0] = (P1 + per_cta - 1) / per_cta;
  a.qtiles[1] = single ? 0 : (P2 + per_cta - 1) / per_cta;
  const int64_t base = N * (a.qtiles[0] + a.qtiles[1]);
  const int64_t Pt = single ? P2 : (P1 > P2 ? P1 : P2);
  const int64_t want = 2 * num_sms();
  int64_t splits = base >= want ? 1 : (want + base - 1) / base;
  const int64_t max_splits = (Pt + kTile - 1) / kTile;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int64_t chunk = (Pt + splits - 1) / splits;
  chunk = (chunk + kTile - 1) / kTile * kTile;
  a.chunk = chunk > 0 ? chunk : kTile;
  a.splits = (Pt + a.chunk - 1) / a.chunk;
  if (a.splits < 1) a.splits = 1;
}

bool layout(int64_t N, int64_t P1, int64_t P2, int32_t pass, Layout& L) {
  L = Layout{};
  Carver c;
  if (pass == 0) {
    L.key0 = c.take(sizeof(unsigned long long) * (size_t)(N * P1));
    L.key1 = c.take(sizeof(unsigned long long) * (size_t)(N * P2));
    L.total = c.used;
    return true;
  }
  const size_t V = (size_t)(N * P1 + N * P2), R = 2 * V;
  L.rows = c.take(sizeof(float) * 3 * R);
  L.nrows = c.take(sizeof(float) * 3 * R);
  L.keys_in = c.take(sizeof(uint32_t) * R);
  L.keys_out = c.take(sizeof(uint32_t) * R);
  L.ids_in = c.take(sizeof(int32_t) * R);
  L.ids_out = c.take(sizeof(int32_t) * R);
  L.offsets = c.take(sizeof(int32_t) * (V + 1));
  const bool sized = run_sort_bytes((int64_t)V, (int64_t)R, L.cub_bytes);
  L.cub = c.take(L.cub_bytes);
  L.total = c.used;
  return sized;
}

int check_args(const char* op, int64_t N, int64_t P1, int64_t P2, int32_t norm, int32_t point_red, int32_t batch_red) {
  if (N < 1 || P1 < 1 || P2 < 1) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": bad sizes");
  if (2 * (N * P1 + N * P2) >= ((int64_t)1 << 31))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": takes 2 (N P1 + N P2) < 2^31 points");
  if (norm != 1 && norm != 2) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": norm must be 1 or 2");
  if (point_red < 0 || point_red > 3 || batch_red < 0 || batch_red > 2 ||
      (point_red == B200R_CHAMFER_POINT_NONE && batch_red != B200R_CHAMFER_BATCH_NONE))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": bad reductions");
  return B200R_OK;
}

LossArgs loss_args(const float* x, const float* y, int64_t N, int64_t P1, int64_t P2, const int64_t* x_lengths,
                   const int64_t* y_lengths, const float* x_normals, const float* y_normals, const float* weights,
                   int32_t point_red, int32_t batch_red, int32_t single, int32_t abs_cosine, const float* dist_x,
                   const int32_t* idx_x, const float* dist_y, const int32_t* idx_y, float* cloud, int32_t* argmax) {
  LossArgs a{};
  a.pts[0] = x;
  a.pts[1] = y;
  const bool nrm = x_normals != nullptr && y_normals != nullptr;
  a.nrm[0] = nrm ? x_normals : nullptr;
  a.nrm[1] = nrm ? y_normals : nullptr;
  a.len[0] = x_lengths;
  a.len[1] = y_lengths;
  a.weights = weights;
  a.N = N;
  a.P[0] = P1;
  a.P[1] = P2;
  a.dist[0] = dist_x;
  a.dist[1] = dist_y;
  a.idx[0] = idx_x;
  a.idx[1] = idx_y;
  a.point_red = point_red;
  a.batch_red = batch_red;
  a.single = single;
  a.abs_cos = abs_cosine;
  a.cloud = cloud;
  a.argmax = argmax;
  return a;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" size_t b200r_chamfer_workspace_bytes(int64_t N, int64_t P1, int64_t P2, int32_t pass) {
  if (N < 1 || P1 < 1 || P2 < 1 || (pass != 0 && pass != 1)) return 0;
  Layout L;
  const bool sized = layout(N, P1, P2, pass, L);
  return workspace_size(sized, L.total);
}

extern "C" int b200r_chamfer_forward(const float* x, const float* y, int64_t N, int64_t P1, int64_t P2,
                                     const int64_t* x_lengths, const int64_t* y_lengths, const float* x_normals,
                                     const float* y_normals, const float* weights, int32_t norm, int32_t point_red,
                                     int32_t batch_red, int32_t single, int32_t abs_cosine, void* workspace,
                                     size_t workspace_bytes, float* dist_x, int32_t* idx_x, float* dist_y,
                                     int32_t* idx_y, float* cloud, int32_t* argmax, float* out_x, float* out_y,
                                     float* out_nx, float* out_ny, int32_t* status, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_args("chamfer_forward", N, P1, P2, norm, point_red, batch_red);
  if (rc != B200R_OK) return rc;
  Layout L;
  layout(N, P1, P2, 0, L);  // the forward's keys need no cub storage
  NNArgs s{};
  plan(N, P1, P2, single != 0, s);
  if (s.splits > 1 && (workspace == nullptr || workspace_bytes < L.total))
    return fail(B200R_ERR_INVALID_ARGUMENT, "chamfer_forward: workspace smaller than b200r_chamfer_workspace_bytes");
  s.pts[0] = x;
  s.pts[1] = y;
  s.len[0] = x_lengths;
  s.len[1] = y_lengths;
  s.N = N;
  s.P[0] = P1;
  s.P[1] = P2;
  s.dist[0] = dist_x;
  s.dist[1] = dist_y;
  s.idx[0] = idx_x;
  s.idx[1] = idx_y;
  if (s.splits > 1) {
    char* ws = static_cast<char*>(workspace);
    s.key[0] = reinterpret_cast<unsigned long long*>(ws + L.key0);
    s.key[1] = reinterpret_cast<unsigned long long*>(ws + L.key1);
    B200R_CUDA_OK(cudaMemsetAsync(ws, 0xff, L.total, stream));
  }
  const unsigned blocks = (unsigned)(N * (s.qtiles[0] + s.qtiles[1]) * s.splits);
  if (norm == 2) nn_search_kernel<2><<<blocks, kThreads, 0, stream>>>(s);
  else nn_search_kernel<1><<<blocks, kThreads, 0, stream>>>(s);
  B200R_LAUNCHED("nn_search_kernel");
  if (s.splits > 1) {
    const dim3 grid = grid_for(N * P1 + (single ? 0 : N * P2));
    if (norm == 2) nn_merge_kernel<2><<<grid, kThreads, 0, stream>>>(s);
    else nn_merge_kernel<1><<<grid, kThreads, 0, stream>>>(s);
    B200R_LAUNCHED("nn_merge_kernel");
  }
  LossArgs a = loss_args(x, y, N, P1, P2, x_lengths, y_lengths, x_normals, y_normals, weights, point_red, batch_red,
                         single, abs_cosine, dist_x, idx_x, dist_y, idx_y, cloud, argmax);
  a.out[0] = out_x;
  a.out[1] = out_y;
  a.out_n[0] = a.nrm[0] != nullptr ? out_nx : nullptr;
  a.out_n[1] = a.nrm[0] != nullptr ? out_ny : nullptr;
  a.status = status;
  cloud_reduce_kernel<<<dim3((unsigned)N, single ? 1 : 2), kThreads, 0, stream>>>(a);
  B200R_LAUNCHED("cloud_reduce_kernel");
  batch_reduce_kernel<<<1, 32, 0, stream>>>(a);
  B200R_LAUNCHED("batch_reduce_kernel");
  return B200R_OK;
}

extern "C" int b200r_chamfer_backward(const float* x, const float* y, int64_t N, int64_t P1, int64_t P2,
                                      const int64_t* x_lengths, const int64_t* y_lengths, const float* x_normals,
                                      const float* y_normals, const float* weights, int32_t norm, int32_t point_red,
                                      int32_t batch_red, int32_t single, int32_t abs_cosine, const int32_t* idx_x,
                                      const int32_t* idx_y, const float* cloud, const int32_t* argmax,
                                      const float* grad_x, const float* grad_y, const float* grad_nx,
                                      const float* grad_ny, void* workspace, size_t workspace_bytes,
                                      float* grad_points, float* grad_normals, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_args("chamfer_backward", N, P1, P2, norm, point_red, batch_red);
  if (rc != B200R_OK) return rc;
  if (grad_points == nullptr && grad_normals == nullptr) return B200R_OK;
  if (grad_normals != nullptr && (x_normals == nullptr || y_normals == nullptr || grad_nx == nullptr))
    return fail(B200R_ERR_INVALID_ARGUMENT, "chamfer_backward: the normals' gradient needs the normals and theirs");
  Layout L;
  const bool sized = layout(N, P1, P2, 1, L);
  rc = check_workspace("chamfer_backward", "b200r_chamfer_workspace_bytes", sized, L.total, workspace, workspace_bytes);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  GradArgs g{};
  g.f = loss_args(x, y, N, P1, P2, x_lengths, y_lengths, x_normals, y_normals, weights, point_red, batch_red, single,
                  abs_cosine, nullptr, idx_x, nullptr, idx_y, const_cast<float*>(cloud), const_cast<int32_t*>(argmax));
  g.g[0] = grad_x;
  g.g[1] = grad_y;
  g.gn[0] = grad_nx;
  g.gn[1] = grad_ny;
  g.norm = norm;
  g.rows = grad_points != nullptr ? reinterpret_cast<float*>(ws + L.rows) : nullptr;
  g.nrows = grad_normals != nullptr ? reinterpret_cast<float*>(ws + L.nrows) : nullptr;
  g.keys = reinterpret_cast<uint32_t*>(ws + L.keys_in);
  g.ids = reinterpret_cast<int32_t*>(ws + L.ids_in);
  uint32_t* keys_out = reinterpret_cast<uint32_t*>(ws + L.keys_out);
  int32_t* ids_out = reinterpret_cast<int32_t*>(ws + L.ids_out);
  int32_t* offsets = reinterpret_cast<int32_t*>(ws + L.offsets);
  const int64_t V = N * P1 + N * P2, R = 2 * V;
  grad_rows_kernel<<<grid_for(V), kThreads, 0, stream>>>(g);
  B200R_LAUNCHED("grad_rows_kernel");
  rc = sort_into_runs(g.keys, keys_out, g.ids, ids_out, R, V, ws + L.cub, L.cub_bytes, offsets, stream);
  if (rc != B200R_OK) return rc;
  if (grad_points != nullptr) {
    segmented_sum_kernel<Mode::kSum>
        <<<grid_for(V), kThreads, 0, stream>>>(offsets, ids_out, V, RowsById{{}, g.rows}, nullptr, grad_points);
    B200R_LAUNCHED("segmented_sum_kernel");
  }
  if (grad_normals != nullptr) {
    segmented_sum_kernel<Mode::kSum>
        <<<grid_for(V), kThreads, 0, stream>>>(offsets, ids_out, V, RowsById{{}, g.nrows}, nullptr, grad_normals);
    B200R_LAUNCHED("segmented_sum_kernel");
  }
  return B200R_OK;
}
