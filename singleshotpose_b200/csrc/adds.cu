// ADD-S / ADD of pose pairs over a mesh and the mesh diameter (reference utils.py:50-64, valid.py:69-72), fp64 throughout.
// The rules and the summation order are in adds_core.h.
//
// adds_kernel: one CTA per (pose pair, block of kQueriesPerBlock query vertices).  Each thread keeps its queries (in the
// estimate's model frame) and their running minimum squared distances in registers and streams the mesh through shared
// memory in tiles of kTile vertices; every thread reads the same vertex at a time (a broadcast).  Brute force: n * Nv^2 pair
// evaluations of 7 fp64 operations each.  The CTA writes one ADD-S and one ADD block sum; adds_finish_kernel adds the block
// sums of a pose in block order.  No atomics, so every pose's result is the same on every launch and in any batch.
//
// diameter_kernel: one CTA per (row tile, column tile >= row tile) of the pair matrix, a running max per row, then a warp max
// and an atomicMax on the bit pattern (non-negative doubles order like their bits), which is order-independent.
#include <limits.h>

#include "ssp_common.cuh"
#include "adds_core.h"

namespace ssp {
using namespace ssp_adds;

__global__ void __launch_bounds__(kThreads) adds_kernel(const double* __restrict__ X /*[nv][3]*/, int nv,
                                                        const double* __restrict__ Rt_est, const double* __restrict__ Rt_gt,
                                                        int nblk, double* __restrict__ sums_adds, double* __restrict__ sums_add) {
  __shared__ double2 s_xy[kTile];
  __shared__ double s_z[kTile];
  __shared__ double s_pose[24];
  __shared__ double s_red[2][kThreads];
  const long long p = blockIdx.x;
  const int blk = blockIdx.y, t = threadIdx.x;
  if (t < 12) s_pose[t] = Rt_est[p * 12 + t];
  else if (t < 24) s_pose[t] = Rt_gt[p * 12 + t - 12];
  __syncthreads();
  double q[kQueriesPerThread][3], m[kQueriesPerThread];
  double add = 0.0;
#pragma unroll
  for (int k = 0; k < kQueriesPerThread; k++) {
    const int i = query_index(blk, k, t);
    m[k] = INFINITY;
    if (i < nv) {
      const double x = X[3LL * i], y = X[3LL * i + 1], z = X[3LL * i + 2];
      model_frame_query(s_pose, s_pose + 12, x, y, z, q[k]);
      add = add + sqrt(sq_dist(q[k], x, y, z));
    } else {
      q[k][0] = q[k][1] = q[k][2] = 0.0;
    }
  }
  for (int base = 0; base < nv; base += kTile) {
    const int cnt = min(kTile, nv - base);
    __syncthreads();                                           // the previous tile has been read
    for (int j = t; j < cnt; j += kThreads) {
      const double* v = X + 3LL * (base + j);
      s_xy[j] = make_double2(v[0], v[1]);
      s_z[j] = v[2];
    }
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < cnt; j++) {
      const double2 xy = s_xy[j];
      const double z = s_z[j];
#pragma unroll
      for (int k = 0; k < kQueriesPerThread; k++) m[k] = fmin(m[k], sq_dist(q[k], xy.x, xy.y, z));
    }
  }
  double adds = 0.0;
#pragma unroll
  for (int k = 0; k < kQueriesPerThread; k++)
    if (query_index(blk, k, t) < nv) adds = adds + sqrt(m[k]);
  s_red[0][t] = adds;
  s_red[1][t] = add;
  for (int stride = kThreads / 2; stride > 0; stride >>= 1) {
    __syncthreads();
    if (t < stride) { tree_step(s_red[0], t, stride); tree_step(s_red[1], t, stride); }
  }
  if (t == 0) {
    sums_adds[p * nblk + blk] = s_red[0][0];
    sums_add[p * nblk + blk] = s_red[1][0];
  }
}

__global__ void adds_finish_kernel(const double* __restrict__ sums_adds, const double* __restrict__ sums_add, int nblk, int nv, long long n,
                                   double* __restrict__ adds_out, double* __restrict__ add_out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  adds_out[p] = finish_mean(sums_adds + p * nblk, nblk, nv);
  if (add_out) add_out[p] = finish_mean(sums_add + p * nblk, nblk, nv);
}

__global__ void __launch_bounds__(kTile) diameter_kernel(const double* __restrict__ X, int nv, unsigned long long* __restrict__ best_bits) {
  const int ti = blockIdx.y, tj = blockIdx.x, t = threadIdx.x;
  if (tj < ti) return;                                         // the distance is symmetric: one triangle of tiles
  __shared__ double s_x[kTile], s_y[kTile], s_z[kTile];
  const int j0 = tj * kTile, cnt = min(kTile, nv - j0);
  for (int j = t; j < cnt; j += kTile) {
    s_x[j] = X[3LL * (j0 + j)]; s_y[j] = X[3LL * (j0 + j) + 1]; s_z[j] = X[3LL * (j0 + j) + 2];
  }
  __syncthreads();
  const int i = ti * kTile + t;
  double best = 0.0;
  if (i < nv) {
    const double x = X[3LL * i], y = X[3LL * i + 1], z = X[3LL * i + 2];
    for (int j = 0; j < cnt; j++) best = fmax(best, diameter_sq(x - s_x[j], y - s_y[j], z - s_z[j]));
  }
  for (int off = 16; off > 0; off >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, off));
  if ((t & 31) == 0) atomicMax(best_bits, (unsigned long long)__double_as_longlong(best));
}

__global__ void diameter_finish_kernel(double* out) {
  *out = sqrt(__longlong_as_double((long long)*reinterpret_cast<const unsigned long long*>(out)));
}

}  // namespace ssp

using namespace ssp;

extern "C" {
long long ssp_adds_work_bytes(int nv, long long n) {
  if (nv < 1 || nv > kMaxVertices || n < 0 || n > INT_MAX) return SSP_ERR_ARG;
  return 2LL * n * query_blocks(nv) * (long long)sizeof(double);
}

int ssp_adds_batched(const double* X, int nv, const double* Rt_est, const double* Rt_gt, long long n, double* adds_out, double* add_out,
                     void* work, long long work_bytes, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!X || !Rt_est || !Rt_gt || !adds_out || !work || nv < 1 || n < 0)
    return fail_msg(SSP_ERR_ARG, "adds_batched: bad argument (null pointer, Nv < 1 or n < 0)");
  if (nv > kMaxVertices) return fail_msg(SSP_ERR_ARG, "adds_batched: more than SSP_ADDS_MAX_VERTICES vertices");
  if (n > INT_MAX) return fail_msg(SSP_ERR_ARG, "adds_batched: more than 2^31 - 1 pose pairs");
  if (work_bytes < ssp_adds_work_bytes(nv, n)) return fail_msg(SSP_ERR_ARG, "adds_batched: work buffer smaller than ssp_adds_work_bytes()");
  if (n == 0) return SSP_OK;
  const int nblk = query_blocks(nv);
  double* sums_adds = static_cast<double*>(work);
  double* sums_add = sums_adds + n * nblk;
  adds_kernel<<<dim3((unsigned)n, (unsigned)nblk), kThreads, 0, s>>>(X, nv, Rt_est, Rt_gt, nblk, sums_adds, sums_add);
  SSP_CHECK_LAUNCH();
  adds_finish_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(sums_adds, sums_add, nblk, nv, n, adds_out, add_out);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

int ssp_mesh_diameter(const double* X, int nv, double* out, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!X || !out || nv < 1) return fail_msg(SSP_ERR_ARG, "mesh_diameter: bad argument (null pointer or Nv < 1)");
  if (nv > kMaxVertices) return fail_msg(SSP_ERR_ARG, "mesh_diameter: more than SSP_ADDS_MAX_VERTICES vertices");
  const cudaError_t e = cudaMemsetAsync(out, 0, sizeof(double), s);          // +0.0: the identity of the max
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  const unsigned tiles = (unsigned)((nv + kTile - 1) / kTile);
  diameter_kernel<<<dim3(tiles, tiles), kTile, 0, s>>>(X, nv, reinterpret_cast<unsigned long long*>(out));
  SSP_CHECK_LAUNCH();
  diameter_finish_kernel<<<1, 1, 0, s>>>(out);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
