// Batched PnP pose recovery (replaces the per-image cv2.solvePnP(ITERATIVE) + cv2.Rodrigues loop of reference
// utils.py:86-100 as called from valid.py:152-153) and batched compute_projection (utils.py:40-45).
//
// One problem per thread, all arithmetic in fp64 like OpenCV:
//   1. normalise the 2-D points with K (zero distortion);
//   2. DLT initialisation exactly as cvFindExtrinsicCameraParams2 poses it: the 2N x 12 system on the RAW 3-D coordinates,
//      unit-norm constraint over all 12 entries, i.e. the eigenvector of the smallest eigenvalue of the 12x12 normal matrix
//      L^T L = [[S, 0, -Sx], [0, S, -Sy], [-Sx, -Sy, Sq]] (S = sum XX^T, Sx = sum x XX^T, ..., X = [X Y Z 1]); cyclic Jacobi in
//      fp64.  (Round 1 eliminated p1, p2 analytically on Hartley-normalised points: the same minimiser for exact data but a
//      different constraint under noise, so garbage keypoints -- what a random-init network emits -- could start LM in another
//      basin than OpenCV.  With the exact formulation the kernel tracks cv2 at every noise level, sigma = 80 px included.)
//   3. nearest rotation by polar decomposition, OpenCV's scale fix for t, Rodrigues -> rvec;
//   4. Levenberg-Marquardt in pixel space with OpenCV's CvLevMarq schedule (lambda = 10^k, k0 = -3, diagonal
//      scaling (1+lambda), reject => k++, accept => k--, <= max_iter accepted steps, eps = FLT_EPSILON).
// The kernel is fp64-ALU / local-memory bound: ~1.6e4 flop per Jacobi sweep (6-9 sweeps), ~3e3 per LM evaluation, 120 B of HBM
// traffic per problem.
#include "ssp_common.cuh"
#include "pnp_core.h"

namespace ssp {

// kCounted: problem id = g * per_group + m is solved only when m < count[g] (count in device memory); the others get zero R, t
template <bool kCounted>
__global__ void __launch_bounds__(128) pnp_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                  const float* __restrict__ Kmat, int np, long long n, int max_iter,
                                                  double* __restrict__ R_out, double* __restrict__ t_out, int* __restrict__ iters_out,
                                                  int* __restrict__ work_out /*[n][3]: Jacobi sweeps, LM iterations, LM solves; or null*/,
                                                  const int* __restrict__ count, int per_group) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  if (kCounted && id % per_group >= count[id / per_group]) {
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = 0.0;
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = 0.0;
    return;
  }
  int work[3];
  ssp_pnp::pnp_solve_one(P3 + id * p3_stride, uv + id * 2 * np, Kmat, np, max_iter, R_out + id * 9, t_out + id * 3, work);
  if (iters_out) iters_out[id] = work[1];
  if (work_out) { work_out[3 * id] = work[0]; work_out[3 * id + 1] = work[1]; work_out[3 * id + 2] = work[2]; }
}

// compute_projection (utils.py:40-45): uv = K [R|t] X / z for every vertex; fp64 math, fp32 result [n][2][nv]
__global__ void project_points_kernel(const float* __restrict__ X4 /*[4][nv] or [3][nv]*/, int rows, int nv,
                                      const double* __restrict__ Rt /*[n][3][4]*/, const double* __restrict__ Kd /*[9]*/, long long n,
                                      float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * nv) return;
  const long long b = idx / nv; const int v = (int)(idx % nv);
  const double X = X4[v], Y = X4[nv + v], Z = X4[2 * nv + v], Wh = rows == 4 ? (double)X4[3 * nv + v] : 1.0;
  const double* T = Rt + b * 12;
  const double cam[3] = {T[0] * X + T[1] * Y + T[2] * Z + T[3] * Wh, T[4] * X + T[5] * Y + T[6] * Z + T[7] * Wh, T[8] * X + T[9] * Y + T[10] * Z + T[11] * Wh};
  const double px = Kd[0] * cam[0] + Kd[1] * cam[1] + Kd[2] * cam[2];
  const double py = Kd[3] * cam[0] + Kd[4] * cam[1] + Kd[5] * cam[2];
  const double pz = Kd[6] * cam[0] + Kd[7] * cam[1] + Kd[8] * cam[2];
  out[(b * 2 + 0) * nv + v] = (float)(px / pz);
  out[(b * 2 + 1) * nv + v] = (float)(py / pz);
}

// ssp_pnp_batched and ssp_pnp_batched_work (ssp_pnp_batched_counted launches pnp_kernel<true> itself)
static int pnp_batched(const float* P3, int p3_shared, const float* uv, const float* K, int np, long long n, int max_iter,
                       double* R_out, double* t_out, int* iters_out, int* work_out, cudaStream_t s) {
  if (!P3 || !uv || !K || !R_out || !t_out || np < 6 || np > PNP_MAXP || n < 0) return fail_msg(SSP_ERR_ARG, "pnp_batched: bad argument (6 <= points <= 16)");
  if (n == 0) return SSP_OK;
  pnp_kernel<false><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(P3, p3_shared ? 0 : 3LL * np, uv, K, np, n, max_iter, R_out, t_out, iters_out,
                                                                work_out, nullptr, 1);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_pnp_batched(const float* P3, int shared, const float* uv, const float* K, int np, long long n, int max_iter, double* R, double* t, int* iters,
                    void* stream) {
  return pnp_batched(P3, shared, uv, K, np, n, max_iter, R, t, iters, nullptr, (cudaStream_t)stream);
}

int ssp_pnp_batched_work(const float* P3, int shared, const float* uv, const float* K, int np, long long n, int max_iter, double* R, double* t,
                         int* work, void* stream) {
  return pnp_batched(P3, shared, uv, K, np, n, max_iter, R, t, nullptr, work, (cudaStream_t)stream);
}

int ssp_pnp_batched_counted(const float* P3, const float* uv, const float* K, int np, int groups, int per_group, const int* count, int max_iter,
                            double* R, double* t, void* stream) {
  if (!P3 || !uv || !K || !count || !R || !t || np < 6 || np > PNP_MAXP || groups < 0 || per_group < 1)
    return fail_msg(SSP_ERR_ARG, "pnp_batched_counted: bad argument (6 <= points <= 16, groups >= 0, per_group >= 1)");
  const long long n = (long long)groups * per_group;
  if (n == 0) return SSP_OK;
  pnp_kernel<true><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(P3, 3LL * np, uv, K, np, n, max_iter, R, t, nullptr, nullptr,
                                                                                 count, per_group);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_project_points(const float* X, int rows, int nv, const double* Rt, const double* K, long long n, float* out, void* stream) {
  if (!X || !Rt || !K || !out || (rows != 3 && rows != 4)) return fail_msg(SSP_ERR_ARG, "project_points: bad argument");
  const long long total = n * nv;
  if (total == 0) return SSP_OK;
  project_points_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(X, rows, nv, Rt, K, n, out);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
