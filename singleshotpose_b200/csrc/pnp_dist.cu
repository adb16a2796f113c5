// PnP and projection for cameras with lens distortion: OpenCV's model with distCoeffs (k1, k2, p1, p2, k3, k4, k5, k6), the arithmetic
// of pnp_core.h (pnp_solve_one's dist, distort, undistort) and pnp_consensus_core.h (score's dist).  Kernels of their own, so that
// the zero-distortion kernels of pnp.cu and pnp_consensus.cu keep their code; the coefficients are a DEVICE double[8] read in place,
// like K, so a captured graph sees the values at replay time.
//   pnp_dist_kernel         one thread per problem: plain, counted (empty slots get zeros) or warm-started (guess, use_guess);
//   pnp_hyp_dist_kernel     the consensus fan-out of pnp_hyp_kernel, one thread per (problem, hypothesis);
//   pnp_select_dist_kernel  the consensus selection and refinement of pnp_select_kernel;
//   project_dist_kernel     cv2.projectPoints of X under [R|t] for every vertex and pose.
#include <math.h>

#include "ssp_common.cuh"
#include "pnp_consensus_core.h"

namespace ssp {

__global__ void __launch_bounds__(128) pnp_dist_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                       const float* __restrict__ Kmat, const double* __restrict__ dist, int np, long long n,
                                                       int max_iter, const int* __restrict__ count, int per_group,
                                                       const double* __restrict__ guess, const int* __restrict__ use_guess,
                                                       double* __restrict__ R_out, double* __restrict__ t_out,
                                                       double* __restrict__ params_out, int* __restrict__ work_out) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  if (count && id % per_group >= count[id / per_group]) {
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = 0.0;
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = 0.0;
    if (params_out) for (int k = 0; k < 6; k++) params_out[id * 6 + k] = 0.0;
    if (work_out) { work_out[3 * id] = 0; work_out[3 * id + 1] = 0; work_out[3 * id + 2] = 0; }
    return;
  }
  int work[3];
  ssp_pnp::pnp_solve_one(P3 + id * p3_stride, uv + id * 2 * np, Kmat, np, max_iter, R_out + id * 9, t_out + id * 3, work, nullptr,
                         guess && use_guess[id] ? guess + id * 6 : nullptr, params_out ? params_out + id * 6 : nullptr, dist);
  if (work_out) { work_out[3 * id] = work[0]; work_out[3 * id + 1] = work[1]; work_out[3 * id + 2] = work[2]; }
}

__global__ void __launch_bounds__(128) pnp_hyp_dist_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                           const float* __restrict__ Kmat, const double* __restrict__ dist, int np,
                                                           long long n, int max_iter, double thr2, const SubsetTable tab, int H1,
                                                           const int* __restrict__ count, int per_group, double* __restrict__ slots,
                                                           unsigned* __restrict__ hmask) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n * H1) return;
  const long long i = id / H1;
  const int h = (int)(id - i * H1);
  if (count && i % per_group >= count[i / per_group]) return;
  hmask[id] = ssp_pnpc::solve_hypothesis(h, tab.m, P3 + i * p3_stride, uv + i * 2 * np, Kmat, np, thr2, max_iter,
                                         slots + id * ssp_pnpc::kSlotDoubles, dist);
}

__global__ void __launch_bounds__(128) pnp_select_dist_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                              const float* __restrict__ Kmat, const double* __restrict__ dist, int np,
                                                              long long n, int max_iter, const SubsetTable tab, int H1,
                                                              const int* __restrict__ count, int per_group, const double* __restrict__ slots,
                                                              const unsigned* __restrict__ hmask, double* __restrict__ R_out,
                                                              double* __restrict__ t_out, double* __restrict__ params_out,
                                                              int* __restrict__ inliers_out, int* __restrict__ hyp_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (count && i % per_group >= count[i / per_group]) {
    for (int k = 0; k < 9; k++) R_out[i * 9 + k] = 0.0;
    for (int k = 0; k < 3; k++) t_out[i * 3 + k] = 0.0;
    for (int k = 0; k < 6; k++) params_out[i * 6 + k] = 0.0;
    inliers_out[i] = 0;
    hyp_out[i] = 0;
    return;
  }
  const unsigned* hm = hmask + i * H1;
  const int hyp = ssp_pnpc::select(hm, 1, H1);
  const unsigned inl = hyp < 0 ? 0u : hm[hyp];
  const double* s0 = slots + i * H1 * ssp_pnpc::kSlotDoubles;
  ssp_pnpc::finish(hyp, inl, s0 + (hyp < 0 ? 0 : hyp) * ssp_pnpc::kSlotDoubles, s0, tab.m, P3 + i * p3_stride, uv + i * 2 * np, Kmat, np,
                   max_iter, R_out + i * 9, t_out + i * 3, params_out + i * 6, dist);
  inliers_out[i] = (int)inl;
  hyp_out[i] = hyp;
}

// cv2.projectPoints(X, R, t, K, dist) for every vertex under every pose: fp64 math, fp32 result [n][2][nv] (project_points_kernel's
// layout; rows == 4 scales t by the homogeneous coordinate as it does)
__global__ void project_dist_kernel(const float* __restrict__ X4, int rows, int nv, const double* __restrict__ Rt, const double* __restrict__ Kd,
                                    const double* __restrict__ dist, long long n, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * nv) return;
  const long long b = idx / nv; const int v = (int)(idx % nv);
  const double X = X4[v], Y = X4[nv + v], Z = X4[2 * nv + v], Wh = rows == 4 ? (double)X4[3 * nv + v] : 1.0;
  const double* T = Rt + b * 12;
  const double x = T[0] * X + T[1] * Y + T[2] * Z + T[3] * Wh, y = T[4] * X + T[5] * Y + T[6] * Z + T[7] * Wh;
  const double z = T[8] * X + T[9] * Y + T[10] * Z + T[11] * Wh;
  double u, w;
  ssp_pnp::project_distorted(dist, x, y, z, Kd[0], Kd[4], Kd[2], Kd[5], &u, &w);
  out[(b * 2 + 0) * nv + v] = (float)u;
  out[(b * 2 + 1) * nv + v] = (float)w;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_pnp_dist(const float* P3, int shared, const float* uv, const float* K, const double* dist, int np, int groups, int per_group,
                 const int* count, const double* guess, const int* use_guess, int max_iter, double* R, double* t, double* params, int* work,
                 void* stream) {
  if (!P3 || !uv || !K || !dist || !R || !t || np < 6 || np > PNP_MAXP || groups < 0 || per_group < 1)
    return fail_msg(SSP_ERR_ARG, "pnp_dist: bad argument (null pointer, points outside 6..16, groups < 0 or per_group < 1)");
  if (!guess != !use_guess) return fail_msg(SSP_ERR_ARG, "pnp_dist: guess and use_guess are given together or not at all");
  if (guess && !params) return fail_msg(SSP_ERR_ARG, "pnp_dist: a warm-started solve writes params (the final LM vectors)");
  const long long n = (long long)groups * per_group;
  if (n == 0) return SSP_OK;
  pnp_dist_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(P3, shared ? 0 : 3LL * np, uv, K, dist, np, n, max_iter, count,
                                                                               per_group, guess, use_guess, R, t, params, work);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_pnp_consensus_dist(const float* P3, int shared, const float* uv, const float* K, const double* dist, int np, int groups, int per_group,
                           const int* count, const unsigned short* subsets, int H, double thr, int max_iter, double* R, double* t,
                           double* params, int* inliers, int* hyp, void* work, long long work_bytes, void* stream) {
  if (!P3 || !uv || !K || !dist || !subsets || !R || !t || !params || !inliers || !hyp || !work || np < ssp_pnpc::kMinPoints ||
      np > ssp_pnpc::kMaxPoints || groups < 0 || per_group < 1)
    return fail_msg(SSP_ERR_ARG, "pnp_consensus_dist: bad argument (null pointer, points outside 7..10, groups < 0 or per_group < 1)");
  if (!ssp_pnpc::table_ok(subsets, H, np))
    return fail_msg(SSP_ERR_ARG, "pnp_consensus_dist: bad subset table (1..210 masks of exactly 6 bits below the point count)");
  if (!(thr > 0.0) || !isfinite(thr)) return fail_msg(SSP_ERR_ARG, "pnp_consensus_dist: the threshold must be > 0 and finite");
  if (max_iter < 1) return fail_msg(SSP_ERR_ARG, "pnp_consensus_dist: max_iter must be >= 1");
  const long long n = (long long)groups * per_group;
  if (work_bytes < ssp_pnpc::work_bytes(H, n) || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "pnp_consensus_dist: workspace smaller than ssp_pnp_consensus_work_bytes or not 8-B aligned");
  if (n == 0) return SSP_OK;
  SubsetTable tab = {};
  for (int h = 0; h < H; h++) tab.m[h] = subsets[h];
  const int H1 = H + 1;
  const long long stride = shared ? 0 : 3LL * np;
  double* slots = (double*)work;
  unsigned* hmask = (unsigned*)(slots + n * H1 * ssp_pnpc::kSlotDoubles);
  cudaStream_t s = (cudaStream_t)stream;
  const long long nh = n * H1;
  pnp_hyp_dist_kernel<<<(unsigned)((nh + 127) / 128), 128, 0, s>>>(P3, stride, uv, K, dist, np, n, max_iter, thr * thr, tab, H1, count,
                                                                   per_group, slots, hmask);
  SSP_CHECK_LAUNCH();
  pnp_select_dist_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(P3, stride, uv, K, dist, np, n, max_iter, tab, H1, count, per_group,
                                                                     slots, hmask, R, t, params, inliers, hyp);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_project_points_dist(const float* X, int rows, int nv, const double* Rt, const double* K, const double* dist, long long n, float* out,
                            void* stream) {
  if (!X || !Rt || !K || !dist || !out || (rows != 3 && rows != 4) || nv < 0 || n < 0)
    return fail_msg(SSP_ERR_ARG, "project_points_dist: bad argument (null pointer, rows not 3 or 4, nv < 0 or n < 0)");
  const long long total = n * nv;
  if (total == 0) return SSP_OK;
  project_dist_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(X, rows, nv, Rt, K, dist, n, out);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
