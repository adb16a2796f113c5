// Step 1 of ssp_fuse_views (rule: multiview_core.h): every (row, slot)'s cold PnP with its row's camera and the projection of its
// points under that pose.  Built with the default multiply-add contraction, like pnp.cu and pnp_dist.cu, so that each row's R, t
// and corners are the bits ssp_pnp_batched / ssp_pnp_dist and ssp_project_points / ssp_project_points_dist give for that camera;
// one launch for the pinhole cameras' rows and, with a distortion table, one per camera for the cameras with coefficients.  The fusion kernels live in
// multiview.cu (-fmad=false).  The counted variants serve ssp_fuse_instances (multiview_instances.cu), whose empty slots need no solve.
#include "ssp_common.cuh"
#include "multiview_core.h"

namespace ssp {

// the rows whose camera is the pinhole model (no distortion table, or a camera whose 8 coefficients are all zero): pnp_kernel's solve
__global__ void __launch_bounds__(128) fuse_rows_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                        const float* __restrict__ K32, const double* __restrict__ K64,
                                                        const double* __restrict__ dist, int np, int C, int S, long long n, int max_iter,
                                                        double* __restrict__ R_out, double* __restrict__ t_out, float* __restrict__ corners) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (row, slot)
  if (id >= n) return;
  const int c = (int)((id / S) % C);
  if (ssp_mv::cam_dist(dist, c)) return;
  const float* p3 = P3 + id * p3_stride;
  int work[3];
  ssp_pnp::pnp_solve_one(p3, uv + id * 2 * np, K32 + 9 * c, np, max_iter, R_out + id * 9, t_out + id * 3, work);
  const double* R = R_out + id * 9;
  const double* t = t_out + id * 3;
  const double* Kd = K64 + 9 * c;
  for (int v = 0; v < np; v++) {
    // project_points_kernel's expressions with T = [R | t] and the homogeneous weight 1
    const double X = p3[3 * v], Y = p3[3 * v + 1], Z = p3[3 * v + 2];
    const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0], y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    const double px = Kd[0] * x + Kd[1] * y + Kd[2] * z;
    const double py = Kd[3] * x + Kd[4] * y + Kd[5] * z;
    const double pz = Kd[6] * x + Kd[7] * y + Kd[8] * z;
    corners[(id * np + v) * 2] = (float)(px / pz);
    corners[(id * np + v) * 2 + 1] = (float)(py / pz);
  }
}

// the rows of camera `cam` when it has distortion coefficients: pnp_dist_kernel's solve.  One launch per camera, one thread per
// (capture, slot).  Kmat, Kd and coeffs are camera cam's rows of the tables, addressed on the host, and guess, use_guess and
// params_out are always null: the solve's arguments are then the kernel arguments that pnp_dist_kernel passes, so that nvcc
// compiles (and contracts) the inlined solve the same way; pointers it could prove non-null, or constant nulls, change the
// contraction and the rows' last bits
__global__ void __launch_bounds__(128) fuse_rows_dist_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                             const float* __restrict__ Kmat, const double* __restrict__ Kd,
                                                             const double* __restrict__ coeffs, const double* __restrict__ table, int cam,
                                                             int np, int C, int S, long long n, int max_iter, const double* __restrict__ guess,
                                                             const int* __restrict__ use_guess, double* __restrict__ params_out,
                                                             double* __restrict__ R_out, double* __restrict__ t_out, float* __restrict__ corners) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;         // (capture, slot)
  if (i >= n || !ssp_mv::cam_dist(table, cam)) return;
  const long long id = ((i / S) * C + cam) * S + i % S;                        // (row, slot)
  int work[3];
  ssp_pnp::pnp_solve_one(P3 + id * p3_stride, uv + id * 2 * np, Kmat, np, max_iter, R_out + id * 9, t_out + id * 3, work, nullptr,
                         guess && use_guess[id] ? guess + id * 6 : nullptr, params_out ? params_out + id * 6 : nullptr, coeffs);
  const float* p3 = P3 + id * p3_stride;
  const double* R = R_out + id * 9;
  const double* t = t_out + id * 3;
  for (int v = 0; v < np; v++) {
    // project_dist_kernel's expressions with T = [R | t] and the homogeneous weight 1
    const double X = p3[3 * v], Y = p3[3 * v + 1], Z = p3[3 * v + 2];
    const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0], y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    double u, w;
    ssp_pnp::project_distorted(coeffs, x, y, z, Kd[0], Kd[4], Kd[2], Kd[5], &u, &w);
    corners[(id * np + v) * 2] = (float)u;
    corners[(id * np + v) * 2 + 1] = (float)w;
  }
}

// the counted rows of ssp_fuse_instances (multiview_instances.cu): fuse_rows_kernel and fuse_rows_dist_kernel for slot m of row b
// only when m < count[b] (the others are left for the caller to zero), so that empty slots cost no solve; the solve and the
// projection are the same expressions, called the same way
__global__ void __launch_bounds__(128) fuse_rows_counted_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                                const float* __restrict__ K32, const double* __restrict__ K64,
                                                                const double* __restrict__ dist, const int* __restrict__ count, int np, int C,
                                                                int S, long long n, int max_iter, double* __restrict__ R_out,
                                                                double* __restrict__ t_out, float* __restrict__ corners) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (row, slot)
  if (id >= n || id % S >= count[id / S]) return;
  const int c = (int)((id / S) % C);
  if (ssp_mv::cam_dist(dist, c)) return;
  const float* p3 = P3 + id * p3_stride;
  int work[3];
  ssp_pnp::pnp_solve_one(p3, uv + id * 2 * np, K32 + 9 * c, np, max_iter, R_out + id * 9, t_out + id * 3, work);
  const double* R = R_out + id * 9;
  const double* t = t_out + id * 3;
  const double* Kd = K64 + 9 * c;
  for (int v = 0; v < np; v++) {
    const double X = p3[3 * v], Y = p3[3 * v + 1], Z = p3[3 * v + 2];
    const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0], y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    const double px = Kd[0] * x + Kd[1] * y + Kd[2] * z;
    const double py = Kd[3] * x + Kd[4] * y + Kd[5] * z;
    const double pz = Kd[6] * x + Kd[7] * y + Kd[8] * z;
    corners[(id * np + v) * 2] = (float)(px / pz);
    corners[(id * np + v) * 2 + 1] = (float)(py / pz);
  }
}

__global__ void __launch_bounds__(128) fuse_rows_dist_counted_kernel(const float* __restrict__ P3, long long p3_stride,
                                                                     const float* __restrict__ uv, const float* __restrict__ Kmat,
                                                                     const double* __restrict__ Kd, const double* __restrict__ coeffs,
                                                                     const double* __restrict__ table, int cam, const int* __restrict__ count,
                                                                     int np, int C, int S, long long n, int max_iter,
                                                                     const double* __restrict__ guess, const int* __restrict__ use_guess,
                                                                     double* __restrict__ params_out, double* __restrict__ R_out,
                                                                     double* __restrict__ t_out, float* __restrict__ corners) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;         // (capture, slot)
  if (i >= n || !ssp_mv::cam_dist(table, cam)) return;
  const long long id = ((i / S) * C + cam) * S + i % S;                        // (row, slot)
  if (id % S >= count[id / S]) return;
  int work[3];
  ssp_pnp::pnp_solve_one(P3 + id * p3_stride, uv + id * 2 * np, Kmat, np, max_iter, R_out + id * 9, t_out + id * 3, work, nullptr,
                         guess && use_guess[id] ? guess + id * 6 : nullptr, params_out ? params_out + id * 6 : nullptr, coeffs);
  const float* p3 = P3 + id * p3_stride;
  const double* R = R_out + id * 9;
  const double* t = t_out + id * 3;
  for (int v = 0; v < np; v++) {
    const double X = p3[3 * v], Y = p3[3 * v + 1], Z = p3[3 * v + 2];
    const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0], y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    double u, w;
    ssp_pnp::project_distorted(coeffs, x, y, z, Kd[0], Kd[4], Kd[2], Kd[5], &u, &w);
    corners[(id * np + v) * 2] = (float)u;
    corners[(id * np + v) * 2 + 1] = (float)w;
  }
}

// launched by ssp_fuse_instances after its argument checks: launch_fuse_rows over the slots m < count[row]
int launch_fuse_rows_counted(const float* P3, long long p3_stride, const float* uv, const float* K32, const double* K64, const double* dist,
                             const int* count, int np, int C, int S, long long rows, int max_iter, double* R, double* t, float* corners,
                             void* stream) {
  const long long n = rows * S;
  cudaStream_t s = (cudaStream_t)stream;
  fuse_rows_counted_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(P3, p3_stride, uv, K32, K64, dist, count, np, C, S, n, max_iter, R, t,
                                                                       corners);
  SSP_CHECK_LAUNCH();
  if (!dist) return SSP_OK;
  const long long m = n / C;
  for (int c = 0; c < C; c++) {
    fuse_rows_dist_counted_kernel<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(P3, p3_stride, uv, K32 + 9 * c, K64 + 9 * c, dist + 8 * c, dist, c,
                                                                             count, np, C, S, m, max_iter, nullptr, nullptr, nullptr, R, t,
                                                                             corners);
    SSP_CHECK_LAUNCH();
  }
  return SSP_OK;
}

// launched by ssp_fuse_views (multiview.cu) after its argument checks
int launch_fuse_rows(const float* P3, long long p3_stride, const float* uv, const float* K32, const double* K64, const double* dist, int np,
                     int C, int S, long long rows, int max_iter, double* R, double* t, float* corners, void* stream) {
  const long long n = rows * S;
  cudaStream_t s = (cudaStream_t)stream;
  fuse_rows_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(P3, p3_stride, uv, K32, K64, dist, np, C, S, n, max_iter, R, t, corners);
  SSP_CHECK_LAUNCH();
  if (!dist) return SSP_OK;
  const long long m = n / C;
  for (int c = 0; c < C; c++) {
    fuse_rows_dist_kernel<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(P3, p3_stride, uv, K32 + 9 * c, K64 + 9 * c, dist + 8 * c, dist, c, np, C,
                                                                     S, m, max_iter, nullptr, nullptr, nullptr, R, t, corners);
    SSP_CHECK_LAUNCH();
  }
  return SSP_OK;
}

}  // namespace ssp
