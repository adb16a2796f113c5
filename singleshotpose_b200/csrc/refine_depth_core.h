// Refinement of a pose against a registered depth frame: projective point-to-plane ICP, the rule of ssp_refine_depth
// (refine_depth.cu), shared with the CPU test harness (tests/helpers/refine_depth_host.cpp, built with g++ -ffp-contract=off; the
// kernel is built with -fmad=false).  fp64 throughout.
//
// One problem: a pose (R, t), camera from model; the class's model points x_i with unit normals n_i (a zero normal is never used);
// one depth frame D [H][W] uint16 (0: no measurement) with depth_scale mesh units per depth unit; K (fx, fy, cx, cy) and optional
// OpenCV distortion coefficients (pnp_core.h's distort / undistort); the object diameter d; iters and the gate range (s, e) as
// fractions of d.  Iteration k = 0 .. iters-1 runs at the gate tau_k = d * g_k, g_k = s * (e / s)^(k / (iters - 1)) (g_0 = s with
// iters = 1).  The factors g_k are computed by gate_factor on the host, so the kernel and the harness use the same bits.
// For each model point (accumulate_point):
//   p = R x_i + t, m = R n_i; skipped when m . p >= 0 (back-facing, or a zero normal) or p_z <= 0;
//   (u, v): p projected with K (distorted with the coefficients); the nearest pixel (iu, iv) = (floor(u + 0.5), floor(v + 0.5)),
//     pixel centres at integer coordinates as compute_projection and render_core.h have them; skipped outside the frame or at D = 0;
//   q = D * depth_scale * (xh, yh, 1), (xh, yh) = ((iu - cx) / fx, (iv - cy) / fy), or undistort of (iu, iv) with coefficients;
//   the pair is rejected when |p_z - q_z| > tau_k (occluders in front, background behind);
//   r = m . (p - q); under the left perturbation x_cam = exp([dth]x) R x + t + dt_ (pose_filter_core.h), with the normal turning
//     with the pose, J = [ (R x_i) x m + m x (p - q) ; m ];
//   the 21 upper entries of J^T J (row-major), the 6 of J^T r, r^2 and 1 are added to the point's accumulator (kAccDoubles).
// Summation order: 256 virtual threads, thread j adds points j, j + 256, ... in index order into its own accumulator; the 256
// accumulators are combined by a halving tree, a[i] += a[i + s] for s = 128, 64, ..., 1 (tree_reduce).
// Per iteration (solve_update): points = the pair count; fewer than kMinPoints is kFewPoints; rmse = sqrt(sum r^2 / points) before
// the update; (J^T J) delta = -J^T r through spd_inverse6 (pose_filter_core.h: a pivot <= 1e-12 x the largest diagonal entry is
// kSingular); R <- exp([dth]x) R, t <- t + dt_.  The iteration count is fixed: no convergence test.
// A pose that is not finite or has t_z <= 0 is kBadPose before any iteration.  Any status bit stops the problem: the output is
// then the input pose unchanged, points and rmse those of the iteration that stopped (0 for kBadPose).
// Only the libm functions sin and cos (so3_exp) may round differently on the device and the host.
#pragma once
#include <math.h>

#include "pnp_core.h"
#include "pose_filter_core.h"

namespace ssp_rd {

constexpr int kThreads = 256;                 // virtual threads of the summation order, the CTA size of the kernel
constexpr int kMinPoints = 50;                // SSP_REFINE_MIN_POINTS
constexpr int kMaxIters = 100;                // SSP_REFINE_MAX_ITERS
constexpr int kAccDoubles = 21 + 6 + 1 + 1;   // J^T J upper, J^T r, sum r^2, pair count
constexpr int kOffJr = 21, kOffR2 = 27, kOffN = 28;
enum Status { kFewPoints = 1, kSingular = 2, kBadPose = 4 };

struct Camera {
  double fx, fy, cx, cy;
  const double* dist;                         // 8 coefficients, or null
  int W, H;
  double depth_scale;
};

// g_k of iteration k (host only: the kernel reads the factors as a launch argument)
inline double gate_factor(double s, double e, int k, int iters) {
  return iters == 1 ? s : s * pow(e / s, (double)k / (double)(iters - 1));
}

// the scene point q of model point x6 = (x, y, z, nx, ny, nz) under (R, t) and its residual terms; false when the point makes no
// pair.  Out: a = R x, m = R n, p = a + t, q.
SSP_HD bool find_pair(const double* x6, const double R[9], const double t[3], const Camera& cam, const unsigned short* depth, double tau,
                      double a[3], double m[3], double p[3], double q[3]) {
  for (int i = 0; i < 3; i++) {
    a[i] = R[3 * i] * x6[0] + R[3 * i + 1] * x6[1] + R[3 * i + 2] * x6[2];
    m[i] = R[3 * i] * x6[3] + R[3 * i + 1] * x6[4] + R[3 * i + 2] * x6[5];
    p[i] = a[i] + t[i];
  }
  if (!(m[0] * p[0] + m[1] * p[1] + m[2] * p[2] < 0.0) || !(p[2] > 0.0)) return false;
  const double iz = 1.0 / p[2], xn = p[0] * iz, yn = p[1] * iz;
  double u, v;
  if (cam.dist) {
    double xd, yd;
    ssp_pnp::distort(cam.dist, xn, yn, &xd, &yd, nullptr);
    u = xd * cam.fx + cam.cx; v = yd * cam.fy + cam.cy;
  } else {
    u = xn * cam.fx + cam.cx; v = yn * cam.fy + cam.cy;
  }
  const double fu = floor(u + 0.5), fv = floor(v + 0.5);     // NaN fails both range tests
  if (!(fu >= 0.0 && fu < (double)cam.W && fv >= 0.0 && fv < (double)cam.H)) return false;
  const int iu = (int)fu, iv = (int)fv;
  const unsigned short D = depth[(long long)iv * cam.W + iu];
  if (D == 0) return false;
  const double z = (double)D * cam.depth_scale;
  if (fabs(p[2] - z) > tau) return false;
  double xh, yh;
  if (cam.dist) ssp_pnp::undistort(cam.dist, fu, fv, cam.fx, cam.fy, cam.cx, cam.cy, &xh, &yh);
  else { xh = (fu - cam.cx) / cam.fx; yh = (fv - cam.cy) / cam.fy; }
  q[0] = z * xh; q[1] = z * yh; q[2] = z;
  return true;
}

// r = m . (p - q) and J [6] = [a x m + m x (p - q); m]
SSP_HD double point_terms(const double a[3], const double m[3], const double p[3], const double q[3], double J[6]) {
  const double d[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
  J[0] = (a[1] * m[2] - a[2] * m[1]) + (m[1] * d[2] - m[2] * d[1]);
  J[1] = (a[2] * m[0] - a[0] * m[2]) + (m[2] * d[0] - m[0] * d[2]);
  J[2] = (a[0] * m[1] - a[1] * m[0]) + (m[0] * d[1] - m[1] * d[0]);
  J[3] = m[0]; J[4] = m[1]; J[5] = m[2];
  return m[0] * d[0] + m[1] * d[1] + m[2] * d[2];
}

// add model point x6's pair, if it makes one, to acc [kAccDoubles]
SSP_HD void accumulate_point(const double* x6, const double R[9], const double t[3], const Camera& cam, const unsigned short* depth,
                             double tau, double* acc) {
  double a[3], m[3], p[3], q[3], J[6];
  if (!find_pair(x6, R, t, cam, depth, tau, a, m, p, q)) return;
  const double r = point_terms(a, m, p, q, J);
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) acc[k++] += J[i] * J[j];
  for (int i = 0; i < 6; i++) acc[kOffJr + i] += J[i] * r;
  acc[kOffR2] += r * r;
  acc[kOffN] += 1.0;
}

// the halving tree over n = kThreads accumulators a [kThreads][kAccDoubles], result in a[0] (the harness's order; the kernel
// performs the same additions with shared memory and warp shuffles)
inline void tree_reduce(double (*a)[kAccDoubles]) {
  for (int s = kThreads / 2; s >= 1; s /= 2)
    for (int i = 0; i < s; i++)
      for (int k = 0; k < kAccDoubles; k++) a[i][k] += a[i + s][k];
}

SSP_HD bool pose_ok(const double R[9], const double t[3]) {
  for (int i = 0; i < 9; i++) if (!isfinite(R[i])) return false;
  for (int i = 0; i < 3; i++) if (!isfinite(t[i])) return false;
  return t[2] > 0.0;
}

// one iteration's solve and update of (R, t) in place from the reduced acc; returns the status bits (0: updated), points and rmse
SSP_HD int solve_update(const double* acc, double R[9], double t[3], int* points, double* rmse) {
  const double n = acc[kOffN];
  *points = (int)n;
  *rmse = n > 0.0 ? sqrt(acc[kOffR2] / n) : 0.0;
  if (*points < kMinPoints) return kFewPoints;
  double A[6][6], Ai[6][6];
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) { A[i][j] = acc[k]; A[j][i] = acc[k]; k++; }
  if (!ssp_pf::spd_inverse6(A, Ai)) return kSingular;
  double delta[6];
  for (int i = 0; i < 6; i++) {
    double v = 0.0;
    for (int j = 0; j < 6; j++) v += Ai[i][j] * acc[kOffJr + j];
    delta[i] = -v;
  }
  double E[9], Rn[9];
  ssp_pf::so3_exp(delta, E);
  ssp_pf::mat3_mul(E, R, Rn);
  for (int i = 0; i < 9; i++) R[i] = Rn[i];
  for (int i = 0; i < 3; i++) t[i] += delta[3 + i];
  return 0;
}

}  // namespace ssp_rd
