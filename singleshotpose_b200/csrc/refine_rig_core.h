// Refinement of a rig's world poses against every camera's registered depth frame: one projective point-to-plane ICP in world
// axes, the rule of ssp_refine_depth_rig (refine_rig.cu), shared with the CPU test harness (tests/helpers/refine_rig_host.cpp,
// g++ -ffp-contract=off; the kernel is built with -fmad=false) and restated with whole arrays in oracle/refine_rig_ref.py.
// fp64 throughout.  refine_depth_core.h gives the per-pair rule and multiview_core.h the rig; both are used unchanged.
//
// One problem: (capture g, slot s) with a world pose (R_w, t_w), world from object; its class's model points x_i with outward
// normals n_i and diameter d (ssp_refine_depth's model / offsets / diam tables); the rig's C cameras, camera c with extrinsics
// x_c = R_c x_w + t_c, intrinsics from its fp64 K_c (the projection's K, the one ssp_refine_depth reads) and coefficients (all
// zero: pinhole, ssp_mv::cam_dist); camera c's depth frame is row b = g C + c.  Every row has one W x H and one depth_scale.
// Iteration k runs at the gate tau_k = d g_k (gate_factor, computed on the host as for one camera).  Per camera c:
//   the camera pose (R_c R_w, R_c t_w + t_c) is ssp_mv::to_camera of the world pose; find_pair runs with camera c's Camera and
//   that pose, so each camera's gate is along its own ray;
//   a pair's terms are taken in world axes: a_w = R_w x, m_w = R_w n, p_w = a_w + t_w, q_w = R_c^T (q - t_c), then
//   point_terms(a_w, m_w, p_w, q_w): the Jacobian of the left perturbation x_w = exp([dth]x) R_w x + t_w + dt_, the perturbation of
//   world_cov, so solve_update applies the step unchanged.
// Summation order: each camera's pairs go into its own accumulator in refine_depth_core.h's order (256 virtual threads, thread j
// takes points j, j + 256, ..., then the halving tree); the C reduced accumulators are then added in camera order,
// ((acc_0 + acc_1) + acc_2) + ...  With C = 1 and identity extrinsics every product by 1 and every sum with 0 is exact, so the rule
// performs ssp_refine_depth's arithmetic and its outputs are those of ssp_refine_depth bit for bit.
// Outputs: the pose, points and rmse of the last iteration over all cameras (the kMinPoints test is on the total), and per camera
// view_points / view_rmse of the last iteration from its own accumulator (rmse 0: no pairs).  Status: kBadPose when the world pose
// is not finite or its fusion status has SSP_FUSE_NO_VALID or SSP_FUSE_NO_VIEW (no t_z test: the pose is in world axes, and every
// camera skips the points behind it); kFewPoints and kSingular as for one camera.  With a status bit the output pose is the input.
// corners: the output pose projected into every row's camera by ssp_mv::project, ssp_fuse_views' arithmetic for corners_world,
// with zeros where the fusion has no pose (SSP_FUSE_NO_VALID / NO_VIEW) or the class is unknown; so a problem with a status bit
// reproduces corners_world bit for bit.
// Only the libm functions sin and cos (so3_exp) may round differently on the device and the host.
#pragma once
#include <math.h>

#include "multiview_core.h"
#include "refine_depth_core.h"

namespace ssp_rr {

constexpr int kMaxViews = ssp_mv::kMaxViews;
constexpr int kAcc = ssp_rd::kAccDoubles;

// the rig as the refinement reads it: K [C][9] fp64, dist [C][8] or null, R [C][9], t [C][3]; the depth frames' size and scale
struct Rig {
  const double* K;
  const double* dist;
  const double* R;
  const double* t;
  int C, W, H;
  double depth_scale;
};

// camera c's depth Camera (fp64 K) and its extrinsics as ssp_mv reads them
SSP_HD ssp_rd::Camera depth_camera(const Rig& rig, int c) {
  const double* K = rig.K + 9 * c;
  return ssp_rd::Camera{K[0], K[4], K[2], K[5], ssp_mv::cam_dist(rig.dist, c), rig.W, rig.H, rig.depth_scale};
}
SSP_HD ssp_mv::Cam extrinsics(const Rig& rig, int c) {
  const double* K = rig.K + 9 * c;
  return ssp_mv::Cam{K[0], K[4], K[2], K[5], ssp_mv::cam_dist(rig.dist, c), rig.R + 9 * c, rig.t + 3 * c};
}

// the world-axis terms r, J of model point x6's pair in camera `ext` (camera pose (Rc, tc) of the world pose (R, t)) and its
// scene point qw in world axes: false when it makes none
SSP_HD bool world_pair(const double* x6, const double R[9], const double t[3], const double Rc[9], const double tc[3], const ssp_mv::Cam& ext,
                       const ssp_rd::Camera& cam, const unsigned short* depth, double tau, double* r, double J[6], double qw[3]) {
  double a[3], m[3], p[3], q[3];
  if (!ssp_rd::find_pair(x6, Rc, tc, cam, depth, tau, a, m, p, q)) return false;
  double aw[3], mw[3], pw[3];
  for (int i = 0; i < 3; i++) {
    aw[i] = R[3 * i] * x6[0] + R[3 * i + 1] * x6[1] + R[3 * i + 2] * x6[2];
    mw[i] = R[3 * i] * x6[3] + R[3 * i + 1] * x6[4] + R[3 * i + 2] * x6[5];
    pw[i] = aw[i] + t[i];
  }
  const double d[3] = {q[0] - ext.t[0], q[1] - ext.t[1], q[2] - ext.t[2]};
  for (int i = 0; i < 3; i++) qw[i] = ext.R[i] * d[0] + ext.R[3 + i] * d[1] + ext.R[6 + i] * d[2];
  *r = ssp_rd::point_terms(aw, mw, pw, qw, J);
  return true;
}

// add model point x6's world-axis pair in one camera, if it makes one, to acc [kAcc] (accumulate_point's additions)
SSP_HD void accumulate_point(const double* x6, const double R[9], const double t[3], const double Rc[9], const double tc[3], const ssp_mv::Cam& ext,
                             const ssp_rd::Camera& cam, const unsigned short* depth, double tau, double* acc) {
  double r, J[6], qw[3];
  if (!world_pair(x6, R, t, Rc, tc, ext, cam, depth, tau, &r, J, qw)) return;
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) acc[k++] += J[i] * J[j];
  for (int i = 0; i < 6; i++) acc[ssp_rd::kOffJr + i] += J[i] * r;
  acc[ssp_rd::kOffR2] += r * r;
  acc[ssp_rd::kOffN] += 1.0;
}

// the input status of a world pose: kBadPose when it is not finite or the fusion left no pose
SSP_HD int input_status(const double R[9], const double t[3], int fuse_status) {
  for (int i = 0; i < 9; i++) if (!isfinite(R[i])) return ssp_rd::kBadPose;
  for (int i = 0; i < 3; i++) if (!isfinite(t[i])) return ssp_rd::kBadPose;
  return (fuse_status & (ssp_mv::kNoValid | ssp_mv::kNoView)) ? ssp_rd::kBadPose : 0;
}

// a camera's pair count and RMS residual from its reduced accumulator
SSP_HD void view_stats(const double* acc, int* points, double* rmse) {
  const double n = acc[ssp_rd::kOffN];
  *points = (int)n;
  *rmse = n > 0.0 ? sqrt(acc[ssp_rd::kOffR2] / n) : 0.0;
}

// sum [kAcc] of the C reduced accumulators (acc(c) returns camera c's), added in camera order
template <class F>
SSP_HD void sum_views(F acc, int C, double* sum) {
  const double* a0 = acc(0);
  for (int i = 0; i < kAcc; i++) sum[i] = a0[i];
  for (int c = 1; c < C; c++) {
    const double* a = acc(c);
    for (int i = 0; i < kAcc; i++) sum[i] += a[i];
  }
}

// the np points of X [np][3] under the world pose (R, t) in camera c's frame, at out [np][2]; zeros with `none`
SSP_HD void project_view(const Rig& rig, int c, const double R[9], const double t[3], const float* X, int np, bool none, float* out) {
  const ssp_mv::Cam ext = extrinsics(rig, c);
  double Rw[9], tw[3];
  ssp_mv::to_camera(ext, R, t, Rw, tw);
  for (int i = 0; i < np; i++) {
    if (none) { out[2 * i] = 0.f; out[2 * i + 1] = 0.f; continue; }
    ssp_mv::project(Rw, tw, X[3 * i], X[3 * i + 1], X[3 * i + 2], rig.K + 9 * c, ext.dist, out + 2 * i, out + 2 * i + 1);
  }
}

}  // namespace ssp_rr
