// Fusing the poses of several calibrated cameras into one world pose: the rule of ssp_fuse_views (multiview_rows.cu, multiview.cu),
// shared with the CPU test harness (tests/helpers/multiview_host.cpp, g++ -ffp-contract=off; multiview.cu is built with
// -fmad=false) and restated with whole arrays in oracle/multiview_ref.py.  fp64 throughout.
//
// Rig.  C calibrated cameras (1 <= C <= kMaxViews); camera c has K_c (fp32 as the PnP reads it), OpenCV distortion dist_c (8
// values; all zero, or no table, is the pinhole model) and extrinsics camera-from-world x_c = R_c x_w + t_c.  World-from-object
// is x_w = R x + t.  A capture g is the rows b = g C + c, c = 0..C-1, row b seen by camera c; each row has S slots (objects).
// The rule runs per (capture g, slot s) over the views c whose slot is valid (the caller's flag: detected, or conf > thresh).
//   1. Per-view solve.  Every row solves its cold PnP with its own camera, pnp_solve_one(K_c, dist_c, max_iter), valid or not,
//      and projects its points under that pose (ssp_project_points' / ssp_project_points_dist's arithmetic).
//   2. Hypotheses.  Hypothesis v (a valid view) is view v's pose in the world frame: R = R_v^T R_(v), t = R_v^T (t_(v) - t_v).
//   3. Agreement.  View w agrees with a world pose at threshold thr when every point lies at camera-w depth > 0 and the mean of
//      its points' squared raw-pixel reprojection errors (distorted model, every operation rounded on its own, the arithmetic of
//      pnp_consensus_core.h's score) is <= thr^2.  Hypothesis h is scored in two stages: A = the valid views that agree with h
//      at `gate`, fit A from h; A' = the valid views that agree with that fit at `reproj_thresh`; if A' != A, fit A' from the
//      first fit.  Check: while a view of the set no longer agrees with the fit at reproj_thresh, it leaves the set and the rest
//      is fitted again from the last fit (the set only shrinks, so at most C fits), so every fused view ends within
//      reproj_thresh of the fused pose.  A fit of a set of one view w is w's hypothesis (no LM: a one-camera rig reproduces its per-view pose bit for
//      bit); a fit of more views is the LM below.  An empty A or A' keeps no view.
//      Why two thresholds: a one-view hypothesis is off along its own viewing ray, where the keypoints constrain it least.
//      Projected into a camera 90 degrees away that offset is a lateral one, tens of pixels even when both views are right, so
//      reproj_thresh applied to the raw hypothesis would refuse to fuse exactly the rigs that gain the most.  The wide gate
//      only decides which views the first fit may use; the tight threshold is applied to the fused pose.
//   4. Selection.  The hypothesis with the most views in its final set wins, then the lower final cost (the sum of squared
//      residuals over the final set; lower by more than the relative margin kCostTie), then the lower index.  The fused pose is the
//      winner's own final pose.  When the same hypothesis wins with and without a wrong view marked invalid, and its stages never
//      admitted that view, the fused pose has the same bits in both calls (the stages read only the views they admit).  A wrong
//      view that stage one admitted has pulled the first fit: if it is dropped later, the fit reaches the same minimum from
//      another start, and the bits differ.
//   5. LM.  Parameters: the world pose under the left perturbation, x_c = R_c (exp([dth]x) R X + t + dt_) + t_c.  A point's
//      Jacobian is pose_jacobian (pose_filter_core.h) at the camera pose (R_c R, R_c t + t_c) times diag(R_c, R_c).  Each step
//      solves (A + lambda diag A) delta = -g (A = J^T J, g = J^T r, Cholesky), lambda from 1e-3, / 10 on an accepted step (lower
//      cost, every point in front of every camera), x 10 on a rejected one or a failed factorisation; at most max_iter steps,
//      stopping at |delta| < 1e-12.  The update is R <- exp([dth]x) R, t <- t + dt_.
//   Outputs per (g, s): the world pose, world_cov = sigma^2 (sum J^T J)^-1 over the final views (spd_inverse6; singular: zeros and
//   kSingular), the final views, each valid view's RMS error under the fused pose (-1 for the others), the winning hypothesis
//   and the status; with kNoValid or kNoView the pose is zeros, no view is set, every view_err is -1 and fuse_hyp is -1.  The
//   fused pose projected into every row's camera (ssp_project_points' arithmetic with K_c in fp64) gives corners_world; zeros
//   without a fused pose.
// Of the operations here only the libm functions sin and cos (so3_exp in the LM update) may round differently on the device and
// the host; the per-view solve (step 1) is built with multiply-add contraction on the device, as pnp.cu is.
#pragma once
#include <math.h>

#include "pnp_consensus_core.h"
#include "pose_filter_core.h"

namespace ssp_mv {

constexpr int kMaxViews = 16, kMinPoints = 7, kMaxPoints = 10;
constexpr int kHypDoubles = 14;                   // per hypothesis in the workspace: R [9], t [3], final cost, final view set
// step 4's cost comparison: a cost counts as lower only below (1 - kCostTie) x the best so far.  Hypotheses that converge to the
// same minimum differ in the last bits of their cost; with this margin the lower index wins among them, whatever the rounding.
constexpr double kCostTie = 1e-9;
enum FuseStatus { kNoValid = 1, kNoView = 2, kSingular = 4 };

// workspace: [groups][slots][views][kHypDoubles] fp64
SSP_HD long long work_bytes(long long groups, int views, int slots) { return groups * slots * views * kHypDoubles * 8; }

SSP_HD int popc(unsigned v) { return ssp_pnpc::popc(v); }

// one camera of the rig: fx, fy, cx, cy of the fp32 K (as the PnP reads it), dist (8) or null for the pinhole model, R [9], t [3]
struct Cam {
  double fx, fy, cx, cy;
  const double* dist;
  const double* R;
  const double* t;
};

// the rig's tables: K [C][9] fp32, dist [C][8] or null, R [C][9], t [C][3]
struct Rig {
  const float* K;
  const double* dist;
  const double* R;
  const double* t;
  int C;
};

// camera c's coefficients, or null when they are all zero
SSP_HD const double* cam_dist(const double* dist, int c) {
  if (!dist) return nullptr;
  const double* d = dist + 8 * c;
  for (int k = 0; k < 8; k++)
    if (d[k] != 0.0) return d;
  return nullptr;
}

SSP_HD Cam camera(const Rig& rig, int c) {
  const float* K = rig.K + 9 * c;
  return Cam{(double)K[0], (double)K[4], (double)K[2], (double)K[5], cam_dist(rig.dist, c), rig.R + 9 * c, rig.t + 3 * c};
}

// the points of the C views of one (capture, slot): view c's np object points at p3 + c * p3_stride, its keypoints at uv + c * uv_stride
struct Views {
  const float* p3;
  long long p3_stride;
  const float* uv;
  long long uv_stride;
  int np;
};

// camera pose of a world pose: Rw = Rc R, tw = Rc t + tc
SSP_HD void to_camera(const Cam& cam, const double R[9], const double t[3], double Rw[9], double tw[3]) {
  ssp_pf::mat3_mul(cam.R, R, Rw);
  for (int i = 0; i < 3; i++) tw[i] = cam.R[3 * i] * t[0] + cam.R[3 * i + 1] * t[1] + cam.R[3 * i + 2] * t[2] + cam.t[i];
}

// world pose of a camera pose (step 2): R = Rc^T Rv, t = Rc^T (tv - tc)
SSP_HD void to_world(const Cam& cam, const double Rv[9], const double tv[3], double R[9], double t[3]) {
  const double* Rc = cam.R;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[3 * i + j] = Rc[i] * Rv[j] + Rc[3 + i] * Rv[3 + j] + Rc[6 + i] * Rv[6 + j];
  const double d[3] = {tv[0] - cam.t[0], tv[1] - cam.t[1], tv[2] - cam.t[2]};
  for (int i = 0; i < 3; i++) t[i] = Rc[i] * d[0] + Rc[3 + i] * d[1] + Rc[6 + i] * d[2];
}

// the mean squared reprojection error of view w's points under its camera pose (Rw, tw), every operation rounded on its own in
// score's order (pnp_consensus_core.h); returns false when a point lies at depth <= 0 (the mean is still written)
SSP_HD bool view_mse(const Cam& cam, const double Rw[9], const double tw[3], const float* p3, const float* uv, int np, double* mse) {
  using namespace ssp_pnpc;
  bool front = true;
  double s = 0.0;
  for (int i = 0; i < np; i++) {
    const double X = p3[3 * i], Y = p3[3 * i + 1], Z = p3[3 * i + 2];
    const double x = add(add(add(mul(Rw[0], X), mul(Rw[1], Y)), mul(Rw[2], Z)), tw[0]);
    const double y = add(add(add(mul(Rw[3], X), mul(Rw[4], Y)), mul(Rw[5], Z)), tw[1]);
    const double z = add(add(add(mul(Rw[6], X), mul(Rw[7], Y)), mul(Rw[8], Z)), tw[2]);
    if (!(z > 0.0)) front = false;
    const double iz = rcp(z);
    double du, dv;
    if (cam.dist) {
      double xd, yd;
      distort_rn(cam.dist, mul(x, iz), mul(y, iz), &xd, &yd);
      du = sub(add(mul(xd, cam.fx), cam.cx), (double)uv[2 * i]);
      dv = sub(add(mul(yd, cam.fy), cam.cy), (double)uv[2 * i + 1]);
    } else {
      du = sub(add(mul(mul(cam.fx, x), iz), cam.cx), (double)uv[2 * i]);
      dv = sub(add(mul(mul(cam.fy, y), iz), cam.cy), (double)uv[2 * i + 1]);
    }
    s = add(s, add(mul(du, du), mul(dv, dv)));
  }
  *mse = s / (double)np;
  return front;
}

// the valid views that agree with the world pose (R, t) at thr2 = thr^2 (step 3)
SSP_HD unsigned agree(const Rig& rig, const Views& v, unsigned valid, const double R[9], const double t[3], double thr2) {
  unsigned set = 0;
  for (int c = 0; c < rig.C; c++) {
    if (!((valid >> c) & 1u)) continue;
    const Cam cam = camera(rig, c);
    double Rw[9], tw[3], mse;
    to_camera(cam, R, t, Rw, tw);
    if (view_mse(cam, Rw, tw, v.p3 + c * v.p3_stride, v.uv + c * v.uv_stride, v.np, &mse) && mse <= thr2) set |= 1u << c;
  }
  return set;
}

// the pixel rows wu, wv [6] of point X's Jacobian with respect to the world pose's (dth, dt_): pose_jacobian at the camera pose
// (Rw, tw) = (Rc R, Rc t + tc), times diag(Rc, Rc)
SSP_HD void world_jacobian(const Cam& cam, const double Rw[9], const double tw[3], const double X[3], double wu[6], double wv[6]) {
  double ju[6], jv[6];
  ssp_pf::pose_jacobian(X, Rw, tw, cam.fx, cam.fy, cam.dist, ju, jv);
  for (int j = 0; j < 3; j++) {
    wu[j] = ju[0] * cam.R[j] + ju[1] * cam.R[3 + j] + ju[2] * cam.R[6 + j];
    wv[j] = jv[0] * cam.R[j] + jv[1] * cam.R[3 + j] + jv[2] * cam.R[6 + j];
    wu[3 + j] = ju[3] * cam.R[j] + ju[4] * cam.R[3 + j] + ju[5] * cam.R[6 + j];
    wv[3 + j] = jv[3] * cam.R[j] + jv[4] * cam.R[3 + j] + jv[5] * cam.R[6 + j];
  }
}

// the cost (sum of squared pixel residuals) of the views in `set` at the world pose (R, t) and, with A non-null, A = J^T J and
// g = J^T r in world axes (step 5); false when a point lies at depth <= 0
SSP_HD bool normal_equations(const Rig& rig, const Views& v, unsigned set, const double R[9], const double t[3], double* cost,
                             double (*A)[6], double* g) {
  if (A)
    for (int a = 0; a < 6; a++) {
      g[a] = 0.0;
      for (int b = 0; b < 6; b++) A[a][b] = 0.0;
    }
  double e = 0.0;
  for (int c = 0; c < rig.C; c++) {
    if (!((set >> c) & 1u)) continue;
    const Cam cam = camera(rig, c);
    double Rw[9], tw[3];
    to_camera(cam, R, t, Rw, tw);
    const float* p3 = v.p3 + c * v.p3_stride;
    const float* uv = v.uv + c * v.uv_stride;
    for (int i = 0; i < v.np; i++) {
      const double X[3] = {(double)p3[3 * i], (double)p3[3 * i + 1], (double)p3[3 * i + 2]};
      const double x = Rw[0] * X[0] + Rw[1] * X[1] + Rw[2] * X[2] + tw[0];
      const double y = Rw[3] * X[0] + Rw[4] * X[1] + Rw[5] * X[2] + tw[1];
      const double z = Rw[6] * X[0] + Rw[7] * X[1] + Rw[8] * X[2] + tw[2];
      if (!(z > 0.0)) return false;
      const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
      double u, w;
      if (cam.dist) {
        double xd, yd;
        ssp_pnp::distort(cam.dist, xn, yn, &xd, &yd, nullptr);
        u = xd * cam.fx + cam.cx; w = yd * cam.fy + cam.cy;
      } else {
        u = cam.fx * xn + cam.cx; w = cam.fy * yn + cam.cy;
      }
      const double eu = u - (double)uv[2 * i], ev = w - (double)uv[2 * i + 1];
      e += eu * eu + ev * ev;
      if (!A) continue;
      double wu[6], wv[6];
      world_jacobian(cam, Rw, tw, X, wu, wv);
      for (int a = 0; a < 6; a++) {
        g[a] += wu[a] * eu + wv[a] * ev;
        for (int b = a; b < 6; b++) A[a][b] += wu[a] * wu[b] + wv[a] * wv[b];
      }
    }
  }
  if (A)
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < a; b++) A[a][b] = A[b][a];
  *cost = e;
  return true;
}

// the LM of step 5 over `set` from (R, t), in place; returns the final cost
SSP_HD double lm(const Rig& rig, const Views& v, unsigned set, double R[9], double t[3], int max_iter) {
  double A[6][6], g[6], cost;
  if (!normal_equations(rig, v, set, R, t, &cost, A, g)) return INFINITY;
  double lam = 1e-3;
  for (int it = 0; it < max_iter; it++) {
    double M[6][6], d[6];
    for (int a = 0; a < 6; a++) {
      for (int b = 0; b < 6; b++) M[a][b] = A[a][b];
      M[a][a] += lam * A[a][a];
      d[a] = -g[a];
    }
    if (!ssp_pnp::chol_solve<6>(M, d)) { lam *= 10.0; continue; }
    double dn = 0.0;
    for (int a = 0; a < 6; a++) dn += d[a] * d[a];
    if (sqrt(dn) < 1e-12) break;
    double E[9], Rn[9], tn[3], An[6][6], gn[6], cn;
    ssp_pf::so3_exp(d, E);
    ssp_pf::mat3_mul(E, R, Rn);
    for (int i = 0; i < 3; i++) tn[i] = t[i] + d[3 + i];
    if (normal_equations(rig, v, set, Rn, tn, &cn, An, gn) && cn < cost) {
      for (int i = 0; i < 9; i++) R[i] = Rn[i];
      for (int i = 0; i < 3; i++) t[i] = tn[i];
      for (int a = 0; a < 6; a++) {
        g[a] = gn[a];
        for (int b = 0; b < 6; b++) A[a][b] = An[a][b];
      }
      cost = cn;
      lam /= 10.0;
    } else {
      lam *= 10.0;
    }
  }
  return cost;
}

// the per-view poses of one (capture, slot): view c's camera-frame R at R + c * r_stride, t at t + c * t_stride
struct RowPoses {
  const double* R;
  long long r_stride;
  const double* t;
  long long t_stride;
};

SSP_HD void hypothesis(const Rig& rig, const RowPoses& rows, int h, double R[9], double t[3]) {
  to_world(camera(rig, h), rows.R + h * rows.r_stride, rows.t + h * rows.t_stride, R, t);
}

// a fit of `set` from (R, t), in place: one view's hypothesis, or the LM
SSP_HD void fit(const Rig& rig, const Views& v, const RowPoses& rows, unsigned set, double R[9], double t[3], int max_iter) {
  if (popc(set) == 1) {
    int w = 0;
    while (!((set >> w) & 1u)) w++;
    hypothesis(rig, rows, w, R, t);
    return;
  }
  lm(rig, v, set, R, t, max_iter);
}

// steps 2-3 for hypothesis h: slot [kHypDoubles] = R, t, final cost, final set (as a double); returns the final set
SSP_HD unsigned score_hypothesis(const Rig& rig, const Views& v, const RowPoses& rows, unsigned valid, int h, double gate2, double thr2,
                                 int max_iter, double* slot) {
  double* R = slot;
  double* t = slot + 9;
  unsigned set = 0;
  double cost = INFINITY;
  for (int i = 0; i < 9; i++) R[i] = 0.0;
  for (int i = 0; i < 3; i++) t[i] = 0.0;
  if ((valid >> h) & 1u) {
    hypothesis(rig, rows, h, R, t);
    const unsigned A = agree(rig, v, valid, R, t, gate2);
    if (A) {
      fit(rig, v, rows, A, R, t, max_iter);
      unsigned A2 = agree(rig, v, valid, R, t, thr2);
      if (A2 != A && A2) fit(rig, v, rows, A2, R, t, max_iter);
      for (int k = 0; k < rig.C && A2; k++) {                 // the check: the fused views that left reproj_thresh go
        const unsigned A3 = agree(rig, v, A2, R, t, thr2);
        if (A3 == A2) break;
        A2 = A3;
        if (A2) fit(rig, v, rows, A2, R, t, max_iter);
      }
      set = A2;
      if (set && !normal_equations(rig, v, set, R, t, &cost, nullptr, nullptr)) cost = INFINITY;
    }
  }
  slot[12] = cost;
  slot[13] = (double)set;
  return set;
}

// step 4 over the C hypothesis slots (kHypDoubles apart): the winner, or -1 when none kept a view
SSP_HD int select(const double* slots, int C) {
  int best = -1, best_n = 0;
  double best_cost = 0.0;
  for (int h = 0; h < C; h++) {
    const double* s = slots + h * kHypDoubles;
    const int n = popc((unsigned)s[13]);
    if (n > best_n || (n == best_n && n > 0 && s[12] < best_cost * (1.0 - kCostTie))) { best = h; best_n = n; best_cost = s[12]; }
  }
  return best;
}

// ssp_project_points' pixel of X under the camera pose (Rw, tw) with the fp64 K [9], or cv2.projectPoints' with dist
SSP_HD void project(const double Rw[9], const double tw[3], double X, double Y, double Z, const double* Kd, const double* dist, float* u, float* v) {
  const double cam[3] = {Rw[0] * X + Rw[1] * Y + Rw[2] * Z + tw[0], Rw[3] * X + Rw[4] * Y + Rw[5] * Z + tw[1], Rw[6] * X + Rw[7] * Y + Rw[8] * Z + tw[2]};
  if (dist) {
    double pu, pv;
    ssp_pnp::project_distorted(dist, cam[0], cam[1], cam[2], Kd[0], Kd[4], Kd[2], Kd[5], &pu, &pv);
    *u = (float)pu; *v = (float)pv;
    return;
  }
  const double px = Kd[0] * cam[0] + Kd[1] * cam[1] + Kd[2] * cam[2];
  const double py = Kd[3] * cam[0] + Kd[4] * cam[1] + Kd[5] * cam[2];
  const double pz = Kd[6] * cam[0] + Kd[7] * cam[1] + Kd[8] * cam[2];
  *u = (float)(px / pz); *v = (float)(py / pz);
}

// step 5's outputs of one (capture, slot) from its hypothesis slots: R [9], t [3], cov [36], views [C] (0/1), view_err [C],
// *hyp, *status, and corners [C][np][2] (view c's points under the fused pose in camera c, at corners + c * corners_stride);
// K64 [C][9] the fp64 intrinsics of the projection
SSP_HD void finish(const Rig& rig, const Views& v, unsigned valid, const double* slots, double sigma, const double* K64, double* R, double* t, double* cov, unsigned char* views, double* view_err, int* hyp, int* status,
                   float* corners, long long corners_stride) {
  const int best = valid ? select(slots, rig.C) : -1;
  const unsigned set = best < 0 ? 0u : (unsigned)slots[best * kHypDoubles + 13];
  int st = !valid ? kNoValid : (best < 0 ? kNoView : 0);
  for (int i = 0; i < 9; i++) R[i] = best < 0 ? 0.0 : slots[best * kHypDoubles + i];
  for (int i = 0; i < 3; i++) t[i] = best < 0 ? 0.0 : slots[best * kHypDoubles + 9 + i];
  for (int c = 0; c < rig.C; c++) views[c] = (unsigned char)((set >> c) & 1u);
  *hyp = best;
  double A[6][6], Ai[6][6], g[6], cost;
  const bool usable = best >= 0 && normal_equations(rig, v, set, R, t, &cost, A, g) && ssp_pf::spd_inverse6(A, Ai);
  if (best >= 0 && !usable) st |= kSingular;
  const double s2 = sigma * sigma;
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) cov[6 * a + b] = usable ? s2 * Ai[a][b] : 0.0;
  *status = st;
  for (int c = 0; c < rig.C; c++) {
    const Cam cam = camera(rig, c);
    const float* p3 = v.p3 + c * v.p3_stride;
    float* out = corners + c * corners_stride;
    double Rw[9], tw[3];
    to_camera(cam, R, t, Rw, tw);
    double mse;
    view_mse(cam, Rw, tw, p3, v.uv + c * v.uv_stride, v.np, &mse);
    view_err[c] = best >= 0 && ((valid >> c) & 1u) ? sqrt(mse) : -1.0;
    for (int i = 0; i < v.np; i++) {
      if (best < 0) { out[2 * i] = 0.f; out[2 * i + 1] = 0.f; continue; }
      project(Rw, tw, p3[3 * i], p3[3 * i + 1], p3[3 * i + 2], K64 + 9 * c, cam.dist, out + 2 * i, out + 2 * i + 1);
    }
  }
}

}  // namespace ssp_mv
