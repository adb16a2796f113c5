// Calibrating an RGB-D rig against depth: a point-to-plane bundle adjustment of the extrinsics and the observations' world poses,
// the rule of ssp_calibrate_rig_depth (calibrate_rig_depth.cu), shared with the CPU test harness
// (tests/helpers/calibrate_rig_depth_host.cpp, g++ -ffp-contract=off; the kernels are built with -fmad=false) and restated with
// whole arrays in oracle/calibrate_rig_depth_ref.py.  fp64 throughout.  refine_depth_core.h (find_pair, point_terms, gate_factor,
// kMinPoints, the 256-thread halving tree), refine_rig_core.h (the world-axis pair terms, depth_camera, extrinsics),
// multiview_core.h (to_camera), calibrate_rig_core.h (tree_sum, chol_pivot / chol_entry / chol_subst) and pose_filter_core.h
// (spd_inverse6, so3_exp) are used unchanged.
//
// Inputs: ssp_calibrate_rig's outputs -- C cameras (fp64 K, optional coefficients) with extrinsics (R_c, t_c), camera-from-world,
// cam_status (SSP_CALIB_UNCONNECTED) and the reference camera (R = I, t = 0); observations o = g S + s with world poses (R_o, t_o),
// views [o][c] and linked [o].  One mesh (vertices x_i, outward normals n_i, diameter d) for every observation.  Depth row g C + c
// is camera c's frame of capture g; every row has one W x H and one depth_scale.  Iteration k runs at the gate tau_k = d g_k.
// A camera is free when it is connected and is not the reference.  A view (o, c) is active when linked[o], views[o][c], camera c
// is connected and observation o has not stopped.
// Iteration k:
//   1. Per active view: for each model point, find_pair in camera c at the camera pose to_camera(R_o, t_o); r = m_c . (p_c - q_c);
//      J_obs the world-axis terms of refine_rig_core.h's world_pair (left perturbation x_w = exp([dth]x) R_o x + t_o + dt_), and for
//      a free camera J_cam = point_terms(a, m_c, p_c, q_c) with a = R_c (R_o x + t_o) (left perturbation in the camera frame,
//      x_c = exp([dth]x) R_c x_w + t_c + dt_, ssp_calibrate_rig's).  The view's accumulator (kAcc doubles): U = 21 upper entries of
//      J_cam J_cam^T, V = 21 of J_obs J_obs^T, W = 36 of J_cam J_obs^T (row-major), g_c = J_cam r, g_o = J_obs r, r^2, n, summed in
//      refine_depth_core.h's order (256 virtual threads, then the halving tree).  A camera that is not free adds no U, W, g_c.
//   2. Per linked observation that has not stopped: n_o, V_o, g_o, r^2 over its active views, the first view's entries copied and
//      the others added in camera order (refine_rig_core.h's sum_views); points = n_o, rmse = sqrt(r^2 / n_o) (0 without pairs).
//      n_o < kMinPoints stops it with kFewPoints, a failed spd_inverse6 (V_o) with kSingular (ssp_refine_depth's bits).  Otherwise
//      q_o = V_o^-1 g_o and, per active view of a free camera, Z_oc = V_o^-1 W_oc^T, in solve_update's product order.
//   3. The views of the observations that did not stop are this iteration's active views.  Per connected camera n_c and r^2_c over
//      them; a free camera with n_c < kMinPoints is held (kCamFewPoints) this iteration.  Over the solved cameras (free, not held)
//      in increasing index: S_c1c2 = [c1 == c2] U_c - sum_o W_oc1 Z_oc2, rhs_c = sum_o (W_oc q_o - g_oc).  Every sum over
//      observations: 256 lane partials (lane l takes o = l, l + 256, ... in increasing o), then tree_sum.  S is factored by
//      calibrate_rig_core.h's Cholesky, undamped; a failure stops the whole call (kCamSingular in the global status, and every
//      output pose is its input).  iter_rmse[k] = sqrt(sum_c r^2_c / sum_c n_c) over the connected cameras in camera order.
//   4. dc = S^-1 rhs (chol_subst); do = -(q_o + sum_c Z_oc dc_c), the solved cameras of o's active views in increasing index;
//      R <- exp([dth]x) R, t <- t + dt_ for each solved camera and each observation that did not stop.  The reference, held and
//      unconnected cameras keep their bits.
// Outputs: per camera R, t; cam_points, cam_rmse over its active views of the last iteration run; cam_cov = iter_rmse^2 times the
// camera's block of the last iteration's S^-1 (zeros for the reference, held and unconnected cameras); cam_status (SSP_CALIB_DEPTH_*).
// Per observation R_world, t_world (the input pose when it stopped or is not linked), obs_points, obs_rmse of its last iteration,
// obs_status (SSP_REFINE_FEW_POINTS / SSP_REFINE_SINGULAR).  Global: status, iter_rmse [iters] (0 for iterations not run).
// With no camera free (or held) the per-observation arithmetic is refine_rig_core.h's: with every view but the reference camera's
// switched off, each observation's outputs are ssp_refine_depth_rig's on the one-camera rig of the reference camera, bit for bit.
// Only the libm functions sin and cos (so3_exp) may round differently on the device and the host.
#pragma once
#include <math.h>

#include "calibrate_rig_core.h"
#include "refine_rig_core.h"

namespace ssp_cd {

constexpr int kMaxViews = ssp_mv::kMaxViews;
constexpr int kThreads = ssp_rd::kThreads;
constexpr int kLanes = ssp_cal::kLanes;
constexpr int kU = 0, kV = 21, kW = 42, kGc = 78, kGo = 84, kR2 = 90, kN = 91, kAcc = 92;
constexpr int kBlockDiag = 80;                 // entries of a diagonal camera block: W Z [36], U [36], rhs [6], n, r^2
enum CamStatus { kCamUnconnected = 1, kCamFewPoints = 2, kCamSingular = 4 };
enum Ctl { kStop, kSolved, kHeld, kCtl = 4 };  // control block: global stop, the solved and held camera masks

// the workspace, in doubles
struct Layout {
  long long acc, Z, q, obs, flag, blocks, diag, cam, dcam, ctl, total;
};
SSP_HD Layout layout(long long O, int C) {
  Layout L;
  long long at = 0;
  L.acc = at; at += O * C * kAcc;
  L.Z = at; at += O * C * 36;
  L.q = at; at += O * 6;
  L.obs = at; at += O * 12;                    // R [9], t [3] per observation
  L.flag = at; at += O;                        // the status that stopped the observation, 0 while it runs
  L.blocks = at; at += (long long)C * C * 36;  // sum_o W_oc1 Z_oc2 of the pair c1 < c2 at [c1][c2]
  L.diag = at; at += (long long)C * (kBlockDiag - 36);   // per camera: U [36], rhs [6], n, r^2
  L.cam = at; at += C * 12;                    // R [C][9], then t [C][3]
  L.dcam = at; at += C * 6;
  L.ctl = at; at += kCtl;
  L.total = at;
  return L;
}

struct Problem {
  const unsigned short* depth;                 // [G C][H][W]
  ssp_rr::Rig rig;                             // R, t: the current extrinsics in the workspace
  const double* model;                         // [nv][6] vertices and outward normals
  int nv;
  double diam;
  const unsigned char* views;                  // [O][C]
  const unsigned char* linked;                 // [O]
  const int* status_in;                        // [C] ssp_calibrate_rig's cam_status
  int ref, S;                                  // S observations per capture: o = g S + s
  long long O;
  double* w;
  Layout L;
};

SSP_HD int C_of(const Problem& P) { return P.rig.C; }
SSP_HD bool connected(const Problem& P, int c) { return !(P.status_in[c] & ssp_cal::kUnconnected); }
SSP_HD bool is_free(const Problem& P, int c) { return c != P.ref && connected(P, c); }
SSP_HD double* ctl(const Problem& P) { return P.w + P.L.ctl; }
SSP_HD bool stopped(const Problem& P, long long o) { return P.w[P.L.flag + o] != 0.0; }
SSP_HD bool view_on(const Problem& P, long long o, int c) { return P.linked[o] && P.views[o * C_of(P) + c] && connected(P, c); }
SSP_HD bool active(const Problem& P, long long o, int c) { return view_on(P, o, c) && !stopped(P, o); }
SSP_HD double* acc_of(const Problem& P, long long o, int c) { return P.w + P.L.acc + (o * C_of(P) + c) * kAcc; }
SSP_HD double* Z_of(const Problem& P, long long o, int c) { return P.w + P.L.Z + (o * C_of(P) + c) * 36; }
SSP_HD double* obs_pose(const Problem& P, long long o) { return P.w + P.L.obs + o * 12; }
SSP_HD const unsigned short* frame(const Problem& P, long long o, int c) {
  return P.depth + ((o / P.S) * C_of(P) + c) * (long long)P.rig.H * P.rig.W;
}
SSP_HD int upper(int a, int b) { return a * 6 - a * (a - 1) / 2 + (b - a); }      // packed index of (a, b), a <= b

// the state from the inputs: extrinsics, world poses, flags and the control block
SSP_HD void init_cams(const Problem& P, const double* R_in, const double* t_in) {
  double* R = P.w + P.L.cam;
  double* t = R + 9 * C_of(P);
  for (int k = 0; k < 9 * C_of(P); k++) R[k] = R_in[k];
  for (int k = 0; k < 3 * C_of(P); k++) t[k] = t_in[k];
  for (int k = 0; k < kCtl; k++) ctl(P)[k] = 0.0;
}
SSP_HD void init_obs(const Problem& P, long long o, const double* R_in, const double* t_in) {
  double* x = obs_pose(P, o);
  for (int k = 0; k < 9; k++) x[k] = R_in[o * 9 + k];
  for (int k = 0; k < 3; k++) x[9 + k] = t_in[o * 3 + k];
  P.w[P.L.flag + o] = 0.0;
}

// ---------------------------------------------------------------------------------------------------- step 1
// the pair of model point x6 in camera `ext` at the world pose (R, t), whose camera pose is (Rp, tp): r = m_c . (p_c - q_c), the
// observation's world-axis terms Jo and, with cam_terms, the camera's terms Jc; false when the point makes no pair
SSP_HD bool pair_terms(const double* x6, const double R[9], const double t[3], const double Rp[9], const double tp[3], const ssp_mv::Cam& ext,
                       const ssp_rd::Camera& cam, const unsigned short* depth, double tau, bool cam_terms, double* r, double Jo[6], double Jc[6]) {
  double a[3], m[3], p[3], q[3];
  if (!ssp_rd::find_pair(x6, Rp, tp, cam, depth, tau, a, m, p, q)) return false;
  double aw[3], mw[3], pw[3], qw[3];                          // world_pair's world-axis terms
  for (int i = 0; i < 3; i++) {
    aw[i] = R[3 * i] * x6[0] + R[3 * i + 1] * x6[1] + R[3 * i + 2] * x6[2];
    mw[i] = R[3 * i] * x6[3] + R[3 * i + 1] * x6[4] + R[3 * i + 2] * x6[5];
    pw[i] = aw[i] + t[i];
  }
  const double d[3] = {q[0] - ext.t[0], q[1] - ext.t[1], q[2] - ext.t[2]};
  for (int i = 0; i < 3; i++) qw[i] = ext.R[i] * d[0] + ext.R[3 + i] * d[1] + ext.R[6 + i] * d[2];
  ssp_rd::point_terms(aw, mw, pw, qw, Jo);
  double ac[3];                                               // R_c x_w: the camera's lever arm
  for (int i = 0; i < 3; i++) ac[i] = cam_terms ? ext.R[3 * i] * pw[0] + ext.R[3 * i + 1] * pw[1] + ext.R[3 * i + 2] * pw[2] : a[i];
  *r = ssp_rd::point_terms(ac, m, p, q, Jc);
  return true;
}

// add model point x6's pair, if it makes one, to the accumulator whose entry i is acc[i * stride]
SSP_HD void accumulate_point(const double* x6, const double R[9], const double t[3], const double Rp[9], const double tp[3], const ssp_mv::Cam& ext,
                             const ssp_rd::Camera& cam, const unsigned short* depth, double tau, bool cam_terms, double* acc, int stride) {
  double r, Jo[6], Jc[6];
  if (!pair_terms(x6, R, t, Rp, tp, ext, cam, depth, tau, cam_terms, &r, Jo, Jc)) return;
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++, k++) {
      acc[(kV + k) * stride] += Jo[i] * Jo[j];
      if (cam_terms) acc[(kU + k) * stride] += Jc[i] * Jc[j];
    }
  if (cam_terms) {
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) acc[(kW + 6 * i + j) * stride] += Jc[i] * Jo[j];
    for (int i = 0; i < 6; i++) acc[(kGc + i) * stride] += Jc[i] * r;
  }
  for (int i = 0; i < 6; i++) acc[(kGo + i) * stride] += Jo[i] * r;
  acc[kR2 * stride] += r * r;
  acc[kN * stride] += 1.0;
}

// virtual thread j's accumulator of view (o, c) at gate tau (entry i at acc[i * stride], zeroed here): model points j, j + kThreads, ...
SSP_HD void view_thread(const Problem& P, long long o, int c, double tau, int j, double* acc, int stride) {
  for (int i = 0; i < kAcc; i++) acc[i * stride] = 0.0;
  const double* x = obs_pose(P, o);
  double R[9], t[3];
  for (int k = 0; k < 9; k++) R[k] = x[k];
  for (int k = 0; k < 3; k++) t[k] = x[9 + k];
  const ssp_mv::Cam ext = ssp_rr::extrinsics(P.rig, c);
  const ssp_rd::Camera cam = ssp_rr::depth_camera(P.rig, c);
  double Rp[9], tp[3];
  ssp_mv::to_camera(ext, R, t, Rp, tp);
  const unsigned short* D = frame(P, o, c);
  const bool ct = is_free(P, c);
  for (int i = j; i < P.nv; i += kThreads) accumulate_point(P.model + (long long)i * 6, R, t, Rp, tp, ext, cam, D, tau, ct, acc, stride);
}

// ---------------------------------------------------------------------------------------------------- step 2
// linked observation o's sums, solve and status (0, or the ssp_refine_depth bit that stops it, also kept in its flag); q_o and Z_oc
// into the workspace.  points, rmse: its pairs and RMS residual of this iteration.
SSP_HD int obs_solve(const Problem& P, long long o, int* points, double* rmse) {
  const int C = C_of(P);
  double V[21], g[6], r2 = 0.0, n = 0.0;
  bool any = false;
  for (int i = 0; i < 21; i++) V[i] = 0.0;
  for (int i = 0; i < 6; i++) g[i] = 0.0;
  for (int c = 0; c < C; c++) {
    if (!active(P, o, c)) continue;
    const double* a = acc_of(P, o, c);
    if (!any) {
      for (int i = 0; i < 21; i++) V[i] = a[kV + i];
      for (int i = 0; i < 6; i++) g[i] = a[kGo + i];
      r2 = a[kR2]; n = a[kN];
    } else {
      for (int i = 0; i < 21; i++) V[i] += a[kV + i];
      for (int i = 0; i < 6; i++) g[i] += a[kGo + i];
      r2 += a[kR2]; n += a[kN];
    }
    any = true;
  }
  *points = (int)n;
  *rmse = n > 0.0 ? sqrt(r2 / n) : 0.0;
  int status = 0;
  double A[6][6], Ai[6][6];
  if (*points < ssp_rd::kMinPoints) {
    status = ssp_rd::kFewPoints;
  } else {
    int k = 0;
    for (int i = 0; i < 6; i++)
      for (int j = i; j < 6; j++) { A[i][j] = V[k]; A[j][i] = V[k]; k++; }
    if (!ssp_pf::spd_inverse6(A, Ai)) status = ssp_rd::kSingular;
  }
  if (status) { P.w[P.L.flag + o] = (double)status; return status; }
  double* q = P.w + P.L.q + o * 6;
  for (int i = 0; i < 6; i++) {
    double v = 0.0;
    for (int j = 0; j < 6; j++) v += Ai[i][j] * g[j];
    q[i] = v;
  }
  for (int c = 0; c < C; c++) {
    if (!active(P, o, c) || !is_free(P, c)) continue;
    const double* W = acc_of(P, o, c) + kW;
    double* Z = Z_of(P, o, c);
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < 6; b++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += Ai[a][k] * W[6 * b + k];
        Z[6 * a + b] = s;
      }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------- step 3
// the entries [block_first, block_entries) of the camera-block pair (c1 <= c2) that are summed: a diagonal block of a connected
// camera that is not free has only n and r^2
SSP_HD int block_entries(const Problem& P, int c1, int c2) {
  if (c1 != c2) return is_free(P, c1) && is_free(P, c2) ? 36 : 0;
  return connected(P, c1) ? kBlockDiag : 0;
}
SSP_HD int block_first(const Problem& P, int c1) { return is_free(P, c1) ? 0 : 78; }

// entry e of observation o's contribution to the camera-block pair (c1 <= c2), or false when it contributes nothing.  Entries
// 0..35: (W_oc1 Z_oc2)[a][b]; on the diagonal also 36..71: U_oc [a][b], 72..77: (W_oc q_o - g_oc)[a], 78: n_oc, 79: r^2_oc (the
// last two for every connected camera, the others for free cameras)
SSP_HD bool block_term(const Problem& P, long long o, int c1, int c2, int e, double* val) {
  if (!active(P, o, c1) || !active(P, o, c2)) return false;
  const double* a1 = acc_of(P, o, c1);
  if (e >= 78) { *val = a1[e == 78 ? kN : kR2]; return true; }
  if (!is_free(P, c1)) return false;
  if (e < 36) {
    const double* W = a1 + kW;
    const double* Z = Z_of(P, o, c2);
    const int a = e / 6, b = e % 6;
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += W[6 * a + k] * Z[6 * k + b];
    *val = s;
  } else if (e < 72) {
    const int a = (e - 36) / 6, b = (e - 36) % 6;
    *val = a1[kU + (a <= b ? upper(a, b) : upper(b, a))];
  } else {
    const int a = e - 72;
    const double* W = a1 + kW;
    const double* q = P.w + P.L.q + o * 6;
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += W[6 * a + k] * q[k];
    *val = s - a1[kGc + a];
  }
  return true;
}

// lane l's partial sum of entry e of block (c1, c2)
SSP_HD double block_partial(const Problem& P, int c1, int c2, int e, int lane) {
  double acc = 0.0, v;
  for (long long o = lane; o < P.O; o += kLanes)
    if (block_term(P, o, c1, c2, e, &v)) acc += v;
  return acc;
}

SSP_HD double* block_slot(const Problem& P, int c1, int c2, int e) {
  if (e < 36 && c1 != c2) return P.w + P.L.blocks + ((long long)c1 * C_of(P) + c2) * 36 + e;
  if (e < 36) return P.w + P.L.blocks + ((long long)c1 * C_of(P) + c1) * 36 + e;
  return P.w + P.L.diag + (long long)c1 * (kBlockDiag - 36) + (e - 36);
}
SSP_HD double cam_n(const Problem& P, int c) { return P.w[P.L.diag + (long long)c * (kBlockDiag - 36) + 42]; }
SSP_HD double cam_r2(const Problem& P, int c) { return P.w[P.L.diag + (long long)c * (kBlockDiag - 36) + 43]; }

// this iteration's solved cameras (free with n_c >= kMinPoints) in increasing index, their count; the solved and held masks
SSP_HD int solve_list(const Problem& P, int* cams, unsigned* held) {
  int n = 0;
  *held = 0;
  for (int c = 0; c < C_of(P); c++) {
    if (!is_free(P, c)) continue;
    if (cam_n(P, c) < (double)ssp_rd::kMinPoints) *held |= 1u << c;
    else cams[n++] = c;
  }
  return n;
}

// the RMS residual over every active view of the iteration, the connected cameras in camera order
SSP_HD double overall_rmse(const Problem& P) {
  double r2 = 0.0, n = 0.0;
  for (int c = 0; c < C_of(P); c++)
    if (connected(P, c)) { r2 += cam_r2(P, c); n += cam_n(P, c); }
  return n > 0.0 ? sqrt(r2 / n) : 0.0;
}

// entry (I, J) of the reduced system over the solved cameras cams
SSP_HD double reduced_entry(const Problem& P, const int* cams, int I, int J) {
  int i = I / 6, j = J / 6, a = I % 6, b = J % 6;
  if (i > j) { int s = i; i = j; j = s; s = a; a = b; b = s; }
  const int c1 = cams[i], c2 = cams[j];
  const double sw = P.w[P.L.blocks + ((long long)c1 * C_of(P) + c2) * 36 + 6 * a + b];
  if (c1 != c2) return -sw;
  return P.w[P.L.diag + (long long)c1 * (kBlockDiag - 36) + 6 * a + b] - sw;
}

SSP_HD double rhs_entry(const Problem& P, const int* cams, int I) {
  return P.w[P.L.diag + (long long)cams[I / 6] * (kBlockDiag - 36) + 36 + I % 6];
}

// ---------------------------------------------------------------------------------------------------- step 4
// the solved cameras' update from dc [6 n] (in solve order) into the state and dcam [c][6]
SSP_HD void camera_update(const Problem& P, const int* cams, int n, const double* dc) {
  double* R = P.w + P.L.cam;
  double* t = R + 9 * C_of(P);
  for (int i = 0; i < n; i++) {
    const int c = cams[i];
    double E[9], Rn[9];
    for (int k = 0; k < 6; k++) P.w[P.L.dcam + 6 * c + k] = dc[6 * i + k];
    ssp_pf::so3_exp(dc + 6 * i, E);
    ssp_pf::mat3_mul(E, R + 9 * c, Rn);
    for (int k = 0; k < 9; k++) R[9 * c + k] = Rn[k];
    for (int k = 0; k < 3; k++) t[3 * c + k] += dc[6 * i + 3 + k];
  }
}

// observation o's update, when it did not stop: do = -(q_o + sum_c Z_oc dc_c) over the solved cameras (mask) of its active views
SSP_HD void obs_update(const Problem& P, long long o, unsigned solved) {
  if (!P.linked[o] || stopped(P, o)) return;
  const double* q = P.w + P.L.q + o * 6;
  double d[6];
  for (int a = 0; a < 6; a++) {
    double s = q[a];
    for (int c = 0; c < C_of(P); c++) {
      if (!((solved >> c) & 1u) || !active(P, o, c)) continue;
      const double* Z = Z_of(P, o, c);
      const double* dc = P.w + P.L.dcam + 6 * c;
      for (int b = 0; b < 6; b++) s += Z[6 * a + b] * dc[b];
    }
    d[a] = -s;
  }
  double* x = obs_pose(P, o);
  double E[9], Rn[9];
  ssp_pf::so3_exp(d, E);
  ssp_pf::mat3_mul(E, x, Rn);
  for (int k = 0; k < 9; k++) x[k] = Rn[k];
  for (int k = 0; k < 3; k++) x[9 + k] += d[3 + k];
}

// camera c's status bits after an iteration: held, unconnected passed through, and kCamSingular for a free camera on a global stop
SSP_HD int cam_status_bits(const Problem& P, int c) {
  const double* k = ctl(P);
  const unsigned held = (unsigned)k[kHeld];
  return (connected(P, c) ? 0 : kCamUnconnected) | (((held >> c) & 1u) ? kCamFewPoints : 0) |
         (is_free(P, c) && k[kStop] != 0.0 ? kCamSingular : 0);
}

}  // namespace ssp_cd
