// Pose covariance of a PnP solution and a constant-velocity pose filter per track slot: the rules of ssp_pose_covariance,
// ssp_track_predict and ssp_track_filter_update (pose_filter.cu), shared with the CPU test harness (tests/helpers/pose_filter_host.cpp,
// built with g++ -ffp-contract=off; the kernels are built with -fmad=false).  fp64 throughout.
//
// Perturbation.  A pose (R, t) is perturbed on the left: x_cam = exp([dth]x) R X + t + dt_, so the error of an estimate against the
// truth is (log(R_true R^T), t_true - t) -- the camera-frame rotation vector and the translation difference.
//
// Covariance of a PnP solution.  J (2P x 6) is the pixel projection of the P points with respect to (dth, dt_): its camera-frame
// part is d x_cam / d dth = -[R X]x and d x_cam / d dt_ = I, then d(x', y')/d x_cam of the normalisation and, with distortion
// coefficients, distort()'s chain rule (pnp_core.h), so the covariance belongs to the model the LM fitted.  Sigma = sigma^2 (J^T J)^-1
// with sigma the keypoint noise in pixels.  The inverse comes from a 6 x 6 Cholesky factorisation; a pivot <= 1e-12 x the largest
// diagonal entry of J^T J makes Sigma unusable (kCovSingular), and so does a point at camera depth <= 0 (kCovDepth).
//
// The filter: an error-state extended Kalman filter per (stream, track slot).  Nominal state: R, t, the angular velocity w (rad/s,
// camera frame, on the left: R(t + dt) = exp([w dt]x) R(t)) and the linear velocity v (mesh units / s); a 12 x 12 covariance P over
// (dth, dt_, dw, dv).  Layout of one slot, kFilterDoubles doubles: R [9], t [3], w [3], v [3], P [144] row-major, valid [1] (1 once
// the slot has been started from a usable measurement).
//   predict(dt):  R <- exp([w dt]x) R, t <- t + v dt;  P <- F P F^T + Q, F = I12 + dt (E(dth, dw) + E(dt_, dv)).  This F is first
//                 order in the rotation: it leaves out the rotation of dth by exp([w dt]x) and the SO(3) Jacobian of the velocity
//                 step, both 1 + O(|w| dt).  Q is white-noise acceleration: per axis q [[dt^3/3, dt^2/2], [dt^2/2, dt]] on (pose,
//                 velocity) with q = accel_sigma_rot^2 for the rotation axes and accel_sigma_trans^2 for the translation axes.
//   update(R_m, t_m, Sigma_m):  y = (log(R_m R^T), t_m - t), H = [I6 0], S = P[0:6, 0:6] + Sigma_m.  If Sigma_m is unusable, S is
//                 not positive definite (same pivot rule as above) or y^T S^-1 y > gate, the slot is re-initialised from the
//                 measurement instead (a mirrored or flipped PnP solution, or a track that jumped).  Else K = P H^T S^-1, the
//                 correction is K y, applied as R <- exp([dth]x) R, t += dt_, w += dw, v += dv (the reset Jacobian of the error
//                 state is taken as the identity), and P = (I - K H) P (I - K H)^T + K Sigma_m K^T (Joseph form), then symmetrised.
//   init(R_m, t_m, Sigma_m):  R, t from the measurement, w = v = 0; P = 0 except P[0:6, 0:6] = Sigma_m and the velocity variances
//                 init_velocity_sigma_rot^2, init_velocity_sigma_trans^2.  An unusable Sigma_m leaves the slot not valid: it is
//                 started again from the next usable measurement.
// Only the libm functions sin, cos (exp of so(3)), atan2 and acos (its log) may round differently on the device and the host.
#pragma once
#include <math.h>

#include "pnp_core.h"
#include "track_core.h"

namespace ssp_pf {

constexpr int kFilterDoubles = 9 + 3 + 3 + 3 + 144 + 1;     // R, t, w, v, P, valid
constexpr int kOffR = 0, kOffT = 9, kOffW = 12, kOffV = 15, kOffP = 18, kOffValid = 162;
enum CovStatus { kCovSingular = 1, kCovDepth = 2 };          // status bits of ssp_pose_covariance
enum FilterResult { kUpdated = 1, kReinit = 2 };              // what update() did

// R = exp([w]x) (Rodrigues' formula, the identity below machine epsilon)
SSP_HD void so3_exp(const double w[3], double R[9]) { ssp_pnp::rodrigues(w, R, nullptr); }

// w = log(R), |w| in [0, pi]: the axis from the antisymmetric part and the angle atan2(sin, cos), exact down to the smallest angles
// (a filter's innovations are small: cv2.Rodrigues' acos and its zero below 1e-5 rad would lose them); near pi the axis comes from
// the symmetric part, as cv2.Rodrigues takes it
SSP_HD void so3_log(const double R[9], double w[3]) {
  const double rv[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
  const double s = sqrt((rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]) * 0.25);
  double c = (R[0] + R[4] + R[8] - 1.0) * 0.5;
  c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
  if (s == 0.0 && c > 0) { w[0] = w[1] = w[2] = 0.0; return; }
  if (s < 1e-5 && c <= 0) {
    double tx = sqrt(fmax((R[0] + 1) * 0.5, 0.0));
    double ty = sqrt(fmax((R[4] + 1) * 0.5, 0.0)) * (R[1] < 0 ? -1.0 : 1.0);
    double tz = sqrt(fmax((R[8] + 1) * 0.5, 0.0)) * (R[2] < 0 ? -1.0 : 1.0);
    if (fabs(tx) < fabs(ty) && fabs(tx) < fabs(tz) && ((R[5] > 0) != (ty * tz > 0))) tz = -tz;
    const double nn = acos(c) / sqrt(tx * tx + ty * ty + tz * tz);
    w[0] = tx * nn; w[1] = ty * nn; w[2] = tz * nn;
    return;
  }
  const double f = 0.5 / s * atan2(s, c);
  w[0] = rv[0] * f; w[1] = rv[1] * f; w[2] = rv[2] * f;
}

SSP_HD void mat3_mul(const double A[9], const double B[9], double C[9]) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// the two pixel rows of J for object point X under (R, t): ju, jv [6] = d(u, v)/d(dth, dt_).  K: fx, fy, cx, cy; dist (8) or null.
// false when the point lies at camera depth <= 0
SSP_HD bool pose_jacobian(const double X[3], const double R[9], const double t[3], double fx, double fy, const double* dist, double ju[6],
                          double jv[6]) {
  const double a[3] = {R[0] * X[0] + R[1] * X[1] + R[2] * X[2], R[3] * X[0] + R[4] * X[1] + R[5] * X[2], R[6] * X[0] + R[7] * X[1] + R[8] * X[2]};
  const double x = a[0] + t[0], y = a[1] + t[1], z = a[2] + t[2];
  if (!(z > 0.0)) return false;
  const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
  // d x_cam / d(dth, dt_): columns of -[a]x, then I
  const double dc[3][6] = {{0.0, a[2], -a[1], 1.0, 0.0, 0.0}, {-a[2], 0.0, a[0], 0.0, 1.0, 0.0}, {a[1], -a[0], 0.0, 0.0, 0.0, 1.0}};
  double gx[6], gy[6];                                        // d(x', y') / d(dth, dt_)
  for (int j = 0; j < 6; j++) { gx[j] = (dc[0][j] - xn * dc[2][j]) * iz; gy[j] = (dc[1][j] - yn * dc[2][j]) * iz; }
  if (dist) {
    double xd, yd, D[4];
    ssp_pnp::distort(dist, xn, yn, &xd, &yd, D);
    for (int j = 0; j < 6; j++) { ju[j] = fx * (D[0] * gx[j] + D[1] * gy[j]); jv[j] = fy * (D[2] * gx[j] + D[3] * gy[j]); }
  } else {
    for (int j = 0; j < 6; j++) { ju[j] = fx * gx[j]; jv[j] = fy * gy[j]; }
  }
  return true;
}

// A^-1 of a symmetric 6 x 6 matrix from its Cholesky factor, symmetric by construction (A^-1 = L^-T L^-1); false when a pivot is
// <= 1e-12 x the largest diagonal entry (or not a number), and then Ai is not written
SSP_HD bool spd_inverse6(const double A[6][6], double Ai[6][6]) {
  double L[6][6], dmax = 0.0;
  for (int i = 0; i < 6; i++) dmax = fmax(dmax, A[i][i]);
  for (int j = 0; j < 6; j++) {
    double d = A[j][j];
    for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k];
    if (!(d > 1e-12 * dmax)) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 6; i++) {
      double v = A[i][j];
      for (int k = 0; k < j; k++) v -= L[i][k] * L[j][k];
      L[i][j] = v / L[j][j];
    }
  }
  double Li[6][6];                                            // L^-1, lower triangular
  for (int c = 0; c < 6; c++)
    for (int i = 0; i < 6; i++) {
      if (i < c) { Li[i][c] = 0.0; continue; }
      double v = i == c ? 1.0 : 0.0;
      for (int k = c; k < i; k++) v -= L[i][k] * Li[k][c];
      Li[i][c] = v / L[i][i];
    }
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) {
      double v = 0.0;
      for (int k = j; k < 6; k++) v += Li[k][i] * Li[k][j];
      Ai[i][j] = v; Ai[j][i] = v;
    }
  return true;
}

// Sigma [36] of the pose (R, t) of np object points p3 [np][3] (fp32, as the PnP reads them) with keypoint noise sigma px;
// returns the status bits (0: usable).  An unusable Sigma is written as zeros.
SSP_HD int pose_covariance(const float* p3, int np, double fx, double fy, const double* dist, const double R[9], const double t[3],
                           double sigma, double* cov) {
  double A[6][6];
  for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) A[a][b] = 0.0;
  int status = 0;
  for (int i = 0; i < np; i++) {
    const double X[3] = {(double)p3[3 * i], (double)p3[3 * i + 1], (double)p3[3 * i + 2]};
    double ju[6], jv[6];
    if (!pose_jacobian(X, R, t, fx, fy, dist, ju, jv)) { status |= kCovDepth; continue; }
    for (int a = 0; a < 6; a++)
      for (int b = a; b < 6; b++) A[a][b] += ju[a] * ju[b] + jv[a] * jv[b];
  }
  for (int a = 0; a < 6; a++) for (int b = 0; b < a; b++) A[a][b] = A[b][a];
  double Ai[6][6];
  if (!status && !spd_inverse6(A, Ai)) status |= kCovSingular;
  const double s2 = sigma * sigma;
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) cov[6 * a + b] = status ? 0.0 : s2 * Ai[a][b];
  return status;
}

// ---------------------------------------------------------------------------------------------------------------- the filter
struct FilterParams {
  double q_rot, q_trans;          // accel_sigma^2: white-noise angular and linear acceleration
  double v0_rot, v0_trans;        // init_velocity_sigma^2
  double gate;                    // chi^2 threshold of y^T S^-1 y
};

// predict the slot f [kFilterDoubles] over dt seconds, in place
SSP_HD void predict(double* f, double dt, const FilterParams& p) {
  double* P = f + kOffP;
  const double wd[3] = {f[kOffW] * dt, f[kOffW + 1] * dt, f[kOffW + 2] * dt};
  double E[9], R[9];
  so3_exp(wd, E);
  mat3_mul(E, f + kOffR, R);
  for (int i = 0; i < 9; i++) f[kOffR + i] = R[i];
  for (int i = 0; i < 3; i++) f[kOffT + i] += f[kOffV + i] * dt;
  // F P F^T with F = I + dt (rows 0..5 get dt x row r + 6), column-wise likewise
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 12; c++) P[12 * r + c] += dt * P[12 * (r + 6) + c];
  for (int r = 0; r < 12; r++)
    for (int c = 0; c < 6; c++) P[12 * r + c] += dt * P[12 * r + c + 6];
  const double d2 = dt * dt, d3 = d2 * dt;
  for (int a = 0; a < 6; a++) {
    const double q = a < 3 ? p.q_rot : p.q_trans;
    P[12 * a + a] += q * d3 / 3.0;
    P[12 * a + a + 6] += q * d2 / 2.0;
    P[12 * (a + 6) + a] += q * d2 / 2.0;
    P[12 * (a + 6) + a + 6] += q * dt;
  }
  for (int r = 0; r < 12; r++)
    for (int c = r + 1; c < 12; c++) { const double m = 0.5 * (P[12 * r + c] + P[12 * c + r]); P[12 * r + c] = m; P[12 * c + r] = m; }
}

// start the slot from the measurement; valid only with a usable Sigma_m
SSP_HD void init(double* f, const double Rm[9], const double tm[3], const double* Sm, bool usable, const FilterParams& p) {
  for (int i = 0; i < 9; i++) f[kOffR + i] = Rm[i];
  for (int i = 0; i < 3; i++) { f[kOffT + i] = tm[i]; f[kOffW + i] = 0.0; f[kOffV + i] = 0.0; }
  double* P = f + kOffP;
  for (int i = 0; i < 144; i++) P[i] = 0.0;
  for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) P[12 * a + b] = usable ? Sm[6 * a + b] : 0.0;
  for (int a = 0; a < 3; a++) { P[12 * (6 + a) + 6 + a] = p.v0_rot; P[12 * (9 + a) + 9 + a] = p.v0_trans; }
  f[kOffValid] = usable ? 1.0 : 0.0;
}

// fold the measurement (R_m, t_m, Sigma_m) into the slot: kUpdated, or kReinit when it was started from the measurement instead
SSP_HD int update(double* f, const double Rm[9], const double tm[3], const double* Sm, bool usable, const FilterParams& p) {
  if (!usable || f[kOffValid] != 1.0) { init(f, Rm, tm, Sm, usable, p); return kReinit; }
  double* P = f + kOffP;
  double S[6][6], Si[6][6];
  for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) S[a][b] = P[12 * a + b] + Sm[6 * a + b];
  double y[6], Rt[9], D[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rt[3 * i + j] = f[kOffR + 3 * j + i];
  mat3_mul(Rm, Rt, D);
  so3_log(D, y);
  for (int i = 0; i < 3; i++) y[3 + i] = tm[i] - f[kOffT + i];
  if (!spd_inverse6(S, Si)) { init(f, Rm, tm, Sm, usable, p); return kReinit; }
  double d2 = 0.0;                                            // y^T S^-1 y
  for (int a = 0; a < 6; a++) { double v = 0.0; for (int b = 0; b < 6; b++) v += Si[a][b] * y[b]; d2 += y[a] * v; }
  if (!(d2 <= p.gate)) { init(f, Rm, tm, Sm, usable, p); return kReinit; }
  double K[12][6];                                            // P H^T S^-1 = P[:, 0:6] S^-1
  for (int r = 0; r < 12; r++)
    for (int c = 0; c < 6; c++) { double v = 0.0; for (int k = 0; k < 6; k++) v += P[12 * r + k] * Si[k][c]; K[r][c] = v; }
  double dx[12];
  for (int r = 0; r < 12; r++) { double v = 0.0; for (int k = 0; k < 6; k++) v += K[r][k] * y[k]; dx[r] = v; }
  double E[9], R[9];
  so3_exp(dx, E);
  mat3_mul(E, f + kOffR, R);
  for (int i = 0; i < 9; i++) f[kOffR + i] = R[i];
  for (int i = 0; i < 3; i++) { f[kOffT + i] += dx[3 + i]; f[kOffW + i] += dx[6 + i]; f[kOffV + i] += dx[9 + i]; }
  // Joseph form: A = I - K H;  AP = P - K P[0:6, :];  P' = AP - AP[:, 0:6] K^T + K Sigma_m K^T
  double AP[12][12];
  for (int r = 0; r < 12; r++)
    for (int c = 0; c < 12; c++) { double v = P[12 * r + c]; for (int k = 0; k < 6; k++) v -= K[r][k] * P[12 * k + c]; AP[r][c] = v; }
  double KS[12][6];
  for (int r = 0; r < 12; r++)
    for (int c = 0; c < 6; c++) { double v = 0.0; for (int k = 0; k < 6; k++) v += K[r][k] * Sm[6 * k + c]; KS[r][c] = v; }
  for (int r = 0; r < 12; r++)
    for (int c = 0; c < 12; c++) {
      double v = AP[r][c];
      for (int k = 0; k < 6; k++) v += (KS[r][k] - AP[r][k]) * K[c][k];
      P[12 * r + c] = v;
    }
  for (int r = 0; r < 12; r++)
    for (int c = r + 1; c < 12; c++) { const double m = 0.5 * (P[12 * r + c] + P[12 * c + r]); P[12 * r + c] = m; P[12 * c + r] = m; }
  return kUpdated;
}

// the predicted corner rectangle of a slot: the 8 corners p3[1..8] of its class under (R, t), projected with K [9] (fp64, row-major;
// ssp_project_points' arithmetic) or, with dist, cv2.projectPoints' model, rounded to fp32 as those kernels round; false when a
// corner lies at depth <= 0
SSP_HD bool predicted_rect(const float* p3, const double R[9], const double t[3], const double* K, const double* dist, float uv[18]) {
  uv[0] = uv[1] = 0.f;
  for (int k = 1; k < 9; k++) {
    const double X = p3[3 * k], Y = p3[3 * k + 1], Z = p3[3 * k + 2];
    const double cam[3] = {R[0] * X + R[1] * Y + R[2] * Z + t[0], R[3] * X + R[4] * Y + R[5] * Z + t[1], R[6] * X + R[7] * Y + R[8] * Z + t[2]};
    if (!(cam[2] > 0.0)) return false;
    if (dist) {
      double u, v;
      ssp_pnp::project_distorted(dist, cam[0], cam[1], cam[2], K[0], K[4], K[2], K[5], &u, &v);
      uv[2 * k] = (float)u; uv[2 * k + 1] = (float)v;
    } else {
      const double px = K[0] * cam[0] + K[1] * cam[1] + K[2] * cam[2];
      const double py = K[3] * cam[0] + K[4] * cam[1] + K[5] * cam[2];
      const double pz = K[6] * cam[0] + K[7] * cam[1] + K[8] * cam[2];
      uv[2 * k] = (float)(px / pz); uv[2 * k + 1] = (float)(py / pz);
    }
  }
  return true;
}

// ssp_track_predict for one (stream, track slot): st [kFields] the slot's int fields, rect [4] / pose [6] its last rectangle and LM
// vector, f its filter, dt the stream's frame interval, P3 [num_classes][9][3]
SSP_HD void predict_slot(const int* st, const float* rect, const double* pose, double* f, double dt, const float* P3, int num_classes,
                         const double* K, const double* dist, const FilterParams& p, double* pred_pose, float* pred_rect) {
  const int c = st[ssp_trk::kCls];
  if (!st[ssp_trk::kAlive] || f[kOffValid] != 1.0 || c < 0 || c >= num_classes) {
    for (int k = 0; k < 6; k++) pred_pose[k] = pose[k];
    for (int k = 0; k < 4; k++) pred_rect[k] = rect[k];
    return;
  }
  predict(f, dt, p);
  so3_log(f + kOffR, pred_pose);
  for (int k = 0; k < 3; k++) pred_pose[3 + k] = f[kOffT + k];
  float uv[18];
  if (predicted_rect(P3 + (long long)c * 27, f + kOffR, f + kOffT, K, dist, uv)) {
    const ssp_det::Rect r = ssp_det::corner_rect(uv);
    pred_rect[0] = r.x0; pred_rect[1] = r.y0; pred_rect[2] = r.x1; pred_rect[3] = r.y1;
  } else {
    for (int k = 0; k < 4; k++) pred_rect[k] = rect[k];
  }
}

// ssp_track_filter_update for one detection slot: f the filter of its track slot, or null (an empty or untracked detection slot:
// zero outputs); R [9], t [3] the PnP, cov [36] / cov_status its covariance; out R_filt [9], t_filt [3], pose_cov [36], velocity [6]
SSP_HD void update_slot(double* f, bool matched, const double* R, const double* t, const double* cov, int cov_status, const FilterParams& p,
                        double* R_filt, double* t_filt, double* pose_cov, double* velocity, int* reinit) {
  if (!f) {
    for (int k = 0; k < 9; k++) R_filt[k] = 0.0;
    for (int k = 0; k < 3; k++) t_filt[k] = 0.0;
    for (int k = 0; k < 36; k++) pose_cov[k] = 0.0;
    for (int k = 0; k < 6; k++) velocity[k] = 0.0;
    *reinit = 0;
    return;
  }
  double Rm[9], tm[3], Sm[36];
  for (int k = 0; k < 9; k++) Rm[k] = R[k];
  for (int k = 0; k < 3; k++) tm[k] = t[k];
  for (int k = 0; k < 36; k++) Sm[k] = cov[k];
  const bool usable = cov_status == 0;
  int res = kReinit;
  if (matched) res = update(f, Rm, tm, Sm, usable, p);
  else init(f, Rm, tm, Sm, usable, p);
  for (int k = 0; k < 9; k++) R_filt[k] = f[kOffR + k];
  for (int k = 0; k < 3; k++) t_filt[k] = f[kOffT + k];
  for (int a = 0; a < 6; a++)
    for (int k = 0; k < 6; k++) pose_cov[6 * a + k] = f[kOffP + 12 * a + k];
  for (int k = 0; k < 3; k++) { velocity[k] = f[kOffW + k]; velocity[3 + k] = f[kOffV + k]; }
  *reinit = res == kReinit;
}

}  // namespace ssp_pf
