// Host harness of the pose covariance and the pose filter (singleshotpose_b200/csrc/pose_filter_core.h): the loops of the kernels
// of pose_filter.cu run serially over the same per-problem and per-slot functions.  Built with -ffp-contract=off, as the kernels are
// built with -fmad=false.  Test infrastructure: built by tests/test_pose_filter_cpu.py into a temporary .so; never loaded by the product.
#include "../../singleshotpose_b200/csrc/pose_filter_core.h"

using namespace ssp_pf;

extern "C" {
// ssp_pose_covariance without groups: n problems, points p3 shared or [n][np][3]
int h_pose_covariance(const float* p3, int shared, const float* K, const double* dist, int np, long long n, const double* R, const double* t,
                      double sigma, double* cov, int* status) {
  if (np < 3 || np > PNP_MAXP || !(sigma > 0.0)) return -1;
  for (long long i = 0; i < n; i++)
    status[i] = pose_covariance(p3 + (shared ? 0 : i * 3 * np), np, K[0], K[4], dist, R + i * 9, t + i * 3, sigma, cov + i * 36);
  return 0;
}

// J [2][6] of one point (the rows d u / d(dth, dt_), d v / d(dth, dt_)); -1 when it lies at depth <= 0
int h_pose_jacobian(const double* X, const double* R, const double* t, double fx, double fy, const double* dist, double* J) {
  return pose_jacobian(X, R, t, fx, fy, dist, J, J + 6) ? 0 : -1;
}

void h_so3_log(const double* R, double* w) { so3_log(R, w); }

// ssp_track_predict (host arrays)
int h_track_predict(int B, int T, const int* tracks, const float* rects, const double* poses, double* filter, const double* dt, const float* P3,
                    int num_classes, const double* K, const double* dist, double accel_rot, double accel_trans, double* pred_poses,
                    float* pred_rects) {
  const FilterParams p = {accel_rot * accel_rot, accel_trans * accel_trans, 0.0, 0.0, 0.0};
  for (long long ts = 0; ts < (long long)B * T; ts++)
    predict_slot(tracks + ts * ssp_trk::kFields, rects + ts * 4, poses + ts * 6, filter + ts * kFilterDoubles, dt[ts / T], P3, num_classes, K,
                 dist, p, pred_poses + ts * 6, pred_rects + ts * 4);
  return 0;
}

// ssp_track_filter_update (host arrays)
int h_track_filter_update(int B, int T, int M, const int* count, const int* slot, const int* use_guess, const double* R, const double* t,
                          const double* cov, const int* cov_status, double* filter, double v0_rot, double v0_trans, double gate,
                          double* R_filt, double* t_filt, double* pose_cov, double* velocity, int* reinit) {
  const FilterParams p = {0.0, 0.0, v0_rot * v0_rot, v0_trans * v0_trans, gate};
  for (long long o = 0; o < (long long)B * M; o++) {
    const int b = (int)(o / M), m = (int)(o % M);
    const int s = m < count[b] ? slot[o] : -1;
    update_slot(s < 0 ? nullptr : filter + ((long long)b * T + s) * kFilterDoubles, use_guess[o] != 0, R + o * 9, t + o * 3, cov + o * 36,
                cov_status[o], p, R_filt + o * 9, t_filt + o * 3, pose_cov + o * 36, velocity + o * 6, reinit + o);
  }
  return 0;
}
}
