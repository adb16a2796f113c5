// Pose covariance of PnP solutions and the constant-velocity pose filter of tracked instances (rules: pose_filter_core.h).  All three
// kernels run one thread per problem or slot and read everything from device memory, so a graph replay needs no host read-back:
//   pose_cov_kernel       one thread per PnP problem: Sigma = sigma^2 (J^T J)^-1 at the solved pose, and its status bits;
//   track_predict_kernel  one thread per (stream, track slot): the filter of an alive, started slot moves to this frame's time in
//                         place; out the predicted LM vector and corner rectangle, which ssp_track_associate reads in place of the
//                         last ones (a slot without a started filter, or a predicted corner behind the camera, passes the last ones on);
//   track_update_kernel   one thread per detection slot with a track slot: a new track starts its filter, a matched one is gated and
//                         updated; out the filtered pose, its covariance, the velocity and whether the filter was (re)started.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <math.h>

#include "ssp_common.cuh"
#include "pose_filter_core.h"

namespace ssp {

static_assert(ssp_pf::kFilterDoubles == SSP_FILTER_DOUBLES, "include/ssp_b200.h's SSP_FILTER_DOUBLES is the filter layout of pose_filter_core.h");
static_assert(ssp_pf::kCovSingular == SSP_POSE_COV_SINGULAR && ssp_pf::kCovDepth == SSP_POSE_COV_DEPTH, "the covariance status bits");

__global__ void __launch_bounds__(128) pose_cov_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ Kmat,
                                                       const double* __restrict__ dist, int np, long long n, const int* __restrict__ count,
                                                       int per_group, const double* __restrict__ R, const double* __restrict__ t,
                                                       double sigma, double* __restrict__ cov, int* __restrict__ status) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  if (count && id % per_group >= count[id / per_group]) {
    for (int k = 0; k < 36; k++) cov[id * 36 + k] = 0.0;
    status[id] = 0;
    return;
  }
  double Ri[9], ti[3];
  for (int k = 0; k < 9; k++) Ri[k] = R[id * 9 + k];
  for (int k = 0; k < 3; k++) ti[k] = t[id * 3 + k];
  status[id] = ssp_pf::pose_covariance(P3 + id * p3_stride, np, Kmat[0], Kmat[4], dist, Ri, ti, sigma, cov + id * 36);
}

__global__ void __launch_bounds__(128) track_predict_kernel(int B, int T, const int* __restrict__ tracks, const float* __restrict__ rects,
                                                            const double* __restrict__ poses, double* __restrict__ filter,
                                                            const double* __restrict__ dt, const float* __restrict__ P3, int num_classes,
                                                            const double* __restrict__ Kd, const double* __restrict__ dist,
                                                            const ssp_pf::FilterParams p, double* __restrict__ pred_poses,
                                                            float* __restrict__ pred_rects) {
  const long long ts = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (ts >= (long long)B * T) return;
  ssp_pf::predict_slot(tracks + ts * ssp_trk::kFields, rects + ts * 4, poses + ts * 6, filter + ts * ssp_pf::kFilterDoubles, dt[ts / T], P3,
                       num_classes, Kd, dist, p, pred_poses + ts * 6, pred_rects + ts * 4);
}

__global__ void __launch_bounds__(128) track_update_kernel(int B, int T, int M, const int* __restrict__ count, const int* __restrict__ slot,
                                                           const int* __restrict__ use_guess, const double* __restrict__ R,
                                                           const double* __restrict__ t, const double* __restrict__ cov,
                                                           const int* __restrict__ cov_status, double* __restrict__ filter,
                                                           const ssp_pf::FilterParams p, double* __restrict__ R_filt,
                                                           double* __restrict__ t_filt, double* __restrict__ pose_cov,
                                                           double* __restrict__ velocity, int* __restrict__ reinit) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)B * M) return;
  const int b = (int)(o / M), m = (int)(o % M);
  const int s = m < count[b] ? slot[o] : -1;
  ssp_pf::update_slot(s < 0 ? nullptr : filter + ((long long)b * T + s) * ssp_pf::kFilterDoubles, use_guess[o] != 0, R + o * 9, t + o * 3,
                      cov + o * 36, cov_status[o], p, R_filt + o * 9, t_filt + o * 3, pose_cov + o * 36, velocity + o * 6, reinit + o);
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_pose_covariance(const float* P3, int shared, const float* K, const double* dist, int np, int groups, int per_group, const int* count,
                        const double* R, const double* t, double sigma, double* cov, int* status, void* stream) {
  if (!P3 || !K || !R || !t || !cov || !status || np < 3 || np > PNP_MAXP || groups < 0 || per_group < 1)
    return fail_msg(SSP_ERR_ARG, "pose_covariance: bad argument (null pointer, points outside 3..16, groups < 0 or per_group < 1)");
  if (!positive_finite(sigma)) return fail_msg(SSP_ERR_ARG, "pose_covariance: keypoint sigma must be > 0 and finite");
  const long long n = (long long)groups * per_group;
  if (n == 0) return SSP_OK;
  pose_cov_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(P3, shared ? 0 : 3LL * np, K, dist, np, n, count, per_group,
                                                                               R, t, sigma, cov, status);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_track_predict(int B, int max_tracks, const int* tracks, const float* rects, const double* poses, double* filter, const double* dt,
                      const float* points3d_table, int num_classes, const double* K, const double* dist, double accel_sigma_rot,
                      double accel_sigma_trans, double* pred_poses, float* pred_rects, void* stream) {
  if (!tracks || !rects || !poses || !filter || !dt || !points3d_table || !K || !pred_poses || !pred_rects)
    return fail_msg(SSP_ERR_ARG, "track_predict: null pointer");
  if (B < 0 || max_tracks < 1 || max_tracks > ssp_trk::kMaxTracks || num_classes < 1)
    return fail_msg(SSP_ERR_ARG, "track_predict: bad argument (B >= 0, 1 <= max_tracks <= 256, num_classes >= 1)");
  if (!positive_finite(accel_sigma_rot) || !positive_finite(accel_sigma_trans))
    return fail_msg(SSP_ERR_ARG, "track_predict: the acceleration sigmas must be > 0 and finite");
  const long long n = (long long)B * max_tracks;
  if (n == 0) return SSP_OK;
  ssp_pf::FilterParams p = {accel_sigma_rot * accel_sigma_rot, accel_sigma_trans * accel_sigma_trans, 0.0, 0.0, 0.0};
  track_predict_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(B, max_tracks, tracks, rects, poses, filter, dt,
                                                                                     points3d_table, num_classes, K, dist, p, pred_poses,
                                                                                     pred_rects);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_track_filter_update(int B, int max_tracks, int max_det, const int* count, const int* slot, const int* use_guess, const double* R,
                            const double* t, const double* cov, const int* cov_status, double* filter, double init_velocity_sigma_rot,
                            double init_velocity_sigma_trans, double gate, double* R_filt, double* t_filt, double* pose_cov,
                            double* velocity, int* reinit, void* stream) {
  if (!count || !slot || !use_guess || !R || !t || !cov || !cov_status || !filter || !R_filt || !t_filt || !pose_cov || !velocity || !reinit)
    return fail_msg(SSP_ERR_ARG, "track_filter_update: null pointer");
  if (B < 0 || max_tracks < 1 || max_tracks > ssp_trk::kMaxTracks || max_det < 1 || max_det > ssp_det::kMaxInstances)
    return fail_msg(SSP_ERR_ARG, "track_filter_update: bad argument (B >= 0, 1 <= max_tracks <= 256, 1 <= max_det <= 256)");
  if (!positive_finite(init_velocity_sigma_rot) || !positive_finite(init_velocity_sigma_trans) || !positive_finite(gate))
    return fail_msg(SSP_ERR_ARG, "track_filter_update: the initial velocity sigmas and the gate must be > 0 and finite");
  const long long n = (long long)B * max_det;
  if (n == 0) return SSP_OK;
  ssp_pf::FilterParams p = {0.0, 0.0, init_velocity_sigma_rot * init_velocity_sigma_rot,
                            init_velocity_sigma_trans * init_velocity_sigma_trans, gate};
  track_update_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(B, max_tracks, max_det, count, slot, use_guess, R, t,
                                                                                    cov, cov_status, filter, p, R_filt, t_filt, pose_cov,
                                                                                    velocity, reinit);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
