// Fusing several calibrated cameras' poses into one world pose (rule: multiview_core.h).  ssp_fuse_views runs three stages:
//   fuse_rows_kernel     (multiview_rows.cu) one thread per (row, slot): the per-view PnP and projection, one launch for the
//                        pinhole cameras and, with a distortion table, one per camera (fuse_rows_dist_kernel);
//   fuse_hyp_kernel      one thread per (capture, slot, hypothesis): agreement, the two fits, the final set and cost;
//   fuse_finish_kernel   one thread per (capture, slot): selection, covariance, per-view errors and the fused corners.
// This file is built with -fmad=false, as the host harness is built with -ffp-contract=off, so the fusion stages equal the harness
// bit for bit when it starts from the same per-row poses.
#include <math.h>

#include "ssp_common.cuh"
#include "multiview_core.h"

namespace ssp {

static_assert(ssp_mv::kMaxViews == SSP_RIG_MAX_VIEWS, "include/ssp_b200.h's view limit");
static_assert(ssp_mv::kNoValid == SSP_FUSE_NO_VALID && ssp_mv::kNoView == SSP_FUSE_NO_VIEW && ssp_mv::kSingular == SSP_FUSE_SINGULAR,
              "the fusion status bits");

int launch_fuse_rows(const float* P3, long long p3_stride, const float* uv, const float* K32, const double* K64, const double* dist, int np,
                     int C, int S, long long rows, int max_iter, double* R, double* t, float* corners, void* stream);

struct FuseArgs {
  const float* P3;
  long long p3_stride;          // between (row, slot)s: 0 shared, else 3 np
  const float* uv;
  const unsigned char* valid;   // [rows][S]
  int np, C, S;
  long long groups;
  ssp_mv::Rig rig;
  const double* R_rows;         // [rows][S][9], [rows][S][3]: step 1's poses
  const double* t_rows;
};

// the views of (capture g, slot s), their valid set and their per-view poses
__device__ inline ssp_mv::Views views_of(const FuseArgs& a, long long g, int s) {
  const long long r0 = (g * a.C) * a.S + s;                       // (row g C, slot s)
  return ssp_mv::Views{a.P3 + r0 * a.p3_stride, a.S * a.p3_stride, a.uv + r0 * 2 * a.np, (long long)a.S * 2 * a.np, a.np};
}
__device__ inline unsigned valid_of(const FuseArgs& a, long long g, int s) {
  unsigned m = 0;
  for (int c = 0; c < a.C; c++) m |= (a.valid[(g * a.C + c) * a.S + s] ? 1u : 0u) << c;
  return m;
}

__global__ void __launch_bounds__(128) fuse_hyp_kernel(const FuseArgs a, double gate2, double thr2, int max_iter, double* __restrict__ slots) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (g, s, h)
  if (id >= a.groups * a.S * a.C) return;
  const int h = (int)(id % a.C);
  const long long gs = id / a.C;
  const int s = (int)(gs % a.S);
  const long long g = gs / a.S;
  const long long r0 = (g * a.C) * a.S + s;
  const ssp_mv::RowPoses rows = {a.R_rows + r0 * 9, (long long)a.S * 9, a.t_rows + r0 * 3, (long long)a.S * 3};
  ssp_mv::score_hypothesis(a.rig, views_of(a, g, s), rows, valid_of(a, g, s), h, gate2, thr2, max_iter, slots + id * ssp_mv::kHypDoubles);
}

__global__ void __launch_bounds__(128) fuse_finish_kernel(const FuseArgs a, const double* __restrict__ slots, double sigma,
                                                          const double* __restrict__ K64, double* __restrict__ R_world,
                                                          double* __restrict__ t_world, double* __restrict__ cov,
                                                          unsigned char* __restrict__ views, double* __restrict__ view_err,
                                                          int* __restrict__ hyp, int* __restrict__ status, float* __restrict__ corners) {
  const long long gs = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (g, s)
  if (gs >= a.groups * a.S) return;
  const int s = (int)(gs % a.S);
  const long long g = gs / a.S;
  const long long r0 = (g * a.C) * a.S + s;
  ssp_mv::finish(a.rig, views_of(a, g, s), valid_of(a, g, s), slots + gs * a.C * ssp_mv::kHypDoubles, sigma, K64, R_world + gs * 9,
                 t_world + gs * 3, cov + gs * 36, views + gs * a.C, view_err + gs * a.C, hyp + gs, status + gs, corners + r0 * 2 * a.np,
                 (long long)a.S * 2 * a.np);
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_fuse_views_work_bytes(int groups, int views, int slots, long long* bytes_out) {
  if (!bytes_out || groups < 0 || views < 1 || views > ssp_mv::kMaxViews || slots < 1)
    return fail_msg(SSP_ERR_ARG, "fuse_views_work_bytes: bad size (groups >= 0, 1 <= views <= 16, slots >= 1)");
  *bytes_out = ssp_mv::work_bytes(groups, views, slots);
  return SSP_OK;
}

int ssp_fuse_views(const float* points3d, int points3d_shared, const float* points2d, const unsigned char* valid, int num_points, int groups,
                   int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null, const double* R_rig,
                   const double* t_rig, double gate, double reproj_thresh, double keypoint_sigma, int max_iter, double* R_out,
                   double* t_out, float* corners_out, double* R_world, double* t_world, double* world_cov, unsigned char* views_out,
                   double* view_err, int* fuse_hyp, int* fuse_status, float* corners_world, void* work, long long work_bytes,
                   void* stream) {
  if (!points3d || !points2d || !valid || !K3x3_f32 || !K3x3 || !R_rig || !t_rig || !R_out || !t_out || !corners_out || !R_world ||
      !t_world || !world_cov || !views_out || !view_err || !fuse_hyp || !fuse_status || !corners_world || !work)
    return fail_msg(SSP_ERR_ARG, "fuse_views: null pointer");
  if (views < 1 || views > ssp_mv::kMaxViews || num_points < ssp_mv::kMinPoints || num_points > ssp_mv::kMaxPoints || groups < 0 ||
      slots < 1 || max_iter < 1)
    return fail_msg(SSP_ERR_ARG, "fuse_views: bad size (1 <= views <= 16, 7 <= points <= 10, groups >= 0, slots >= 1, max_iter >= 1)");
  if (!positive_finite(gate) || !positive_finite(reproj_thresh) || !positive_finite(keypoint_sigma))
    return fail_msg(SSP_ERR_ARG, "fuse_views: gate, reproj_thresh and keypoint_sigma must be > 0 and finite");
  if (gate < reproj_thresh) return fail_msg(SSP_ERR_ARG, "fuse_views: the gate must be >= reproj_thresh");
  if (work_bytes < ssp_mv::work_bytes(groups, views, slots) || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "fuse_views: workspace smaller than ssp_fuse_views_work_bytes or not 8-B aligned");
  if (groups == 0) return SSP_OK;
  const long long rows = (long long)groups * views;
  const long long p3_stride = points3d_shared ? 0 : 3LL * num_points;
  int rc = launch_fuse_rows(points3d, p3_stride, points2d, K3x3_f32, K3x3, dist8_or_null, num_points, views, slots, rows, max_iter, R_out,
                            t_out, corners_out, stream);
  if (rc != SSP_OK) return rc;
  const FuseArgs a = {points3d, p3_stride, points2d, valid, num_points, views, slots, groups,
                      ssp_mv::Rig{K3x3_f32, dist8_or_null, R_rig, t_rig, views}, R_out, t_out};
  double* slots_buf = (double*)work;
  cudaStream_t s = (cudaStream_t)stream;
  const long long nh = (long long)groups * slots * views, ng = (long long)groups * slots;
  fuse_hyp_kernel<<<(unsigned)((nh + 127) / 128), 128, 0, s>>>(a, gate * gate, reproj_thresh * reproj_thresh, max_iter, slots_buf);
  SSP_CHECK_LAUNCH();
  fuse_finish_kernel<<<(unsigned)((ng + 127) / 128), 128, 0, s>>>(a, slots_buf, keypoint_sigma, K3x3, R_world, t_world, world_cov, views_out,
                                                                  view_err, fuse_hyp, fuse_status, corners_world);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
