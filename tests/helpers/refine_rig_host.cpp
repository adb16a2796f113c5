// Host harness of the rig refinement (singleshotpose_b200/csrc/refine_rig_core.h): the work of refine_rig.cu's cluster runs serially
// over the header's functions -- per camera 256 virtual threads and the halving tree, the cameras' sums in camera order, the
// solve and update.  Built with -ffp-contract=off, as the kernel is built with -fmad=false.  Test infrastructure: built by the
// tests into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/refine_rig_core.h"

using namespace ssp_rr;

extern "C" {
// ssp_refine_depth_rig on host arrays; -1 for the arguments the entry point refuses
int h_refine_depth_rig(const unsigned short* depth, int W, int H, double depth_scale, int C, const double* K, const double* dist,
                       const double* Rr, const double* tr, const double* model, const int* offsets, const double* diam,
                       const float* table, int np, int num_classes, const int* cls, int groups, int slots, const int* count,
                       const int* fuse_status, const double* R_in, const double* t_in, int iters, double s, double e, double* R_out,
                       double* t_out, int* points_out, double* rmse_out, int* status_out, int* view_points, double* view_rmse,
                       float* corners) {
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || C < 1 || C > kMaxViews || np < ssp_mv::kMinPoints || np > ssp_mv::kMaxPoints ||
      num_classes < 1 || groups < 0 || slots < 1 || iters < 1 || iters > ssp_rd::kMaxIters || !(s > 0.0) || !(e > 0.0) || e > s ||
      !(depth_scale > 0.0))
    return -1;
  const Rig rig = {K, dist, Rr, tr, C, W, H, depth_scale};
  std::vector<double> g(iters), acc((size_t)C * ssp_rd::kThreads * kAcc);
  for (int k = 0; k < iters; k++) g[k] = ssp_rd::gate_factor(s, e, k, iters);
  for (long long id = 0; id < (long long)groups * slots; id++) {
    const long long grp = id / slots;
    const int m = (int)(id % slots);
    const int c_ = cls[id];
    const bool known = c_ >= 0 && c_ < num_classes;
    const int fs = fuse_status ? fuse_status[id] : 0;
    float* crn = corners + (grp * C * slots + m) * 2LL * np;              // (row g C, slot m)
    const long long cstride = (long long)slots * 2 * np;
    if (count && m >= count[grp]) {
      for (int k = 0; k < 9; k++) R_out[id * 9 + k] = 0.0;
      for (int k = 0; k < 3; k++) t_out[id * 3 + k] = 0.0;
      points_out[id] = 0; rmse_out[id] = 0.0; status_out[id] = 0;
      for (int c = 0; c < C; c++) {
        view_points[id * C + c] = 0; view_rmse[id * C + c] = 0.0;
        for (int i = 0; i < 2 * np; i++) crn[c * cstride + i] = 0.f;
      }
      continue;
    }
    double R[9], t[3];
    for (int k = 0; k < 9; k++) R[k] = R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) t[k] = t_in[id * 3 + k];
    const int begin = known ? offsets[c_] : 0, end = known ? offsets[c_ + 1] : 0;
    const double d = known ? diam[c_] : 0.0;
    int status = input_status(R, t, fs), points = 0;
    double rmse = 0.0;
    std::vector<int> vp(C, 0);
    std::vector<double> vr(C, 0.0);
    for (int k = 0; k < iters && status == 0; k++) {
      const double tau = d * g[k];
      for (int c = 0; c < C; c++) {
        const ssp_mv::Cam ext = extrinsics(rig, c);
        const ssp_rd::Camera cam = depth_camera(rig, c);
        double Rc[9], tc[3];
        ssp_mv::to_camera(ext, R, t, Rc, tc);
        const unsigned short* D = depth + (grp * C + c) * (long long)H * W;
        double (*a)[kAcc] = (double (*)[kAcc])(acc.data() + (size_t)c * ssp_rd::kThreads * kAcc);
        for (int j = 0; j < ssp_rd::kThreads; j++) {
          for (int i = 0; i < kAcc; i++) a[j][i] = 0.0;
          for (int i = begin + j; i < end; i += ssp_rd::kThreads) accumulate_point(model + (long long)i * 6, R, t, Rc, tc, ext, cam, D, tau, a[j]);
        }
        ssp_rd::tree_reduce(a);
        view_stats(a[0], &vp[c], &vr[c]);
      }
      double sum[kAcc];
      sum_views([&](int c) { return (const double*)(acc.data() + (size_t)c * ssp_rd::kThreads * kAcc); }, C, sum);
      status = ssp_rd::solve_update(sum, R, t, &points, &rmse);
    }
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = status ? R_in[id * 9 + k] : R[k];
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = status ? t_in[id * 3 + k] : t[k];
    points_out[id] = points; rmse_out[id] = rmse; status_out[id] = status;
    for (int c = 0; c < C; c++) { view_points[id * C + c] = vp[c]; view_rmse[id * C + c] = vr[c]; }
    const bool none = !known || (fs & (ssp_mv::kNoValid | ssp_mv::kNoView));
    const float* X = table + (known ? c_ : 0) * 3LL * np;
    for (int c = 0; c < C; c++) project_view(rig, c, R_out + id * 9, t_out + id * 3, X, np, none, crn + c * cstride);
  }
  return 0;
}

// the world-axis pair of model point x6 in camera c of the rig under the world pose (R, t) at gate tau: 1 and r, J [6], q_w [3]
// when it makes one, else 0
int h_world_pair(const double* x6, const double* R, const double* t, const unsigned short* depth, int W, int H, double depth_scale,
                 int C, const double* K, const double* dist, const double* Rr, const double* tr, int c, double tau, double* r, double* J,
                 double* qw) {
  const Rig rig = {K, dist, Rr, tr, C, W, H, depth_scale};
  const ssp_mv::Cam ext = extrinsics(rig, c);
  double Rc[9], tc[3];
  ssp_mv::to_camera(ext, R, t, Rc, tc);
  return world_pair(x6, R, t, Rc, tc, ext, depth_camera(rig, c), depth, tau, r, J, qw) ? 1 : 0;
}
}
