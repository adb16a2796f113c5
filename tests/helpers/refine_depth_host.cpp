// Host harness of the depth refinement (singleshotpose_b200/csrc/refine_depth_core.h): the loops of refine_depth.cu's kernel run
// serially over the header's functions -- 256 virtual threads per iteration, the halving tree, the solve and update.  Built with
// -ffp-contract=off, as the kernel is built with -fmad=false.  Test infrastructure: built by the tests into a temporary .so; never
// loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/refine_depth_core.h"

using namespace ssp_rd;

extern "C" {
// ssp_refine_depth on host arrays (K [9] fp64, dist [8] or null); -1 for the arguments the entry point refuses
int h_refine_depth(const unsigned short* depth, int W, int H, double depth_scale, const double* K, const double* dist, const double* model,
                   const int* offsets, const double* diam, int num_classes, const int* cls, int groups, int per_group, const int* count,
                   const double* R_in, const double* t_in, int iters, double s, double e, double* R_out, double* t_out, int* points_out,
                   double* rmse_out, int* status_out) {
  if (W < 1 || H < 1 || iters < 1 || iters > kMaxIters || !(s > 0.0) || !(e > 0.0) || e > s || !(depth_scale > 0.0)) return -1;
  const Camera cam = {K[0], K[4], K[2], K[5], dist, W, H, depth_scale};
  std::vector<double> g(iters);
  for (int k = 0; k < iters; k++) g[k] = gate_factor(s, e, k, iters);
  static double acc[kThreads][kAccDoubles];
  for (long long id = 0; id < (long long)groups * per_group; id++) {
    const int grp = (int)(id / per_group), m = (int)(id % per_group);
    if (count && m >= count[grp]) {
      for (int k = 0; k < 9; k++) R_out[id * 9 + k] = 0.0;
      for (int k = 0; k < 3; k++) t_out[id * 3 + k] = 0.0;
      points_out[id] = 0; rmse_out[id] = 0.0; status_out[id] = 0;
      continue;
    }
    double R[9], t[3];
    for (int k = 0; k < 9; k++) R[k] = R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) t[k] = t_in[id * 3 + k];
    const int c = cls[id];
    const bool known = c >= 0 && c < num_classes;
    const int begin = known ? offsets[c] : 0, end = known ? offsets[c + 1] : 0;
    const double d = known ? diam[c] : 0.0;
    int status = pose_ok(R, t) ? 0 : kBadPose, points = 0;
    double rmse = 0.0;
    const unsigned short* D = depth + (long long)grp * H * W;
    for (int k = 0; k < iters && status == 0; k++) {
      const double tau = d * g[k];
      for (int j = 0; j < kThreads; j++) {
        for (int i = 0; i < kAccDoubles; i++) acc[j][i] = 0.0;
        for (int i = begin + j; i < end; i += kThreads) accumulate_point(model + (long long)i * 6, R, t, cam, D, tau, acc[j]);
      }
      tree_reduce(acc);
      status = solve_update(acc[0], R, t, &points, &rmse);
    }
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = status ? R_in[id * 9 + k] : R[k];
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = status ? t_in[id * 3 + k] : t[k];
    points_out[id] = points; rmse_out[id] = rmse; status_out[id] = status;
  }
  return 0;
}

// the pair of one model point x6 under (R, t) at gate tau: 1 and r, J [6], q [3] when it makes one, else 0
int h_point_pair(const double* x6, const double* R, const double* t, const unsigned short* depth, int W, int H, double depth_scale,
                 const double* K, const double* dist, double tau, double* r, double* J, double* q) {
  const Camera cam = {K[0], K[4], K[2], K[5], dist, W, H, depth_scale};
  double a[3], m[3], p[3];
  if (!find_pair(x6, R, t, cam, depth, tau, a, m, p, q)) return 0;
  *r = point_terms(a, m, p, q, J);
  return 1;
}
}
