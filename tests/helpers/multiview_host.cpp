// Host harness of the multi-view fusion (singleshotpose_b200/csrc/multiview_core.h): the three launches of ssp_fuse_views run
// serially over the header's functions.  Built with -ffp-contract=off, as multiview.cu is built with -fmad=false.  Test
// infrastructure: built by the tests into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/multiview_core.h"

using namespace ssp_mv;

extern "C" {
// ssp_fuse_views on host arrays; rows_given != 0 takes R_out, t_out as step 1's poses (the device's, say) instead of solving them
// (corners_out is then not written); -1 for the arguments the entry point refuses
int h_fuse_views(const float* P3, int shared, const float* uv, const unsigned char* valid, int np, int groups, int C, int S, const float* K32,
                 const double* K64, const double* dist, const double* Rr, const double* tr, double gate, double thr, double sigma, int max_iter,
                 int rows_given, double* R_out, double* t_out, float* corners_out, double* R_world, double* t_world, double* cov,
                 unsigned char* views, double* view_err, int* hyp, int* status, float* corners_world) {
  if (C < 1 || C > kMaxViews || np < kMinPoints || np > kMaxPoints || groups < 0 || S < 1 || max_iter < 1 || !(gate > 0.0) ||
      !(thr > 0.0) || !(sigma > 0.0) || gate < thr)
    return -1;
  const long long p3_stride = shared ? 0 : 3LL * np;
  const long long n = (long long)groups * C * S;
  if (!rows_given)
    for (long long id = 0; id < n; id++) {
      const int c = (int)((id / S) % C);
      const double* d = cam_dist(dist, c);
      const float* p3 = P3 + id * p3_stride;
      int work[3];
      ssp_pnp::pnp_solve_one(p3, uv + id * 2 * np, K32 + 9 * c, np, max_iter, R_out + id * 9, t_out + id * 3, work, nullptr, nullptr, nullptr, d);
      double Rw[9], tw[3];
      for (int k = 0; k < 9; k++) Rw[k] = R_out[id * 9 + k];
      for (int k = 0; k < 3; k++) tw[k] = t_out[id * 3 + k];
      for (int v = 0; v < np; v++)
        project(Rw, tw, p3[3 * v], p3[3 * v + 1], p3[3 * v + 2], K64 + 9 * c, d, corners_out + (id * np + v) * 2, corners_out + (id * np + v) * 2 + 1);
    }
  const Rig rig = {K32, dist, Rr, tr, C};
  std::vector<double> slots((size_t)C * kHypDoubles);
  for (long long g = 0; g < groups; g++)
    for (int s = 0; s < S; s++) {
      const long long r0 = (g * C) * S + s, gs = g * S + s;
      const Views v = {P3 + r0 * p3_stride, S * p3_stride, uv + r0 * 2 * np, (long long)S * 2 * np, np};
      const RowPoses rows = {R_out + r0 * 9, (long long)S * 9, t_out + r0 * 3, (long long)S * 3};
      unsigned m = 0;
      for (int c = 0; c < C; c++) m |= (valid[(g * C + c) * S + s] ? 1u : 0u) << c;
      for (int h = 0; h < C; h++) score_hypothesis(rig, v, rows, m, h, gate * gate, thr * thr, max_iter, slots.data() + h * kHypDoubles);
      finish(rig, v, m, slots.data(), sigma, K64, R_world + gs * 9, t_world + gs * 3, cov + gs * 36, views + gs * C, view_err + gs * C,
             hyp + gs, status + gs, corners_world + r0 * 2 * np, (long long)S * 2 * np);
    }
  return 0;
}

// world_jacobian of one point X for camera (K32 [9], dist [8] or null, Rc [9], tc [3]) at the world pose (R, t)
void h_world_jacobian(const float* K32, const double* dist, const double* Rc, const double* tc, const double* R, const double* t,
                      const double* X, double* wu, double* wv) {
  const Rig rig = {K32, dist, Rc, tc, 1};
  const Cam cam = camera(rig, 0);
  double Rw[9], tw[3];
  to_camera(cam, R, t, Rw, tw);
  world_jacobian(cam, Rw, tw, X, wu, wv);
}
}
