// Host harness of the depth calibration of a rig (singleshotpose_b200/csrc/calibrate_rig_depth_core.h): the work of
// calibrate_rig_depth.cu's kernels runs serially over the header's functions -- per active view 256 virtual threads and the halving
// tree, per observation the solve, per camera-block pair the 256 lane partials and tree_sum, then the factorisation and the
// updates.  Built with -ffp-contract=off, as the kernels are built with -fmad=false.  Test infrastructure: built by the tests into
// a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/calibrate_rig_depth_core.h"

using namespace ssp_cd;

extern "C" {
// ssp_calibrate_rig_depth on host arrays; -1 for the arguments the entry point refuses
int h_calibrate_rig_depth(const unsigned short* depth, int W, int H, double depth_scale, int C, const double* K, const double* dist,
                          int reference, const int* status_in, const double* R_cam_in, const double* t_cam_in, const double* model, int nv,
                          double diam, int groups, int slots, const unsigned char* views, const unsigned char* linked,
                          const double* R_in, const double* t_in, int iters, double s, double e, double* R_cam, double* t_cam,
                          double* cam_cov, int* cam_points, double* cam_rmse, int* cam_status, double* R_out, double* t_out,
                          int* obs_points, double* obs_rmse, int* obs_status, int* status, double* iter_rmse) {
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || C < 2 || C > kMaxViews || reference < 0 || reference >= C || nv < 1 || !(diam > 0.0) ||
      groups < 0 || slots < 1 || iters < 1 || iters > ssp_rd::kMaxIters || !(s > 0.0) || !(e > 0.0) || e > s || !(depth_scale > 0.0))
    return -1;
  const long long O = (long long)groups * slots;
  const Layout L = layout(O, C);
  std::vector<double> w(L.total, 0.0), g(iters);
  for (int k = 0; k < iters; k++) g[k] = ssp_rd::gate_factor(s, e, k, iters);
  const Problem P = {depth, ssp_rr::Rig{K, dist, w.data() + L.cam, w.data() + L.cam + 9 * C, C, W, H, depth_scale}, model, nv, diam, views,
                     linked, status_in, reference, slots, O, w.data(), L};
  init_cams(P, R_cam_in, t_cam_in);
  for (long long o = 0; o < O; o++) {
    init_obs(P, o, R_in, t_in);
    obs_points[o] = 0; obs_rmse[o] = 0.0; obs_status[o] = 0;
  }
  for (int k = 0; k < 36 * C; k++) cam_cov[k] = 0.0;
  for (int c = 0; c < C; c++) { cam_points[c] = 0; cam_rmse[c] = 0.0; cam_status[c] = cam_status_bits(P, c); }
  for (int k = 0; k < iters; k++) iter_rmse[k] = 0.0;
  std::vector<double> a((size_t)kThreads * kAcc), A(90 * 90), X(90 * 90), lanes(kLanes);
  for (int k = 0; k < iters && ctl(P)[kStop] == 0.0; k++) {
    const double tau = diam * g[k];
    // step 1
    for (long long o = 0; o < O; o++)
      for (int c = 0; c < C; c++) {
        if (!active(P, o, c)) continue;
        double (*t)[kAcc] = (double (*)[kAcc])a.data();
        for (int j = 0; j < kThreads; j++) view_thread(P, o, c, tau, j, t[j], 1);
        for (int h = kThreads / 2; h >= 1; h /= 2)
          for (int j = 0; j < h; j++)
            for (int i = 0; i < kAcc; i++) t[j][i] += t[j + h][i];
        for (int i = 0; i < kAcc; i++) acc_of(P, o, c)[i] = t[0][i];
      }
    // step 2
    for (long long o = 0; o < O; o++) {
      if (!linked[o] || stopped(P, o)) continue;
      obs_status[o] = obs_solve(P, o, &obs_points[o], &obs_rmse[o]);
    }
    // step 3: the block sums, the reduced system, its factorisation
    for (int c1 = 0; c1 < C; c1++)
      for (int c2 = c1; c2 < C; c2++)
        for (int e2 = block_first(P, c1); e2 < block_entries(P, c1, c2); e2++) {
          for (int l = 0; l < kLanes; l++) lanes[l] = block_partial(P, c1, c2, e2, l);
          *block_slot(P, c1, c2, e2) = ssp_cal::tree_sum(lanes.data());
        }
    int cams[kMaxViews];
    unsigned held;
    const int n = 6 * solve_list(P, cams, &held);
    ctl(P)[kHeld] = (double)held;
    iter_rmse[k] = overall_rmse(P);
    for (int I = 0; I < n * n; I++) A[I] = reduced_entry(P, cams, I / n, I % n);
    bool ok = true;
    for (int j = 0; j < n && ok; j++) {
      ok = ssp_cal::chol_pivot(A.data(), n, j);
      for (int i = j + 1; ok && i < n; i++) ssp_cal::chol_entry(A.data(), n, j, i);
    }
    for (int c = 0; c < C; c++) {
      const double cn = connected(P, c) ? cam_n(P, c) : 0.0;
      cam_points[c] = (int)cn;
      cam_rmse[c] = cn > 0.0 ? sqrt(cam_r2(P, c) / cn) : 0.0;
    }
    if (!ok) {
      ctl(P)[kStop] = 1.0;
      for (int c = 0; c < C; c++) cam_status[c] = cam_status_bits(P, c);
      break;
    }
    double dc[90];
    for (int I = 0; I < n; I++) dc[I] = rhs_entry(P, cams, I);
    ssp_cal::chol_subst(A.data(), n, dc);
    if (k == iters - 1) {
      const double s2 = iter_rmse[k] * iter_rmse[k];
      for (int j = 0; j < n; j++) {
        double* x = X.data() + j * n;
        for (int i = 0; i < n; i++) x[i] = i == j ? 1.0 : 0.0;
        ssp_cal::chol_subst(A.data(), n, x);
        const int c = cams[j / 6], b = j % 6;
        for (int r = 0; r < 6; r++) cam_cov[c * 36 + 6 * r + b] = s2 * x[(j / 6) * 6 + r];
      }
    }
    // step 4
    unsigned solved = 0;
    for (int i = 0; i < n / 6; i++) solved |= 1u << cams[i];
    ctl(P)[kSolved] = (double)solved;
    camera_update(P, cams, n / 6, dc);
    for (long long o = 0; o < O; o++) obs_update(P, o, solved);
    for (int c = 0; c < C; c++) cam_status[c] = cam_status_bits(P, c);
  }
  const bool stop = ctl(P)[kStop] != 0.0;
  for (int c = 0; c < C; c++) {
    for (int k = 0; k < 9; k++) R_cam[9 * c + k] = stop ? R_cam_in[9 * c + k] : P.rig.R[9 * c + k];
    for (int k = 0; k < 3; k++) t_cam[3 * c + k] = stop ? t_cam_in[3 * c + k] : P.rig.t[3 * c + k];
  }
  for (long long o = 0; o < O; o++) {
    const bool keep = stop || !linked[o] || stopped(P, o);
    for (int k = 0; k < 9; k++) R_out[o * 9 + k] = keep ? R_in[o * 9 + k] : obs_pose(P, o)[k];
    for (int k = 0; k < 3; k++) t_out[o * 3 + k] = keep ? t_in[o * 3 + k] : obs_pose(P, o)[9 + k];
  }
  *status = stop ? kCamSingular : 0;
  return 0;
}

// the pair of model point x6 in camera c at the world pose (R, t) and gate tau: 1 and r, the observation's terms Jo [6], the
// camera's terms Jc [6] and q_c [3] (the scene point in camera c's frame) when it makes one, else 0
int h_pair_terms(const double* x6, const double* R, const double* t, const unsigned short* depth, int W, int H, double depth_scale, int C,
                 const double* K, const double* dist, const double* Rr, const double* tr, int c, double tau, double* r, double* Jo, double* Jc,
                 double* qc) {
  const ssp_rr::Rig rig = {K, dist, Rr, tr, C, W, H, depth_scale};
  const ssp_mv::Cam ext = ssp_rr::extrinsics(rig, c);
  double Rp[9], tp[3], a[3], m[3], p[3];
  ssp_mv::to_camera(ext, R, t, Rp, tp);
  if (!ssp_rd::find_pair(x6, Rp, tp, ssp_rr::depth_camera(rig, c), depth, tau, a, m, p, qc)) return 0;
  return pair_terms(x6, R, t, Rp, tp, ext, ssp_rr::depth_camera(rig, c), depth, tau, true, r, Jo, Jc) ? 1 : 0;
}
}
