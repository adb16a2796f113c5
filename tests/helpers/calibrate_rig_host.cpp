// Host harness of the rig calibration (singleshotpose_b200/csrc/calibrate_rig_core.h): the launches of ssp_calibrate_rig run
// serially over the header's functions, each CTA's lanes and fixed-order trees as loops.  Built with -ffp-contract=off, as
// calibrate_rig.cu is built with -fmad=false.  Test infrastructure: built by the tests into a temporary .so; never loaded by the
// product.
#include <vector>

#include "../../singleshotpose_b200/csrc/calibrate_rig_core.h"

using namespace ssp_cal;

namespace {

// kLanes partials of f(lane), reduced by the fixed tree
template <class F>
double lane_sum(F f) {
  double p[kLanes];
  for (int l = 0; l < kLanes; l++) p[l] = f(l);
  return tree_sum(p);
}

// factor_reduced on the host: false when a pivot fails
bool factor(const Problem& P, const int* cams, int n, double lam, std::vector<double>& A) {
  A.assign((size_t)n * n, 0.0);
  for (int e = 0; e < n * n; e++) A[e] = reduced_entry(P, cams, e / n, e % n, lam);
  for (int j = 0; j < n; j++) {
    if (!chol_pivot(A.data(), n, j)) return false;
    for (int i = j + 1; i < n; i++) chol_entry(A.data(), n, j, i);
  }
  return true;
}

void blocks(const Problem& P) {
  const unsigned fr = free_cams(P);
  for (int c1 = 0; c1 < P.C; c1++)
    for (int c2 = c1; c2 < P.C; c2++) {
      if (!((fr >> c1) & 1u) || !((fr >> c2) & 1u)) continue;
      for (int e = 0; e < block_entries(c1, c2); e++) *block_slot(P, c1, c2, e) = lane_sum([&](int l) { return block_partial(P, c1, c2, e, l); });
    }
}

}  // namespace

extern "C" {
// ssp_calibrate_rig on host arrays; rows_given != 0 takes R_rows, t_rows as step 1's poses (the device's, say) instead of solving
// them; tree_only != 0 stops after step 3 (R_cam, t_cam, tree_parent and edge_agree are written); -1 for the arguments the entry
// point refuses
int h_calibrate_rig(const float* P3, int shared, const float* uv, const unsigned char* valid, int np, int groups, int C, int S, const float* K32,
                    const double* dist, int reference, double gate, double thr, double sigma, int max_iter, int rows_given, double* R_rows,
                    double* t_rows, double* R_cam, double* t_cam, double* cam_cov, int* cam_obs, double* cam_rmse, int* tree_parent,
                    int* edge_agree, int* cam_status, double* R_world, double* t_world, unsigned char* views, double* view_err,
                    unsigned char* linked, int* rounds, int* iterations, double* cost, int tree_only) {
  if (C < 1 || C > ssp_mv::kMaxViews || np < ssp_mv::kMinPoints || np > ssp_mv::kMaxPoints || groups < 0 || S < 1 || max_iter < 1 ||
      !(gate > 0.0) || !(thr > 0.0) || !(sigma > 0.0) || gate < thr || reference < 0 || reference >= C)
    return -1;
  const long long p3_stride = shared ? 0 : 3LL * np;
  const long long n_rows = (long long)groups * C * S;
  if (!rows_given)
    for (long long id = 0; id < n_rows; id++) {
      const int c = (int)((id / S) % C);
      int work[3];
      ssp_pnp::pnp_solve_one(P3 + id * p3_stride, uv + id * 2 * np, K32 + 9 * c, np, max_iter, R_rows + id * 9, t_rows + id * 3, work, nullptr,
                             nullptr, nullptr, ssp_mv::cam_dist(dist, c));
    }
  const Layout L = layout(groups, C, S, np);
  std::vector<double> w((size_t)L.total, 0.0);
  const Problem P = {P3, p3_stride, uv, valid, np, C, S, reference, (long long)groups, K32, dist, gate * gate, thr * thr, max_iter,
                     R_rows, t_rows, R_cam, t_cam, w.data(), L};
  const long long O = num_obs(P);
  const int npairs = num_pairs(C);
  for (int p = 0; p < npairs; p++) pair_list(P, p);
  for (int p = 0; p < npairs; p++)
    for (int i = 0; i < kMaxPairHyp; i++) pair_score(P, p, i);
  std::vector<int> win(npairs + 1);
  for (int p = 0; p < npairs; p++) win[p] = pair_winner(P, p);
  tree(P, win.data(), tree_parent, edge_agree);
  if (tree_only) return 0;
  double* k = ctl(P);
  std::vector<double> A, X;
  for (int r = 0; r <= kRounds; r++) {
    if (k[kStop] != 0.0) break;
    for (long long o = 0; o < O; o++)
      for (int h = 0; h < C; h++) fuse_hyp(P, o, h);
    for (long long o = 0; o < O; o++) fuse_obs(P, o, R_world + o * 9, t_world + o * 3, views + o * C, view_err + o * C, linked + o);
    bool changed = k[kRoundsRun] == 0.0;
    for (long long o = 0; o < O; o++) changed = changed || key_changed(P, o);
    if (!changed || r == kRounds) { k[kStop] = 1.0; break; }
    bool front = true;
    for (long long o = 0; o < O; o++) {
      round_obs(P, o, R_world + o * 9, t_world + o * 3);
      if (is_linked(P, o) && w[L.front_o + o] == 0.0) front = false;
    }
    round_start(P, lane_sum([&](int l) { return obs_partial(P, L.cost_o, l); }), front);
    int cams[ssp_mv::kMaxViews];
    const int n = 6 * free_list(P, cams);
    for (int it = 0; it < max_iter; it++) {
      if (k[kDone] != 0.0) break;
      for (long long o = 0; o < O; o++)
        if (is_linked(P, o) && !obs_terms(P, o, k[kLam])) k[kFail] = 1.0;
      if (k[kFail] == 0.0) {
        blocks(P);
        if (!factor(P, cams, n, k[kLam], A)) k[kFail] = 1.0;
        else {
          double* dc = w.data() + L.dcam;
          for (int i = 0; i < n; i++) dc[i] = w[L.rhs + cams[i / 6] * 6 + i % 6];
          chol_subst(A.data(), n, dc);
          camera_candidates(P, cams, n, dc);
          for (long long o = 0; o < O; o++)
            if (is_linked(P, o)) obs_step(P, o, cams, n);
        }
      }
      bool fr = true;
      for (long long o = 0; o < O; o++)
        if (is_linked(P, o) && w[L.front_o + o] == 0.0) fr = false;
      const double c_new = lane_sum([&](int l) { return obs_partial(P, L.cost_o, l); });
      const double dn = lane_sum([&](int l) { return obs_partial(P, L.dn_o, l); });
      if (accept(P, cams, n, c_new, dn, fr))
        for (long long o = 0; o < O; o++)
          if (is_linked(P, o))
            for (int j = 0; j < 12; j++) w[L.obs + o * 12 + j] = w[L.cand + o * 12 + j];
    }
    // the covariance
    for (int e = 0; e < C * 36; e++) cam_cov[e] = 0.0;
    for (long long o = 0; o < O; o++)
      if (is_linked(P, o) && !obs_terms(P, o, 0.0)) k[kSingular] = 1.0;
    if (k[kSingular] != 0.0) continue;
    blocks(P);
    if (!factor(P, cams, n, 0.0, A)) { k[kSingular] = 1.0; continue; }
    X.assign((size_t)n, 0.0);
    for (int j = 0; j < n; j++) {
      for (int i = 0; i < n; i++) X[i] = i == j ? 1.0 : 0.0;
      chol_subst(A.data(), n, X.data());
      const int c = cams[j / 6], b = j % 6;
      for (int a = 0; a < 6; a++) cam_cov[c * 36 + 6 * a + b] = sigma * sigma * X[(j / 6) * 6 + a];
    }
  }
  const unsigned conn = connected(P), fr = free_cams(P);
  for (int c = 0; c < C; c++) {
    const double cnt = lane_sum([&](int l) {
      double a = 0.0;
      for (long long o = l; o < O; o += kLanes)
        if (is_linked(P, o) && views[o * C + c]) a += 1.0;
      return a;
    });
    const double s = lane_sum([&](int l) {
      double a = 0.0;
      for (long long o = l; o < O; o += kLanes)
        if (is_linked(P, o) && views[o * C + c]) a += view_err[o * C + c] * view_err[o * C + c];
      return a;
    });
    cam_obs[c] = (int)cnt;
    cam_rmse[c] = cnt > 0.0 ? sqrt(s / cnt) : -1.0;
    cam_status[c] = (((conn >> c) & 1u) ? 0 : kUnconnected) | (((fr >> c) & 1u) && k[kSingular] != 0.0 ? kSingularCov : 0);
  }
  *rounds = (int)k[kRoundsRun];
  *iterations = (int)k[kIters];
  *cost = k[kCost];
  return 0;
}

// the camera block's Jacobian rows of point X (object frame) of an observation at world pose (R, t) seen by camera (K32, dist, Rc,
// tc): cu, cv [6], d(u, v)/d(dth, dt_) of the camera's left perturbation
void h_camera_jacobian(const float* K32, const double* dist, const double* Rc, const double* tc, const double* R, const double* t,
                       const double* X, double* cu, double* cv) {
  const double Xw[3] = {R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0], R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1],
                        R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2]};
  ssp_pf::pose_jacobian(Xw, Rc, tc, (double)K32[0], (double)K32[4], dist, cu, cv);
}
}
