// Fusing every detected instance across the cameras of a rig: the rule of ssp_fuse_instances (multiview_instances.cu), shared
// with the CPU test harness (tests/helpers/multiview_instances_host.cpp, g++ -ffp-contract=off; multiview_instances.cu is built
// with -fmad=false) and restated with whole arrays in oracle/fuse_instances_ref.py.  fp64 throughout.  It generalises
// multiview_core.h's view consensus from "which views agree" to "which detection in each view agrees", and reuses that header's
// view_mse, agree, lm, normal_equations, to_world / to_camera, kCostTie and spd_inverse6 unchanged.
//
// Per capture g (rows b = g C + c, each with M detection slots): detection d = (view c, slot m) exists when m < count[b] and its
// class k_d = cls[b][m] is in [0, num_classes); its index is i(d) = c M + m, its points the class table's, its keypoints the
// row's, its pose the per-row solve of step 1 (multiview_core.h step 1).  Every detection starts in the available set U.
//   assign(R, t, k, thr, U): in each view, the available detection of class k with every point in front of the camera and the
//     lowest view_mse under the world pose (R, t) (ties: the lower slot); the view joins when that mse is <= thr^2.  With at most
//     one detection of class k per view this is agree().
//   Scoring hypothesis h in U (the stages of multiview_core.h's score_hypothesis, the chosen detections as each view's keypoints):
//     1. h's pose in the world frame; A = assign(., gate).
//     2. Fit A: one view takes its chosen detection's own world pose, more views run the LM.
//     3. A' = assign(fit, reproj_thresh); if A' differs from A in its views or in a chosen detection and A' is not empty, fit A'
//        from the first fit.
//     4. Check, the chosen detections held fixed: while a member lies beyond reproj_thresh it leaves and the rest is refitted.
//     5. The cost is the summed squared residual of the final set.
//   Greedy extraction: each class's candidate is multiview_core.h's select() over the available hypotheses of that class in
//   index order (most views, then a cost lower by the relative margin kCostTie, then the lower index); the winner is select()'s
//   rule again over the class candidates in index order.  Its final pose is emitted as a world instance with world_cov =
//   sigma^2 (J^T J)^-1 over its members (finish's arithmetic), its members leave U, and the extraction repeats until no
//   hypothesis keeps a view or M instances are out; the detections left in U are `unfused`.  The margin is not transitive, so
//   the scan order is part of the rule; scanning per class first makes each class's candidate exactly select() over that class,
//   whatever the other classes hold, so with at most one detection per class per view a class's first world instance is
//   ssp_fuse_views' fused pose for that class, bit for bit (another class's emission never touches this class's hypotheses).
//   Reuse of scores: a hypothesis is rescored only when a removed detection was the argmin of one of its two assign calls in its
//   view; otherwise every argmin, hence every stage, is unchanged.  The result equals rescoring everything, bit for bit.
// Why greedy rather than a global assignment: the objective of a global assignment (views per instance against residuals) has
// no natural weighting, and an exact one is combinatorial in C and M; the greedy rule takes the best-supported instance first,
// and every instance it emits is one that multiview_core.h's rule would fuse from those detections alone.  The worst case: two
// same-class instances on nearly one viewing ray of one camera project to nearly the same keypoints there, so that camera's
// detections can be swapped between them; the other views decide which instance gets the views they agree with, and a swap
// costs that camera's pixel error only, not a wrong view in the fit of an instance the other views pin down.
#pragma once
#include "multiview_core.h"

namespace ssp_mvi {

using ssp_mv::Cam;
using ssp_mv::kMaxPoints;
using ssp_mv::kMaxViews;
using ssp_mv::Rig;
using ssp_mv::Views;

// per hypothesis in the workspace: R [9], t [3], cost, view set (as a double), then sel, dep0, dep1 [kMaxViews] int each
constexpr int kHypDoubles = 14 + 3 * kMaxViews / 2;
// per capture in the workspace: the hypotheses, their keypoint scratch ([C][kMaxPoints][2] float each, the final set's chosen
// detections), and the bytes avail, stale, candidate [C M] (rounded up to 8 B)
SSP_HD long long capture_bytes(int C, int M) {
  const long long H = (long long)C * M;
  return H * kHypDoubles * 8 + H * C * kMaxPoints * 2 * 4 + ((3 * H + 7) / 8) * 8;
}
// the workspace: the gathered points [groups C][M][kMaxPoints][3] float, then each capture's block
SSP_HD long long points_bytes(long long groups, int C, int M) { return ((groups * C * M * kMaxPoints * 3 * 4 + 7) / 8) * 8; }
SSP_HD long long work_bytes(long long groups, int C, int M) { return points_bytes(groups, C, M) + groups * capture_bytes(C, M); }

// the detections of one capture: C rows of M slots
struct Dets {
  const float* table;     // [num_classes][np][3] the class points
  int num_classes;
  const int* cls;         // [C][M]
  const int* count;       // [C]
  const float* uv;        // [C][M][np][2]
  const double* R_rows;   // [C][M][9], [C][M][3]: step 1's poses
  const double* t_rows;
  int M, np;
};

SSP_HD bool exists(const Dets& d, int i) {
  const int c = i / d.M, m = i % d.M;
  return m < d.count[c] && d.cls[i] >= 0 && d.cls[i] < d.num_classes;
}

// one hypothesis's record in the workspace
struct Hyp {
  double* R;    // [9], t [3], cost, set: the slot's doubles
  int* sel;     // [kMaxViews] the final set's chosen slot per view (-1 for none)
  int* dep;     // [2][kMaxViews] the argmin slots of the two assign calls per view (-1 for none)
  float* uv;    // [C][kMaxPoints][2] the chosen detections' keypoints
};

SSP_HD Hyp hyp_at(double* slots, float* uvs, int h, int C) {
  double* s = slots + (long long)h * kHypDoubles;
  int* ints = (int*)(s + 14);
  return Hyp{s, ints, ints + kMaxViews, uvs + (long long)h * C * kMaxPoints * 2};
}

// the views of hypothesis record H's chosen detections of class k: view c's keypoints at H.uv + c * 2 np
SSP_HD Views chosen_views(const Dets& d, const Hyp& H, int k) {
  return Views{d.table + (long long)k * d.np * 3, 0, H.uv, 2LL * d.np, d.np};
}

SSP_HD void gather(const Dets& d, const Hyp& H, unsigned set, const int* sel, int C) {
  for (int c = 0; c < C; c++) {
    if (!((set >> c) & 1u)) continue;
    const float* src = d.uv + ((long long)c * d.M + sel[c]) * 2 * d.np;
    for (int j = 0; j < 2 * d.np; j++) H.uv[c * 2 * d.np + j] = src[j];
  }
}

// assign(R, t, k, thr2, U): the joined views; sel[c] the chosen slot of a joined view (else -1), arg[c] the argmin (or -1)
SSP_HD unsigned assign(const Rig& rig, const Dets& d, const unsigned char* avail, const double R[9], const double t[3], int k, double thr2,
                       int* sel, int* arg) {
  unsigned set = 0;
  const float* p3 = d.table + (long long)k * d.np * 3;
  for (int c = 0; c < rig.C; c++) {
    const Cam cam = ssp_mv::camera(rig, c);
    double Rw[9], tw[3];
    ssp_mv::to_camera(cam, R, t, Rw, tw);
    int best = -1;
    double best_mse = 0.0;
    for (int m = 0; m < d.M; m++) {
      const int i = c * d.M + m;
      if (!avail[i] || d.cls[i] != k) continue;
      double mse;
      if (ssp_mv::view_mse(cam, Rw, tw, p3, d.uv + (long long)i * 2 * d.np, d.np, &mse) && (best < 0 || mse < best_mse)) {
        best = m;
        best_mse = mse;
      }
    }
    arg[c] = best;
    sel[c] = -1;
    if (best >= 0 && best_mse <= thr2) { set |= 1u << c; sel[c] = best; }
  }
  return set;
}

// a fit of `set` (the chosen detections in H.uv) from (R, t), in place: one view's chosen detection's own world pose, or the LM
SSP_HD void fit(const Rig& rig, const Dets& d, const Hyp& H, int k, unsigned set, const int* sel, double R[9], double t[3], int max_iter) {
  if (ssp_mv::popc(set) == 1) {
    int w = 0;
    while (!((set >> w) & 1u)) w++;
    const long long i = (long long)w * d.M + sel[w];
    ssp_mv::to_world(ssp_mv::camera(rig, w), d.R_rows + i * 9, d.t_rows + i * 3, R, t);
    return;
  }
  ssp_mv::lm(rig, chosen_views(d, H, k), set, R, t, max_iter);
}

// the scoring of hypothesis h (available) into its record; returns the final set
SSP_HD unsigned score(const Rig& rig, const Dets& d, const unsigned char* avail, int h, double gate2, double thr2, int max_iter, const Hyp& H) {
  const int C = rig.C, k = d.cls[h];
  double* R = H.R;
  double* t = H.R + 9;
  int s1[kMaxViews], s2[kMaxViews];
  for (int c = 0; c < kMaxViews; c++) { H.sel[c] = -1; H.dep[c] = -1; H.dep[kMaxViews + c] = -1; }
  ssp_mv::to_world(ssp_mv::camera(rig, h / d.M), d.R_rows + (long long)h * 9, d.t_rows + (long long)h * 3, R, t);
  unsigned set = 0;
  double cost = INFINITY;
  const unsigned A = assign(rig, d, avail, R, t, k, gate2, s1, H.dep);
  if (A) {
    gather(d, H, A, s1, C);
    fit(rig, d, H, k, A, s1, R, t, max_iter);
    unsigned A2 = assign(rig, d, avail, R, t, k, thr2, s2, H.dep + kMaxViews);
    bool differs = A2 != A;
    for (int c = 0; c < C; c++) differs = differs || (((A2 >> c) & 1u) && s2[c] != s1[c]);
    if (differs && A2) {
      gather(d, H, A2, s2, C);
      fit(rig, d, H, k, A2, s2, R, t, max_iter);
    }
    const Views v = chosen_views(d, H, k);
    for (int it = 0; it < C && A2; it++) {                          // the check: the members beyond reproj_thresh go
      const unsigned A3 = ssp_mv::agree(rig, v, A2, R, t, thr2);
      if (A3 == A2) break;
      A2 = A3;
      if (A2) fit(rig, d, H, k, A2, s2, R, t, max_iter);
    }
    set = A2;
    for (int c = 0; c < C; c++) H.sel[c] = ((set >> c) & 1u) ? s2[c] : -1;
    if (set && !ssp_mv::normal_equations(rig, v, set, R, t, &cost, nullptr, nullptr)) cost = INFINITY;
  }
  H.R[12] = cost;
  H.R[13] = (double)set;
  return set;
}

// select()'s step over one more hypothesis record s: true when it beats the best so far (best_n, best_cost)
SSP_HD bool beats(const double* s, int best_n, double best_cost) {
  const int n = ssp_mv::popc((unsigned)s[13]);
  return n > best_n || (n == best_n && n > 0 && s[12] < best_cost * (1.0 - ssp_mv::kCostTie));
}

// class k's candidate: select() over the available hypotheses of class k in index order; -1 when none keeps a view
SSP_HD int class_candidate(const Dets& d, const unsigned char* avail, const double* slots, int H, int k) {
  int best = -1, best_n = 0;
  double best_cost = 0.0;
  for (int h = 0; h < H; h++) {
    if (!avail[h] || d.cls[h] != k) continue;
    const double* s = slots + (long long)h * kHypDoubles;
    if (beats(s, best_n, best_cost)) { best = h; best_n = ssp_mv::popc((unsigned)s[13]); best_cost = s[12]; }
  }
  return best;
}

// the winner: select() over the class candidates (cand[h] != 0) in index order; -1 for none
SSP_HD int pick(const unsigned char* cand, const double* slots, int H) {
  int best = -1, best_n = 0;
  double best_cost = 0.0;
  for (int h = 0; h < H; h++) {
    if (!cand[h]) continue;
    const double* s = slots + (long long)h * kHypDoubles;
    if (beats(s, best_n, best_cost)) { best = h; best_n = ssp_mv::popc((unsigned)s[13]); best_cost = s[12]; }
  }
  return best;
}

// the world instance of the winning record H (class k): R [9], t [3], cov [36] (finish's arithmetic over the members), members
// [C] (the chosen slot, -1 for other views), view_err [C] (RMS px of the members, -1 for the others), *status (kSingular or 0)
SSP_HD void emit(const Rig& rig, const Dets& d, const Hyp& H, int k, double sigma, double* R, double* t, double* cov, int* members,
                 double* view_err, int* status) {
  const unsigned set = (unsigned)H.R[13];
  for (int i = 0; i < 9; i++) R[i] = H.R[i];
  for (int i = 0; i < 3; i++) t[i] = H.R[9 + i];
  const Views v = chosen_views(d, H, k);
  double A[6][6], Ai[6][6], g[6], cost;
  const bool usable = ssp_mv::normal_equations(rig, v, set, R, t, &cost, A, g) && ssp_pf::spd_inverse6(A, Ai);
  const double s2 = sigma * sigma;
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) cov[6 * a + b] = usable ? s2 * Ai[a][b] : 0.0;
  *status = usable ? 0 : ssp_mv::kSingular;
  for (int c = 0; c < rig.C; c++) {
    const bool in = (set >> c) & 1u;
    members[c] = in ? H.sel[c] : -1;
    view_err[c] = -1.0;
    if (!in) continue;
    const Cam cam = ssp_mv::camera(rig, c);
    double Rw[9], tw[3], mse;
    ssp_mv::to_camera(cam, R, t, Rw, tw);
    ssp_mv::view_mse(cam, Rw, tw, v.p3, v.uv + c * v.uv_stride, v.np, &mse);
    view_err[c] = sqrt(mse);
  }
}

// whether record H must be rescored after the detections (c, sel[c]), c in `removed`, left U: one was an argmin of its assigns
SSP_HD bool touched(const Hyp& H, unsigned removed, const int* sel, int C) {
  for (int c = 0; c < C; c++)
    if (((removed >> c) & 1u) && (H.dep[c] == sel[c] || H.dep[kMaxViews + c] == sel[c])) return true;
  return false;
}

}  // namespace ssp_mvi
