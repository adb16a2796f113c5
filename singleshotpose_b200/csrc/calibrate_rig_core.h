// Calibrating a camera rig from the object it sees: the rule of ssp_calibrate_rig (calibrate_rig.cu), shared with the CPU test
// harness (tests/helpers/calibrate_rig_host.cpp, g++ -ffp-contract=off; calibrate_rig.cu is built with -fmad=false) and restated
// with whole arrays in oracle/calibrate_rig_ref.py.  fp64 throughout.  It reuses multiview_core.h (ssp_mv) unchanged.
//
// Inputs.  C cameras (1 <= C <= kMaxViews), camera c with K_c (fp32, as the PnP reads it) and optional distortion dist_c; the
// extrinsics are unknown.  Rows b = g C + c for G captures, S object slots per row, np = 7..10 points per slot, the 3-D points
// shared or given per (row, slot); valid [B][S] flags the views that take part.  Observation o = g S + s (O = G S of them); view
// (o, c) is row (g C + c), slot s.
//   1. Per-view solve.  Every (row, slot) solves its cold PnP with its own camera: ssp_fuse_views' step 1 (multiview_rows.cu).
//   2. Pair hypotheses.  For each camera pair a < b (pair index p in lexicographic order), the co-observations are the o valid in
//      both, in increasing o (n of them).  Hypothesis i < min(n, kMaxPairHyp) comes from co-observation floor(i n / kMaxPairHyp)
//      when n > kMaxPairHyp, else from co-observation i: T_ba = T_b,o T_a,o^-1, R_ba = R_b R_a^T, t_ba = t_b - R_ba t_a (b's
//      frame from a's).  It is scored over every co-observation o': view a's solved pose carried into camera b (R_ba R_a,o',
//      R_ba t_a,o' + t_ba) against b's keypoints, and view b's pose carried into camera a (R_ba^T R_b,o', R_ba^T (t_b,o' - t_ba))
//      against a's, each with ssp_mv::view_mse; o' agrees when both lie in front and both means are <= gate^2.  Its cost is the
//      sum over the agreeing o' of (mse in b + mse in a), in increasing o'.  The pair's winner has the most agreements, then the
//      lower cost by more than the relative margin ssp_mv::kCostTie, then the lower index.
//   3. Initial rig.  Prim's maximum spanning tree from camera `reference`: while an edge joins a camera of the tree to one outside
//      it with agreements >= kMinAgree, the edge with the most agreements joins (ties: the lower pair index).  The reference camera
//      is the world frame (R = I, t = 0 exactly); a child b of a gets R_b = R_ba R_a, t_b = R_ba t_a + t_ba, a child a of b gets
//      R_a = R_ba^T R_b, t_a = R_ba^T (t_b - t_ba).  A camera the tree does not reach is UNCONNECTED, with zero extrinsics, and takes
//      no further part.  The connected cameras other than the reference are the free cameras.
//   4. Per-observation fusion.  ssp_mv::score_hypothesis and ssp_mv::select, unchanged, with the current rig, over the views that
//      are valid and connected: each observation's world pose and fused view set.  An observation whose set has >= 2 cameras is
//      linked; only linked observations enter step 5.
//   5. Bundle adjustment.  LM over the free cameras' extrinsics and the linked observations' world poses (starting from step 4's
//      fused poses), residuals the pixel residuals of each fused view's points (ssp_mv::normal_equations' model).  A camera is
//      perturbed on the left in its own frame, x_c = exp([dth]x) R_c x_w + t_c + dt_ (its Jacobian is ssp_pf::pose_jacobian at the
//      world point with (R_c, t_c)); an observation by ssp_mv's world perturbation (ssp_mv::world_jacobian).  Damping lambda diag
//      on both blocks; lambda from 1e-3, / 10 on an accepted step (lower cost, every point in front of every camera of its set),
//      x 10 on a rejected one or a failed factorisation; at most max_iter steps, stopping at |delta| < 1e-12 (delta the whole step,
//      cameras then observations).  A step by the Schur complement: per linked observation V_o, g_o (obs block) and, per free camera
//      c of its set, U_o,c = J_c^T J_c, g_o,c = J_c^T r, W_o,c = J_c^T J_o; V_o* = V_o + lambda diag V_o inverted by spd_inverse6
//      (a failure is a failed factorisation), Z_o,c = V_o*^-1 W_o,c^T, q_o = V_o*^-1 g_o.  The reduced system over the free cameras
//      in increasing index: S_c1c2 = [c1 == c2] (U_c + lambda diag U_c) - sum_o W_o,c1 Z_o,c2, rhs_c = sum_o (W_o,c q_o - g_o,c);
//      S is factored by Cholesky (the column order of ssp_pnp::chol_solve), dc = S^-1 rhs, then do = -(q_o + sum_c Z_o,c dc_c)
//      (the cameras in increasing index, each camera's 6 terms in order).  Updates: R <- exp([dth]x) R, t <- t + dt_.
//      Order of the sums over observations: every such sum (U, W Z, rhs, the cost, |do|^2, cam_rmse) is taken as 256 partial sums,
//      lane l summing its terms over o = l, l + 256, ... in increasing o (observations that do not contribute are skipped), then the
//      fixed binary tree p[i] += p[i + h] for h = 128, 64, .., 1 (tree_sum).  |delta|^2 = the cameras' sum (increasing camera, then
//      component) + the observations' tree sum.
//   6. Rounds.  Step 4 runs again with the refined rig.  If no observation's (linked ? fused set : none) changed, stop; else run
//      step 5 again; at most kRounds runs of step 5, and step 4 always runs after the last one, so the outputs are the fusion under
//      the final rig.
// Outputs.  Per camera: R, t (camera-from-world), cam_cov = keypoint_sigma^2 times the camera's block of S^-1 at lambda = 0 at the
// last step 5's final state (columns of S^-1 solved one by one; zeros and kSingularCov when a factorisation fails, zeros for the
// reference and the unconnected cameras), cam_obs (linked observations the camera takes part in, by the final fusion), cam_rmse
// (RMS px over those views, -1 without one), tree_parent (-1 for the root and the unconnected), edge_agree (the tree edge's
// agreements, 0 for those), cam_status.  Per observation: R_world, t_world, views, view_err (as ssp_fuse_views defines them), linked.
// Global: rounds (runs of step 5), iterations (LM steps taken over all rounds) and the last step 5's final cost.
// Of the operations here only the libm functions sin and cos (so3_exp) may round differently on the device and the host.
#pragma once
#include <math.h>

#include "multiview_core.h"

namespace ssp_cal {

using ssp_mv::Cam;
using ssp_mv::Rig;
using ssp_mv::Views;

constexpr int kMaxPairHyp = 256, kMinAgree = 3, kRounds = 4, kLanes = 256;
constexpr int kHyp = ssp_mv::kHypDoubles;                     // pair slot: R_ba [9], t_ba [3], cost, agreements
constexpr int kTerm = 114;                                    // per (o, c): U [36], g_c [6], W [36], Z [36]
enum CalibStatus { kUnconnected = 1, kSingularCov = 2 };
// control block (doubles): lambda, cost, done, stop, fail, rounds, iterations, connected mask, singular flag
enum Ctl { kLam, kCost, kDone, kStop, kFail, kRoundsRun, kIters, kConnected, kSingular, kCtl = 16 };

SSP_HD int num_pairs(int C) { return C * (C - 1) / 2; }
SSP_HD void pair_cams(int C, int p, int* a, int* b) {
  int i = 0;
  while (p >= C - 1 - i) { p -= C - 1 - i; i++; }
  *a = i; *b = i + 1 + p;
}
SSP_HD int pair_index(int C, int a, int b) { return a * (2 * C - a - 1) / 2 + (b - a - 1); }

// the workspace, in doubles (ints packed two to a double)
struct Layout {
  long long corners, colist, ncol, pair_slots, fuse_slots, key_new, key_old, obs, cand, terms, q, cost_o, dn_o, front_o, blocks, udiag,
      rhs, dcam, cam_cand, ctl, total;
};
SSP_HD Layout layout(long long G, int C, int S, int np) {
  const long long O = G * S, B = G * C * S, P = num_pairs(C);
  Layout L;
  long long at = 0;
  L.corners = at; at += (B * np * 2 + 1) / 2;
  L.colist = at; at += (P * O + 1) / 2;
  L.ncol = at; at += (P + 1) / 2;
  L.pair_slots = at; at += P * kMaxPairHyp * kHyp;
  L.fuse_slots = at; at += O * C * kHyp;
  L.key_new = at; at += (O + 1) / 2;
  L.key_old = at; at += (O + 1) / 2;
  L.obs = at; at += O * 12;
  L.cand = at; at += O * 12;
  L.terms = at; at += O * C * kTerm;
  L.q = at; at += O * 6;
  L.cost_o = at; at += O;
  L.dn_o = at; at += O;
  L.front_o = at; at += O;
  L.blocks = at; at += (long long)C * C * 36;
  L.udiag = at; at += C * 36;
  L.rhs = at; at += C * 6;
  L.dcam = at; at += C * 6;
  L.cam_cand = at; at += C * 12;
  L.ctl = at; at += kCtl;
  L.total = at;
  return L;
}

// the problem: inputs, the current rig (R_cam, t_cam: outputs updated in place) and the workspace w
struct Problem {
  const float* P3;
  long long p3_stride;          // between (row, slot)s: 0 shared, else 3 np
  const float* uv;
  const unsigned char* valid;   // [rows][S]
  int np, C, S, ref;
  long long G;
  const float* K32;
  const double* dist;
  double gate2, thr2;
  int max_iter;
  const double* R_rows;         // [rows][S][9], [rows][S][3]: step 1's poses
  const double* t_rows;
  double* R_cam;                // [C][9], [C][3]
  double* t_cam;
  double* w;
  Layout L;
};

SSP_HD long long num_obs(const Problem& P) { return P.G * P.S; }
SSP_HD long long view_id(const Problem& P, long long o, int c) { return ((o / P.S) * P.C + c) * P.S + o % P.S; }   // (row, slot)
SSP_HD bool view_valid(const Problem& P, long long o, int c) { return P.valid[view_id(P, o, c)] != 0; }
SSP_HD int* colist(const Problem& P, int p) { return (int*)(P.w + P.L.colist) + (long long)p * num_obs(P); }
SSP_HD int* ncol(const Problem& P) { return (int*)(P.w + P.L.ncol); }
SSP_HD int* key_new(const Problem& P) { return (int*)(P.w + P.L.key_new); }
SSP_HD int* key_old(const Problem& P) { return (int*)(P.w + P.L.key_old); }
SSP_HD double* ctl(const Problem& P) { return P.w + P.L.ctl; }
SSP_HD unsigned connected(const Problem& P) { return (unsigned)ctl(P)[kConnected]; }
SSP_HD unsigned free_cams(const Problem& P) { return connected(P) & ~(1u << P.ref); }
SSP_HD Cam intrinsics(const Problem& P, int c) {
  const float* K = P.K32 + 9 * c;
  return Cam{(double)K[0], (double)K[4], (double)K[2], (double)K[5], ssp_mv::cam_dist(P.dist, c), nullptr, nullptr};
}
SSP_HD Rig rig_of(const Problem& P, const double* R, const double* t) { return Rig{P.K32, P.dist, R, t, P.C}; }
SSP_HD Views views_of(const Problem& P, long long o) {
  const long long r0 = view_id(P, o, 0);
  return Views{P.P3 + r0 * P.p3_stride, P.S * P.p3_stride, P.uv + r0 * 2 * P.np, (long long)P.S * 2 * P.np, P.np};
}

// the fixed reduction tree over kLanes partial sums, in place; returns p[0]
SSP_HD double tree_sum(double* p) {
  for (int h = kLanes / 2; h > 0; h >>= 1)
    for (int i = 0; i < h; i++) p[i] += p[i + h];
  return p[0];
}

// ---------------------------------------------------------------------------------------------------- step 2
// the co-observation list of pair p, in increasing o
SSP_HD void pair_list(const Problem& P, int p) {
  int a, b;
  pair_cams(P.C, p, &a, &b);
  int* list = colist(P, p);
  int n = 0;
  for (long long o = 0; o < num_obs(P); o++)
    if (view_valid(P, o, a) && view_valid(P, o, b)) list[n++] = (int)o;
  ncol(P)[p] = n;
}

SSP_HD int pair_hyps(const Problem& P, int p) { const int n = ncol(P)[p]; return n < kMaxPairHyp ? n : kMaxPairHyp; }

// hypothesis i of pair p, scored: slot = R_ba, t_ba, cost, agreements
SSP_HD void pair_score(const Problem& P, int p, int i) {
  double* slot = P.w + P.L.pair_slots + ((long long)p * kMaxPairHyp + i) * kHyp;
  const int n = ncol(P)[p];
  if (i >= pair_hyps(P, p)) { slot[12] = INFINITY; slot[13] = 0.0; return; }
  int a, b;
  pair_cams(P.C, p, &a, &b);
  const int* list = colist(P, p);
  const long long o = list[n > kMaxPairHyp ? (int)((long long)i * n / kMaxPairHyp) : i];
  const double* Ra = P.R_rows + view_id(P, o, a) * 9;
  const double* ta = P.t_rows + view_id(P, o, a) * 3;
  const double* Rb = P.R_rows + view_id(P, o, b) * 9;
  const double* tb = P.t_rows + view_id(P, o, b) * 3;
  double* R = slot;
  double* t = slot + 9;
  for (int r = 0; r < 3; r++)
    for (int k = 0; k < 3; k++) R[3 * r + k] = Rb[3 * r] * Ra[3 * k] + Rb[3 * r + 1] * Ra[3 * k + 1] + Rb[3 * r + 2] * Ra[3 * k + 2];
  for (int r = 0; r < 3; r++) t[r] = tb[r] - (R[3 * r] * ta[0] + R[3 * r + 1] * ta[1] + R[3 * r + 2] * ta[2]);
  const Cam ca = intrinsics(P, a), cb = intrinsics(P, b);
  int agree = 0;
  double cost = 0.0;
  for (int k = 0; k < n; k++) {
    const long long q = list[k];
    const long long ia = view_id(P, q, a), ib = view_id(P, q, b);
    double Rw[9], tw[3], ma, mb;
    // view a's pose in camera b
    ssp_pf::mat3_mul(R, P.R_rows + ia * 9, Rw);
    const double* tq = P.t_rows + ia * 3;
    for (int r = 0; r < 3; r++) tw[r] = R[3 * r] * tq[0] + R[3 * r + 1] * tq[1] + R[3 * r + 2] * tq[2] + t[r];
    const bool fb = ssp_mv::view_mse(cb, Rw, tw, P.P3 + ib * P.p3_stride, P.uv + ib * 2 * P.np, P.np, &mb);
    // view b's pose in camera a
    const double* Rq = P.R_rows + ib * 9;
    const double* tr = P.t_rows + ib * 3;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) Rw[3 * r + c] = R[r] * Rq[c] + R[3 + r] * Rq[3 + c] + R[6 + r] * Rq[6 + c];
    const double d[3] = {tr[0] - t[0], tr[1] - t[1], tr[2] - t[2]};
    for (int r = 0; r < 3; r++) tw[r] = R[r] * d[0] + R[3 + r] * d[1] + R[6 + r] * d[2];
    const bool fa = ssp_mv::view_mse(ca, Rw, tw, P.P3 + ia * P.p3_stride, P.uv + ia * 2 * P.np, P.np, &ma);
    if (fa && fb && ma <= P.gate2 && mb <= P.gate2) { agree++; cost += mb + ma; }
  }
  slot[12] = cost;
  slot[13] = (double)agree;
}

// the winner of pair p (step 2), -1 without a hypothesis
SSP_HD int pair_winner(const Problem& P, int p) {
  const double* s0 = P.w + P.L.pair_slots + (long long)p * kMaxPairHyp * kHyp;
  int best = -1, best_n = 0;
  double best_cost = 0.0;
  for (int i = 0; i < pair_hyps(P, p); i++) {
    const double* s = s0 + i * kHyp;
    const int n = (int)s[13];
    if (best < 0 || n > best_n || (n == best_n && s[12] < best_cost * (1.0 - ssp_mv::kCostTie))) { best = i; best_n = n; best_cost = s[12]; }
  }
  return best;
}

// ---------------------------------------------------------------------------------------------------- step 3
// the tree and the initial rig into R_cam, t_cam; parent [C], edge_agree [C]; win [num_pairs] the pairs' winners (pair_winner).
// Also starts the control block: the connected mask, no round run yet.
SSP_HD void tree(const Problem& P, const int* win, int* parent, int* edge_agree) {
  const int C = P.C;
  for (int c = 0; c < C; c++) {
    parent[c] = -1;
    edge_agree[c] = 0;
    for (int k = 0; k < 9; k++) P.R_cam[9 * c + k] = 0.0;
    for (int k = 0; k < 3; k++) P.t_cam[3 * c + k] = 0.0;
  }
  for (int k = 0; k < 3; k++) P.R_cam[9 * P.ref + 4 * k] = 1.0;
  unsigned in = 1u << P.ref;
  for (;;) {
    int best = -1, best_n = 0;
    for (int p = 0; p < num_pairs(C); p++) {
      int a, b;
      pair_cams(C, p, &a, &b);
      if (((in >> a) & 1u) == ((in >> b) & 1u) || win[p] < 0) continue;
      const int n = (int)P.w[P.L.pair_slots + ((long long)p * kMaxPairHyp + win[p]) * kHyp + 13];
      if (n >= kMinAgree && n > best_n) { best = p; best_n = n; }
    }
    if (best < 0) break;
    int a, b;
    pair_cams(C, best, &a, &b);
    const double* s = P.w + P.L.pair_slots + ((long long)best * kMaxPairHyp + win[best]) * kHyp;
    const double* Rba = s;
    const double* tba = s + 9;
    if ((in >> a) & 1u) {                                     // b joins below a: R_b = R_ba R_a, t_b = R_ba t_a + t_ba
      const double* Ra = P.R_cam + 9 * a;
      const double* ta = P.t_cam + 3 * a;
      ssp_pf::mat3_mul(Rba, Ra, P.R_cam + 9 * b);
      for (int r = 0; r < 3; r++) P.t_cam[3 * b + r] = Rba[3 * r] * ta[0] + Rba[3 * r + 1] * ta[1] + Rba[3 * r + 2] * ta[2] + tba[r];
      parent[b] = a; edge_agree[b] = best_n; in |= 1u << b;
    } else {                                                  // a joins below b: R_a = R_ba^T R_b, t_a = R_ba^T (t_b - t_ba)
      const double* Rb = P.R_cam + 9 * b;
      const double* tb = P.t_cam + 3 * b;
      double* Ra = P.R_cam + 9 * a;
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) Ra[3 * r + c] = Rba[r] * Rb[c] + Rba[3 + r] * Rb[3 + c] + Rba[6 + r] * Rb[6 + c];
      const double d[3] = {tb[0] - tba[0], tb[1] - tba[1], tb[2] - tba[2]};
      for (int r = 0; r < 3; r++) P.t_cam[3 * a + r] = Rba[r] * d[0] + Rba[3 + r] * d[1] + Rba[6 + r] * d[2];
      parent[a] = b; edge_agree[a] = best_n; in |= 1u << a;
    }
  }
  double* k = ctl(P);
  for (int i = 0; i < kCtl; i++) k[i] = 0.0;
  k[kConnected] = (double)in;
}

// ---------------------------------------------------------------------------------------------------- step 4
SSP_HD unsigned fuse_valid(const Problem& P, long long o) {
  unsigned m = 0;
  for (int c = 0; c < P.C; c++) m |= (view_valid(P, o, c) ? 1u : 0u) << c;
  return m & connected(P);
}

SSP_HD ssp_mv::RowPoses row_poses(const Problem& P, long long o) {
  const long long r0 = view_id(P, o, 0);
  return ssp_mv::RowPoses{P.R_rows + r0 * 9, (long long)P.S * 9, P.t_rows + r0 * 3, (long long)P.S * 3};
}

// hypothesis h of observation o under the current rig
SSP_HD void fuse_hyp(const Problem& P, long long o, int h) {
  ssp_mv::score_hypothesis(rig_of(P, P.R_cam, P.t_cam), views_of(P, o), row_poses(P, o), fuse_valid(P, o), h, P.gate2, P.thr2, P.max_iter,
                           P.w + P.L.fuse_slots + (o * P.C + h) * kHyp);
}

// observation o's fused outputs and its key (the fused set when linked, else 0) in key_new
SSP_HD void fuse_obs(const Problem& P, long long o, double* R, double* t, unsigned char* views, double* view_err, unsigned char* linked) {
  const unsigned valid = fuse_valid(P, o);
  const double* slots = P.w + P.L.fuse_slots + o * P.C * kHyp;
  const int best = valid ? ssp_mv::select(slots, P.C) : -1;
  const unsigned set = best < 0 ? 0u : (unsigned)slots[best * kHyp + 13];
  for (int i = 0; i < 9; i++) R[i] = best < 0 ? 0.0 : slots[best * kHyp + i];
  for (int i = 0; i < 3; i++) t[i] = best < 0 ? 0.0 : slots[best * kHyp + 9 + i];
  const Rig rig = rig_of(P, P.R_cam, P.t_cam);
  const Views v = views_of(P, o);
  for (int c = 0; c < P.C; c++) {
    views[c] = (unsigned char)((set >> c) & 1u);
    view_err[c] = -1.0;
    if (best < 0 || !((valid >> c) & 1u)) continue;
    const Cam cam = ssp_mv::camera(rig, c);
    double Rw[9], tw[3], mse;
    ssp_mv::to_camera(cam, R, t, Rw, tw);
    ssp_mv::view_mse(cam, Rw, tw, v.p3 + c * v.p3_stride, v.uv + c * v.uv_stride, v.np, &mse);
    view_err[c] = sqrt(mse);
  }
  const bool link = ssp_mv::popc(set) >= 2;
  *linked = link ? 1 : 0;
  key_new(P)[o] = link ? (int)set : 0;
}

// ---------------------------------------------------------------------------------------------------- step 5
SSP_HD bool is_linked(const Problem& P, long long o) { return key_new(P)[o] != 0; }
SSP_HD unsigned obs_set(const Problem& P, long long o) { return (unsigned)key_new(P)[o]; }

// observation o's cost at world pose (R, t) under the rig (Rc, tc); false when a point lies behind a camera of its set
SSP_HD bool obs_cost(const Problem& P, long long o, const double* Rc, const double* tc, const double* R, const double* t, double* cost) {
  return ssp_mv::normal_equations(rig_of(P, Rc, tc), views_of(P, o), obs_set(P, o), R, t, cost, nullptr, nullptr);
}

// observation o's terms at the current state with damping lam: q, and per free camera c of its set U, g_c, W, Z; false when V_o*
// cannot be inverted (or a point lies behind a camera)
SSP_HD bool obs_terms(const Problem& P, long long o, double lam) {
  const Rig rig = rig_of(P, P.R_cam, P.t_cam);
  const Views v = views_of(P, o);
  const unsigned set = obs_set(P, o), fr = free_cams(P);
  const double* R = P.w + P.L.obs + o * 12;
  const double* t = R + 9;
  double* T = P.w + P.L.terms + o * P.C * kTerm;
  double V[6][6], go[6];
  for (int a = 0; a < 6; a++) { go[a] = 0.0; for (int b = 0; b < 6; b++) V[a][b] = 0.0; }
  for (int c = 0; c < P.C; c++) {
    if (!((set >> c) & 1u)) continue;
    const bool f = (fr >> c) & 1u;
    double* U = T + c * kTerm;
    double* gc = U + 36;
    double* W = U + 42;
    if (f)
      for (int k = 0; k < 78; k++) U[k] = 0.0;
    const Cam cam = ssp_mv::camera(rig, c);
    double Rw[9], tw[3];
    ssp_mv::to_camera(cam, R, t, Rw, tw);
    const float* p3 = v.p3 + c * v.p3_stride;
    const float* uv = v.uv + c * v.uv_stride;
    for (int i = 0; i < v.np; i++) {
      const double X[3] = {(double)p3[3 * i], (double)p3[3 * i + 1], (double)p3[3 * i + 2]};
      const double x = Rw[0] * X[0] + Rw[1] * X[1] + Rw[2] * X[2] + tw[0];
      const double y = Rw[3] * X[0] + Rw[4] * X[1] + Rw[5] * X[2] + tw[1];
      const double z = Rw[6] * X[0] + Rw[7] * X[1] + Rw[8] * X[2] + tw[2];
      if (!(z > 0.0)) return false;
      const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
      double u, w;
      if (cam.dist) {
        double xd, yd;
        ssp_pnp::distort(cam.dist, xn, yn, &xd, &yd, nullptr);
        u = xd * cam.fx + cam.cx; w = yd * cam.fy + cam.cy;
      } else {
        u = cam.fx * xn + cam.cx; w = cam.fy * yn + cam.cy;
      }
      const double eu = u - (double)uv[2 * i], ev = w - (double)uv[2 * i + 1];
      double ou[6], ov[6];
      ssp_mv::world_jacobian(cam, Rw, tw, X, ou, ov);
      for (int a = 0; a < 6; a++) {
        go[a] += ou[a] * eu + ov[a] * ev;
        for (int b = a; b < 6; b++) V[a][b] += ou[a] * ou[b] + ov[a] * ov[b];
      }
      if (!f) continue;
      const double Xw[3] = {R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0], R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1],
                            R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2]};
      double cu[6], cv[6];
      if (!ssp_pf::pose_jacobian(Xw, cam.R, cam.t, cam.fx, cam.fy, cam.dist, cu, cv)) return false;
      for (int a = 0; a < 6; a++) {
        gc[a] += cu[a] * eu + cv[a] * ev;
        for (int b = a; b < 6; b++) U[6 * a + b] += cu[a] * cu[b] + cv[a] * cv[b];
        for (int b = 0; b < 6; b++) W[6 * a + b] += cu[a] * ou[b] + cv[a] * ov[b];
      }
    }
    if (f)
      for (int a = 0; a < 6; a++)
        for (int b = 0; b < a; b++) U[6 * a + b] = U[6 * b + a];
  }
  double Vs[6][6], Vi[6][6];
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) {
      const double e = a <= b ? V[a][b] : V[b][a];
      Vs[a][b] = a == b ? e + lam * e : e;
    }
  if (!ssp_pf::spd_inverse6(Vs, Vi)) return false;
  double* q = P.w + P.L.q + o * 6;
  for (int a = 0; a < 6; a++) {
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += Vi[a][k] * go[k];
    q[a] = s;
  }
  for (int c = 0; c < P.C; c++) {
    if (!((set >> c) & 1u) || !((fr >> c) & 1u)) continue;
    const double* W = T + c * kTerm + 42;
    double* Z = T + c * kTerm + 78;
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < 6; b++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += Vi[a][k] * W[6 * b + k];
        Z[6 * a + b] = s;
      }
  }
  // g_o is kept for the back-substitution's |do| only through q; U, g_c, W, Z are in T
  return true;
}

// entry e of observation o's contribution to the camera-block pair (c1 <= c2), or false when it contributes nothing.  Entries
// 0..35: (W_o,c1 Z_o,c2)[a][b]; on the diagonal also 36..71: U_o,c [a][b] and 72..77: (W_o,c q_o - g_o,c)[a]
SSP_HD bool block_term(const Problem& P, long long o, int c1, int c2, int e, double* val) {
  if (!is_linked(P, o)) return false;
  const unsigned set = obs_set(P, o);
  if (!((set >> c1) & 1u) || !((set >> c2) & 1u)) return false;
  const double* T = P.w + P.L.terms + o * P.C * kTerm;
  if (e < 36) {
    const double* W = T + c1 * kTerm + 42;
    const double* Z = T + c2 * kTerm + 78;
    const int a = e / 6, b = e % 6;
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += W[6 * a + k] * Z[6 * k + b];
    *val = s;
  } else if (e < 72) {
    *val = T[c1 * kTerm + (e - 36)];
  } else {
    const int a = e - 72;
    const double* W = T + c1 * kTerm + 42;
    const double* q = P.w + P.L.q + o * 6;
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += W[6 * a + k] * q[k];
    *val = s - T[c1 * kTerm + 36 + a];
  }
  return true;
}

SSP_HD int block_entries(int c1, int c2) { return c1 == c2 ? 78 : 36; }

// lane l's partial sum of entry e of block (c1, c2)
SSP_HD double block_partial(const Problem& P, int c1, int c2, int e, int lane) {
  double acc = 0.0, v;
  for (long long o = lane; o < num_obs(P); o += kLanes)
    if (block_term(P, o, c1, c2, e, &v)) acc += v;
  return acc;
}

// where the reduced entry e of block (c1, c2) is stored
SSP_HD double* block_slot(const Problem& P, int c1, int c2, int e) {
  if (e < 36) return P.w + P.L.blocks + ((long long)c1 * P.C + c2) * 36 + e;
  if (e < 72) return P.w + P.L.udiag + c1 * 36 + (e - 36);
  return P.w + P.L.rhs + c1 * 6 + (e - 72);
}

// the free cameras in increasing index: count and their order
SSP_HD int free_list(const Problem& P, int* cams) {
  const unsigned fr = free_cams(P);
  int n = 0;
  for (int c = 0; c < P.C; c++)
    if ((fr >> c) & 1u) cams[n++] = c;
  return n;
}

// the reduced system S [n][n] (n = 6 free cameras, row-major, leading dimension n) and rhs [n] at damping lam
SSP_HD double reduced_entry(const Problem& P, const int* cams, int I, int J, double lam) {
  int i = I / 6, j = J / 6, a = I % 6, b = J % 6;
  if (i > j) { int s = i; i = j; j = s; s = a; a = b; b = s; }
  const int c1 = cams[i], c2 = cams[j];
  const double sw = P.w[P.L.blocks + ((long long)c1 * P.C + c2) * 36 + 6 * a + b];
  if (c1 != c2) return -sw;
  const double* U = P.w + P.L.udiag + c1 * 36;
  double u = U[6 * a + b];
  if (a == b) u += lam * U[6 * a + a];
  return u - sw;
}

// the Cholesky factorisation's two parts, column j of A [n][n] (row-major; the lower triangle is read and written): the pivot
// (false when it is not > 0) and entry i > j.  Column j's entries may be computed in any order once its pivot is.
SSP_HD bool chol_pivot(double* A, int n, int j) {
  double d = A[j * n + j];
  for (int k = 0; k < j; k++) d -= A[j * n + k] * A[j * n + k];
  if (!(d > 0.0)) return false;
  A[j * n + j] = sqrt(d);
  return true;
}
SSP_HD void chol_entry(double* A, int n, int j, int i) {
  double v = A[i * n + j];
  for (int k = 0; k < j; k++) v -= A[i * n + k] * A[j * n + k];
  A[i * n + j] = v / A[j * n + j];
}
// L L^T x = b in place (ssp_pnp::chol_solve's substitutions)
SSP_HD void chol_subst(const double* A, int n, double* b) {
  for (int i = 0; i < n; i++) { double v = b[i]; for (int k = 0; k < i; k++) v -= A[i * n + k] * b[k]; b[i] = v / A[i * n + i]; }
  for (int i = n - 1; i >= 0; i--) { double v = b[i]; for (int k = i + 1; k < n; k++) v -= A[k * n + i] * b[k]; b[i] = v / A[i * n + i]; }
}

// the free cameras' candidate extrinsics from dc [n] into cam_cand (R [C][9], then t [C][3]); the others copy the current rig
SSP_HD void camera_candidates(const Problem& P, const int* cams, int n, const double* dc) {
  double* Rc = P.w + P.L.cam_cand;
  double* tc = Rc + 9 * P.C;
  for (int c = 0; c < P.C; c++) {
    for (int k = 0; k < 9; k++) Rc[9 * c + k] = P.R_cam[9 * c + k];
    for (int k = 0; k < 3; k++) tc[3 * c + k] = P.t_cam[3 * c + k];
  }
  for (int i = 0; i < n / 6; i++) {
    const int c = cams[i];
    double E[9];
    ssp_pf::so3_exp(dc + 6 * i, E);
    ssp_pf::mat3_mul(E, P.R_cam + 9 * c, Rc + 9 * c);
    for (int k = 0; k < 3; k++) tc[3 * c + k] = P.t_cam[3 * c + k] + dc[6 * i + 3 + k];
  }
}

// linked observation o's step from dcam [n] (the free cameras' step, cams their order), its candidate pose, |do|^2, its cost at
// the candidate (under the candidate rig cam_cand) and whether every point lies in front
SSP_HD void obs_step(const Problem& P, long long o, const int* cams, int n) {
  const double* dc = P.w + P.L.dcam;
  const double* Rc = P.w + P.L.cam_cand;
  const double* tc = Rc + 9 * P.C;
  const unsigned set = obs_set(P, o);
  const double* T = P.w + P.L.terms + o * P.C * kTerm;
  const double* q = P.w + P.L.q + o * 6;
  double d[6];
  for (int a = 0; a < 6; a++) {
    double s = q[a];
    for (int i = 0; i < n / 6; i++) {
      const int c = cams[i];
      if (!((set >> c) & 1u)) continue;
      const double* Z = T + c * kTerm + 78;
      for (int b = 0; b < 6; b++) s += Z[6 * a + b] * dc[6 * i + b];
    }
    d[a] = -s;
  }
  double dn = 0.0;
  for (int a = 0; a < 6; a++) dn += d[a] * d[a];
  const double* R = P.w + P.L.obs + o * 12;
  double* Rn = P.w + P.L.cand + o * 12;
  double E[9];
  ssp_pf::so3_exp(d, E);
  ssp_pf::mat3_mul(E, R, Rn);
  for (int k = 0; k < 3; k++) Rn[9 + k] = R[9 + k] + d[3 + k];
  double cost = 0.0;
  const bool front = obs_cost(P, o, Rc, tc, Rn, Rn + 9, &cost);
  P.w[P.L.cost_o + o] = cost;
  P.w[P.L.dn_o + o] = dn;
  P.w[P.L.front_o + o] = front ? 1.0 : 0.0;
}

// lane l's partial sums over the linked observations of the per-observation doubles at `off` (cost_o or dn_o)
SSP_HD double obs_partial(const Problem& P, long long off, int lane) {
  double acc = 0.0;
  for (long long o = lane; o < num_obs(P); o += kLanes)
    if (is_linked(P, o)) acc += P.w[off + o];
  return acc;
}

// the decision of one LM step from the reduced sums: applies the camera candidates (the caller copies the observations' candidates
// when this returns true), updates lambda, the done flag and the iteration count
SSP_HD bool accept(const Problem& P, const int* cams, int n, double cost_new, double dn_obs, bool front) {
  double* k = ctl(P);
  k[kIters] += 1.0;
  if (k[kFail] != 0.0) { k[kLam] *= 10.0; k[kFail] = 0.0; return false; }
  const double* dc = P.w + P.L.dcam;
  double dn = 0.0;
  for (int i = 0; i < n; i++) dn += dc[i] * dc[i];
  dn += dn_obs;
  if (sqrt(dn) < 1e-12) { k[kDone] = 1.0; return false; }
  if (front && cost_new < k[kCost]) {
    const double* Rc = P.w + P.L.cam_cand;
    const double* tc = Rc + 9 * P.C;
    for (int i = 0; i < n / 6; i++) {
      const int c = cams[i];
      for (int j = 0; j < 9; j++) P.R_cam[9 * c + j] = Rc[9 * c + j];
      for (int j = 0; j < 3; j++) P.t_cam[3 * c + j] = tc[3 * c + j];
    }
    k[kCost] = cost_new;
    k[kLam] /= 10.0;
    return true;
  }
  k[kLam] *= 10.0;
  return false;
}

// ---------------------------------------------------------------------------------------------------- step 6
// whether observation o's key differs from the last round's
SSP_HD bool key_changed(const Problem& P, long long o) { return key_new(P)[o] != key_old(P)[o]; }

// a round's start for observation o: its key is kept and, when linked, step 5 starts from the fused pose (R, t); its cost under
// the current rig and whether it lies in front go to cost_o, front_o
SSP_HD void round_obs(const Problem& P, long long o, const double* R, const double* t) {
  key_old(P)[o] = key_new(P)[o];
  if (!is_linked(P, o)) return;
  double* x = P.w + P.L.obs + o * 12;
  for (int k = 0; k < 9; k++) x[k] = R[k];
  for (int k = 0; k < 3; k++) x[9 + k] = t[k];
  double cost = 0.0;
  const bool front = obs_cost(P, o, P.R_cam, P.t_cam, x, x + 9, &cost);
  P.w[P.L.cost_o + o] = cost;
  P.w[P.L.front_o + o] = front ? 1.0 : 0.0;
}

// a round's start from the reduced cost: lambda 1e-3, the initial cost (infinite, and no step, when a point lies behind a camera)
SSP_HD void round_start(const Problem& P, double cost, bool front) {
  double* k = ctl(P);
  k[kLam] = 1e-3;
  k[kCost] = front ? cost : INFINITY;
  k[kDone] = front ? 0.0 : 1.0;
  k[kFail] = 0.0;
  k[kSingular] = 0.0;
  k[kRoundsRun] += 1.0;
}

}  // namespace ssp_cal
