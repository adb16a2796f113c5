// Host harness of the instance fusion (singleshotpose_b200/csrc/multiview_instances_core.h): the launches of ssp_fuse_instances run
// serially over the header's functions.  Built with -ffp-contract=off, as multiview_instances.cu is built with -fmad=false.  Test
// infrastructure: built by the tests into a temporary .so; never loaded by the product.
#include <cstring>
#include <vector>

#include "../../singleshotpose_b200/csrc/multiview_instances_core.h"

using namespace ssp_mvi;

extern "C" {
// ssp_fuse_instances on host arrays; rows_given != 0 takes R_out, t_out as step 1's poses (the device's, say) instead of solving
// them (corners_out is then not written); rescore_all != 0 rescores every available hypothesis in every round instead of only the
// touched ones; -1 for the arguments the entry point refuses
int h_fuse_instances(const float* table, int num_classes, const float* uv, const int* cls, const int* count, int np, int groups, int C, int M,
                     const float* K32, const double* K64, const double* dist, const double* Rr, const double* tr, double gate, double thr,
                     double sigma, int max_iter, int rows_given, int rescore_all, double* R_out, double* t_out, float* corners_out,
                     int* world_count, int* unfused, int* world_cls, double* R_world, double* t_world, double* cov, int* members,
                     double* view_err, int* fuse_hyp, int* fuse_status, int* world_index, float* corners_world) {
  if (C < 1 || C > kMaxViews || np < ssp_mv::kMinPoints || np > kMaxPoints || groups < 0 || M < 1 || M > 256 || num_classes < 1 ||
      max_iter < 1 || !(gate > 0.0) || !(thr > 0.0) || !(sigma > 0.0) || gate < thr)
    return -1;
  const long long rows = (long long)groups * C, n = rows * M;
  for (long long id = 0; id < n; id++) {
    const long long b = id / M;
    const int c = (int)(b % C), m = (int)(id % M);
    if (m >= count[b]) {
      for (int j = 0; j < 9; j++) R_out[id * 9 + j] = 0.0;
      for (int j = 0; j < 3; j++) t_out[id * 3 + j] = 0.0;
      for (int j = 0; j < 2 * np; j++) corners_out[id * 2 * np + j] = 0.f;
      continue;
    }
    if (rows_given) continue;
    const int k = cls[id] < 0 ? 0 : (cls[id] >= num_classes ? num_classes - 1 : cls[id]);
    const float* p3 = table + (long long)k * np * 3;
    const double* d = ssp_mv::cam_dist(dist, c);
    int work[3];
    ssp_pnp::pnp_solve_one(p3, uv + id * 2 * np, K32 + 9 * c, np, max_iter, R_out + id * 9, t_out + id * 3, work, nullptr, nullptr, nullptr, d);
    double Rw[9], tw[3];
    for (int j = 0; j < 9; j++) Rw[j] = R_out[id * 9 + j];
    for (int j = 0; j < 3; j++) tw[j] = t_out[id * 3 + j];
    for (int v = 0; v < np; v++)
      ssp_mv::project(Rw, tw, p3[3 * v], p3[3 * v + 1], p3[3 * v + 2], K64 + 9 * c, d, corners_out + (id * np + v) * 2,
                      corners_out + (id * np + v) * 2 + 1);
  }
  const Rig rig = {K32, dist, Rr, tr, C};
  const int H = C * M;
  std::vector<double> slots((size_t)H * kHypDoubles);
  std::vector<float> uvs((size_t)H * C * kMaxPoints * 2);
  std::vector<unsigned char> avail(H), stale(H), cand(H);
  for (long long g = 0; g < groups; g++) {
    const long long b0 = g * C;
    const Dets d = {table, num_classes, cls + b0 * M, count + b0, uv + b0 * M * 2 * np, R_out + b0 * M * 9, t_out + b0 * M * 3, M, np};
    for (int i = 0; i < H; i++) {
      avail[i] = stale[i] = exists(d, i);
      world_index[b0 * M + i] = -1;
    }
    for (int w = 0; w < M; w++) {
      const long long gw = g * M + w;
      world_cls[gw] = -1;
      fuse_hyp[gw] = -1;
      fuse_status[gw] = 0;
      for (int j = 0; j < 9; j++) R_world[gw * 9 + j] = 0.0;
      for (int j = 0; j < 3; j++) t_world[gw * 3 + j] = 0.0;
      for (int j = 0; j < 36; j++) cov[gw * 36 + j] = 0.0;
      for (int c = 0; c < C; c++) { members[gw * C + c] = -1; view_err[gw * C + c] = -1.0; }
    }
    int nw = 0;
    for (; nw < M; nw++) {
      for (int h = 0; h < H; h++) {
        cand[h] = 0;
        if (avail[h] && (stale[h] || rescore_all)) score(rig, d, avail.data(), h, gate * gate, thr * thr, max_iter, hyp_at(slots.data(), uvs.data(), h, C));
        stale[h] = 0;
      }
      for (int k = 0; k < num_classes; k++) {
        const int w = class_candidate(d, avail.data(), slots.data(), H, k);
        if (w >= 0) cand[w] = 1;
      }
      const int win = pick(cand.data(), slots.data(), H);
      if (win < 0) break;
      const long long gw = g * M + nw;
      const Hyp W = hyp_at(slots.data(), uvs.data(), win, C);
      emit(rig, d, W, d.cls[win], sigma, R_world + gw * 9, t_world + gw * 3, cov + gw * 36, members + gw * C, view_err + gw * C, fuse_status + gw);
      world_cls[gw] = d.cls[win];
      fuse_hyp[gw] = win;
      for (int c = 0; c < C; c++)
        if (W.sel[c] >= 0) {
          avail[c * M + W.sel[c]] = 0;
          world_index[b0 * M + c * M + W.sel[c]] = nw;
        }
      for (int h = 0; h < H; h++)
        if (avail[h] && touched(hyp_at(slots.data(), uvs.data(), h, C), (unsigned)W.R[13], W.sel, C)) stale[h] = 1;
    }
    int left = 0;
    for (int i = 0; i < H; i++) left += avail[i];
    world_count[g] = nw;
    unfused[g] = left;
    for (int c = 0; c < C; c++)
      for (int w = 0; w < M; w++)
        for (int p = 0; p < np; p++) {
          float* out = corners_world + ((b0 + c) * M + w) * 2 * np + 2 * p;
          if (w >= nw) { out[0] = 0.f; out[1] = 0.f; continue; }
          const long long gw = g * M + w;
          const ssp_mv::Cam cam = ssp_mv::camera(rig, c);
          double Rw[9], tw[3];
          ssp_mv::to_camera(cam, R_world + gw * 9, t_world + gw * 3, Rw, tw);
          const float* X = table + ((long long)world_cls[gw] * np + p) * 3;
          ssp_mv::project(Rw, tw, X[0], X[1], X[2], K64 + 9 * c, cam.dist, out, out + 1);
        }
  }
  return 0;
}
// the reuse criterion of one capture, pair by pair: for every detection h and every other detection e, h's record scored with
// all detections available and with e removed.  Returns the pairs whose record changed although touched() says h needs no
// rescoring (0 when the criterion is exact); *changed counts the pairs whose record changed, *refit_only those among them where e
// was the argmin of the refit's assign only (not of the first assign) in its view
int h_reuse_check(const float* table, int num_classes, const float* uv, const int* cls, const int* count, int np, int C, int M,
                  const float* K32, const double* dist, const double* Rr, const double* tr, const double* R_rows, const double* t_rows,
                  double gate, double thr, int max_iter, int* changed, int* refit_only) {
  const Rig rig = {K32, dist, Rr, tr, C};
  const Dets d = {table, num_classes, cls, count, uv, R_rows, t_rows, M, np};
  const int H = C * M;
  std::vector<double> slots(2 * kHypDoubles);
  std::vector<float> uvs(2 * C * kMaxPoints * 2);
  std::vector<unsigned char> avail(H);
  int bad = 0;
  *changed = *refit_only = 0;
  for (int h = 0; h < H; h++) {
    if (!exists(d, h)) continue;
    for (int i = 0; i < H; i++) avail[i] = exists(d, i);
    const Hyp A = hyp_at(slots.data(), uvs.data(), 0, C), B = hyp_at(slots.data(), uvs.data(), 1, C);
    score(rig, d, avail.data(), h, gate * gate, thr * thr, max_iter, A);
    for (int e = 0; e < H; e++) {
      if (e == h || !exists(d, e)) continue;
      avail[e] = 0;
      score(rig, d, avail.data(), h, gate * gate, thr * thr, max_iter, B);
      avail[e] = 1;
      // a record that keeps no view never wins, whatever its pose: the set and cost decide, and the pose and choices when kept
      const bool differ = std::memcmp(A.R + 12, B.R + 12, 2 * sizeof(double)) != 0 ||
                          (A.R[13] != 0.0 && (std::memcmp(A.R, B.R, 12 * sizeof(double)) != 0 || std::memcmp(A.sel, B.sel, C * sizeof(int)) != 0));
      const int c = e / M;
      int sel[kMaxViews];
      for (int k = 0; k < kMaxViews; k++) sel[k] = -1;
      sel[c] = e % M;
      if (!differ) continue;
      (*changed)++;
      if (A.dep[c] != sel[c] && A.dep[kMaxViews + c] == sel[c]) (*refit_only)++;
      if (!touched(A, 1u << c, sel, C)) bad++;
    }
  }
  return bad;
}
}
