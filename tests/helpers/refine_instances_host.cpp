// Host harness of the refinement of a rig's world instances (singleshotpose_b200/csrc/refine_instances_core.h): the work of
// refine_instances.cu runs serially over the header's functions -- per iteration every drawn slot's faces into the owner buffers,
// then per problem and camera 256 virtual threads and the halving tree, the cameras' sums in camera order, the solve and update.
// Built with -ffp-contract=off, as the kernels are built with -fmad=false.  Test infrastructure: built by the tests into a
// temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/refine_instances_core.h"

using namespace ssp_ri;

namespace {

struct Problem {
  bool out, known;
  int cls, fs;
};

// every drawn slot of capture g at the poses P [slots][12] into the owner buffers O [C][H][W]
void draw_capture(const ssp_rr::Rig& rig, const double* model, const int* offsets, const int* faces, const int* face_offsets,
                  const std::vector<Problem>& pr, const double* R_in, const double* t_in, const double* P, long long g, int slots,
                  unsigned long long* O) {
  const long long frame = (long long)rig.H * rig.W;
  for (long long i = 0; i < (long long)rig.C * frame; i++) O[i] = kNobody;
  for (int w = 0; w < slots; w++) {
    const long long id = g * slots + w;
    const Problem& p = pr[id];
    if (p.out || !p.known || !drawn(false, R_in + id * 9, t_in + id * 3, p.fs)) continue;
    for (int c = 0; c < rig.C; c++) {
      const ssp_mv::Cam ext = ssp_rr::extrinsics(rig, c);
      double Rc[9], tc[3];
      ssp_mv::to_camera(ext, P + id * 12, P + id * 12 + 9, Rc, tc);
      unsigned long long* Oc = O + c * frame;
      for (int f = face_offsets[p.cls]; f < face_offsets[p.cls + 1]; f++)
        draw_model_face(model + (long long)offsets[p.cls] * 6, faces + (long long)f * 3, Rc, tc, rig.K + 9 * c, ext.dist, rig.W, rig.H,
                        [&](long long px, double z) {
                          const unsigned long long k = owner_key(z, w);
                          if (k < Oc[px]) Oc[px] = k;
                        });
    }
  }
}

}  // namespace

extern "C" {
// ssp_refine_instances_rig on host arrays; -1 for the arguments the entry point refuses
int h_refine_instances_rig(const unsigned short* depth, int W, int H, double depth_scale, int C, const double* K, const double* dist,
                           const double* Rr, const double* tr, const double* model, const int* offsets, const double* diam, const int* faces,
                           const int* face_offsets, const float* table, int np, int num_classes, const int* cls, int groups, int slots,
                           const int* count, const int* fuse_status, const double* R_in, const double* t_in, int iters, double s, double e,
                           double* R_out, double* t_out, int* points_out, double* rmse_out, int* status_out, int* view_points,
                           double* view_rmse, int* view_hidden, float* corners, short* instance_map) {
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || C < 1 || C > ssp_rr::kMaxViews || np < ssp_mv::kMinPoints || np > ssp_mv::kMaxPoints ||
      num_classes < 1 || groups < 0 || slots < 1 || slots > 256 || iters < 1 || iters > ssp_rd::kMaxIters || !(s > 0.0) || !(e > 0.0) ||
      e > s || !(depth_scale > 0.0))
    return -1;
  const ssp_rr::Rig rig = {K, dist, Rr, tr, C, W, H, depth_scale};
  const long long n = (long long)groups * slots, frame = (long long)H * W;
  std::vector<Problem> pr(n);
  std::vector<double> P(n * 12), acc((size_t)C * ssp_rd::kThreads * kAcc);
  std::vector<unsigned long long> O(C * frame);
  for (long long id = 0; id < n; id++) {
    Problem& p = pr[id];
    p.out = count && (int)(id % slots) >= count[id / slots];
    p.cls = cls[id];
    p.known = p.cls >= 0 && p.cls < num_classes;
    p.fs = fuse_status ? fuse_status[id] : 0;
    for (int k = 0; k < 12; k++) P[id * 12 + k] = p.out ? 0.0 : (k < 9 ? R_in[id * 9 + k] : t_in[id * 3 + k - 9]);
    status_out[id] = p.out ? 0 : ssp_rr::input_status(R_in + id * 9, t_in + id * 3, p.fs);
    points_out[id] = 0;
    rmse_out[id] = 0.0;
    for (int c = 0; c < C; c++) { view_points[id * C + c] = 0; view_rmse[id * C + c] = 0.0; view_hidden[id * C + c] = 0; }
  }
  for (int k = 0; k < iters; k++) {
    const double gk = ssp_rd::gate_factor(s, e, k, iters);
    for (long long g = 0; g < groups; g++) {
      draw_capture(rig, model, offsets, faces, face_offsets, pr, R_in, t_in, P.data(), g, slots, O.data());
      for (int w = 0; w < slots; w++) {
        const long long id = g * slots + w;
        const Problem& p = pr[id];
        if (p.out || status_out[id] != 0) continue;
        const int begin = p.known ? offsets[p.cls] : 0, end = p.known ? offsets[p.cls + 1] : 0;
        const double tau = (p.known ? diam[p.cls] : 0.0) * gk;
        double R[9], t[3];
        for (int i = 0; i < 9; i++) R[i] = P[id * 12 + i];
        for (int i = 0; i < 3; i++) t[i] = P[id * 12 + 9 + i];
        for (int c = 0; c < C; c++) {
          const ssp_mv::Cam ext = ssp_rr::extrinsics(rig, c);
          const ssp_rd::Camera cam = ssp_rr::depth_camera(rig, c);
          double Rc[9], tc[3];
          ssp_mv::to_camera(ext, R, t, Rc, tc);
          const unsigned short* D = depth + (g * C + c) * frame;
          double (*a)[kAcc] = (double (*)[kAcc])(acc.data() + (size_t)c * ssp_rd::kThreads * kAcc);
          for (int j = 0; j < ssp_rd::kThreads; j++) {
            for (int i = 0; i < kAcc; i++) a[j][i] = 0.0;
            for (int i = begin + j; i < end; i += ssp_rd::kThreads)
              accumulate_point(model + (long long)i * 6, R, t, Rc, tc, ext, cam, D, O.data() + c * frame, w, tau, a[j]);
          }
          for (int st = ssp_rd::kThreads / 2; st >= 1; st /= 2)            // ssp_rd::tree_reduce over kAcc doubles
            for (int i = 0; i < st; i++)
              for (int q = 0; q < kAcc; q++) a[i][q] += a[i + st][q];
          ssp_rr::view_stats(a[0], &view_points[id * C + c], &view_rmse[id * C + c]);
          view_hidden[id * C + c] = (int)a[0][kOffHidden];
        }
        double sum[ssp_rr::kAcc];
        ssp_rr::sum_views([&](int c) { return (const double*)(acc.data() + (size_t)c * ssp_rd::kThreads * kAcc); }, C, sum);
        const int st = ssp_rd::solve_update(sum, R, t, &points_out[id], &rmse_out[id]);
        status_out[id] = st;
        for (int i = 0; i < 9; i++) P[id * 12 + i] = st ? R_in[id * 9 + i] : R[i];
        for (int i = 0; i < 3; i++) P[id * 12 + 9 + i] = st ? t_in[id * 3 + i] : t[i];
      }
    }
  }
  for (long long g = 0; g < groups; g++) {
    draw_capture(rig, model, offsets, faces, face_offsets, pr, R_in, t_in, P.data(), g, slots, O.data());
    for (long long i = 0; i < C * frame; i++) instance_map[g * C * frame + i] = map_entry(O[i]);
  }
  for (long long id = 0; id < n; id++) {
    const Problem& p = pr[id];
    const long long g = id / slots;
    const int m = (int)(id % slots);
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = P[id * 12 + k];
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = P[id * 12 + 9 + k];
    const bool none = p.out || !p.known || (p.fs & (ssp_mv::kNoValid | ssp_mv::kNoView));
    const float* X = table + (p.known ? p.cls : 0) * 3LL * np;
    float* crn = corners + (g * C * slots + m) * 2LL * np;
    for (int c = 0; c < C; c++) ssp_rr::project_view(rig, c, R_out + id * 9, t_out + id * 3, X, np, none, crn + c * (long long)slots * 2 * np);
  }
  return 0;
}

// the pair of model point x6 of slot w in camera c under the world pose (R, t) at gate tau against the owner buffer O [H][W]:
// 0 no pair, 1 a kept pair with r, J [6] and its scene point q_w [3], 2 a pair dropped for ownership
int h_owned_pair(const double* x6, const double* R, const double* t, const unsigned short* depth, const unsigned long long* O, int w, int W,
                 int H, double depth_scale, int C, const double* K, const double* dist, const double* Rr, const double* tr, int c, double tau,
                 double* r, double* J, double* qw) {
  const ssp_rr::Rig rig = {K, dist, Rr, tr, C, W, H, depth_scale};
  const ssp_mv::Cam ext = ssp_rr::extrinsics(rig, c);
  double Rc[9], tc[3], acc[kAcc] = {0.0};
  ssp_mv::to_camera(ext, R, t, Rc, tc);
  accumulate_point(x6, R, t, Rc, tc, ext, ssp_rr::depth_camera(rig, c), depth, O, w, tau, acc);
  if (acc[kOffHidden] > 0.0) return 2;
  if (acc[ssp_rd::kOffN] == 0.0) return 0;
  ssp_rr::world_pair(x6, R, t, Rc, tc, ext, ssp_rr::depth_camera(rig, c), depth, tau, r, J, qw);
  return 1;
}
}
