// Fusing every detected instance across the cameras of a rig (rule: multiview_instances_core.h).  ssp_fuse_instances runs three
// stages:
//   gather_points_kernel   one thread per point of a (row, slot): the slot's class's points from the class table, into the
//                          workspace (an unknown class reads class 0's or the last class's; such a slot is solved but joins nothing);
//   launch_fuse_rows_counted (multiview_rows.cu) the per-row PnP and projection of ssp_fuse_views' step 1, for the slots m < count;
//   fuse_instances_kernel  one CTA per capture: empty slots' rows zeroed, then rounds of scoring (threads over the C M
//                          hypotheses, only those whose argmins a removal touched), per-class candidates (threads over the
//                          classes), the winner (one thread, select()'s ordered scan), its emission, separated by barriers; then
//                          every world instance drawn in every camera of the capture.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off, so the fusion equals the harness bit for bit when
// it starts from the same per-row poses.
#include <math.h>

#include "ssp_common.cuh"
#include "multiview_instances_core.h"

namespace ssp {

int launch_fuse_rows_counted(const float* P3, long long p3_stride, const float* uv, const float* K32, const double* K64, const double* dist,
                             const int* count, int np, int C, int S, long long rows, int max_iter, double* R, double* t, float* corners,
                             void* stream);

__global__ void __launch_bounds__(256) gather_points_kernel(const float* __restrict__ table, int num_classes, const int* __restrict__ cls,
                                                            int np, long long n, float* __restrict__ P3) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (row, slot, coordinate)
  if (id >= n * np * 3) return;
  const long long rs = id / (np * 3);
  const int k = min(max(cls[rs], 0), num_classes - 1);
  P3[id] = table[(long long)k * np * 3 + id % (np * 3)];
}

struct InstArgs {
  const float* table;
  int num_classes;
  const int* cls;               // [rows][M]
  const int* count;             // [rows]
  const float* uv;              // [rows][M][np][2]
  int np, C, M;
  ssp_mv::Rig rig;
  const double* K64;
  double gate2, thr2, sigma;
  int max_iter;
  double* R_rows;               // [rows][M][9], [rows][M][3], [rows][M][np][2]: step 1's outputs
  double* t_rows;
  float* corners;
  int* world_count;             // [groups]
  int* unfused;
  int* world_cls;               // [groups][M]
  double* R_world;              // [groups][M][9]
  double* t_world;
  double* world_cov;
  int* members;                 // [groups][M][C]
  double* view_err;
  int* fuse_hyp;                // [groups][M]
  int* fuse_status;
  int* world_index;             // [rows][M]
  float* corners_world;         // [rows][M][np][2]
  char* work;                   // the captures' blocks
};

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) fuse_instances_kernel(const InstArgs a) {
  const int g = blockIdx.x, tid = threadIdx.x, C = a.C, M = a.M, np = a.np, H = C * M;
  const long long b0 = (long long)g * C;                        // the capture's first row
  const ssp_mvi::Dets d = {a.table, a.num_classes, a.cls + b0 * M, a.count + b0, a.uv + b0 * M * 2 * np, a.R_rows + b0 * M * 9,
                           a.t_rows + b0 * M * 3, M, np};
  char* blk = a.work + g * ssp_mvi::capture_bytes(C, M);
  double* slots = (double*)blk;
  float* uvs = (float*)(slots + (long long)H * ssp_mvi::kHypDoubles);
  unsigned char* avail = (unsigned char*)(uvs + (long long)H * C * ssp_mv::kMaxPoints * 2);
  unsigned char* stale = avail + H;
  unsigned char* cand = stale + H;
  for (int i = tid; i < H; i += kThreads) {
    const bool e = ssp_mvi::exists(d, i);
    avail[i] = e;
    stale[i] = e;
    a.world_index[b0 * M + i] = -1;
    if (i % M < d.count[i / M]) continue;
    const long long r = b0 * M + i;                              // an empty slot: zero pose and corners
    for (int j = 0; j < 9; j++) a.R_rows[r * 9 + j] = 0.0;
    for (int j = 0; j < 3; j++) a.t_rows[r * 3 + j] = 0.0;
    for (int j = 0; j < 2 * np; j++) a.corners[r * 2 * np + j] = 0.f;
  }
  for (int w = tid; w < M; w += kThreads) {
    const long long gw = (long long)g * M + w;
    a.world_cls[gw] = -1;
    a.fuse_hyp[gw] = -1;
    a.fuse_status[gw] = 0;
    for (int j = 0; j < 9; j++) a.R_world[gw * 9 + j] = 0.0;
    for (int j = 0; j < 3; j++) a.t_world[gw * 3 + j] = 0.0;
    for (int j = 0; j < 36; j++) a.world_cov[gw * 36 + j] = 0.0;
    for (int c = 0; c < C; c++) { a.members[gw * C + c] = -1; a.view_err[gw * C + c] = -1.0; }
  }
  __shared__ int s_win;
  __syncthreads();
  int nw = 0;
  for (; nw < M; nw++) {
    for (int h = tid; h < H; h += kThreads) {
      cand[h] = 0;
      if (!avail[h] || !stale[h]) continue;
      ssp_mvi::score(a.rig, d, avail, h, a.gate2, a.thr2, a.max_iter, ssp_mvi::hyp_at(slots, uvs, h, C));
      stale[h] = 0;
    }
    __syncthreads();
    for (int k = tid; k < a.num_classes; k += kThreads) {
      const int w = ssp_mvi::class_candidate(d, avail, slots, H, k);
      if (w >= 0) cand[w] = 1;
    }
    __syncthreads();
    if (tid == 0) {
      const int win = ssp_mvi::pick(cand, slots, H);
      s_win = win;
      if (win >= 0) {
        const long long gw = (long long)g * M + nw;
        const ssp_mvi::Hyp W = ssp_mvi::hyp_at(slots, uvs, win, C);
        ssp_mvi::emit(a.rig, d, W, d.cls[win], a.sigma, a.R_world + gw * 9, a.t_world + gw * 3, a.world_cov + gw * 36, a.members + gw * C,
                      a.view_err + gw * C, a.fuse_status + gw);
        a.world_cls[gw] = d.cls[win];
        a.fuse_hyp[gw] = win;
        for (int c = 0; c < C; c++)
          if (W.sel[c] >= 0) {
            avail[c * M + W.sel[c]] = 0;
            a.world_index[b0 * M + c * M + W.sel[c]] = nw;
          }
      }
    }
    __syncthreads();
    const int win = s_win;
    if (win < 0) break;
    const ssp_mvi::Hyp W = ssp_mvi::hyp_at(slots, uvs, win, C);
    const unsigned removed = (unsigned)W.R[13];
    for (int h = tid; h < H; h += kThreads)
      if (avail[h] && ssp_mvi::touched(ssp_mvi::hyp_at(slots, uvs, h, C), removed, W.sel, C)) stale[h] = 1;
    __syncthreads();
  }
  if (tid == 0) {
    int left = 0;
    for (int i = 0; i < H; i++) left += avail[i];
    a.world_count[g] = nw;
    a.unfused[g] = left;
  }
  // every world instance in every camera of the capture: (view c, world slot w, point p)
  for (long long e = tid; e < (long long)C * M * np; e += kThreads) {
    const int p = (int)(e % np), w = (int)((e / np) % M), c = (int)(e / ((long long)np * M));
    float* out = a.corners_world + ((b0 + c) * M + w) * 2 * np + 2 * p;
    if (w >= nw) { out[0] = 0.f; out[1] = 0.f; continue; }
    const long long gw = (long long)g * M + w;
    const ssp_mv::Cam cam = ssp_mv::camera(a.rig, c);
    double Rw[9], tw[3];
    ssp_mv::to_camera(cam, a.R_world + gw * 9, a.t_world + gw * 3, Rw, tw);
    const float* X = a.table + ((long long)a.world_cls[gw] * np + p) * 3;
    ssp_mv::project(Rw, tw, X[0], X[1], X[2], a.K64 + 9 * c, cam.dist, out, out + 1);
  }
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_fuse_instances_work_bytes(int groups, int views, int slots, long long* bytes_out) {
  if (!bytes_out || groups < 0 || views < 1 || views > ssp_mv::kMaxViews || slots < 1 || slots > SSP_FUSE_MAX_SLOTS)
    return fail_msg(SSP_ERR_ARG, "fuse_instances_work_bytes: bad size (groups >= 0, 1 <= views <= 16, 1 <= slots <= 256)");
  *bytes_out = ssp_mvi::work_bytes(groups, views, slots);
  return SSP_OK;
}

int ssp_fuse_instances(const float* points3d_table, int num_classes, const float* points2d, const int* cls, const int* count, int num_points,
                       int groups, int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null,
                       const double* R_rig, const double* t_rig, double gate, double reproj_thresh, double keypoint_sigma, int max_iter,
                       double* R_out, double* t_out, float* corners_out, int* world_count, int* unfused, int* world_cls, double* R_world,
                       double* t_world, double* world_cov, int* members, double* view_err, int* fuse_hyp, int* fuse_status,
                       int* world_index, float* corners_world, void* work, long long work_bytes, void* stream) {
  if (!points3d_table || !points2d || !cls || !count || !K3x3_f32 || !K3x3 || !R_rig || !t_rig || !R_out || !t_out || !corners_out ||
      !world_count || !unfused || !world_cls || !R_world || !t_world || !world_cov || !members || !view_err || !fuse_hyp || !fuse_status ||
      !world_index || !corners_world || !work)
    return fail_msg(SSP_ERR_ARG, "fuse_instances: null pointer");
  if (views < 1 || views > ssp_mv::kMaxViews || num_points < ssp_mv::kMinPoints || num_points > ssp_mv::kMaxPoints || groups < 0 ||
      slots < 1 || slots > SSP_FUSE_MAX_SLOTS || num_classes < 1 || max_iter < 1)
    return fail_msg(SSP_ERR_ARG, "fuse_instances: bad size (1 <= views <= 16, 7 <= points <= 10, groups >= 0, 1 <= slots <= 256, "
                                 "num_classes >= 1, max_iter >= 1)");
  if (!positive_finite(gate) || !positive_finite(reproj_thresh) || !positive_finite(keypoint_sigma))
    return fail_msg(SSP_ERR_ARG, "fuse_instances: gate, reproj_thresh and keypoint_sigma must be > 0 and finite");
  if (gate < reproj_thresh) return fail_msg(SSP_ERR_ARG, "fuse_instances: the gate must be >= reproj_thresh");
  if (work_bytes < ssp_mvi::work_bytes(groups, views, slots) || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "fuse_instances: workspace smaller than ssp_fuse_instances_work_bytes or not 8-B aligned");
  if (groups == 0) return SSP_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const long long rows = (long long)groups * views, n = rows * slots;
  float* P3 = (float*)work;
  gather_points_kernel<<<(unsigned)((n * num_points * 3 + 255) / 256), 256, 0, s>>>(points3d_table, num_classes, cls, num_points, n, P3);
  SSP_CHECK_LAUNCH();
  int rc = launch_fuse_rows_counted(P3, 3LL * num_points, points2d, K3x3_f32, K3x3, dist8_or_null, count, num_points, views, slots, rows,
                                    max_iter, R_out, t_out, corners_out, stream);
  if (rc != SSP_OK) return rc;
  const InstArgs a = {points3d_table, num_classes, cls, count, points2d, num_points, views, slots,
                      ssp_mv::Rig{K3x3_f32, dist8_or_null, R_rig, t_rig, views}, K3x3, gate * gate, reproj_thresh * reproj_thresh,
                      keypoint_sigma, max_iter, R_out, t_out, corners_out, world_count, unfused, world_cls, R_world, t_world, world_cov,
                      members, view_err, fuse_hyp, fuse_status, world_index, corners_world,
                      (char*)work + ssp_mvi::points_bytes(groups, views, slots)};
  fuse_instances_kernel<<<(unsigned)groups, kThreads, 0, s>>>(a);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
