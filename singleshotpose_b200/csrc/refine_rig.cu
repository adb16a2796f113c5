// Refinement of a rig's world poses against every camera's depth frame (rule: refine_rig_core.h).  One thread-block cluster per
// problem runs every iteration in one launch: the cluster has min(C, 8) CTAs of 256 threads, and CTA r takes the cameras r, r + 8,
// ...  For each of its cameras a CTA accumulates the pairs of model points j, j + 256, ... in thread j, combines the 256
// accumulators by the halving tree of refine_depth.cu (shared memory for the strides 128, 64, 32, warp shuffles for 16 .. 1) and
// keeps the result in its shared memory.  After a cluster barrier thread 0 of the leader CTA reads the C accumulators over
// distributed shared memory in camera order, adds them, solves and updates the pose; after a second barrier every CTA reads the
// pose back.  A one-camera call therefore costs about what ssp_refine_depth's one CTA costs, not C times it.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <cooperative_groups.h>
#include <math.h>

#include "ssp_common.cuh"
#include "refine_rig_core.h"

namespace cg = cooperative_groups;

namespace ssp {

constexpr int kRigCtas = 8;                                              // the portable cluster size
constexpr int kViewsPerCta = (ssp_rr::kMaxViews + kRigCtas - 1) / kRigCtas;

struct RigGates {
  double g[ssp_rd::kMaxIters];                // the rule's factors g_k, computed on the host (gate_factor)
};

struct RigRefineArgs {
  const unsigned short* depth;                // [groups * C][H][W]
  ssp_rr::Rig rig;
  const double* model;
  const int* offsets;
  const double* diam;
  const float* table;                         // [num_classes][np][3]
  int np, num_classes, slots, iters;
  const int* cls;                             // [groups][slots]
  const int* count;                           // [groups] or null
  const int* fuse_status;                     // [groups][slots] or null
  const double* R_in;
  const double* t_in;
  double* R_out;
  double* t_out;
  int* points_out;
  double* rmse_out;
  int* status_out;
  int* view_points;                           // [groups][slots][C]
  double* view_rmse;
  float* corners;                             // [groups * C][slots][np][2]
};

// the halving tree of refine_depth.cu over the CTA's 256 accumulators; the result in thread 0's acc
__device__ __forceinline__ void cta_tree(double* acc, double (*red)[ssp_rd::kThreads / 2], int tid) {
  constexpr int NA = ssp_rr::kAcc;
#pragma unroll
  for (int s = ssp_rd::kThreads / 2; s >= 32; s /= 2) {       // a[i] += a[i + s], i < s, through shared memory
    if (tid >= s && tid < 2 * s)
      for (int i = 0; i < NA; i++) red[i][tid - s] = acc[i];
    __syncthreads();
    if (tid < s)
      for (int i = 0; i < NA; i++) acc[i] += red[i][tid];
    __syncthreads();
  }
  if (tid < 32) {
#pragma unroll
    for (int s = 16; s >= 1; s /= 2)
      for (int i = 0; i < NA; i++) acc[i] += __shfl_down_sync(0xffffffffu, acc[i], s);
  }
}

__global__ void __launch_bounds__(ssp_rd::kThreads, 1) refine_rig_kernel(const RigRefineArgs a, const RigGates gates) {
  constexpr int NA = ssp_rr::kAcc;
  __shared__ double red[NA][ssp_rd::kThreads / 2];
  __shared__ double s_acc[kViewsPerCta][NA];                   // this CTA's cameras' reduced accumulators
  __shared__ double sR[9], st[3];
  __shared__ double s_rmse, s_diam, s_vr[ssp_rr::kMaxViews];
  __shared__ int s_status, s_points, s_begin, s_end, s_vp[ssp_rr::kMaxViews];
  cg::cluster_group cluster = cg::this_cluster();
  const int ctas = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, C = a.rig.C, np = a.np;
  const long long id = blockIdx.x / ctas;
  const long long g = id / a.slots;
  const int m = (int)(id % a.slots);
  const int c_ = a.cls[id];
  const bool known = c_ >= 0 && c_ < a.num_classes;
  const int fs = a.fuse_status ? a.fuse_status[id] : 0;
  const long long cstride = (long long)a.slots * 2 * np;        // between the rows of one capture
  float* crn = a.corners + (g * C * a.slots + m) * 2LL * np;   // (row g C, slot m)
  if (a.count && m >= a.count[g]) {                            // the whole cluster leaves: no barrier is pending
    if (rank == 0) {
      if (tid < 9) a.R_out[id * 9 + tid] = 0.0;
      if (tid < 3) a.t_out[id * 3 + tid] = 0.0;
      if (tid < C) { a.view_points[id * C + tid] = 0; a.view_rmse[id * C + tid] = 0.0; }
      if (tid == 0) { a.points_out[id] = 0; a.rmse_out[id] = 0.0; a.status_out[id] = 0; }
    }
    for (int c = rank; c < C; c += ctas)
      if (tid < 2 * np) crn[c * cstride + tid] = 0.f;
    return;
  }
  if (tid == 0) {
    for (int k = 0; k < 9; k++) sR[k] = a.R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) st[k] = a.t_in[id * 3 + k];
    s_begin = known ? a.offsets[c_] : 0;
    s_end = known ? a.offsets[c_ + 1] : 0;
    s_diam = known ? a.diam[c_] : 0.0;
    s_status = ssp_rr::input_status(sR, st, fs);
    s_points = 0;
    s_rmse = 0.0;
  }
  if (tid < ssp_rr::kMaxViews) { s_vp[tid] = 0; s_vr[tid] = 0.0; }
  __syncthreads();
  for (int k = 0; k < a.iters && s_status == 0; k++) {
    const double tau = s_diam * gates.g[k];
    double R[9], t[3];
    for (int i = 0; i < 9; i++) R[i] = sR[i];
    for (int i = 0; i < 3; i++) t[i] = st[i];
    for (int j = 0, c = rank; c < C; j++, c += ctas) {
      const ssp_mv::Cam ext = ssp_rr::extrinsics(a.rig, c);
      const ssp_rd::Camera cam = ssp_rr::depth_camera(a.rig, c);
      double Rc[9], tc[3], acc[NA];
      ssp_mv::to_camera(ext, R, t, Rc, tc);
      const unsigned short* D = a.depth + (g * C + c) * (long long)a.rig.H * a.rig.W;
      for (int i = 0; i < NA; i++) acc[i] = 0.0;
      for (int i = s_begin + tid; i < s_end; i += ssp_rd::kThreads)
        ssp_rr::accumulate_point(a.model + (long long)i * 6, R, t, Rc, tc, ext, cam, D, tau, acc);
      cta_tree(acc, red, tid);
      if (tid == 0)
        for (int i = 0; i < NA; i++) s_acc[j][i] = acc[i];
    }
    cluster.sync();                                            // every camera's accumulator is in its CTA's shared memory
    if (rank == 0 && tid == 0) {
      double sum[NA];
      auto view = [&](int c) { return (const double*)cluster.map_shared_rank(&s_acc[c / ctas][0], c % ctas); };
      for (int c = 0; c < C; c++) {
        int p;
        double r;
        ssp_rr::view_stats(view(c), &p, &r);
        s_vp[c] = p;
        s_vr[c] = r;
      }
      ssp_rr::sum_views(view, C, sum);
      int pts;
      double rmse;
      s_status = ssp_rd::solve_update(sum, sR, st, &pts, &rmse);
      s_points = pts;
      s_rmse = rmse;
    }
    cluster.sync();                                            // the leader's pose and status are written
    if (rank != 0 && tid == 0) {
      const double* lR = cluster.map_shared_rank(sR, 0);
      const double* lt = cluster.map_shared_rank(st, 0);
      for (int i = 0; i < 9; i++) sR[i] = lR[i];
      for (int i = 0; i < 3; i++) st[i] = lt[i];
      s_status = *cluster.map_shared_rank(&s_status, 0);
    }
    __syncthreads();
  }
  cluster.sync();                                              // no CTA leaves while another still reads its shared memory
  const bool ok = s_status == 0;
  if (rank == 0 && tid == 0) {
    for (int k = 0; k < 9; k++) a.R_out[id * 9 + k] = ok ? sR[k] : a.R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) a.t_out[id * 3 + k] = ok ? st[k] : a.t_in[id * 3 + k];
    a.points_out[id] = s_points;
    a.rmse_out[id] = s_rmse;
    a.status_out[id] = s_status;
  }
  if (rank == 0 && tid < C) { a.view_points[id * C + tid] = s_vp[tid]; a.view_rmse[id * C + tid] = s_vr[tid]; }
  const int c = rank + ctas * (tid / 32);                      // warp w's lane 0 draws camera rank + w ctas
  if (tid % 32 == 0 && c < C) {
    double R[9], t[3];
    for (int k = 0; k < 9; k++) R[k] = ok ? sR[k] : a.R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) t[k] = ok ? st[k] : a.t_in[id * 3 + k];
    const bool none = !known || (fs & (ssp_mv::kNoValid | ssp_mv::kNoView));
    ssp_rr::project_view(a.rig, c, R, t, a.table + (known ? c_ : 0) * 3LL * np, np, none, crn + c * cstride);
  }
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_refine_depth_rig(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                         const double* dist8_or_null, const double* R_rig, const double* t_rig, const double* model, const int* offsets,
                         const double* diam, const float* points3d_table, int num_points, int num_classes, const int* cls, int groups,
                         int slots, const int* count_or_null, const int* fuse_status_or_null, const double* R_world,
                         const double* t_world, int iters, double gate_start, double gate_end, double* R_out, double* t_out,
                         int* points_out, double* rmse_out, int* status_out, int* view_points, double* view_rmse,
                         float* corners_world_ref, void* stream) {
  if (!depth || !K3x3 || !R_rig || !t_rig || !model || !offsets || !diam || !points3d_table || !cls || !R_world || !t_world || !R_out ||
      !t_out || !points_out || !rmse_out || !status_out || !view_points || !view_rmse || !corners_world_ref)
    return fail_msg(SSP_ERR_ARG, "refine_depth_rig: null pointer");
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || num_classes < 1 || groups < 0 || slots < 1 || iters < 1 || iters > ssp_rd::kMaxIters)
    return fail_msg(SSP_ERR_ARG, "refine_depth_rig: bad size (W, H in 1..16384, num_classes >= 1, groups >= 0, slots >= 1, iters in 1..100)");
  if (views < 1 || views > ssp_rr::kMaxViews || num_points < ssp_mv::kMinPoints || num_points > ssp_mv::kMaxPoints)
    return fail_msg(SSP_ERR_ARG, "refine_depth_rig: bad size (1 <= views <= 16, 7 <= num_points <= 10)");
  if (!positive_finite(gate_start) || !positive_finite(gate_end) || gate_end > gate_start)
    return fail_msg(SSP_ERR_ARG, "refine_depth_rig: the gate range needs 0 < gate_end <= gate_start < inf");
  if (!positive_finite(depth_scale)) return fail_msg(SSP_ERR_ARG, "refine_depth_rig: depth_scale must be > 0 and finite");
  const long long n = (long long)groups * slots;
  if (n == 0) return SSP_OK;
  const int ctas = views < kRigCtas ? views : kRigCtas;
  if (n * ctas > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "refine_depth_rig: more than 2^31 - 1 CTAs");
  RigGates gates;
  for (int k = 0; k < ssp_rd::kMaxIters; k++) gates.g[k] = k < iters ? ssp_rd::gate_factor(gate_start, gate_end, k, iters) : 0.0;
  const RigRefineArgs a = {depth, ssp_rr::Rig{K3x3, dist8_or_null, R_rig, t_rig, views, W, H, depth_scale}, model, offsets, diam,
                           points3d_table, num_points, num_classes, slots, iters, cls, count_or_null, fuse_status_or_null, R_world,
                           t_world, R_out, t_out, points_out, rmse_out, status_out, view_points, view_rmse, corners_world_ref};
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(n * ctas));
  cfg.blockDim = dim3(ssp_rd::kThreads);
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)ctas;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, refine_rig_kernel, a, gates);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
