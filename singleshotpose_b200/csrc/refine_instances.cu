// Refinement of every world instance of a rig's capture against every camera's depth frame, each depth pixel owned by the
// instance drawn in front of it (rule: refine_instances_core.h).  The iteration count is fixed, and per iteration the host enqueues
// without synchronising:
//   1. a memset of the owner buffers [groups * C][H][W] uint64 to all ones;
//   2. ri_draw_kernel: one CTA per (problem, camera) and face block, one thread per face of a drawn instance; thread 0 maps the
//      instance's pose to the camera once, every thread projects its face's three vertices and atomicMin's its 64-bit keys;
//   3. ri_step_kernel: refine_rig.cu's cluster of min(C, 8) CTAs per problem, one iteration per launch.  The pose is carried
//      between launches in fp64 device state (the workspace) and points, rmse, status and the per-camera counts in the outputs, so
//      nothing is rounded in between; a stopped problem's state is reset to its input pose, which is the pose it is drawn at.
// A last memset and draw under the output poses, ri_map_kernel (owner -> int16) and ri_finish_kernel (the output poses and their
// corners) end the call.  Every launch is capturable in a CUDA graph.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <cooperative_groups.h>
#include <math.h>

#include "ssp_common.cuh"
#include "refine_instances_core.h"

namespace cg = cooperative_groups;

namespace ssp {

constexpr int kRiCtas = 8;                                               // the portable cluster size
constexpr int kRiViewsPerCta = (ssp_rr::kMaxViews + kRiCtas - 1) / kRiCtas;
constexpr int kRiDrawThreads = 256;
constexpr int kRiState = 12;                                             // doubles of pose state per problem: R [9], t [3]

struct InstanceRefineArgs {
  const unsigned short* depth;                // [groups * C][H][W]
  ssp_rr::Rig rig;
  const double* model;
  const int* offsets;
  const double* diam;
  const int* faces;                           // [total faces][3] class-local vertex indices
  const int* face_offsets;                    // [num_classes + 1]
  const float* table;                         // [num_classes][np][3]
  int np, num_classes, slots;
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
  int* view_hidden;
  float* corners;                             // [groups * C][slots][np][2]
  short* instance_map;                        // [groups * C][H][W]
  unsigned long long* owner;                  // [groups * C][H][W] (workspace)
  double* state;                              // [groups][slots][kRiState] (workspace)
};

__device__ __forceinline__ bool ri_known(const InstanceRefineArgs& a, long long id) {
  return a.cls[id] >= 0 && a.cls[id] < a.num_classes;
}
__device__ __forceinline__ bool ri_counted_out(const InstanceRefineArgs& a, long long id) {
  return a.count && (int)(id % a.slots) >= a.count[id / a.slots];
}
__device__ __forceinline__ int ri_fuse_status(const InstanceRefineArgs& a, long long id) { return a.fuse_status ? a.fuse_status[id] : 0; }

// the pose state and the outputs before the first iteration: the input pose, its input status, zero counts
__global__ void ri_init_kernel(const InstanceRefineArgs a, long long n) {
  const long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (id >= n) return;
  const int C = a.rig.C;
  const bool out = ri_counted_out(a, id);
  double* s = a.state + id * kRiState;
  for (int k = 0; k < 9; k++) s[k] = out ? 0.0 : a.R_in[id * 9 + k];
  for (int k = 0; k < 3; k++) s[9 + k] = out ? 0.0 : a.t_in[id * 3 + k];
  a.status_out[id] = out ? 0 : ssp_rr::input_status(a.R_in + id * 9, a.t_in + id * 3, ri_fuse_status(a, id));
  a.points_out[id] = 0;
  a.rmse_out[id] = 0.0;
  for (int c = 0; c < C; c++) { a.view_points[id * C + c] = 0; a.view_rmse[id * C + c] = 0.0; a.view_hidden[id * C + c] = 0; }
}

// one CTA per (problem, camera) = blockIdx.x and face block blockIdx.y: every face of the drawn instance into the owner buffer
__global__ void __launch_bounds__(kRiDrawThreads) ri_draw_kernel(const InstanceRefineArgs a) {
  __shared__ double sRc[9], stc[3];
  const int C = a.rig.C;
  const long long id = blockIdx.x / C;
  const int c = (int)(blockIdx.x % C);
  if (ri_counted_out(a, id) || !ri_known(a, id)) return;
  if (!ssp_ri::drawn(false, a.R_in + id * 9, a.t_in + id * 3, ri_fuse_status(a, id))) return;
  const ssp_mv::Cam ext = ssp_rr::extrinsics(a.rig, c);
  if (threadIdx.x == 0) ssp_mv::to_camera(ext, a.state + id * kRiState, a.state + id * kRiState + 9, sRc, stc);
  __syncthreads();
  const int cl = a.cls[id], w = (int)(id % a.slots);
  const long long g = id / a.slots;
  const int f0 = a.face_offsets[cl], nf = a.face_offsets[cl + 1] - f0;
  const double* model = a.model + (long long)a.offsets[cl] * 6;
  unsigned long long* O = a.owner + (g * C + c) * (long long)a.rig.H * a.rig.W;
  double Rc[9], tc[3];
  for (int i = 0; i < 9; i++) Rc[i] = sRc[i];
  for (int i = 0; i < 3; i++) tc[i] = stc[i];
  for (int f = blockIdx.y * kRiDrawThreads + threadIdx.x; f < nf; f += gridDim.y * kRiDrawThreads)
    ssp_ri::draw_model_face(model, a.faces + (long long)(f0 + f) * 3, Rc, tc, a.rig.K + 9 * c, ext.dist, a.rig.W, a.rig.H,
                            [&](long long p, double z) { atomicMin(O + p, ssp_ri::owner_key(z, w)); });
}

// the halving tree of refine_depth.cu over the CTA's 256 accumulators of NA doubles; the result in thread 0's acc
template <int NA>
__device__ __forceinline__ void ri_cta_tree(double* acc, double (*red)[ssp_rd::kThreads / 2], int tid) {
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

// one iteration of every running problem at the gate factor gk: one cluster of min(C, 8) CTAs per problem, CTA r takes the
// cameras r, r + 8, ...; the leader CTA adds the cameras' accumulators in camera order over distributed shared memory and solves
__global__ void __launch_bounds__(ssp_rd::kThreads, 1) ri_step_kernel(const InstanceRefineArgs a, double gk) {
  constexpr int NA = ssp_ri::kAcc;
  __shared__ double red[NA][ssp_rd::kThreads / 2];
  __shared__ double s_acc[kRiViewsPerCta][NA];
  cg::cluster_group cluster = cg::this_cluster();
  const int ctas = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, C = a.rig.C;
  const long long id = blockIdx.x / ctas;
  if (ri_counted_out(a, id) || a.status_out[id] != 0) return;     // the same for the whole cluster: no barrier is pending
  const long long g = id / a.slots;
  const int w = (int)(id % a.slots), c_ = a.cls[id];
  const bool known = c_ >= 0 && c_ < a.num_classes;
  const int begin = known ? a.offsets[c_] : 0, end = known ? a.offsets[c_ + 1] : 0;
  const double tau = (known ? a.diam[c_] : 0.0) * gk;
  double R[9], t[3];
  for (int i = 0; i < 9; i++) R[i] = a.state[id * kRiState + i];
  for (int i = 0; i < 3; i++) t[i] = a.state[id * kRiState + 9 + i];
  const long long frame = (long long)a.rig.H * a.rig.W;
  for (int j = 0, c = rank; c < C; j++, c += ctas) {
    const ssp_mv::Cam ext = ssp_rr::extrinsics(a.rig, c);
    const ssp_rd::Camera cam = ssp_rr::depth_camera(a.rig, c);
    double Rc[9], tc[3], acc[NA];
    ssp_mv::to_camera(ext, R, t, Rc, tc);
    const unsigned short* D = a.depth + (g * C + c) * frame;
    const unsigned long long* O = a.owner + (g * C + c) * frame;
    for (int i = 0; i < NA; i++) acc[i] = 0.0;
    for (int i = begin + tid; i < end; i += ssp_rd::kThreads)
      ssp_ri::accumulate_point(a.model + (long long)i * 6, R, t, Rc, tc, ext, cam, D, O, w, tau, acc);
    ri_cta_tree<NA>(acc, red, tid);
    if (tid == 0)
      for (int i = 0; i < NA; i++) s_acc[j][i] = acc[i];
  }
  cluster.sync();                                              // every camera's accumulator is in its CTA's shared memory
  if (rank == 0 && tid == 0) {
    auto view = [&](int c) { return (const double*)cluster.map_shared_rank(&s_acc[c / ctas][0], c % ctas); };
    for (int c = 0; c < C; c++) {
      int p;
      double r;
      ssp_rr::view_stats(view(c), &p, &r);
      a.view_points[id * C + c] = p;
      a.view_rmse[id * C + c] = r;
      a.view_hidden[id * C + c] = (int)view(c)[ssp_ri::kOffHidden];
    }
    double sum[ssp_rr::kAcc];
    ssp_rr::sum_views(view, C, sum);
    int pts;
    double rmse;
    const int st = ssp_rd::solve_update(sum, R, t, &pts, &rmse);
    a.points_out[id] = pts;
    a.rmse_out[id] = rmse;
    a.status_out[id] = st;
    for (int i = 0; i < 9; i++) a.state[id * kRiState + i] = st ? a.R_in[id * 9 + i] : R[i];
    for (int i = 0; i < 3; i++) a.state[id * kRiState + 9 + i] = st ? a.t_in[id * 3 + i] : t[i];
  }
  cluster.sync();                                              // no CTA leaves while the leader still reads its shared memory
}

// the instance map of every pixel of every frame
__global__ void ri_map_kernel(const InstanceRefineArgs a, long long pixels) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < pixels; p += (long long)gridDim.x * blockDim.x)
    a.instance_map[p] = ssp_ri::map_entry(a.owner[p]);
}

// the output poses (the state: the refined pose, or the input pose with a status bit) and their corners in every camera
__global__ void ri_finish_kernel(const InstanceRefineArgs a, long long n) {
  const long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (id >= n) return;
  const int C = a.rig.C, np = a.np;
  const long long g = id / a.slots;
  const int m = (int)(id % a.slots);
  const bool out = ri_counted_out(a, id), known = ri_known(a, id);
  const double* R = a.state + id * kRiState;
  const double* t = R + 9;
  for (int k = 0; k < 9; k++) a.R_out[id * 9 + k] = R[k];
  for (int k = 0; k < 3; k++) a.t_out[id * 3 + k] = t[k];
  const bool none = out || !known || (ri_fuse_status(a, id) & (ssp_mv::kNoValid | ssp_mv::kNoView));
  const long long cstride = (long long)a.slots * 2 * np;
  float* crn = a.corners + (g * C * a.slots + m) * 2LL * np;
  for (int c = 0; c < C; c++)
    ssp_rr::project_view(a.rig, c, R, t, a.table + (known ? a.cls[id] : 0) * 3LL * np, np, none, crn + c * cstride);
}

static inline bool ri_positive_finite(double x) { return x > 0.0 && isfinite(x); }

static long long ri_owner_bytes(long long groups, int views, int W, int H) { return groups * views * (long long)W * H * 8; }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_refine_instances_rig_work_bytes(int groups, int views, int slots, int W, int H, long long* bytes_out) {
  if (!bytes_out || groups < 0 || views < 1 || views > ssp_rr::kMaxViews || slots < 1 || slots > SSP_FUSE_MAX_SLOTS || W < 1 || H < 1 ||
      W > 16384 || H > 16384)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig_work_bytes: bad size (groups >= 0, views in 1..16, slots in 1..256, W, H in 1..16384)");
  *bytes_out = ri_owner_bytes(groups, views, W, H) + (long long)groups * slots * kRiState * 8;
  return SSP_OK;
}

int ssp_refine_instances_rig(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                             const double* dist8_or_null, const double* R_rig, const double* t_rig, const double* model, const int* offsets,
                             const double* diam, const int* faces, const int* face_offsets, int max_faces, const float* points3d_table,
                             int num_points, int num_classes, const int* world_cls, int groups, int slots, const int* world_count_or_null,
                             const int* fuse_status_or_null, const double* R_world, const double* t_world, int iters, double gate_start,
                             double gate_end, double* R_out, double* t_out, int* points_out, double* rmse_out, int* status_out,
                             int* view_points, double* view_rmse, int* view_hidden, float* corners_world_ref, short* instance_map,
                             void* work, long long work_bytes, void* stream) {
  if (!depth || !K3x3 || !R_rig || !t_rig || !model || !offsets || !diam || !faces || !face_offsets || !points3d_table || !world_cls ||
      !R_world || !t_world || !R_out || !t_out || !points_out || !rmse_out || !status_out || !view_points || !view_rmse || !view_hidden ||
      !corners_world_ref || !instance_map || !work)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: null pointer");
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || num_classes < 1 || groups < 0 || slots < 1 || slots > SSP_FUSE_MAX_SLOTS || iters < 1 ||
      iters > ssp_rd::kMaxIters || max_faces < 0)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: bad size (W, H in 1..16384, num_classes >= 1, groups >= 0, slots in 1..256, "
                                 "iters in 1..100, max_faces >= 0)");
  if (views < 1 || views > ssp_rr::kMaxViews || num_points < ssp_mv::kMinPoints || num_points > ssp_mv::kMaxPoints)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: bad size (1 <= views <= 16, 7 <= num_points <= 10)");
  if (!ri_positive_finite(gate_start) || !ri_positive_finite(gate_end) || gate_end > gate_start)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: the gate range needs 0 < gate_end <= gate_start < inf");
  if (!ri_positive_finite(depth_scale)) return fail_msg(SSP_ERR_ARG, "refine_instances_rig: depth_scale must be > 0 and finite");
  const long long n = (long long)groups * slots;
  const long long owner_bytes = ri_owner_bytes(groups, views, W, H);
  if (work_bytes < owner_bytes + n * kRiState * 8 || ((unsigned long long)work & 7))
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: short or misaligned workspace (ssp_refine_instances_rig_work_bytes)");
  if (n == 0) return SSP_OK;
  const int ctas = views < kRiCtas ? views : kRiCtas;
  if (n * ctas > 0x7fffffffLL || n * views > 0x7fffffffLL)
    return fail_msg(SSP_ERR_ARG, "refine_instances_rig: more than 2^31 - 1 CTAs");
  unsigned long long* owner = (unsigned long long*)work;
  const InstanceRefineArgs a = {depth, ssp_rr::Rig{K3x3, dist8_or_null, R_rig, t_rig, views, W, H, depth_scale}, model, offsets, diam,
                                faces, face_offsets, points3d_table, num_points, num_classes, slots, world_cls, world_count_or_null,
                                fuse_status_or_null, R_world, t_world, R_out, t_out, points_out, rmse_out, status_out, view_points,
                                view_rmse, view_hidden, corners_world_ref, instance_map, owner, (double*)((char*)work + owner_bytes)};
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((n + 127) / 128);
  const long long fblocks = (max_faces + kRiDrawThreads - 1) / kRiDrawThreads;
  const dim3 draw_grid((unsigned)(n * views), (unsigned)(fblocks < 1 ? 1 : fblocks > 65535 ? 65535 : fblocks));
  auto draw = [&]() -> int {
    cudaError_t e = cudaMemsetAsync(owner, 0xff, (size_t)owner_bytes, s);
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    ri_draw_kernel<<<draw_grid, kRiDrawThreads, 0, s>>>(a);
    SSP_CHECK_LAUNCH();
    return SSP_OK;
  };
  ri_init_kernel<<<blocks, 128, 0, s>>>(a, n);
  SSP_CHECK_LAUNCH();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(n * ctas));
  cfg.blockDim = dim3(ssp_rd::kThreads);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)ctas;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  for (int k = 0; k < iters; k++) {
    const int rc = draw();
    if (rc != SSP_OK) return rc;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, ri_step_kernel, a, ssp_rd::gate_factor(gate_start, gate_end, k, iters));
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    SSP_CHECK_LAUNCH();
  }
  const int rc = draw();
  if (rc != SSP_OK) return rc;
  const long long pixels = owner_bytes / 8;
  const long long mblocks = (pixels + 255) / 256;
  ri_map_kernel<<<(unsigned)(mblocks > 65535 * 16 ? 65535 * 16 : mblocks), 256, 0, s>>>(a, pixels);
  SSP_CHECK_LAUNCH();
  ri_finish_kernel<<<blocks, 128, 0, s>>>(a, n);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
