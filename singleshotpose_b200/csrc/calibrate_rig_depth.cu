// Calibrating an RGB-D rig against depth (rule: calibrate_rig_depth_core.h).  ssp_calibrate_rig_depth runs, on one stream and
// with no synchronisation, so the call can be captured in a CUDA graph:
//   cd_init_kernel        one CTA: the state (extrinsics, world poses) from the inputs, the outputs of an iteration not run
//   per iteration (a stopped call's kernels return at once):
//     cd_pair_kernel      one 256-thread CTA per (observation, camera), active views only: thread j adds the pairs of model points
//                         j, j + 256, ... into its column of a [kAcc][256] accumulator in dynamic shared memory (184 KB, opted
//                         in, so no accumulator lives in registers), then the halving tree a[j] += a[j + s], s = 128 .. 1, the
//                         harness's order
//     cd_obs_kernel       one thread per observation: the sums over its views, the stop test, q_o and Z_oc
//     cd_block_kernel     one 256-thread CTA per camera-block pair c1 <= c2: each entry's 256 lane partials and tree_sum
//     cd_factor_kernel    one CTA: the solved cameras, the reduced system in dynamic shared memory factored by columns, dc, the
//                         cameras' update, the camera outputs and, on the last iteration, cam_cov
//     cd_update_kernel    one thread per observation: do and the world pose, and its output pose
//   cd_restore_kernel     after a global stop, every output pose back to its input
// This file is built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <math.h>

#include "ssp_common.cuh"
#include "calibrate_rig_depth_core.h"

namespace ssp {
namespace {

static_assert(ssp_cd::kCamUnconnected == SSP_CALIB_DEPTH_UNCONNECTED && ssp_cd::kCamFewPoints == SSP_CALIB_DEPTH_FEW_POINTS &&
              ssp_cd::kCamSingular == SSP_CALIB_DEPTH_SINGULAR && ssp_cd::kCamUnconnected == SSP_CALIB_UNCONNECTED,
              "the depth calibration's status bits");
static_assert(ssp_cd::kLanes == 256 && ssp_cd::kThreads == 256, "the reductions run one CTA of 256 threads");

using ssp_cd::Problem;

constexpr size_t kPairSmem = (size_t)ssp_cd::kAcc * ssp_cd::kThreads * sizeof(double);
constexpr int kMaxN = 6 * (ssp_cd::kMaxViews - 1);
constexpr size_t kFactorSmem = (size_t)2 * kMaxN * kMaxN * sizeof(double);

struct Outputs {
  const double* R_cam_in;
  const double* t_cam_in;
  const double* R_in;
  const double* t_in;
  double* R_cam;
  double* t_cam;
  double* cam_cov;
  int* cam_points;
  double* cam_rmse;
  int* cam_status;
  double* R_out;
  double* t_out;
  int* obs_points;
  double* obs_rmse;
  int* obs_status;
  int* status;
  double* iter_rmse;
  int iters;
};

__device__ inline bool halted(const Problem& P) { return ssp_cd::ctl(P)[ssp_cd::kStop] != 0.0; }

// the fixed tree over the CTA's 256 partials in shared memory; every thread gets the sum
__device__ double cta_tree_sum(double* red, double v) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = ssp_cd::kLanes / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double s = red[0];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(256) cd_init_kernel(const Problem P, const Outputs out) {
  const int C = ssp_cd::C_of(P);
  if (threadIdx.x == 0) ssp_cd::init_cams(P, out.R_cam_in, out.t_cam_in);
  for (long long o = threadIdx.x; o < P.O; o += blockDim.x) {
    ssp_cd::init_obs(P, o, out.R_in, out.t_in);
    for (int k = 0; k < 9; k++) out.R_out[o * 9 + k] = out.R_in[o * 9 + k];
    for (int k = 0; k < 3; k++) out.t_out[o * 3 + k] = out.t_in[o * 3 + k];
    out.obs_points[o] = 0; out.obs_rmse[o] = 0.0; out.obs_status[o] = 0;
  }
  for (int k = threadIdx.x; k < 36 * C; k += blockDim.x) out.cam_cov[k] = 0.0;
  for (int k = threadIdx.x; k < 9 * C; k += blockDim.x) out.R_cam[k] = out.R_cam_in[k];
  for (int k = threadIdx.x; k < 3 * C; k += blockDim.x) out.t_cam[k] = out.t_cam_in[k];
  for (int k = threadIdx.x; k < out.iters; k += blockDim.x) out.iter_rmse[k] = 0.0;
  if ((int)threadIdx.x < C) {
    const int c = threadIdx.x;
    out.cam_points[c] = 0; out.cam_rmse[c] = 0.0;
    out.cam_status[c] = ssp_cal::kUnconnected & P.status_in[c];
  }
  if (threadIdx.x == 0) *out.status = 0;
}

__global__ void __launch_bounds__(256, 1) cd_pair_kernel(const Problem P, double tau) {
  extern __shared__ double acc[];                                  // [kAcc][256]: thread j's column
  const int C = ssp_cd::C_of(P);
  const long long o = blockIdx.x / C;
  const int c = (int)(blockIdx.x % C);
  if (halted(P) || !ssp_cd::active(P, o, c)) return;
  const int tid = threadIdx.x;
  ssp_cd::view_thread(P, o, c, tau, tid, acc + tid, ssp_cd::kThreads);
  __syncthreads();
  for (int s = ssp_cd::kThreads / 2; s >= 1; s /= 2) {
    if (tid < s)
      for (int i = 0; i < ssp_cd::kAcc; i++) acc[i * ssp_cd::kThreads + tid] += acc[i * ssp_cd::kThreads + tid + s];
    __syncthreads();
  }
  double* dst = ssp_cd::acc_of(P, o, c);
  for (int i = tid; i < ssp_cd::kAcc; i += ssp_cd::kThreads) dst[i] = acc[i * ssp_cd::kThreads];
}

__global__ void __launch_bounds__(128) cd_obs_kernel(const Problem P, const Outputs out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (halted(P) || o >= P.O || !P.linked[o] || ssp_cd::stopped(P, o)) return;
  int pts;
  double rmse;
  const int st = ssp_cd::obs_solve(P, o, &pts, &rmse);
  out.obs_status[o] = st;
  out.obs_points[o] = pts;
  out.obs_rmse[o] = rmse;
  if (st) {                                                        // a stopped observation's output is its input pose
    for (int k = 0; k < 9; k++) out.R_out[o * 9 + k] = out.R_in[o * 9 + k];
    for (int k = 0; k < 3; k++) out.t_out[o * 3 + k] = out.t_in[o * 3 + k];
  }
}

__global__ void __launch_bounds__(256) cd_block_kernel(const Problem P) {
  __shared__ double red[ssp_cd::kLanes];
  if (halted(P)) return;
  const int C = ssp_cd::C_of(P);
  int c1, c2;
  if ((int)blockIdx.x < C) { c1 = c2 = blockIdx.x; }
  else ssp_cal::pair_cams(C, blockIdx.x - C, &c1, &c2);
  for (int e = ssp_cd::block_first(P, c1); e < ssp_cd::block_entries(P, c1, c2); e++) {
    const double s = cta_tree_sum(red, ssp_cd::block_partial(P, c1, c2, e, threadIdx.x));
    if (threadIdx.x == 0) *ssp_cd::block_slot(P, c1, c2, e) = s;
  }
}

__global__ void __launch_bounds__(256) cd_factor_kernel(const Problem P, const Outputs out, int k) {
  extern __shared__ double A[];
  __shared__ int cams[ssp_cd::kMaxViews], ok, n;
  __shared__ double dc[kMaxN];
  double* ctl = ssp_cd::ctl(P);
  if (halted(P)) return;
  const int C = ssp_cd::C_of(P);
  if (threadIdx.x == 0) {
    unsigned held;
    n = 6 * ssp_cd::solve_list(P, cams, &held);
    ctl[ssp_cd::kHeld] = (double)held;
    out.iter_rmse[k] = ssp_cd::overall_rmse(P);
    ok = 1;
  }
  if ((int)threadIdx.x < C) {
    const int c = threadIdx.x;
    const double cn = ssp_cd::connected(P, c) ? ssp_cd::cam_n(P, c) : 0.0;
    out.cam_points[c] = (int)cn;
    out.cam_rmse[c] = cn > 0.0 ? sqrt(ssp_cd::cam_r2(P, c) / cn) : 0.0;
  }
  __syncthreads();
  const int N = n;
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) A[e] = ssp_cd::reduced_entry(P, cams, e / N, e % N);
  __syncthreads();
  for (int j = 0; j < N; j++) {
    if (threadIdx.x == 0 && !ssp_cal::chol_pivot(A, N, j)) ok = 0;
    __syncthreads();
    if (!ok) break;
    for (int i = j + 1 + threadIdx.x; i < N; i += blockDim.x) ssp_cal::chol_entry(A, N, j, i);
    __syncthreads();
  }
  if (!ok) {                                                       // every output is the input: cd_init_kernel wrote them
    __syncthreads();
    if (threadIdx.x == 0) { ctl[ssp_cd::kStop] = 1.0; *out.status = ssp_cd::kCamSingular; }
    __syncthreads();
    if ((int)threadIdx.x < C) out.cam_status[threadIdx.x] = ssp_cd::cam_status_bits(P, threadIdx.x);
    return;
  }
  if (k == out.iters - 1) {                                        // cam_cov: one column of S^-1 per thread
    double* X = A + N * N;
    const double s2 = out.iter_rmse[k] * out.iter_rmse[k];
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      double* x = X + j * N;
      for (int i = 0; i < N; i++) x[i] = i == j ? 1.0 : 0.0;
      ssp_cal::chol_subst(A, N, x);
      const int c = cams[j / 6], b = j % 6;
      for (int a = 0; a < 6; a++) out.cam_cov[c * 36 + 6 * a + b] = s2 * x[(j / 6) * 6 + a];
    }
  }
  if (threadIdx.x == 0) {
    for (int I = 0; I < N; I++) dc[I] = ssp_cd::rhs_entry(P, cams, I);
    ssp_cal::chol_subst(A, N, dc);
    unsigned solved = 0;
    for (int i = 0; i < N / 6; i++) solved |= 1u << cams[i];
    ctl[ssp_cd::kSolved] = (double)solved;
    ssp_cd::camera_update(P, cams, N / 6, dc);
  }
  __syncthreads();
  if ((int)threadIdx.x < C) {
    const int c = threadIdx.x;
    for (int i = 0; i < 9; i++) out.R_cam[9 * c + i] = P.rig.R[9 * c + i];
    for (int i = 0; i < 3; i++) out.t_cam[3 * c + i] = P.rig.t[3 * c + i];
    out.cam_status[c] = ssp_cd::cam_status_bits(P, c);
  }
}

__global__ void __launch_bounds__(128) cd_update_kernel(const Problem P, const Outputs out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (halted(P) || o >= P.O || !P.linked[o] || ssp_cd::stopped(P, o)) return;
  ssp_cd::obs_update(P, o, (unsigned)ssp_cd::ctl(P)[ssp_cd::kSolved]);
  const double* x = ssp_cd::obs_pose(P, o);
  for (int k = 0; k < 9; k++) out.R_out[o * 9 + k] = x[k];
  for (int k = 0; k < 3; k++) out.t_out[o * 3 + k] = x[9 + k];
}

// a global stop returns every pose to its input: the world poses an earlier iteration wrote, and the cameras
__global__ void __launch_bounds__(128) cd_restore_kernel(const Problem P, const Outputs out) {
  if (!halted(P)) return;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o < P.O) {
    for (int k = 0; k < 9; k++) out.R_out[o * 9 + k] = out.R_in[o * 9 + k];
    for (int k = 0; k < 3; k++) out.t_out[o * 3 + k] = out.t_in[o * 3 + k];
  }
  if (blockIdx.x == 0)
    for (int k = threadIdx.x; k < 12 * ssp_cd::C_of(P); k += blockDim.x) {
      if (k < 9 * ssp_cd::C_of(P)) out.R_cam[k] = out.R_cam_in[k];
      else out.t_cam[k - 9 * ssp_cd::C_of(P)] = out.t_cam_in[k - 9 * ssp_cd::C_of(P)];
    }
}

inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }
inline unsigned grid(long long n, int b) { return (unsigned)(n > 0 ? (n + b - 1) / b : 1); }

}  // namespace
}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_calibrate_rig_depth_work_bytes(int groups, int views, int slots, long long* bytes_out) {
  if (!bytes_out || groups < 0 || views < 2 || views > ssp_cd::kMaxViews || slots < 1)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth_work_bytes: bad size (groups >= 0, 2 <= views <= 16, slots >= 1)");
  *bytes_out = ssp_cd::layout((long long)groups * slots, views).total * 8;
  return SSP_OK;
}

int ssp_calibrate_rig_depth(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                            const double* dist8_or_null, int reference, const int* cam_status_in, const double* R_cam_in,
                            const double* t_cam_in, const double* model, int num_vertices, double diam, int groups, int slots,
                            const unsigned char* obs_views, const unsigned char* linked, const double* R_world_in,
                            const double* t_world_in, int iters, double gate_start, double gate_end, double* R_cam, double* t_cam,
                            double* cam_cov, int* cam_points, double* cam_rmse, int* cam_status, double* R_world, double* t_world,
                            int* obs_points, double* obs_rmse, int* obs_status, int* status, double* iter_rmse, void* work,
                            long long work_bytes, void* stream) {
  if (!depth || !K3x3 || !cam_status_in || !R_cam_in || !t_cam_in || !model || !obs_views || !linked || !R_world_in || !t_world_in ||
      !R_cam || !t_cam || !cam_cov || !cam_points || !cam_rmse || !cam_status || !R_world || !t_world || !obs_points || !obs_rmse ||
      !obs_status || !status || !iter_rmse || !work)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: null pointer");
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || groups < 0 || slots < 1 || iters < 1 || iters > ssp_rd::kMaxIters || num_vertices < 1)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: bad size (W, H in 1..16384, groups >= 0, slots >= 1, iters in 1..100, num_vertices >= 1)");
  if (views < 2 || views > ssp_cd::kMaxViews) return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: bad size (2 <= views <= 16)");
  if (reference < 0 || reference >= views) return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: the reference camera must be in 0..views-1");
  if (!positive_finite(gate_start) || !positive_finite(gate_end) || gate_end > gate_start)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: the gate range needs 0 < gate_end <= gate_start < inf");
  if (!positive_finite(depth_scale)) return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: depth_scale must be > 0 and finite");
  if (!positive_finite(diam)) return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: the mesh diameter must be > 0 and finite");
  const long long O = (long long)groups * slots;
  const ssp_cd::Layout L = ssp_cd::layout(O, views);
  if (work_bytes < L.total * 8 || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: workspace smaller than ssp_calibrate_rig_depth_work_bytes or not 8-B aligned");
  if (O * views > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "calibrate_rig_depth: more than 2^31 - 1 views");
  double* w = (double*)work;
  const Problem P = {depth, ssp_rr::Rig{K3x3, dist8_or_null, w + L.cam, w + L.cam + 9 * views, views, W, H, depth_scale}, model,
                     num_vertices, diam, obs_views, linked, cam_status_in, reference, slots, O, w, L};
  const Outputs out = {R_cam_in, t_cam_in, R_world_in, t_world_in, R_cam, t_cam, cam_cov, cam_points, cam_rmse, cam_status, R_world,
                       t_world, obs_points, obs_rmse, obs_status, status, iter_rmse, iters};
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(cd_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPairSmem) != cudaSuccess ||
        cudaFuncSetAttribute(cd_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFactorSmem) != cudaSuccess)
      SSP_CHECK_LAUNCH();
    attr = true;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int blocks = views + ssp_cal::num_pairs(views);
  const int n = 6 * (views - 1);
  const size_t smem_factor = (size_t)2 * n * n * sizeof(double);
  cd_init_kernel<<<1, 256, 0, s>>>(P, out);
  SSP_CHECK_LAUNCH();
  for (int k = 0; k < iters; k++) {
    if (O > 0) {
      const double tau = diam * ssp_rd::gate_factor(gate_start, gate_end, k, iters);      // the harness's bits
      cd_pair_kernel<<<(unsigned)(O * views), ssp_cd::kThreads, kPairSmem, s>>>(P, tau);
      SSP_CHECK_LAUNCH();
    }
    cd_obs_kernel<<<grid(O, 128), 128, 0, s>>>(P, out);
    SSP_CHECK_LAUNCH();
    cd_block_kernel<<<blocks, ssp_cd::kLanes, 0, s>>>(P);
    SSP_CHECK_LAUNCH();
    cd_factor_kernel<<<1, 256, smem_factor, s>>>(P, out, k);
    SSP_CHECK_LAUNCH();
    cd_update_kernel<<<grid(O, 128), 128, 0, s>>>(P, out);
    SSP_CHECK_LAUNCH();
  }
  cd_restore_kernel<<<grid(O, 128), 128, 0, s>>>(P, out);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
