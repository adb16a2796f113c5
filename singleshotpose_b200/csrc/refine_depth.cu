// Pose refinement against registered depth frames (rule: refine_depth_core.h).  One 256-thread CTA per problem runs every
// iteration in one launch: thread j accumulates the pairs of model points j, j + 256, ..., the 256 accumulators are combined by the
// halving tree of the rule (shared memory for the strides 128, 64, 32, warp shuffles for 16 .. 1, the same additions as
// tree_reduce), thread 0 solves and updates the pose in shared memory, and a barrier separates the iterations.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <math.h>

#include "ssp_common.cuh"
#include "refine_depth_core.h"

namespace ssp {

static_assert(ssp_rd::kMinPoints == SSP_REFINE_MIN_POINTS && ssp_rd::kMaxIters == SSP_REFINE_MAX_ITERS, "include/ssp_b200.h's limits");
static_assert(ssp_rd::kFewPoints == SSP_REFINE_FEW_POINTS && ssp_rd::kSingular == SSP_REFINE_SINGULAR && ssp_rd::kBadPose == SSP_REFINE_BAD_POSE,
              "the refinement status bits");

struct RefineGates {
  double g[ssp_rd::kMaxIters];                // the rule's factors g_k, computed on the host (gate_factor)
};

__global__ void __launch_bounds__(ssp_rd::kThreads, 1)
refine_depth_kernel(const unsigned short* __restrict__ depth, int W, int H, double depth_scale, const double* __restrict__ Kd,
                    const double* __restrict__ dist, const double* __restrict__ model, const int* __restrict__ offsets,
                    const double* __restrict__ diam, int num_classes, const int* __restrict__ cls, int per_group,
                    const int* __restrict__ count, const double* __restrict__ R_in, const double* __restrict__ t_in, int iters,
                    const RefineGates gates, double* __restrict__ R_out, double* __restrict__ t_out, int* __restrict__ points_out,
                    double* __restrict__ rmse_out, int* __restrict__ status_out) {
  constexpr int NA = ssp_rd::kAccDoubles;
  __shared__ double red[NA][ssp_rd::kThreads / 2];
  __shared__ double sR[9], st[3];
  __shared__ int s_status, s_points, s_begin, s_end;
  __shared__ double s_rmse, s_diam;
  const long long id = blockIdx.x;
  const int tid = threadIdx.x;
  const int g = (int)(id / per_group), m = (int)(id % per_group);
  if (count && m >= count[g]) {
    if (tid < 9) R_out[id * 9 + tid] = 0.0;
    if (tid < 3) t_out[id * 3 + tid] = 0.0;
    if (tid == 0) { points_out[id] = 0; rmse_out[id] = 0.0; status_out[id] = 0; }
    return;
  }
  if (tid == 0) {
    for (int k = 0; k < 9; k++) sR[k] = R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) st[k] = t_in[id * 3 + k];
    const int c = cls[id];
    const bool known = c >= 0 && c < num_classes;
    s_begin = known ? offsets[c] : 0;
    s_end = known ? offsets[c + 1] : 0;
    s_diam = known ? diam[c] : 0.0;
    s_status = ssp_rd::pose_ok(sR, st) ? 0 : ssp_rd::kBadPose;
    s_points = 0;
    s_rmse = 0.0;
  }
  __syncthreads();
  const ssp_rd::Camera cam = {Kd[0], Kd[4], Kd[2], Kd[5], dist, W, H, depth_scale};
  const unsigned short* D = depth + (long long)g * H * W;
  for (int k = 0; k < iters && s_status == 0; k++) {
    const double tau = s_diam * gates.g[k];
    double R[9], t[3], acc[NA];
    for (int i = 0; i < 9; i++) R[i] = sR[i];
    for (int i = 0; i < 3; i++) t[i] = st[i];
    for (int i = 0; i < NA; i++) acc[i] = 0.0;
    for (int i = s_begin + tid; i < s_end; i += ssp_rd::kThreads) ssp_rd::accumulate_point(model + (long long)i * 6, R, t, cam, D, tau, acc);
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
    if (tid == 0) {
      int pts;
      double rmse;
      s_status = ssp_rd::solve_update(acc, sR, st, &pts, &rmse);
      s_points = pts;
      s_rmse = rmse;
    }
    __syncthreads();
  }
  if (tid == 0) {
    const bool ok = s_status == 0;
    for (int k = 0; k < 9; k++) R_out[id * 9 + k] = ok ? sR[k] : R_in[id * 9 + k];
    for (int k = 0; k < 3; k++) t_out[id * 3 + k] = ok ? st[k] : t_in[id * 3 + k];
    points_out[id] = s_points;
    rmse_out[id] = s_rmse;
    status_out[id] = s_status;
  }
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_refine_depth(const unsigned short* depth, int W, int H, double depth_scale, const double* K3x3, const double* dist8_or_null,
                     const double* model, const int* offsets, const double* diam, int num_classes, const int* cls, int groups,
                     int per_group, const int* count_or_null, const double* R, const double* t, int iters, double gate_start,
                     double gate_end, double* R_out, double* t_out, int* points_out, double* rmse_out, int* status_out, void* stream) {
  if (!depth || !K3x3 || !model || !offsets || !diam || !cls || !R || !t || !R_out || !t_out || !points_out || !rmse_out || !status_out)
    return fail_msg(SSP_ERR_ARG, "refine_depth: null pointer");
  if (W < 1 || H < 1 || W > 16384 || H > 16384 || num_classes < 1 || groups < 0 || per_group < 1 || iters < 1 ||
      iters > ssp_rd::kMaxIters)
    return fail_msg(SSP_ERR_ARG, "refine_depth: bad size (W, H in 1..16384, num_classes >= 1, groups >= 0, per_group >= 1, iters in 1..100)");
  if (!positive_finite(gate_start) || !positive_finite(gate_end) || gate_end > gate_start)
    return fail_msg(SSP_ERR_ARG, "refine_depth: the gate range needs 0 < gate_end <= gate_start < inf");
  if (!positive_finite(depth_scale)) return fail_msg(SSP_ERR_ARG, "refine_depth: depth_scale must be > 0 and finite");
  const long long n = (long long)groups * per_group;
  if (n == 0) return SSP_OK;
  if (n > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "refine_depth: more than 2^31 - 1 problems");
  RefineGates gates;
  for (int k = 0; k < ssp_rd::kMaxIters; k++) gates.g[k] = k < iters ? ssp_rd::gate_factor(gate_start, gate_end, k, iters) : 0.0;
  refine_depth_kernel<<<(unsigned)n, ssp_rd::kThreads, 0, (cudaStream_t)stream>>>(depth, W, H, depth_scale, K3x3, dist8_or_null, model,
                                                                                 offsets, diam, num_classes, cls, per_group, count_or_null,
                                                                                 R, t, iters, gates, R_out, t_out, points_out, rmse_out,
                                                                                 status_out);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
