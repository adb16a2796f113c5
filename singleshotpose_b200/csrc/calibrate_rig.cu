// Calibrating a camera rig from the object it sees (rule: calibrate_rig_core.h).  ssp_calibrate_rig runs, on one stream and with
// no synchronisation:
//   launch_fuse_rows       (multiview_rows.cu) step 1, ssp_fuse_views' per-row stage
//   pair_list_kernel       one thread per camera pair: its co-observations
//   pair_score_kernel      one thread per (pair, hypothesis) over the pair's co-observations
//   tree_kernel            one thread per pair picks its winner, then one thread builds the tree and the initial rig
//   per round (kRounds + 1 at most; a stopped round's kernels return at once):
//     fuse_hyp_kernel      one thread per (observation, hypothesis): ssp_mv::score_hypothesis under the current rig
//     fuse_obs_kernel      one thread per observation: selection, the fused outputs and the observation's key
//     round_kernel         one CTA: stop when no key changed, else start step 5 from the fused poses
//     max_iter LM steps, each: obs_terms_kernel (one thread per observation), block_kernel (one CTA per camera-block pair
//                          c1 <= c2, the fixed-order sums), factor_kernel (one CTA: the reduced system in shared memory),
//                          backsub_kernel (one thread per observation), accept_kernel (one CTA: the decision, lambda on the
//                          device).  Steps after convergence return at once.
//     the covariance: obs_terms_kernel and block_kernel at lambda = 0, cov_kernel (one CTA)
//   finish_kernel          one CTA per camera: cam_obs, cam_rmse, cam_status and the global outputs
// This file is built with -fmad=false, as the host harness is built with -ffp-contract=off, so every stage after step 1 equals the
// harness bit for bit when it starts from the same per-row poses.
#include <math.h>

#include "ssp_common.cuh"
#include "calibrate_rig_core.h"

namespace ssp {

static_assert(ssp_cal::kUnconnected == SSP_CALIB_UNCONNECTED && ssp_cal::kSingularCov == SSP_CALIB_SINGULAR, "the calibration status bits");
static_assert(ssp_cal::kLanes == 256, "the reductions run one CTA of kLanes threads");

int launch_fuse_rows(const float* P3, long long p3_stride, const float* uv, const float* K32, const double* K64, const double* dist, int np,
                     int C, int S, long long rows, int max_iter, double* R, double* t, float* corners, void* stream);

using ssp_cal::Problem;

__device__ inline bool halted(const Problem& P) { const double* k = ssp_cal::ctl(P); return k[ssp_cal::kStop] != 0.0 || k[ssp_cal::kDone] != 0.0; }

// the fixed tree over the CTA's kLanes partials in shared memory; every thread gets the sum
__device__ double cta_tree_sum(double* red, double v) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = ssp_cal::kLanes / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double s = red[0];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(128) pair_list_kernel(const Problem P) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < ssp_cal::num_pairs(P.C)) ssp_cal::pair_list(P, p);
}

__global__ void __launch_bounds__(128) pair_score_kernel(const Problem P) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (pair, hypothesis)
  if (id >= (long long)ssp_cal::num_pairs(P.C) * ssp_cal::kMaxPairHyp) return;
  ssp_cal::pair_score(P, (int)(id / ssp_cal::kMaxPairHyp), (int)(id % ssp_cal::kMaxPairHyp));
}

__global__ void __launch_bounds__(128) tree_kernel(const Problem P, int* __restrict__ parent, int* __restrict__ edge_agree) {
  __shared__ int win[SSP_RIG_MAX_VIEWS * (SSP_RIG_MAX_VIEWS - 1) / 2];
  for (int p = threadIdx.x; p < ssp_cal::num_pairs(P.C); p += blockDim.x) win[p] = ssp_cal::pair_winner(P, p);
  __syncthreads();
  if (threadIdx.x == 0) ssp_cal::tree(P, win, parent, edge_agree);
}

__global__ void __launch_bounds__(128) fuse_hyp_kernel(const Problem P) {
  if (ssp_cal::ctl(P)[ssp_cal::kStop] != 0.0) return;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // (o, h)
  if (id >= ssp_cal::num_obs(P) * P.C) return;
  ssp_cal::fuse_hyp(P, id / P.C, (int)(id % P.C));
}

__global__ void __launch_bounds__(128) fuse_obs_kernel(const Problem P, double* __restrict__ R_world, double* __restrict__ t_world,
                                                       unsigned char* __restrict__ views, double* __restrict__ view_err,
                                                       unsigned char* __restrict__ linked) {
  if (ssp_cal::ctl(P)[ssp_cal::kStop] != 0.0) return;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= ssp_cal::num_obs(P)) return;
  ssp_cal::fuse_obs(P, o, R_world + o * 9, t_world + o * 3, views + o * P.C, view_err + o * P.C, linked + o);
}

__global__ void __launch_bounds__(256) round_kernel(const Problem P, const double* __restrict__ R_world, const double* __restrict__ t_world,
                                                    int last) {
  __shared__ double red[ssp_cal::kLanes];
  __shared__ int changed, front;
  double* k = ssp_cal::ctl(P);
  if (k[ssp_cal::kStop] != 0.0) return;
  if (threadIdx.x == 0) { changed = k[ssp_cal::kRoundsRun] == 0.0; front = 1; }
  __syncthreads();
  const long long O = ssp_cal::num_obs(P);
  for (long long o = threadIdx.x; o < O; o += blockDim.x)
    if (ssp_cal::key_changed(P, o)) changed = 1;
  __syncthreads();
  if (!changed || last) {
    if (threadIdx.x == 0) k[ssp_cal::kStop] = 1.0;
    return;
  }
  for (long long o = threadIdx.x; o < O; o += blockDim.x) {
    ssp_cal::round_obs(P, o, R_world + o * 9, t_world + o * 3);
    if (ssp_cal::is_linked(P, o) && P.w[P.L.front_o + o] == 0.0) front = 0;
  }
  __syncthreads();
  const double cost = cta_tree_sum(red, ssp_cal::obs_partial(P, P.L.cost_o, threadIdx.x));
  if (threadIdx.x == 0) ssp_cal::round_start(P, cost, front != 0);
}

// one LM step's per-observation terms (cov != 0: the covariance's, at lambda = 0, run once after the steps)
__global__ void __launch_bounds__(128) obs_terms_kernel(const Problem P, int cov) {
  double* k = ssp_cal::ctl(P);
  if (cov ? k[ssp_cal::kStop] != 0.0 : halted(P)) return;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= ssp_cal::num_obs(P) || !ssp_cal::is_linked(P, o)) return;
  if (!ssp_cal::obs_terms(P, o, cov ? 0.0 : k[ssp_cal::kLam])) k[cov ? ssp_cal::kSingular : ssp_cal::kFail] = 1.0;
}

// one CTA per camera-block pair (c1 <= c2) of the free cameras: the fixed-order sums of its entries
__global__ void __launch_bounds__(256) block_kernel(const Problem P, int cov) {
  __shared__ double red[ssp_cal::kLanes];
  const double* k = ssp_cal::ctl(P);
  if (cov ? k[ssp_cal::kStop] != 0.0 : (halted(P) || k[ssp_cal::kFail] != 0.0)) return;
  int c1, c2;
  if ((int)blockIdx.x < P.C) { c1 = c2 = blockIdx.x; }
  else ssp_cal::pair_cams(P.C, blockIdx.x - P.C, &c1, &c2);
  const unsigned fr = ssp_cal::free_cams(P);
  if (!((fr >> c1) & 1u) || !((fr >> c2) & 1u)) return;
  for (int e = 0; e < ssp_cal::block_entries(c1, c2); e++) {
    const double s = cta_tree_sum(red, ssp_cal::block_partial(P, c1, c2, e, threadIdx.x));
    if (threadIdx.x == 0) *ssp_cal::block_slot(P, c1, c2, e) = s;
  }
}

// the reduced system S [n][n] at damping lam into shared A, factored by columns; false (to every thread) when a pivot fails
__device__ bool factor_reduced(const Problem& P, const int* cams, int n, double lam, double* A, int* ok) {
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) A[e] = ssp_cal::reduced_entry(P, cams, e / n, e % n, lam);
  if (threadIdx.x == 0) *ok = 1;
  __syncthreads();
  for (int j = 0; j < n; j++) {
    if (threadIdx.x == 0 && !ssp_cal::chol_pivot(A, n, j)) *ok = 0;
    __syncthreads();
    if (!*ok) return false;
    for (int i = j + 1 + threadIdx.x; i < n; i += blockDim.x) ssp_cal::chol_entry(A, n, j, i);
    __syncthreads();
  }
  return true;
}

__global__ void __launch_bounds__(256) factor_kernel(const Problem P) {
  extern __shared__ double A[];
  __shared__ int cams[SSP_RIG_MAX_VIEWS], ok;
  double* k = ssp_cal::ctl(P);
  if (halted(P) || k[ssp_cal::kFail] != 0.0) return;
  const int n = 6 * ssp_cal::free_list(P, cams);
  __syncthreads();
  if (!factor_reduced(P, cams, n, k[ssp_cal::kLam], A, &ok)) {
    if (threadIdx.x == 0) k[ssp_cal::kFail] = 1.0;
    return;
  }
  if (threadIdx.x != 0) return;
  double* dc = P.w + P.L.dcam;
  for (int i = 0; i < n; i++) dc[i] = P.w[P.L.rhs + cams[i / 6] * 6 + i % 6];
  ssp_cal::chol_subst(A, n, dc);
  ssp_cal::camera_candidates(P, cams, n, dc);
}

__global__ void __launch_bounds__(128) backsub_kernel(const Problem P) {
  if (halted(P) || ssp_cal::ctl(P)[ssp_cal::kFail] != 0.0) return;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= ssp_cal::num_obs(P) || !ssp_cal::is_linked(P, o)) return;
  int cams[SSP_RIG_MAX_VIEWS];
  const int n = 6 * ssp_cal::free_list(P, cams);
  ssp_cal::obs_step(P, o, cams, n);
}

__global__ void __launch_bounds__(256) accept_kernel(const Problem P) {
  __shared__ double red[ssp_cal::kLanes];
  __shared__ int front, take;
  if (halted(P)) return;
  if (threadIdx.x == 0) front = 1;
  __syncthreads();
  const long long O = ssp_cal::num_obs(P);
  for (long long o = threadIdx.x; o < O; o += blockDim.x)
    if (ssp_cal::is_linked(P, o) && P.w[P.L.front_o + o] == 0.0) front = 0;
  const double cost = cta_tree_sum(red, ssp_cal::obs_partial(P, P.L.cost_o, threadIdx.x));
  const double dn = cta_tree_sum(red, ssp_cal::obs_partial(P, P.L.dn_o, threadIdx.x));
  if (threadIdx.x == 0) {
    int cams[SSP_RIG_MAX_VIEWS];
    const int n = 6 * ssp_cal::free_list(P, cams);
    take = ssp_cal::accept(P, cams, n, cost, dn, front != 0);
  }
  __syncthreads();
  if (!take) return;
  for (long long o = threadIdx.x; o < O; o += blockDim.x)
    if (ssp_cal::is_linked(P, o))
      for (int j = 0; j < 12; j++) P.w[P.L.obs + o * 12 + j] = P.w[P.L.cand + o * 12 + j];
}

// the covariance of the free cameras: keypoint_sigma^2 times their blocks of S^-1 at lambda = 0, one column of S^-1 per thread
__global__ void __launch_bounds__(256) cov_kernel(const Problem P, double sigma, double* __restrict__ cam_cov) {
  extern __shared__ double A[];
  __shared__ int cams[SSP_RIG_MAX_VIEWS], ok;
  double* k = ssp_cal::ctl(P);
  if (k[ssp_cal::kStop] != 0.0) return;
  for (int e = threadIdx.x; e < P.C * 36; e += blockDim.x) cam_cov[e] = 0.0;
  const int n = 6 * ssp_cal::free_list(P, cams);
  __syncthreads();
  if (k[ssp_cal::kSingular] != 0.0) return;
  if (!factor_reduced(P, cams, n, 0.0, A, &ok)) {
    if (threadIdx.x == 0) k[ssp_cal::kSingular] = 1.0;
    return;
  }
  double* X = A + n * n;
  const double s2 = sigma * sigma;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    double* x = X + j * n;
    for (int i = 0; i < n; i++) x[i] = i == j ? 1.0 : 0.0;
    ssp_cal::chol_subst(A, n, x);
    const int c = cams[j / 6], b = j % 6;
    for (int a = 0; a < 6; a++) cam_cov[c * 36 + 6 * a + b] = s2 * x[(j / 6) * 6 + a];
  }
}

__global__ void __launch_bounds__(256) finish_kernel(const Problem P, const unsigned char* __restrict__ views, const double* __restrict__ view_err,
                                                     int* __restrict__ cam_obs, double* __restrict__ cam_rmse, int* __restrict__ cam_status,
                                                     int* __restrict__ rounds, int* __restrict__ iterations, double* __restrict__ cost) {
  __shared__ double red[ssp_cal::kLanes];
  const int c = blockIdx.x;
  const long long O = ssp_cal::num_obs(P);
  double cnt = 0.0, sum = 0.0;
  for (long long o = threadIdx.x; o < O; o += ssp_cal::kLanes)
    if (ssp_cal::is_linked(P, o) && views[o * P.C + c]) { cnt += 1.0; sum += view_err[o * P.C + c] * view_err[o * P.C + c]; }
  const double n = cta_tree_sum(red, cnt), s = cta_tree_sum(red, sum);
  if (threadIdx.x != 0) return;
  const double* k = ssp_cal::ctl(P);
  cam_obs[c] = (int)n;
  cam_rmse[c] = n > 0.0 ? sqrt(s / n) : -1.0;
  const unsigned conn = ssp_cal::connected(P), fr = ssp_cal::free_cams(P);
  cam_status[c] = (((conn >> c) & 1u) ? 0 : ssp_cal::kUnconnected) | (((fr >> c) & 1u) && k[ssp_cal::kSingular] != 0.0 ? ssp_cal::kSingularCov : 0);
  if (c == 0) { *rounds = (int)k[ssp_cal::kRoundsRun]; *iterations = (int)k[ssp_cal::kIters]; *cost = k[ssp_cal::kCost]; }
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }
static inline unsigned grid(long long n, int b) { return (unsigned)(n > 0 ? (n + b - 1) / b : 1); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_calibrate_rig_work_bytes(int groups, int views, int slots, long long* bytes_out) {
  if (!bytes_out || groups < 0 || views < 1 || views > ssp_mv::kMaxViews || slots < 1)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig_work_bytes: bad size (groups >= 0, 1 <= views <= 16, slots >= 1)");
  *bytes_out = ssp_cal::layout(groups, views, slots, ssp_mv::kMaxPoints).total * 8;
  return SSP_OK;
}

int ssp_calibrate_rig(const float* points3d, int points3d_shared, const float* points2d, const unsigned char* valid, int num_points, int groups,
                      int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null, int reference,
                      double gate, double reproj_thresh, double keypoint_sigma, int max_iter, double* R_rows, double* t_rows,
                      double* R_cam, double* t_cam, double* cam_cov, int* cam_obs, double* cam_rmse, int* tree_parent, int* edge_agree,
                      int* cam_status, double* R_world, double* t_world, unsigned char* views_out, double* view_err,
                      unsigned char* linked, int* rounds, int* iterations, double* cost, void* work, long long work_bytes, void* stream) {
  if (!points3d || !points2d || !valid || !K3x3_f32 || !K3x3 || !R_rows || !t_rows || !R_cam || !t_cam || !cam_cov || !cam_obs ||
      !cam_rmse || !tree_parent || !edge_agree || !cam_status || !R_world || !t_world || !views_out || !view_err || !linked || !rounds ||
      !iterations || !cost || !work)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig: null pointer");
  if (views < 1 || views > ssp_mv::kMaxViews || num_points < ssp_mv::kMinPoints || num_points > ssp_mv::kMaxPoints || groups < 0 ||
      slots < 1 || max_iter < 1)
    return fail_msg(SSP_ERR_ARG, "calibrate_rig: bad size (1 <= views <= 16, 7 <= points <= 10, groups >= 0, slots >= 1, max_iter >= 1)");
  if (reference < 0 || reference >= views) return fail_msg(SSP_ERR_ARG, "calibrate_rig: the reference camera must be in 0..views-1");
  if (!positive_finite(gate) || !positive_finite(reproj_thresh) || !positive_finite(keypoint_sigma))
    return fail_msg(SSP_ERR_ARG, "calibrate_rig: gate, reproj_thresh and keypoint_sigma must be > 0 and finite");
  if (gate < reproj_thresh) return fail_msg(SSP_ERR_ARG, "calibrate_rig: the gate must be >= reproj_thresh");
  const ssp_cal::Layout L = ssp_cal::layout(groups, views, slots, num_points);
  if (work_bytes < L.total * 8 || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "calibrate_rig: workspace smaller than ssp_calibrate_rig_work_bytes or not 8-B aligned");
  const long long rows = (long long)groups * views;
  const long long p3_stride = points3d_shared ? 0 : 3LL * num_points;
  double* w = (double*)work;
  cudaStream_t s = (cudaStream_t)stream;
  if (rows > 0) {
    const int rc = launch_fuse_rows(points3d, p3_stride, points2d, K3x3_f32, K3x3, dist8_or_null, num_points, views, slots, rows, max_iter,
                                    R_rows, t_rows, (float*)(w + L.corners), stream);
    if (rc != SSP_OK) return rc;
  }
  const Problem P = {points3d, p3_stride, points2d, valid, num_points, views, slots, reference, (long long)groups, K3x3_f32, dist8_or_null,
                     gate * gate, reproj_thresh * reproj_thresh, max_iter, R_rows, t_rows, R_cam, t_cam, w, L};
  const int np = ssp_cal::num_pairs(views);
  const long long O = (long long)groups * slots;
  const int n = 6 * (views - 1);
  const size_t smem_factor = (size_t)n * n * 8, smem_cov = (size_t)2 * n * n * 8;
  static bool attr = false;
  if (!attr) {
    const int most = 2 * 90 * 90 * 8;
    if (cudaFuncSetAttribute(factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, most) != cudaSuccess ||
        cudaFuncSetAttribute(cov_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, most) != cudaSuccess)
      SSP_CHECK_LAUNCH();
    attr = true;
  }
  pair_list_kernel<<<grid(np, 128), 128, 0, s>>>(P);
  SSP_CHECK_LAUNCH();
  pair_score_kernel<<<grid((long long)np * ssp_cal::kMaxPairHyp, 128), 128, 0, s>>>(P);
  SSP_CHECK_LAUNCH();
  tree_kernel<<<1, 128, 0, s>>>(P, tree_parent, edge_agree);
  SSP_CHECK_LAUNCH();
  for (int r = 0; r <= ssp_cal::kRounds; r++) {
    fuse_hyp_kernel<<<grid(O * views, 128), 128, 0, s>>>(P);
    SSP_CHECK_LAUNCH();
    fuse_obs_kernel<<<grid(O, 128), 128, 0, s>>>(P, R_world, t_world, views_out, view_err, linked);
    SSP_CHECK_LAUNCH();
    round_kernel<<<1, ssp_cal::kLanes, 0, s>>>(P, R_world, t_world, r == ssp_cal::kRounds);
    SSP_CHECK_LAUNCH();
    if (r == ssp_cal::kRounds) break;
    for (int it = 0; it < max_iter; it++) {
      obs_terms_kernel<<<grid(O, 128), 128, 0, s>>>(P, 0);
      SSP_CHECK_LAUNCH();
      block_kernel<<<views + np, ssp_cal::kLanes, 0, s>>>(P, 0);
      SSP_CHECK_LAUNCH();
      factor_kernel<<<1, ssp_cal::kLanes, smem_factor, s>>>(P);
      SSP_CHECK_LAUNCH();
      backsub_kernel<<<grid(O, 128), 128, 0, s>>>(P);
      SSP_CHECK_LAUNCH();
      accept_kernel<<<1, ssp_cal::kLanes, 0, s>>>(P);
      SSP_CHECK_LAUNCH();
    }
    obs_terms_kernel<<<grid(O, 128), 128, 0, s>>>(P, 1);
    SSP_CHECK_LAUNCH();
    block_kernel<<<views + np, ssp_cal::kLanes, 0, s>>>(P, 1);
    SSP_CHECK_LAUNCH();
    cov_kernel<<<1, ssp_cal::kLanes, smem_cov, s>>>(P, keypoint_sigma, cam_cov);
    SSP_CHECK_LAUNCH();
  }
  finish_kernel<<<views, ssp_cal::kLanes, 0, s>>>(P, views_out, view_err, cam_obs, cam_rmse, cam_status, rounds, iterations, cost);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
