// Consensus PnP over keypoint subsets (rule: pnp_consensus_core.h).  Two launches:
//   pnp_hyp_kernel     one thread per (problem, hypothesis): the cold solve of hypothesis h and its inlier mask, into the workspace;
//   pnp_select_kernel  one thread per problem: the selection over the H + 1 masks and, when the inliers differ from the chosen
//                      hypothesis's own points, the warm LM on the inliers.
// The hypotheses of a problem are neighbours in the thread order, so the fan-out runs them side by side: the consensus solve costs
// about two LM latencies, not H + 1.  The subset table (<= 210 uint16) travels by value in the launch parameters, so a captured
// graph keeps its own copy.  Counted groups as in ssp_pnp_batched_counted: problem (g, m) with m >= count[g] does no work and gets zeros.
#include <math.h>

#include "ssp_common.cuh"
#include "pnp_consensus_core.h"

namespace ssp {


__global__ void __launch_bounds__(128) pnp_hyp_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                      const float* __restrict__ Kmat, int np, long long n, int max_iter, double thr2,
                                                      const SubsetTable tab, int H1, const int* __restrict__ count, int per_group,
                                                      double* __restrict__ slots, unsigned* __restrict__ hmask) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n * H1) return;
  const long long i = id / H1;
  const int h = (int)(id - i * H1);
  if (count && i % per_group >= count[i / per_group]) return;
  hmask[id] = ssp_pnpc::solve_hypothesis(h, tab.m, P3 + i * p3_stride, uv + i * 2 * np, Kmat, np, thr2, max_iter,
                                         slots + id * ssp_pnpc::kSlotDoubles);
}

__global__ void __launch_bounds__(128) pnp_select_kernel(const float* __restrict__ P3, long long p3_stride, const float* __restrict__ uv,
                                                         const float* __restrict__ Kmat, int np, long long n, int max_iter,
                                                         const SubsetTable tab, int H1, const int* __restrict__ count, int per_group,
                                                         const double* __restrict__ slots, const unsigned* __restrict__ hmask,
                                                         double* __restrict__ R_out, double* __restrict__ t_out,
                                                         double* __restrict__ params_out, int* __restrict__ inliers_out,
                                                         int* __restrict__ hyp_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (count && i % per_group >= count[i / per_group]) {
    for (int k = 0; k < 9; k++) R_out[i * 9 + k] = 0.0;
    for (int k = 0; k < 3; k++) t_out[i * 3 + k] = 0.0;
    for (int k = 0; k < 6; k++) params_out[i * 6 + k] = 0.0;
    inliers_out[i] = 0;
    hyp_out[i] = 0;
    return;
  }
  const unsigned* hm = hmask + i * H1;
  const int hyp = ssp_pnpc::select(hm, 1, H1);
  const unsigned inl = hyp < 0 ? 0u : hm[hyp];
  const double* s0 = slots + i * H1 * ssp_pnpc::kSlotDoubles;
  ssp_pnpc::finish(hyp, inl, s0 + (hyp < 0 ? 0 : hyp) * ssp_pnpc::kSlotDoubles, s0, tab.m, P3 + i * p3_stride, uv + i * 2 * np, Kmat, np,
                   max_iter, R_out + i * 9, t_out + i * 3, params_out + i * 6);
  inliers_out[i] = (int)inl;
  hyp_out[i] = hyp;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_pnp_consensus_work_bytes(int num_points, int n_subsets, long long n, long long* bytes_out) {
  if (!bytes_out || num_points < ssp_pnpc::kMinPoints || num_points > ssp_pnpc::kMaxPoints || n_subsets < 1 || n_subsets > ssp_pnpc::kMaxSubsets || n < 0)
    return fail_msg(SSP_ERR_ARG, "pnp_consensus_work_bytes: bad size (7 <= points <= 10, 1 <= subsets <= 210, n >= 0)");
  *bytes_out = ssp_pnpc::work_bytes(n_subsets, n);
  return SSP_OK;
}

int ssp_pnp_consensus(const float* P3, int shared, const float* uv, const float* K, int np, int groups, int per_group, const int* count,
                      const unsigned short* subsets, int H, double thr, int max_iter, double* R, double* t, double* params, int* inliers,
                      int* hyp, void* work, long long work_bytes, void* stream) {
  if (!P3 || !uv || !K || !subsets || !R || !t || !params || !inliers || !hyp || !work || np < ssp_pnpc::kMinPoints ||
      np > ssp_pnpc::kMaxPoints || groups < 0 || per_group < 1)
    return fail_msg(SSP_ERR_ARG, "pnp_consensus: bad argument (null pointer, points outside 7..10, groups < 0 or per_group < 1)");
  if (!ssp_pnpc::table_ok(subsets, H, np))
    return fail_msg(SSP_ERR_ARG, "pnp_consensus: bad subset table (1..210 masks of exactly 6 bits below the point count)");
  if (!(thr > 0.0) || !isfinite(thr)) return fail_msg(SSP_ERR_ARG, "pnp_consensus: the threshold must be > 0 and finite");
  if (max_iter < 1) return fail_msg(SSP_ERR_ARG, "pnp_consensus: max_iter must be >= 1");
  const long long n = (long long)groups * per_group;
  if (work_bytes < ssp_pnpc::work_bytes(H, n) || ((unsigned long long)work & 7u))
    return fail_msg(SSP_ERR_ARG, "pnp_consensus: workspace smaller than ssp_pnp_consensus_work_bytes or not 8-B aligned");
  if (n == 0) return SSP_OK;
  SubsetTable tab = {};
  for (int h = 0; h < H; h++) tab.m[h] = subsets[h];
  const int H1 = H + 1;
  const long long stride = shared ? 0 : 3LL * np;
  double* slots = (double*)work;
  unsigned* hmask = (unsigned*)(slots + n * H1 * ssp_pnpc::kSlotDoubles);
  cudaStream_t s = (cudaStream_t)stream;
  const long long nh = n * H1;
  pnp_hyp_kernel<<<(unsigned)((nh + 127) / 128), 128, 0, s>>>(P3, stride, uv, K, np, n, max_iter, thr * thr, tab, H1, count, per_group,
                                                              slots, hmask);
  SSP_CHECK_LAUNCH();
  pnp_select_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(P3, stride, uv, K, np, n, max_iter, tab, H1, count, per_group, slots,
                                                                hmask, R, t, params, inliers, hyp);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
