// ADD-S (the reference's adi, utils.py:60-64 and multi_obj_pose_estimation/utils_multi.py:66-70) and the mesh diameter
// (calc_pts_diameter, utils.py:50-58): the arithmetic shared by the kernels of adds.cu and the CPU test harness
// (tests/helpers/adds_host.cpp, built with g++).
//
// ADD-S of a pose pair p over a mesh X (Nv vertices, fp64):
//     adds[p] = mean_i min_j || Rt_gt[p] x_i - Rt_est[p] x_j ||
// i.e. adi(pts_est, pts_gt): the nearest-neighbour structure is on the ESTIMATED points, queried with the ground-truth points.
// Both sides are rotated into the estimate's model frame, q_i = R_est^T (R_gt x_i + t_gt - t_est), so that every pose pair
// compares its queries with the same untransformed mesh (the rotation keeps distances).  The same q_i gives the ADD term of
// vertex i, || q_i - x_i || = || Rt_gt x_i - Rt_est x_i ||, at no extra pass over the mesh.
//
// Order of the sums (fixed, so that a pose's result depends on nothing but its own inputs and Nv): queries are grouped in
// blocks of kQueriesPerBlock; within a block thread t owns queries t, t + kThreads, ... and adds their distances in that
// order; the kThreads thread sums are reduced by tree_step with strides kThreads/2, ..., 1; the block sums are added in
// block order by finish_mean, which divides by Nv.
//
// Diameter: the largest squared distance over all vertex pairs, each computed as (dx*dx + dy*dy) + dz*dz with every product
// and sum rounded separately -- the operation sequence of numpy's (d * d).sum(axis=1) on an (n, 3) array -- then one sqrt.
// The maximum does not depend on the order of the pairs, and sqrt is monotonic, so the result is bit-identical to
// calc_pts_diameter on float64 input.
#pragma once
#include <math.h>
#if defined(__CUDACC__)
#define SSP_ADDS_HD __host__ __device__ __forceinline__
#else
#define SSP_ADDS_HD inline
#endif

namespace ssp_adds {

constexpr int kThreads = 256;                                    // threads of a query block
constexpr int kQueriesPerThread = 4;
constexpr int kQueriesPerBlock = kThreads * kQueriesPerThread;
constexpr int kTile = 256;                                       // mesh vertices per shared-memory tile
constexpr int kMaxVertices = 1 << 20;                            // SSP_ADDS_MAX_VERTICES

SSP_ADDS_HD int query_blocks(int nv) { return (nv + kQueriesPerBlock - 1) / kQueriesPerBlock; }
SSP_ADDS_HD int query_index(int block, int k, int t) { return block * kQueriesPerBlock + k * kThreads + t; }

// q = R_est^T (R_gt x + (t_gt - t_est)); est, gt are row-major [3][4] [R | t]
SSP_ADDS_HD void model_frame_query(const double* est, const double* gt, double x, double y, double z, double* q) {
  double c[3];
  for (int r = 0; r < 3; r++) c[r] = fma(gt[4 * r], x, fma(gt[4 * r + 1], y, fma(gt[4 * r + 2], z, gt[4 * r + 3] - est[4 * r + 3])));
  for (int r = 0; r < 3; r++) q[r] = fma(est[r], c[0], fma(est[4 + r], c[1], est[8 + r] * c[2]));
}

SSP_ADDS_HD double sq_dist(const double* q, double px, double py, double pz) {
  const double dx = q[0] - px, dy = q[1] - py, dz = q[2] - pz;
  return fma(dx, dx, fma(dy, dy, dz * dz));
}

// (dx*dx + dy*dy) + dz*dz without contraction into FMAs
SSP_ADDS_HD double diameter_sq(double dx, double dy, double dz) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
#else
  volatile double xx = dx * dx, yy = dy * dy, zz = dz * dz;    // volatile: separate roundings whatever -ffp-contract says
  volatile double s = xx + yy;
  return s + zz;
#endif
}

// one level of the block's fixed reduction tree: s[t] += s[t + stride] for t < stride
SSP_ADDS_HD void tree_step(double* s, int t, int stride) { s[t] = s[t] + s[t + stride]; }

// the block sums of one pose, added in block order, over Nv
SSP_ADDS_HD double finish_mean(const double* block_sums, int nblk, int nv) {
  double s = block_sums[0];
  for (int b = 1; b < nblk; b++) s = s + block_sums[b];
  return s / (double)nv;
}

}  // namespace ssp_adds
