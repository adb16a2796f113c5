// Host harness of the ADD-S / ADD / diameter rules of adds_core.h, driven the way adds_kernel and diameter_kernel (adds.cu)
// drive them, with plain loops: the same queries per thread, the same per-thread order, the same reduction tree and the same
// block order.  Test infrastructure: built by tests/test_adds_cpu.py into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/adds_core.h"

using namespace ssp_adds;

extern "C" {
// X [nv][3]; Rt_est, Rt_gt [n][3][4]; adds_out, add_out [n]
int h_adds_batched(const double* X, int nv, const double* Rt_est, const double* Rt_gt, long long n, double* adds_out, double* add_out) {
  if (nv < 1 || nv > kMaxVertices || n < 0) return -1;
  const int nblk = query_blocks(nv);
  std::vector<double> sums_adds(nblk), sums_add(nblk), red_adds(kThreads), red_add(kThreads);
  for (long long p = 0; p < n; p++) {
    const double* est = Rt_est + 12 * p;
    const double* gt = Rt_gt + 12 * p;
    for (int blk = 0; blk < nblk; blk++) {
      for (int t = 0; t < kThreads; t++) {
        double adds = 0.0, add = 0.0;
        for (int k = 0; k < kQueriesPerThread; k++) {
          const int i = query_index(blk, k, t);
          if (i >= nv) continue;
          const double* x = X + 3LL * i;
          double q[3];
          model_frame_query(est, gt, x[0], x[1], x[2], q);
          add = add + sqrt(sq_dist(q, x[0], x[1], x[2]));
          double m = INFINITY;
          for (int j = 0; j < nv; j++) m = fmin(m, sq_dist(q, X[3LL * j], X[3LL * j + 1], X[3LL * j + 2]));
          adds = adds + sqrt(m);
        }
        red_adds[t] = adds;
        red_add[t] = add;
      }
      for (int stride = kThreads / 2; stride > 0; stride >>= 1)
        for (int t = 0; t < stride; t++) { tree_step(red_adds.data(), t, stride); tree_step(red_add.data(), t, stride); }
      sums_adds[blk] = red_adds[0];
      sums_add[blk] = red_add[0];
    }
    adds_out[p] = finish_mean(sums_adds.data(), nblk, nv);
    add_out[p] = finish_mean(sums_add.data(), nblk, nv);
  }
  return 0;
}

double h_mesh_diameter(const double* X, int nv) {
  double best = 0.0;
  for (int i = 0; i < nv; i++)
    for (int j = i; j < nv; j++) {
      const double d = diameter_sq(X[3LL * i] - X[3LL * j], X[3LL * i + 1] - X[3LL * j + 1], X[3LL * i + 2] - X[3LL * j + 2]);
      if (d > best) best = d;
    }
  return sqrt(best);
}
}
