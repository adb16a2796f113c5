// Host harness of PnP and projection with lens distortion: pnp_core.h (pnp_solve_one's dist, undistort, project_distorted) and
// pnp_consensus_core.h (score's dist) compiled with g++ -ffp-contract=off, the loops of the kernels of pnp_dist.cu run serially.
// Test infrastructure: built by tests/test_pnp_dist_cpu.py into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/pnp_consensus_core.h"

using namespace ssp_pnpc;

extern "C" {
// ssp_pnp_dist without groups: n problems, guess (n x 6) or null (with use_guess), params (n x 6) or null; dist null is the plain solve
int h_pnp_dist(const float* p3, int shared, const float* uv, const float* K, const double* dist, int np, long long n, int max_iter,
               const double* guess, const int* use_guess, double* R, double* t, double* params, int* work) {
  if (np < 6 || np > PNP_MAXP) return -1;
  for (long long i = 0; i < n; i++)
    ssp_pnp::pnp_solve_one(p3 + (shared ? 0 : i * 3 * np), uv + i * 2 * np, K, np, max_iter, R + i * 9, t + i * 3, work + i * 3, nullptr,
                           guess && use_guess[i] ? guess + i * 6 : nullptr, params ? params + i * 6 : nullptr, dist);
  return 0;
}

// cv2.undistortPoints of n pixels uv [n][2] (fp64) -> xy [n][2]
int h_undistort(const double* uv, long long n, const float* K, const double* dist, double* xy) {
  for (long long i = 0; i < n; i++) ssp_pnp::undistort(dist, uv[2 * i], uv[2 * i + 1], K[0], K[4], K[2], K[5], xy + 2 * i, xy + 2 * i + 1);
  return 0;
}

// cv2.projectPoints of X [nv][3] under n poses Rt [n][3][4] with K [9] fp64 -> out [n][2][nv] fp32 (ssp_project_points_dist's layout)
int h_project_dist(const float* X, int nv, const double* Rt, const double* K, const double* dist, long long n, float* out) {
  for (long long b = 0; b < n; b++)
    for (int v = 0; v < nv; v++) {
      const double* T = Rt + b * 12;
      const double x0 = X[3 * v], y0 = X[3 * v + 1], z0 = X[3 * v + 2];
      double u, w;
      ssp_pnp::project_distorted(dist, T[0] * x0 + T[1] * y0 + T[2] * z0 + T[3], T[4] * x0 + T[5] * y0 + T[6] * z0 + T[7],
                                 T[8] * x0 + T[9] * y0 + T[10] * z0 + T[11], K[0], K[4], K[2], K[5], &u, &w);
      out[(b * 2) * nv + v] = (float)u;
      out[(b * 2 + 1) * nv + v] = (float)w;
    }
  return 0;
}

// the consensus rule with distortion for n problems (ssp_pnp_consensus_dist without the groups; host arrays)
int h_pnp_consensus_dist(const float* p3, int shared, const float* uv, const float* K, const double* dist, int np, long long n,
                         const unsigned short* masks, int H, double thr, int max_iter, double* R, double* t, double* params, int* inliers,
                         int* hyp) {
  if (np < kMinPoints || np > kMaxPoints || !table_ok(masks, H, np) || !(thr > 0.0)) return -1;
  std::vector<double> slots((H + 1) * kSlotDoubles);
  std::vector<unsigned> hm(H + 1);
  for (long long i = 0; i < n; i++) {
    const float* P = p3 + (shared ? 0 : i * 3 * np);
    const float* q = uv + i * 2 * np;
    for (int h = 0; h <= H; h++)
      hm[h] = solve_hypothesis(h, masks, P, q, K, np, thr * thr, max_iter, slots.data() + h * kSlotDoubles, dist);
    const int best = select(hm.data(), 1, H + 1);
    const unsigned inl = best < 0 ? 0u : hm[best];
    finish(best, inl, slots.data() + (best < 0 ? 0 : best) * kSlotDoubles, slots.data(), masks, P, q, K, np, max_iter, R + i * 9,
           t + i * 3, params + i * 6, dist);
    inliers[i] = (int)inl;
    hyp[i] = best;
  }
  return 0;
}
}
