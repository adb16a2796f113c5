// Host harness of the consensus PnP (singleshotpose_b200/csrc/pnp_consensus_core.h): the fan-out and the selection of the two kernels of
// pnp_consensus.cu as serial loops, on the same workspace layout.  Built with -ffp-contract=off so the scoring is rounded as the
// kernels round it.  Test infrastructure: built by tests/test_pnp_consensus_cpu.py into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/pnp_consensus_core.h"

using namespace ssp_pnpc;

extern "C" {
// steps 1-2 for n problems (points3d [n][np][3], or shared when shared != 0): slots [n][H+1][15] (R, rvec, t), hmask [n][H+1]
int h_consensus_hyps(const float* p3, int shared, const float* uv, const float* K, int np, long long n, const unsigned short* masks, int H,
                     double thr, int max_iter, double* slots, unsigned* hmask) {
  if (np < kMinPoints || np > kMaxPoints || !table_ok(masks, H, np) || !(thr > 0.0)) return -1;
  for (long long i = 0; i < n; i++)
    for (int h = 0; h <= H; h++)
      hmask[i * (H + 1) + h] = solve_hypothesis(h, masks, p3 + (shared ? 0 : i * 3 * np), uv + i * 2 * np, K, np, thr * thr, max_iter,
                                                slots + (i * (H + 1) + h) * kSlotDoubles);
  return 0;
}

// the whole rule; the arguments are those of ssp_pnp_consensus without the groups (host arrays)
int h_pnp_consensus(const float* p3, int shared, const float* uv, const float* K, int np, long long n, const unsigned short* masks, int H,
                    double thr, int max_iter, double* R, double* t, double* params, int* inliers, int* hyp) {
  if (np < kMinPoints || np > kMaxPoints || !table_ok(masks, H, np) || !(thr > 0.0)) return -1;
  std::vector<double> slots((H + 1) * kSlotDoubles);
  std::vector<unsigned> hm(H + 1);
  for (long long i = 0; i < n; i++) {
    const float* P = p3 + (shared ? 0 : i * 3 * np);
    const float* q = uv + i * 2 * np;
    for (int h = 0; h <= H; h++) hm[h] = solve_hypothesis(h, masks, P, q, K, np, thr * thr, max_iter, slots.data() + h * kSlotDoubles);
    const int best = select(hm.data(), 1, H + 1);
    const unsigned inl = best < 0 ? 0u : hm[best];
    finish(best, inl, slots.data() + (best < 0 ? 0 : best) * kSlotDoubles, slots.data(), masks, P, q, K, np, max_iter, R + i * 9,
           t + i * 3, params + i * 6);
    inliers[i] = (int)inl;
    hyp[i] = best;
  }
  return 0;
}

// the plain solve of ssp_pnp_batched (pnp_solve_one as pnp_kernel calls it), for the invariant
int h_pnp_plain(const float* p3, int shared, const float* uv, const float* K, int np, long long n, int max_iter, double* R, double* t) {
  int work[3];
  for (long long i = 0; i < n; i++)
    ssp_pnp::pnp_solve_one(p3 + (shared ? 0 : i * 3 * np), uv + i * 2 * np, K, np, max_iter, R + i * 9, t + i * 3, work);
  return 0;
}
}
