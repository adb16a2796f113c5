// Consensus PnP of ONE problem: a pose that survives wrong keypoints (a hidden corner, one off the frame, one taken from a neighbouring
// instance), where the plain solve (pnp_core.h) fits all points and one bad point drags the whole pose with it.
// SSP_HD: compiled by nvcc into the kernels of pnp_consensus.cu and by g++ (-ffp-contract=off) into tests/helpers/pnp_consensus_host.cpp.
//
// Inputs: np object points (7 <= np <= 10), np pixel points, K, a threshold thr in pixels (> 0, finite), max_iter, and a table of H
// subset masks (1 <= H <= 210), each with exactly 6 distinct bits below np; the table's order is the tie-break order
// (utils.consensus_subsets lists the 6-subsets in lexicographic order and drops those where the DLT is degenerate).
//   1. Hypotheses.  Hypothesis 0 is the cold solve on all np points: pnp_solve_one exactly as ssp_pnp_batched runs it.  Hypothesis
//      h >= 1 is the cold solve on the 6 points of mask h-1 in ascending index order, cv2.solvePnP(P[S], uv[S], K, None, ITERATIVE).
//   2. Score.  From each hypothesis's final LM vector (rvec, t), with R = rodrigues(rvec) as the solve returns it, every one of the np
//      points gets its camera depth z and squared pixel error, in fp64 with each operation rounded on its own, in this order:
//        x = ((R0*X + R1*Y) + R2*Z) + t0,  y = ((R3*X + R4*Y) + R5*Z) + t1,  z = ((R6*X + R7*Y) + R8*Z) + t2,
//        iz = 1/z,  du = ((fx*x)*iz + cx) - u,  dv = ((fy*y)*iz + cy) - v,  e2 = du*du + dv*dv   (reproj_err's arithmetic).
//      Depth rule: if any point has z <= 0 the hypothesis has no inliers.  The box points are centrally symmetric, so a 6-point
//      solve often lands on the mirrored pose behind the camera, which reprojects every point within a pixel or two.
//      Otherwise point i is an inlier when e2 <= thr*thr (cv2's RANSAC comparison).
//   3. Select the hypothesis with the most inliers, the lower index on a tie (integers only); hyp = -1 when every one has none.
//   4. Result: hyp == -1: hypothesis 0's pose, empty mask.  Inliers == the hypothesis's own point set: its pose, unchanged.
//      Otherwise, >= 6 inliers: a warm LM on the inliers in ascending order from the hypothesis's LM vector,
//      cv2.solvePnP(P[inl], uv[inl], K, None, rvec, tvec, useExtrinsicGuess=True).  Otherwise: the hypothesis's pose, unrefined.
//   Out: R, t, the final LM vector, the inlier mask of the chosen hypothesis (bit i = point i) and hyp.
// Invariant: when hypothesis 0 has all np points as inliers, the result is bit-identical to ssp_pnp_batched.
// With distortion coefficients (dist, 8 values, or null) every solve is cv2.solvePnP(..., distCoeffs) (pnp_solve_one's dist) and step
// 2 scores the distorted reprojection (score); the rule is otherwise the same.
#pragma once
#include "pnp_core.h"

namespace ssp_pnpc {

constexpr int kMinPoints = 7, kMaxPoints = 10, kSubsetSize = 6, kMaxSubsets = 210;
constexpr int kSlotDoubles = 15;        // per hypothesis in the workspace: R[9], then the final LM vector (rvec, t)

// workspace: slots [n][H+1][15] fp64, then masks [n][H+1] uint32; a multiple of 8 B, so that a buffer of fp64 elements fits it exactly
SSP_HD long long work_bytes(int H, long long n) { return (n * (H + 1) * (kSlotDoubles * 8 + 4) + 7) / 8 * 8; }

SSP_HD double mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
SSP_HD double add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SSP_HD double sub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
SSP_HD double rcp(double a) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(1.0, a);
#else
  return 1.0 / a;
#endif
}

SSP_HD int popc(unsigned v) {
  int n = 0;
  for (; v; v &= v - 1) n++;
  return n;
}

// the table is valid for np points: 1 <= H <= 210, every mask has 6 bits, all below np (distinct bits are a property of a bitmask)
SSP_HD bool table_ok(const unsigned short* masks, int H, int np) {
  if (H < 1 || H > kMaxSubsets) return false;
  for (int h = 0; h < H; h++)
    if (popc(masks[h]) != kSubsetSize || (masks[h] >> np) != 0) return false;
  return true;
}

// the point set of hypothesis h (0: all np points)
SSP_HD unsigned hyp_set(int h, const unsigned short* masks, int np) { return h == 0 ? (1u << np) - 1u : (unsigned)masks[h - 1]; }

// the points of `set` in ascending index order -> p3s [n][3], uvs [n][2]; returns n
SSP_HD int gather(const float* p3, const float* uv, int np, unsigned set, float* p3s, float* uvs) {
  int n = 0;
  for (int i = 0; i < np; i++) {
    if (!((set >> i) & 1u)) continue;
    p3s[3 * n] = p3[3 * i]; p3s[3 * n + 1] = p3[3 * i + 1]; p3s[3 * n + 2] = p3[3 * i + 2];
    uvs[2 * n] = uv[2 * i]; uvs[2 * n + 1] = uv[2 * i + 1];
    n++;
  }
  return n;
}

// cv2.projectPoints' lens model (ssp_pnp::distort) with every operation rounded on its own, in the written order
SSP_HD void distort_rn(const double* k, double x, double y, double* xd, double* yd) {
  const double r2 = add(mul(x, x), mul(y, y)), r4 = mul(r2, r2), r6 = mul(r4, r2);
  const double a1 = mul(mul(2.0, x), y), a2 = add(r2, mul(mul(2.0, x), x)), a3 = add(r2, mul(mul(2.0, y), y));
  const double cdist = add(add(add(1.0, mul(k[0], r2)), mul(k[1], r4)), mul(k[4], r6));
  const double icdist2 = rcp(add(add(add(1.0, mul(k[5], r2)), mul(k[6], r4)), mul(k[7], r6)));
  *xd = add(add(mul(mul(x, cdist), icdist2), mul(k[2], a1)), mul(k[3], a2));
  *yd = add(add(mul(mul(y, cdist), icdist2), mul(k[2], a3)), mul(k[3], a1));
}

// step 2: the inlier mask of the pose (R, t) over all np points, 0 if a point has z <= 0.  dist (8, or null): the distorted
// reprojection, xn = x*iz, yn = y*iz, (xd, yd) = distort_rn(xn, yn), du = (xd*fx + cx) - u, dv = (yd*fy + cy) - v
SSP_HD unsigned score(const double R[9], const double t[3], const float* p3, const float* uv, const float* Kmat, int np, double thr2,
                      const double* dist = nullptr) {
  const double fx = Kmat[0], fy = Kmat[4], cx = Kmat[2], cy = Kmat[5];
  unsigned mask = 0;
  for (int i = 0; i < np; i++) {
    const double X = p3[3 * i], Y = p3[3 * i + 1], Z = p3[3 * i + 2];
    const double x = add(add(add(mul(R[0], X), mul(R[1], Y)), mul(R[2], Z)), t[0]);
    const double y = add(add(add(mul(R[3], X), mul(R[4], Y)), mul(R[5], Z)), t[1]);
    const double z = add(add(add(mul(R[6], X), mul(R[7], Y)), mul(R[8], Z)), t[2]);
    if (!(z > 0.0)) return 0u;
    const double iz = rcp(z);
    if (dist) {
      double xd, yd;
      distort_rn(dist, mul(x, iz), mul(y, iz), &xd, &yd);
      const double du = sub(add(mul(xd, fx), cx), (double)uv[2 * i]);
      const double dv = sub(add(mul(yd, fy), cy), (double)uv[2 * i + 1]);
      if (add(mul(du, du), mul(dv, dv)) <= thr2) mask |= 1u << i;
      continue;
    }
    const double du = sub(add(mul(mul(fx, x), iz), cx), (double)uv[2 * i]);
    const double dv = sub(add(mul(mul(fy, y), iz), cy), (double)uv[2 * i + 1]);
    if (add(mul(du, du), mul(dv, dv)) <= thr2) mask |= 1u << i;
  }
  return mask;
}

// steps 1-2 for hypothesis h: slot [15] = R, (rvec, t); returns its inlier mask
SSP_HD unsigned solve_hypothesis(int h, const unsigned short* masks, const float* p3, const float* uv, const float* Kmat, int np,
                                 double thr2, int max_iter, double* slot, const double* dist = nullptr) {
  int work[3];
  double* R = slot;
  double* p = slot + 9;
  // one call site for every h (hypothesis 0 gathers all points, the same values): two inlined solves would double the spills
  float p3s[3 * kMaxPoints], uvs[2 * kMaxPoints];
  const int n = gather(p3, uv, np, hyp_set(h, masks, np), p3s, uvs);
  ssp_pnp::pnp_solve_one(p3s, uvs, Kmat, n, max_iter, R, p + 3, work, nullptr, nullptr, p, dist);
  return score(R, p + 3, p3, uv, Kmat, np, thr2, dist);
}

// step 3 over the H + 1 masks of the hypotheses (stride apart)
SSP_HD int select(const unsigned* hmask, int stride, int H1) {
  int best = -1, best_n = 0;
  for (int h = 0; h < H1; h++) {
    const int n = popc(hmask[(long long)h * stride]);
    if (n > best_n) { best = h; best_n = n; }
  }
  return best;
}

// step 4 for the chosen hypothesis `hyp` (its inlier mask `inl`, slot = its workspace entry; slot0 = hypothesis 0's).
// Writes R [9], t [3], params [6]
SSP_HD void finish(int hyp, unsigned inl, const double* slot, const double* slot0, const unsigned short* masks, const float* p3,
                   const float* uv, const float* Kmat, int np, int max_iter, double* R_out, double* t_out, double* params_out,
                   const double* dist = nullptr) {
  const double* src = hyp < 0 ? slot0 : slot;
  if (hyp >= 0 && inl != hyp_set(hyp, masks, np) && popc(inl) >= kSubsetSize) {
    float p3s[3 * kMaxPoints], uvs[2 * kMaxPoints];
    const int n = gather(p3, uv, np, inl, p3s, uvs);
    int work[3];
    ssp_pnp::pnp_solve_one(p3s, uvs, Kmat, n, max_iter, R_out, t_out, work, nullptr, slot + 9, params_out, dist);
    return;
  }
  for (int i = 0; i < 9; i++) R_out[i] = src[i];
  for (int i = 0; i < 6; i++) params_out[i] = src[9 + i];
  for (int i = 0; i < 3; i++) t_out[i] = src[12 + i];
}

}  // namespace ssp_pnpc

namespace ssp {
struct SubsetTable { unsigned short m[ssp_pnpc::kMaxSubsets]; };       // the subset table, by value in the kernels' launch parameters
}  // namespace ssp
