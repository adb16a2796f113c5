// PnP pose recovery of ONE problem -- cv2.solvePnP(SOLVEPNP_ITERATIVE) + cv2.Rodrigues restated in fp64 (reference utils.py:86-100).
// SSP_HD: the same source is compiled by nvcc into pnp_kernel (pnp.cu, one problem per thread) and by g++ into the CPU test harness
// (tests/helpers/pnp_host.cpp), where it is checked against the reference-generated goldens without a GPU.
//   1. normalise the 2-D points with K (zero distortion);
//   2. DLT initialisation exactly as cvFindExtrinsicCameraParams2 poses it: the 2N x 12 system on the RAW 3-D coordinates,
//      unit-norm constraint over all 12 entries, i.e. the eigenvector of the smallest eigenvalue of the 12x12 normal matrix
//      L^T L = [[S, 0, -Sx], [0, S, -Sy], [-Sx, -Sy, Sq]] (S = sum XX^T, Sx = sum x XX^T, ..., X = [X Y Z 1]); cyclic Jacobi in fp64;
//   3. nearest rotation by polar decomposition, OpenCV's scale fix for t, Rodrigues -> rvec;
//   4. Levenberg-Marquardt in pixel space with OpenCV's CvLevMarq schedule (lambda = 10^k, k0 = -3, diagonal scaling (1+lambda),
//      reject => k++, accept => k--, <= max_iter accepted steps, eps = FLT_EPSILON).
#pragma once
#include <math.h>
#if defined(__CUDACC__)
#define SSP_HD __host__ __device__ inline
#else
#define SSP_HD inline
#endif

namespace ssp_pnp {

#define PNP_MAXP 16

SSP_HD void rodrigues(const double r[3], double R[9], double* J /*27 or null: dR[k]/dr[i] at J[i*9+k]*/) {
  const double th = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
  if (th < 2.220446049250313e-16) {
    for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (J) {
      for (int i = 0; i < 27; i++) J[i] = 0.0;
      J[5] = -1; J[7] = 1; J[9 + 2] = 1; J[9 + 6] = -1; J[18 + 1] = -1; J[18 + 3] = 1;
    }
    return;
  }
  const double c = cos(th), s = sin(th), c1 = 1.0 - c, it = 1.0 / th;
  const double u[3] = {r[0] * it, r[1] * it, r[2] * it};
  const double rrt[9] = {u[0] * u[0], u[0] * u[1], u[0] * u[2], u[1] * u[0], u[1] * u[1], u[1] * u[2], u[2] * u[0], u[2] * u[1], u[2] * u[2]};
  const double rx[9] = {0, -u[2], u[1], u[2], 0, -u[0], -u[1], u[0], 0};
  for (int k = 0; k < 9; k++) R[k] = c * ((k % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[k] + s * rx[k];
  if (!J) return;
  for (int i = 0; i < 3; i++) {
    double drrt[9], drx[9];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) drrt[a * 3 + b] = (a == i ? u[b] : 0.0) + (b == i ? u[a] : 0.0);
    for (int k = 0; k < 9; k++) drx[k] = 0.0;
    if (i == 0) { drx[5] = -1; drx[7] = 1; } else if (i == 1) { drx[2] = 1; drx[6] = -1; } else { drx[1] = -1; drx[3] = 1; }
    const double ri = u[i];
    const double a0 = -s * ri, a1 = (s - 2 * c1 * it) * ri, a2 = c1 * it, a3 = (c - s * it) * ri, a4 = s * it;
    for (int k = 0; k < 9; k++)
      J[i * 9 + k] = a0 * ((k % 4 == 0) ? 1.0 : 0.0) + a1 * rrt[k] + a2 * drrt[k] + a3 * rx[k] + a4 * drx[k];
  }
}

// cyclic Jacobi on a symmetric n x n matrix: A -> diag, V = eigenvectors (columns); returns the number of sweeps.
// Works on the upper triangle only, each rotation through scalar temporaries (the textbook form: the pivot is set to zero and
// the diagonal updated by t*a_pq exactly, symmetry cannot drift), loops kept rolled.  The two-sided form that rotates whole columns and then whole rows in place (jacobi_eig_twosided
// below) is right on the host and as device code at -O0, but as -O3 device code for n = 12 it does not
// converge (128 of 128 problems wrong, negative "eigenvalues" of a PSD matrix, with and without -fmad=false).  The same arithmetic
// with `#pragma unroll 1` on the two pivot loops (variant 1) is right again: nvcc 12.9's unrolling of the pivot loop over the
// overlapping column / row updates is what breaks it.  Variant 2 (this function) is the default.
#ifndef PNP_JACOBI_VARIANT
#define PNP_JACOBI_VARIANT 2
#endif
#if defined(__CUDACC__)
#define PNP_ROLLED _Pragma("unroll 1")
#else
#define PNP_ROLLED
#endif
template <int n>
SSP_HD int jacobi_eig_upper(double A[n][n], double V[n][n]) {
  PNP_ROLLED
  for (int i = 0; i < n; i++) {
    PNP_ROLLED
    for (int j = 0; j < n; j++) V[i][j] = (i == j) ? 1.0 : 0.0;
  }
  int sweep = 0;
  PNP_ROLLED
  for (; sweep < 30; sweep++) {
    double off = 0.0, diag = 0.0;
    PNP_ROLLED
    for (int i = 0; i < n; i++) {
      diag += A[i][i] * A[i][i];
      PNP_ROLLED
      for (int j = i + 1; j < n; j++) off += A[i][j] * A[i][j];
    }
    if (off <= 1e-34 * diag || off == 0.0) break;
    PNP_ROLLED
    for (int p = 0; p < n - 1; p++) {
      PNP_ROLLED
      for (int q = p + 1; q < n; q++) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        A[p][p] -= t * apq; A[q][q] += t * apq; A[p][q] = 0.0;
        PNP_ROLLED
        for (int k = 0; k < n; k++) {
          if (k != p && k != q) {
            // element (k, p) and (k, q) of the symmetric matrix, read from / written to the upper triangle
            double* ep = k < p ? &A[k][p] : &A[p][k];
            double* eq = k < q ? &A[k][q] : &A[q][k];
            const double akp = *ep, akq = *eq;
            *ep = c * akp - s * akq; *eq = s * akp + c * akq;
          }
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
        }
      }
    }
  }
  return sweep;
}

template <int n>
SSP_HD int jacobi_eig_twosided(double A[n][n], double V[n][n]) {
  for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) V[i][j] = (i == j) ? 1.0 : 0.0;
  int sweep = 0;
  for (; sweep < 30; sweep++) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < n; i++) { diag += A[i][i] * A[i][i]; for (int j = i + 1; j < n; j++) off += A[i][j] * A[i][j]; }
    if (off <= 1e-34 * diag || off == 0.0) break;
#if PNP_JACOBI_VARIANT == 1      // probe: the same arithmetic with the pivot loops kept rolled
    PNP_ROLLED
#endif
    for (int p = 0; p < n - 1; p++)
#if PNP_JACOBI_VARIANT == 1
      PNP_ROLLED
#endif
      for (int q = p + 1; q < n; q++) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; k++) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        for (int k = 0; k < n; k++) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < n; k++) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
      }
  }
  return sweep;
}

template <int n>
SSP_HD int jacobi_eig(double A[n][n], double V[n][n]) {
#if PNP_JACOBI_VARIANT == 0 || PNP_JACOBI_VARIANT == 1
  return jacobi_eig_twosided<n>(A, V);
#else
  return jacobi_eig_upper<n>(A, V);
#endif
}

// ------------------------------------------------------------------------------------------------------------------------------
// Smallest eigenpair of the DLT normal matrix WITHOUT touching the 12 x 12 matrix: it is a 3 x 3 arrangement of 4 x 4 blocks,
//     M = [[S, 0, -Sx], [0, S, -Sy], [-Sx, -Sy, Sq]],     S = sum XX^T, Sx = sum x XX^T, Sy = sum y XX^T, Sq = sum (x^2 + y^2) XX^T,
// so (M - mu I) y = b is solved by eliminating the first two block rows (A = S - mu I is SPD, A^-1 from a 4 x 4 Cholesky):
//     C(mu) y3 = b3 + Sx A^-1 b1 + Sy A^-1 b2,   C(mu) = (Sq - mu I) - Sx A^-1 Sx - Sy A^-1 Sy,   y1 = A^-1 (b1 + Sx y3),  y2 likewise.
// Three inverse iterations at mu ~ 0 (M is PSD) pull the iterate towards the smallest eigenvector, Rayleigh-quotient iteration
// (mu = v^T M v, cubic convergence) finishes it to machine precision, and a last block-Cholesky of M - (rho - eps) I PROVES that no
// eigenvalue lies below the one found (Sylvester: A and C(mu) positive definite <=> M - mu I positive definite).  If any step fails --
// a Cholesky that should succeed does not, no convergence, the proof fails -- the caller falls back to the cyclic Jacobi on the full
// 12 x 12 matrix, so the result is the same eigenvector either way (up to sign, fixed by det > 0 below).  Everything lives in
// registers (4 x 4 blocks, static indices): ~4e3 flop instead of ~1e5 flop of local-memory Jacobi -- the single-image latency of
// valid.py's pnp() call is what this is for (round 2: batch-1 inference 2.1 ms with the Jacobi, of which 0.6 ms in this solve).
SSP_HD bool chol4_inv(const double A[4][4], double Ai[4][4]) {       // SPD inverse; false if a pivot is not positive
  double L[4][4];
  for (int j = 0; j < 4; j++) {
    double d = A[j][j];
    for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k];
    if (!(d > 0.0)) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 4; i++) {
      double v = A[i][j];
      for (int k = 0; k < j; k++) v -= L[i][k] * L[j][k];
      L[i][j] = v / L[j][j];
    }
  }
  for (int c = 0; c < 4; c++) {                                       // solve L L^T x = e_c
    double y[4];
    for (int i = 0; i < 4; i++) { double v = (i == c) ? 1.0 : 0.0; for (int k = 0; k < i; k++) v -= L[i][k] * y[k]; y[i] = v / L[i][i]; }
    for (int i = 3; i >= 0; i--) { double v = y[i]; for (int k = i + 1; k < 4; k++) v -= L[k][i] * Ai[k][c]; Ai[i][c] = v / L[i][i]; }
  }
  return true;
}
SSP_HD bool gauss4_solve(const double A[4][4], const double b[4], double x[4]) {     // general 4 x 4, partial pivoting (C(mu) is indefinite / nearly singular in the RQI steps)
  double a[4][5];
  for (int i = 0; i < 4; i++) { for (int j = 0; j < 4; j++) a[i][j] = A[i][j]; a[i][4] = b[i]; }
  for (int c = 0; c < 4; c++) {
    int piv = c; double best = fabs(a[c][c]);
    for (int r = c + 1; r < 4; r++) if (fabs(a[r][c]) > best) { best = fabs(a[r][c]); piv = r; }
    if (best == 0.0) return false;
    for (int j = 0; j < 5; j++) {                                     // row swap through selects: no dynamic register indexing
      double top = a[c][j], oth = top;
      for (int r = c + 1; r < 4; r++) if (r == piv) oth = a[r][j];
      for (int r = c + 1; r < 4; r++) if (r == piv) a[r][j] = top;
      a[c][j] = oth;
    }
    const double inv = 1.0 / a[c][c];
    for (int r = c + 1; r < 4; r++) {
      const double f = a[r][c] * inv;
      for (int j = c; j < 5; j++) a[r][j] -= f * a[c][j];
    }
  }
  for (int i = 3; i >= 0; i--) { double v = a[i][4]; for (int k = i + 1; k < 4; k++) v -= a[i][k] * x[k]; x[i] = v / a[i][i]; }
  return true;
}
SSP_HD void mat4_vec(const double A[4][4], const double v[4], double o[4]) {
  for (int i = 0; i < 4; i++) o[i] = A[i][0] * v[0] + A[i][1] * v[1] + A[i][2] * v[2] + A[i][3] * v[3];
}
struct DltBlocks { double S[4][4], Sx[4][4], Sy[4][4], Sq[4][4]; };
// A^-1 and C(mu); false if S - mu I is not positive definite
SSP_HD bool dlt_factor(const DltBlocks& B, double mu, double Ai[4][4], double C[4][4]) {
  double A[4][4];
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) A[i][j] = B.S[i][j] - (i == j ? mu : 0.0);
  if (!chol4_inv(A, Ai)) return false;
  double Tx[4][4], Ty[4][4];
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < 4; k++) { a += Ai[i][k] * B.Sx[k][j]; b += Ai[i][k] * B.Sy[k][j]; }
    Tx[i][j] = a; Ty[i][j] = b;
  }
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double v = B.Sq[i][j] - (i == j ? mu : 0.0);
    for (int k = 0; k < 4; k++) v -= B.Sx[i][k] * Tx[k][j] + B.Sy[i][k] * Ty[k][j];
    C[i][j] = v;
  }
  return true;
}
SSP_HD bool dlt_solve(const DltBlocks& B, const double Ai[4][4], const double C[4][4], const double b[12], double y[12]) {
  double t1[4], t2[4], u[4], rhs[4];
  mat4_vec(Ai, b, t1); mat4_vec(Ai, b + 4, t2);
  mat4_vec(B.Sx, t1, u); for (int i = 0; i < 4; i++) rhs[i] = b[8 + i] + u[i];
  mat4_vec(B.Sy, t2, u); for (int i = 0; i < 4; i++) rhs[i] += u[i];
  if (!gauss4_solve(C, rhs, y + 8)) return false;
  mat4_vec(B.Sx, y + 8, u); for (int i = 0; i < 4; i++) u[i] += b[i];
  mat4_vec(Ai, u, y);
  mat4_vec(B.Sy, y + 8, u); for (int i = 0; i < 4; i++) u[i] += b[4 + i];
  mat4_vec(Ai, u, y + 4);
  return true;
}
SSP_HD void dlt_matvec(const DltBlocks& B, const double v[12], double o[12]) {
  double a[4], b[4];
  mat4_vec(B.S, v, a); mat4_vec(B.Sx, v + 8, b); for (int i = 0; i < 4; i++) o[i] = a[i] - b[i];
  mat4_vec(B.S, v + 4, a); mat4_vec(B.Sy, v + 8, b); for (int i = 0; i < 4; i++) o[4 + i] = a[i] - b[i];
  mat4_vec(B.Sq, v + 8, o + 8); mat4_vec(B.Sx, v, a); mat4_vec(B.Sy, v + 4, b); for (int i = 0; i < 4; i++) o[8 + i] -= a[i] + b[i];
}
SSP_HD bool normalize12(double v[12]) {
  double n = 0.0; for (int i = 0; i < 12; i++) n += v[i] * v[i];
  if (!(n > 0.0) || !(n < 1e300)) return false;
  n = 1.0 / sqrt(n); for (int i = 0; i < 12; i++) v[i] *= n;
  return true;
}
// v (unit norm) and lambda of the smallest eigenvalue of M; false => use the Jacobi on the full matrix.
// An attempt = 6 inverse iterations at mu ~ 0 (one factorisation), Rayleigh-quotient iteration to convergence, the proof.  When the
// proof fails the pair found is a HIGHER eigenpair (the start vector had too little of the smallest one: ~15 % of the noisy golden
// problems with a single attempt): it is kept, projected out of the next attempt's inverse iterations (deflation), and the next
// attempt starts from another vector.  *steps returns the total number of Rayleigh-quotient steps.
SSP_HD bool dlt_smallest_eigvec(const DltBlocks& B, double v[12], double* lambda, int* steps) {
  double tr = 0.0;
  for (int i = 0; i < 4; i++) tr += 2.0 * B.S[i][i] + B.Sq[i][i];
  if (!(tr > 0.0)) return false;
  double A0[4][4], C0[4][4];
  if (!dlt_factor(B, -1e-13 * tr, A0, C0)) return false;
  double found[2][12];                                                   // higher eigenvectors met on the way
  int nfound = 0, total = 0;
  for (int attempt = 0; attempt < 3; attempt++) {
    double Ai[4][4], C[4][4], y[12];
    for (int i = 0; i < 12; i++) v[i] = attempt == 0 ? 1.0 + 0.0625 * i : (attempt == 1 ? ((i & 1) ? -1.0 : 1.0) * (1.0 + 0.03 * i) : ((i % 3) == 0 ? 1.5 : -0.4) + 0.01 * i);
    normalize12(v);
    for (int it = 0; it < 6; it++) {
      for (int f = 0; f < nfound; f++) { double d = 0.0; for (int i = 0; i < 12; i++) d += v[i] * found[f][i]; for (int i = 0; i < 12; i++) v[i] -= d * found[f][i]; }
      if (!dlt_solve(B, A0, C0, v, y)) return false;
      for (int i = 0; i < 12; i++) v[i] = y[i];
      if (!normalize12(v)) return false;
    }
    double rho = 0.0; bool conv = false;
    for (int k = 0; k < 8 && !conv; k++, total++) {
      dlt_matvec(B, v, y);
      rho = 0.0; for (int i = 0; i < 12; i++) rho += v[i] * y[i];
      double res = 0.0; for (int i = 0; i < 12; i++) { const double r = y[i] - rho * v[i]; res += r * r; }
      if (sqrt(res) <= 2e-15 * tr) { conv = true; break; }
      if (!dlt_factor(B, rho, Ai, C)) return false;
      if (!dlt_solve(B, Ai, C, v, y)) { conv = true; break; }          // exactly singular: rho IS an eigenvalue to the last bit
      for (int i = 0; i < 12; i++) v[i] = y[i];
      if (!normalize12(v)) return false;
    }
    if (!conv) return false;
    // proof: M - (rho - eps) I is positive definite  =>  nothing below rho - eps
    double Ci[4][4];
    if (dlt_factor(B, rho - 1e-10 * tr, Ai, C) && chol4_inv(C, Ci)) { *lambda = rho; *steps = total; return true; }
    if (nfound == 2) return false;
    for (int i = 0; i < 12; i++) found[nfound][i] = v[i];
    nfound++;
  }
  return false;
}

// in-place Cholesky solve of SPD n x n system (n <= 6); returns false if not positive definite
template <int n>
SSP_HD bool chol_solve(double A[n][n], double b[n]) {
  for (int j = 0; j < n; j++) {
    double d = A[j][j];
    for (int k = 0; k < j; k++) d -= A[j][k] * A[j][k];
    if (!(d > 0.0)) return false;
    d = sqrt(d); A[j][j] = d;
    for (int i = j + 1; i < n; i++) {
      double v = A[i][j];
      for (int k = 0; k < j; k++) v -= A[i][k] * A[j][k];
      A[i][j] = v / d;
    }
  }
  for (int i = 0; i < n; i++) { double v = b[i]; for (int k = 0; k < i; k++) v -= A[i][k] * b[k]; b[i] = v / A[i][i]; }
  for (int i = n - 1; i >= 0; i--) { double v = b[i]; for (int k = i + 1; k < n; k++) v -= A[k][i] * b[k]; b[i] = v / A[i][i]; }
  return true;
}

SSP_HD double reproj_err(const double* M, const double* m, int np, const double p[6], double fx, double fy, double cx, double cy) {
  double R[9]; rodrigues(p, R, nullptr);
  double e = 0.0;
  for (int i = 0; i < np; i++) {
    const double X = M[3 * i], Y = M[3 * i + 1], Z = M[3 * i + 2];
    const double x = R[0] * X + R[1] * Y + R[2] * Z + p[3], y = R[3] * X + R[4] * Y + R[5] * Z + p[4], z = R[6] * X + R[7] * Y + R[8] * Z + p[5];
    const double iz = 1.0 / z;
    const double du = fx * x * iz + cx - m[2 * i], dv = fy * y * iz + cy - m[2 * i + 1];
    e += du * du + dv * dv;
  }
  return sqrt(e);
}

// p3: np x 3 object points, q: np x 2 image points (pixels), Kmat: 3x3 row-major intrinsics (float32 like the reference passes them);
// R_out[9], t_out[3] in fp64; work[3] = {Jacobi sweeps of the DLT (0 when started from a guess), accepted LM iterations, LM linear solves}.
// The solve has two stages: the DLT gives the initial LM vector p = (rvec, t), LM refines it.  guess (6, or null): LM starts from this
// (rvec, t) and the DLT is skipped, as cvFindExtrinsicCameraParams2 does with useExtrinsicGuess (same LM, same max_iter, same
// FLT_EPSILON stop).  params_out (6, or null): the final LM vector, what cv2.solvePnP returns as rvec, tvec.  Both stay in this one
// function (not two called ones) because that keeps the code nvcc generates for guess == params_out == null unchanged.
SSP_HD void pnp_solve_one(const float* p3, const float* q, const float* Kmat, int np, int max_iter, double* R_out, double* t_out, int* work,
                          double* dbg = nullptr /*[20]: smallest eigenvalue, its eigenvector, det, initial (rvec, t) -- probes only*/,
                          const double* guess = nullptr, double* params_out = nullptr) {
  const double fx = Kmat[0], fy = Kmat[4], cx = Kmat[2], cy = Kmat[5];
  double M[3 * PNP_MAXP], m[2 * PNP_MAXP];
  for (int i = 0; i < 3 * np; i++) M[i] = (double)p3[i];
  for (int i = 0; i < 2 * np; i++) m[i] = (double)q[i];

  double p[6];
  int sweeps = 0;
  if (guess) {
    for (int i = 0; i < 6; i++) p[i] = guess[i];
  } else {
    // ---- DLT (cvFindExtrinsicCameraParams2, non-planar branch): smallest eigenvector of L^T L on the raw coordinates ----
    // the four 4 x 4 blocks of L^T L; the smallest eigenvector through the block solve (dlt_smallest_eigvec), the cyclic Jacobi on the
    // assembled 12 x 12 matrix only if that declines (PNP_DLT_JACOBI=1 forces it: the two must agree, tests/test_pnp_host.py)
    DltBlocks Bk;
    for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) { Bk.S[a][b] = 0.0; Bk.Sx[a][b] = 0.0; Bk.Sy[a][b] = 0.0; Bk.Sq[a][b] = 0.0; }
    for (int i = 0; i < np; i++) {
      const double X[4] = {M[3 * i], M[3 * i + 1], M[3 * i + 2], 1.0};
      const double x = (m[2 * i] - cx) / fx, y = (m[2 * i + 1] - cy) / fy, qq = x * x + y * y;
      for (int a = 0; a < 4; a++)
        for (int b = 0; b < 4; b++) {
          const double xx = X[a] * X[b];
          Bk.S[a][b] += xx; Bk.Sx[a][b] += x * xx; Bk.Sy[a][b] += y * xx; Bk.Sq[a][b] += qq * xx;
        }
    }
    double ev[12], lam_min = 0.0;
#ifndef PNP_DLT_JACOBI
#define PNP_DLT_JACOBI 0
#endif
    bool have = false;
    if (!PNP_DLT_JACOBI) { int st = 0; have = dlt_smallest_eigvec(Bk, ev, &lam_min, &st); sweeps = -st; }      // work[0] < 0: block-solve steps
    if (!have) {
      double LL[12][12], LV[12][12];
      for (int a = 0; a < 12; a++) for (int b = 0; b < 12; b++) LL[a][b] = 0.0;
      for (int a = 0; a < 4; a++)
        for (int b = 0; b < 4; b++) {
          LL[a][b] = Bk.S[a][b]; LL[4 + a][4 + b] = Bk.S[a][b];
          LL[a][8 + b] = -Bk.Sx[a][b]; LL[4 + a][8 + b] = -Bk.Sy[a][b];
          LL[8 + a][8 + b] = Bk.Sq[a][b];
        }
      for (int a = 0; a < 8; a++) for (int b = 8; b < 12; b++) LL[b][a] = LL[a][b];
      sweeps = jacobi_eig<12>(LL, LV);
      int kmin = 0;
      for (int k = 1; k < 12; k++) if (LL[k][k] < LL[kmin][kmin]) kmin = k;
      for (int i = 0; i < 12; i++) ev[i] = LV[i][kmin];
      lam_min = LL[kmin][kmin];
    }
    double RR[9], tt[3];
    for (int r = 0; r < 3; r++) {
      RR[3 * r] = ev[4 * r]; RR[3 * r + 1] = ev[4 * r + 1]; RR[3 * r + 2] = ev[4 * r + 2];
      tt[r] = ev[4 * r + 3];
    }
    const double det = RR[0] * (RR[4] * RR[8] - RR[5] * RR[7]) - RR[1] * (RR[3] * RR[8] - RR[5] * RR[6]) + RR[2] * (RR[3] * RR[7] - RR[4] * RR[6]);
    if (det < 0) { for (int i = 0; i < 9; i++) RR[i] = -RR[i]; for (int i = 0; i < 3; i++) tt[i] = -tt[i]; }
    double sc = 0; for (int i = 0; i < 9; i++) sc += RR[i] * RR[i];
    sc = sqrt(sc);
    // polar decomposition: R = RR (RR^T RR)^(-1/2)
    double G[3][3], Vg[3][3];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { double v = 0; for (int k = 0; k < 3; k++) v += RR[3 * k + a] * RR[3 * k + b]; G[a][b] = v; }
    jacobi_eig<3>(G, Vg);
    double Gi[3][3];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { double v = 0; for (int k = 0; k < 3; k++) v += Vg[a][k] * Vg[b][k] / sqrt(fmax(G[k][k], 1e-300)); Gi[a][b] = v; }
    double R0[9];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { double v = 0; for (int k = 0; k < 3; k++) v += RR[3 * a + k] * Gi[k][b]; R0[3 * a + b] = v; }
    { const double f = sqrt(3.0) / sc; p[3] = tt[0] * f; p[4] = tt[1] * f; p[5] = tt[2] * f; }
    {  // rotation matrix -> axis-angle (cv2.Rodrigues inverse branch structure)
      const double rv[3] = {R0[7] - R0[5], R0[2] - R0[6], R0[3] - R0[1]};
      const double s = sqrt((rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]) * 0.25);
      double c = (R0[0] + R0[4] + R0[8] - 1.0) * 0.5; c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
      const double th = acos(c);
      if (s < 1e-5) {
        if (c > 0) { p[0] = p[1] = p[2] = 0.0; }
        else {
          double tx = sqrt(fmax((R0[0] + 1) * 0.5, 0.0));
          double ty = sqrt(fmax((R0[4] + 1) * 0.5, 0.0)) * (R0[1] < 0 ? -1.0 : 1.0);
          double tz = sqrt(fmax((R0[8] + 1) * 0.5, 0.0)) * (R0[2] < 0 ? -1.0 : 1.0);
          if (fabs(tx) < fabs(ty) && fabs(tx) < fabs(tz) && ((R0[5] > 0) != (ty * tz > 0))) tz = -tz;
          const double nn = th / sqrt(tx * tx + ty * ty + tz * tz);
          p[0] = tx * nn; p[1] = ty * nn; p[2] = tz * nn;
        }
      } else {
        const double f = 0.5 / s * th;
        p[0] = rv[0] * f; p[1] = rv[1] * f; p[2] = rv[2] * f;
      }
    }

    if (dbg) { dbg[0] = lam_min; for (int i = 0; i < 12; i++) dbg[1 + i] = ev[i]; dbg[13] = det; for (int i = 0; i < 6; i++) dbg[14 + i] = p[i]; }
  }

  // ---- Levenberg-Marquardt (CvLevMarq schedule) ----
  int lam_lg10 = -3, iters = 0, solves = 0;
  double prev_err = 0.0, e = 0.0;
  while (true) {
    double R[9], dR[27];
    rodrigues(p, R, dR);
    double JtJ[6][6] = {}, Jte[6] = {};
    double err2 = 0.0;
    for (int i = 0; i < np; i++) {
      const double X = M[3 * i], Y = M[3 * i + 1], Z = M[3 * i + 2];
      const double x = R[0] * X + R[1] * Y + R[2] * Z + p[3], y = R[3] * X + R[4] * Y + R[5] * Z + p[4], z = R[6] * X + R[7] * Y + R[8] * Z + p[5];
      const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
      const double eu = fx * xn + cx - m[2 * i], ev = fy * yn + cy - m[2 * i + 1];
      err2 += eu * eu + ev * ev;
      double ju[6], jv[6];
      for (int j = 0; j < 3; j++) {
        const double* d = dR + 9 * j;
        const double dx = d[0] * X + d[1] * Y + d[2] * Z, dy = d[3] * X + d[4] * Y + d[5] * Z, dz = d[6] * X + d[7] * Y + d[8] * Z;
        ju[j] = fx * (dx - xn * dz) * iz; jv[j] = fy * (dy - yn * dz) * iz;
      }
      ju[3] = fx * iz; ju[4] = 0.0; ju[5] = -fx * xn * iz;
      jv[3] = 0.0; jv[4] = fy * iz; jv[5] = -fy * yn * iz;
      for (int a = 0; a < 6; a++) {
        Jte[a] += ju[a] * eu + jv[a] * ev;
        for (int b = a; b < 6; b++) JtJ[a][b] += ju[a] * ju[b] + jv[a] * jv[b];
      }
    }
    for (int a = 0; a < 6; a++) for (int b = 0; b < a; b++) JtJ[a][b] = JtJ[b][a];
    if (iters == 0) prev_err = sqrt(err2);
    double prev[6];
    for (int a = 0; a < 6; a++) prev[a] = p[a];
    bool first = true;
    while (true) {
      if (!first) { if (++lam_lg10 > 16) break; }
      first = false;
      const double lam = exp(lam_lg10 * 2.302585092994046);
      double A[6][6], d[6];
      for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) A[a][b] = JtJ[a][b]; A[a][a] *= 1.0 + lam; d[a] = Jte[a]; }
      if (!chol_solve<6>(A, d)) { for (int a = 0; a < 6; a++) d[a] = 0.0; }
      solves++;
      for (int a = 0; a < 6; a++) p[a] = prev[a] - d[a];
      e = reproj_err(M, m, np, p, fx, fy, cx, cy);
      if (!(e > prev_err)) break;
    }
    lam_lg10 = lam_lg10 - 1 < -16 ? -16 : lam_lg10 - 1;
    iters++;
    double dn = 0, pn = 0;
    for (int a = 0; a < 6; a++) { dn += (p[a] - prev[a]) * (p[a] - prev[a]); pn += prev[a] * prev[a]; }
    if (iters >= max_iter || sqrt(dn) < 1.1920929e-07 * sqrt(pn)) break;
    prev_err = e;
  }
  double R[9];
  rodrigues(p, R, nullptr);
  for (int i = 0; i < 9; i++) R_out[i] = R[i];
  for (int i = 0; i < 3; i++) t_out[i] = p[3 + i];
  if (params_out) for (int i = 0; i < 6; i++) params_out[i] = p[i];
  work[0] = sweeps; work[1] = iters; work[2] = solves;
}

}  // namespace ssp_pnp
