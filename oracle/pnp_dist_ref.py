"""Oracle of PnP and projection with lens distortion: cv2.undistortPoints, cv2.projectPoints (with its Jacobian) and
cv2.solvePnP(..., distCoeffs, SOLVEPNP_ITERATIVE), cold and warm, restated in numpy.  TEST INFRASTRUCTURE ONLY.

k = (k1, k2, p1, p2, k3, k4, k5, k6), OpenCV's order (fewer coefficients are zero-padded).  With x' = x/z, y' = y/z,
r2 = x'^2 + y'^2:
    xd = x' (1 + k1 r2 + k2 r4 + k3 r6) / (1 + k4 r2 + k5 r4 + k6 r6) + 2 p1 x'y' + p2 (r2 + 2x'^2),   u = fx xd + cx
    yd = y' (...) / (...) + p1 (r2 + 2y'^2) + 2 p2 x'y',                                               v = fy yd + cy
cv2.solvePnP's ITERATIVE solve (cvFindExtrinsicCameraParams2) runs the DLT of oracle/pnp_ref.py on cv2.undistortPoints'
normalised points -- 5 fixed-point iterations of the inverse model, no convergence test -- and the CvLevMarq refinement on the
raw pixels with the distorted model above."""
from __future__ import annotations

import numpy as np

from .pnp_ref import FLT_EPSILON, dlt_init, rodrigues_vec2mat


def dist8(k):
    """(4|5|8,) coefficients -> (8,) fp64, zero-padded"""
    k = np.asarray(k, np.float64).reshape(-1)
    return np.concatenate([k, np.zeros(8 - len(k))])


def undistort_points(uv, K, k):
    """cv2.undistortPoints(uv, K, k) (no R, no P): (N, 2) pixels -> (N, 2) normalised points"""
    k = dist8(k)
    K = np.asarray(K, np.float64)
    uv = np.asarray(uv, np.float64).reshape(-1, 2)
    x0 = (uv[:, 0] - K[0, 2]) * (1.0 / K[0, 0])
    y0 = (uv[:, 1] - K[1, 2]) * (1.0 / K[1, 1])
    out = np.empty((len(uv), 2))
    for i in range(len(uv)):
        x, y = x0[i], y0[i]
        for _ in range(5):
            r2 = x * x + y * y
            icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
            if icdist < 0:
                x, y = x0[i], y0[i]
                break
            dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x)
            dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y
            x, y = (x0[i] - dx) * icdist, (y0[i] - dy) * icdist
        out[i] = x, y
    return out


def project_points(M, r, t, K, k, jac=False):
    """cv2.projectPoints(M, r, t, K, k): M (N, 3) -> (N, 2) pixels [+ J (2N, 6) = d(u, v)/d(rvec, t), rows u0, v0, u1, ...]"""
    k = dist8(k)
    K = np.asarray(K, np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    M = np.asarray(M, np.float64).reshape(-1, 3)
    R, dRdr = rodrigues_vec2mat(np.asarray(r, np.float64).reshape(3), True)
    P = M @ R.T + np.asarray(t, np.float64).reshape(3)
    iz = 1.0 / P[:, 2]
    x, y = P[:, 0] * iz, P[:, 1] * iz
    r2 = x * x + y * y
    r4, r6 = r2 * r2, r2 * r2 * r2
    cdist = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6
    icdist2 = 1.0 / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6)
    xd = x * cdist * icdist2 + k[2] * 2 * x * y + k[3] * (r2 + 2 * x * x)
    yd = y * cdist * icdist2 + k[2] * (r2 + 2 * y * y) + k[3] * 2 * x * y
    uv = np.stack([xd * fx + cx, yd * fy + cy], 1)
    if not jac:
        return uv
    g = cdist * icdist2
    dg = (k[0] + 2 * k[1] * r2 + 3 * k[4] * r4) * icdist2 - g * icdist2 * (k[5] + 2 * k[6] * r2 + 3 * k[7] * r4)
    d00 = g + 2 * x * x * dg + 2 * k[2] * y + 6 * k[3] * x
    d01 = 2 * x * y * dg + 2 * k[2] * x + 2 * k[3] * y
    d11 = g + 2 * y * y * dg + 6 * k[2] * y + 2 * k[3] * x
    gx, gy = np.zeros((len(M), 6)), np.zeros((len(M), 6))           # d(x', y')/d(rvec, t)
    for j in range(3):
        dP = M @ dRdr[j].reshape(3, 3).T
        gx[:, j] = (dP[:, 0] - x * dP[:, 2]) * iz
        gy[:, j] = (dP[:, 1] - y * dP[:, 2]) * iz
    gx[:, 3], gx[:, 5] = iz, -x * iz
    gy[:, 4], gy[:, 5] = iz, -y * iz
    J = np.zeros((2 * len(M), 6))
    J[0::2] = fx * (d00[:, None] * gx + d01[:, None] * gy)
    J[1::2] = fy * (d01[:, None] * gx + d11[:, None] * gy)
    return uv, J


def solve_pnp_dist(points_3D, points_2D, K, k, rvec=None, tvec=None, max_iter=20):
    """cv2.solvePnP(points_3D, points_2D, K, k, [rvec, tvec, useExtrinsicGuess=True,] flags=SOLVEPNP_ITERATIVE) -> (rvec (3,),
    tvec (3,)) fp64.  Cold (rvec None): the DLT on the undistorted points; warm: LM from (rvec, tvec)."""
    M = np.asarray(points_3D, np.float64).reshape(-1, 3)
    m = np.asarray(points_2D, np.float64).reshape(-1, 2)
    K = np.asarray(K, np.float64)
    if rvec is None:
        r, t = dlt_init(M, undistort_points(m, K, k))
    else:
        r, t = np.asarray(rvec, np.float64).reshape(3), np.asarray(tvec, np.float64).reshape(3)
    p = np.concatenate([r, t])
    lam_lg10, iters = -3, 0

    def step(JtJ, Jte, prev, lg):
        A = JtJ.copy()
        A[np.diag_indices(6)] *= 1.0 + np.exp(lg * np.log(10.0))
        return prev - np.linalg.lstsq(A, Jte, rcond=None)[0]

    while True:
        uv, J = project_points(M, p[:3], p[3:], K, k, jac=True)
        err = (uv - m).reshape(-1)
        JtJ, Jte = J.T @ J, J.T @ err
        prev = p.copy()
        p = step(JtJ, Jte, prev, lam_lg10)
        if iters == 0:
            prev_err = np.linalg.norm(err)
        while True:
            e = np.linalg.norm((project_points(M, p[:3], p[3:], K, k) - m).reshape(-1))
            if e > prev_err:
                lam_lg10 += 1
                if lam_lg10 <= 16:
                    p = step(JtJ, Jte, prev, lam_lg10)
                    continue
            break
        lam_lg10 = max(lam_lg10 - 1, -16)
        iters += 1
        if iters >= max_iter or np.linalg.norm(p - prev) / np.linalg.norm(prev) < FLT_EPSILON:
            break
        prev_err = e
    return p[:3].copy(), p[3:].copy()


def corner_problems(n, seed, K, k, P3, depth=(0.6, 1.0), moved=(40.0, 150.0), W=640, H=480):
    """n seeded consensus problems towards the frame corners: the box depth[0]..depth[1] m away, its centre 60-140 px from a corner of the
    W x H frame, exact distorted keypoints (project_points, float32) of which one, chosen at random, is moved by moved[0]..moved[1]
    px in a random direction -> (uv (n, P, 2) float32, outlier index (n,) int64, rvec (n, 3), t (n, 3))"""
    rng = np.random.default_rng(seed)
    K = np.asarray(K, np.float64)
    uv, out, rv, tv = [], [], [], []
    for _ in range(n):
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        r = ax * rng.uniform(0, np.pi)
        z = rng.uniform(*depth)
        du, dv = rng.uniform(60, 140, size=2)
        u = du if rng.random() < 0.5 else W - du
        v = dv if rng.random() < 0.5 else H - dv
        t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0])
        q = project_points(P3, r, t, K, k)
        j = int(rng.integers(len(q)))
        a = rng.uniform(0, 2 * np.pi)
        q[j] += rng.uniform(*moved) * np.array([np.cos(a), np.sin(a)])
        uv.append(q.astype(np.float32)); out.append(j); rv.append(r); tv.append(t)
    return np.array(uv), np.array(out, np.int64), np.array(rv), np.array(tv)
