"""Oracle of the depth refinement (singleshotpose_b200/csrc/refine_depth_core.h) in numpy, written from the rule's text: whole
arrays per iteration and numpy's summation order where the core sums per virtual thread and by a halving tree.  Also a z-buffered
depth renderer that builds the test scenes.  TEST INFRASTRUCTURE ONLY: the product has no depth renderer.

The rule per iteration k (gate tau_k = d s (e/s)^(k/(iters-1)), d s with iters = 1): p = R x + t, m = R n; a point pairs when
m . p < 0, p_z > 0, its nearest pixel (floor(u + 0.5), floor(v + 0.5)) lies in the frame with D > 0, and |p_z - q_z| <= tau_k with
q = D depth_scale (x^, y^, 1) (undistorted with coefficients); r = m . (p - q), J = [R x  x  m + m x (p - q); m]; fewer than 50
pairs (status 1) or a Cholesky pivot <= 1e-12 x the largest diagonal of J^T J (status 2) stops with the input pose; a pose that
is not finite or has t_z <= 0 is status 4; else delta = -(J^T J)^-1 J^T r, R <- exp([dth]x) R, t <- t + dt_."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import chol_ok, so3_exp
from .render_ref import snap

MIN_POINTS = 50
FEW_POINTS, SINGULAR, BAD_POSE = 1, 2, 4


def distort(k, x, y):
    """OpenCV's model at normalised points (N,) -> (xd, yd)"""
    r2 = x * x + y * y
    g = (1 + k[0] * r2 + k[1] * r2 ** 2 + k[4] * r2 ** 3) / (1 + k[5] * r2 + k[6] * r2 ** 2 + k[7] * r2 ** 3)
    return x * g + 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x), y * g + k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y


def undistort(k, u, v, K):
    """cv2.undistortPoints of pixels (N,): 5 fixed-point iterations of the inverse model, the plain point where icdist < 0"""
    x0, y0 = (u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1]
    x, y = x0.copy(), y0.copy()
    live = np.ones(len(x0), bool)
    for _ in range(5):
        r2 = x * x + y * y
        icd = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
        live &= icd >= 0
        nx = (x0 - (2 * k[2] * x * y + k[3] * (r2 + 2 * x * x))) * icd
        ny = (y0 - (k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y)) * icd
        x, y = np.where(live, nx, x0), np.where(live, ny, y0)
    return x, y


def project(Pc, K, k=None):
    """pixels (u, v) of camera-frame points Pc (N, 3)"""
    x, y = Pc[:, 0] / Pc[:, 2], Pc[:, 1] / Pc[:, 2]
    if k is not None:
        x, y = distort(np.asarray(k, np.float64), x, y)
    return K[0, 0] * x + K[0, 2], K[1, 1] * y + K[1, 2]


def pairs(depth, X, N, R, t, K, tau, depth_scale, k=None):
    """-> (a, m, p, q) of the points that pair at gate tau"""
    depth = np.asarray(depth)
    H, W = depth.shape
    a, m = X @ R.T, N @ R.T
    p = a + t
    ok = ((m * p).sum(1) < 0) & (p[:, 2] > 0)
    a, m, p = a[ok], m[ok], p[ok]
    u, v = project(p, K, k)
    fu, fv = np.floor(u + 0.5), np.floor(v + 0.5)
    ok = (fu >= 0) & (fu < W) & (fv >= 0) & (fv < H)
    a, m, p, fu, fv = a[ok], m[ok], p[ok], fu[ok], fv[ok]
    D = depth[fv.astype(np.int64), fu.astype(np.int64)].astype(np.float64)
    z = D * depth_scale
    ok = (D > 0) & (np.abs(p[:, 2] - z) <= tau)
    a, m, p, fu, fv, z = a[ok], m[ok], p[ok], fu[ok], fv[ok], z[ok]
    if k is None:
        xh, yh = (fu - K[0, 2]) / K[0, 0], (fv - K[1, 2]) / K[1, 1]
    else:
        xh, yh = undistort(np.asarray(k, np.float64), fu, fv, K)
    return a, m, p, np.stack([z * xh, z * yh, z], 1)


def terms(a, m, p, q):
    """r (N,) and J (N, 6)"""
    d = p - q
    return (m * d).sum(1), np.concatenate([np.cross(a, m) + np.cross(m, d), m], 1)


def refine_ref(depth, X, N, K, R, t, diam, depth_scale=0.001, iters=10, gate=(0.5, 0.02), k=None):
    """one problem -> (R, t, points, rmse, status)"""
    R0, t0 = np.asarray(R, np.float64), np.asarray(t, np.float64).reshape(3)
    K = np.asarray(K, np.float64)
    if not (np.isfinite(R0).all() and np.isfinite(t0).all() and t0[2] > 0):
        return R0, t0, 0, 0.0, BAD_POSE
    s, e = gate
    R, t = R0.copy(), t0.copy()
    for it in range(iters):
        tau = diam * (s if iters == 1 else s * (e / s) ** (it / (iters - 1)))
        r, J = terms(*pairs(depth, X, N, R, t, K, tau, depth_scale, k))
        n = len(r)
        rmse = float(np.sqrt((r @ r) / n)) if n else 0.0
        if n < MIN_POINTS:
            return R0, t0, n, rmse, FEW_POINTS
        A = J.T @ J
        if not chol_ok(A):
            return R0, t0, n, rmse, SINGULAR
        delta = -np.linalg.solve(A, J.T @ r)
        R, t = so3_exp(delta[:3]) @ R, t + delta[3:]
    return R, t, n, rmse, 0


def add_error(X, R1, t1, R2, t2):
    """ADD: mean |(R1 x + t1) - (R2 x + t2)| over the points"""
    return float(np.linalg.norm(X @ (np.asarray(R1) - np.asarray(R2)).T + (np.asarray(t1) - np.asarray(t2)).reshape(3), axis=1).mean())


# ---------------------------------------------------------------------------------------------- the test scenes' depth renderer
def render_depth_ref(Pc, faces, K, W, H, depth_scale, k=None):
    """uint16 depth (H, W) of camera-frame vertices Pc (Nv, 3) (every z > 0) and faces (Nf, 3): render_masks_ref's coverage of the
    float32 pixel coordinates (oracle/render_ref.py: 1/256 px snapping, pixel centres at integer coordinates, the top-left rule),
    the depth interpolated perspective-correctly (1/z linear in screen space), the nearest surface winning, rounded to depth
    units of depth_scale (0 where nothing is drawn or beyond 65535 units).  With coefficients k the vertices are projected
    distorted and the triangles stay straight between them."""
    Pc = np.asarray(Pc, np.float64)
    assert (Pc[:, 2] > 0).all()
    u, v = project(Pc, np.asarray(K, np.float64), k)
    s = snap(np.stack([u, v]).astype(np.float32))                      # (2, Nv) int64
    F = np.asarray(faces, np.int64)
    a, b, c = F[:, 0], F[:, 1], F[:, 2]
    area = (s[0, b] - s[0, a]) * (s[1, c] - s[1, a]) - (s[1, b] - s[1, a]) * (s[0, c] - s[0, a])
    keep = area != 0
    a, b, c, area = a[keep], b[keep], c[keep], area[keep]
    flip = area < 0
    b, c = np.where(flip, c, b), np.where(flip, b, c)
    area = np.abs(area)
    V = np.stack([a, b, c], 1)                                         # (T, 3) clockwise on screen
    X, Y = s[0, V], s[1, V]
    x0 = np.maximum(-((-X.min(1)) // 256), 0); x1 = np.minimum(X.max(1) // 256, W - 1)
    y0 = np.maximum(-((-Y.min(1)) // 256), 0); y1 = np.minimum(Y.max(1) // 256, H - 1)
    keep = (x0 <= x1) & (y0 <= y1)
    V, X, Y, area, x0, x1, y0, y1 = V[keep], X[keep], Y[keep], area[keep], x0[keep], x1[keep], y0[keep], y1[keep]
    zbuf = np.full(H * W, np.inf)
    iz = 1.0 / Pc[:, 2]
    w, h = x1 - x0 + 1, y1 - y0 + 1
    cnt = w * h
    for lo in range(0, len(V), 4096):                                  # bounded memory for the large triangles of a plane
        sl = slice(lo, lo + 4096)
        tri = np.repeat(np.arange(len(V))[sl], cnt[sl])
        off = np.arange(cnt[sl].sum()) - np.repeat(np.cumsum(cnt[sl]) - cnt[sl], cnt[sl])
        xx, yy = x0[tri] + off % w[tri], y0[tri] + off // w[tri]
        px, py = xx * 256, yy * 256
        inside = np.ones(len(tri), bool)
        lam = np.zeros((len(tri), 3))
        for i, j in ((0, 1), (1, 2), (2, 0)):
            ax, ay = X[tri, i], Y[tri, i]
            dx, dy = X[tri, j] - ax, Y[tri, j] - ay
            e = dx * (py - ay) - dy * (px - ax)
            top_left = ((dy == 0) & (dx > 0)) | (dy < 0)
            inside &= (e > 0) | ((e == 0) & top_left)
            lam[:, 3 - i - j] = e / area[tri]                          # the weight of the vertex opposite edge (i, j)
        tri, xx, yy, lam = tri[inside], xx[inside], yy[inside], lam[inside]
        z = 1.0 / (lam * iz[V[tri]]).sum(1)
        np.minimum.at(zbuf, yy * W + xx, z)
    units = np.rint(zbuf / depth_scale)
    return np.where(np.isfinite(units) & (units <= 65535), units, 0).astype(np.uint16).reshape(H, W)
