"""Oracle of the pose covariance and the constant-velocity pose filter (singleshotpose_b200/csrc/pose_filter_core.h) in numpy, with
whole matrices where the core works element by element.  TEST INFRASTRUCTURE ONLY.

A pose (R, t) is perturbed on the left, x_cam = exp([dth]x) R X + t + dt_.  The covariance of a PnP pose is
Sigma = sigma^2 (J^T J)^-1, J (2N x 6) = d(u, v)/d(dth, dt_) of the N points.  The filter per track: state R, t, w, v and P (12 x 12) over
(dth, dt_, dw, dv); predict with F = I + dt (E(dth, dw) + E(dt_, dv)) and white-noise-acceleration Q; update with H = [I6 0], a chi^2
gate on y^T S^-1 y and the Joseph form; a gated or unusable measurement re-initialises the filter."""
from __future__ import annotations

import numpy as np

from .pnp_ref import rodrigues_vec2mat

SINGULAR, DEPTH = 1, 2
PIVOT = 1e-12


def skew(a):
    return np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], np.float64)


def so3_exp(w):
    return rodrigues_vec2mat(np.asarray(w, np.float64))


def so3_log(R):
    """the rotation vector of R, |w| in [0, pi]: angle atan2(sin, cos), the axis from R - R^T (near pi from R + I)"""
    R = np.asarray(R, np.float64)
    rv = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.sqrt(rv @ rv * 0.25)
    c = np.clip((np.trace(R) - 1.0) * 0.5, -1.0, 1.0)
    if s == 0.0 and c > 0:
        return np.zeros(3)
    if s < 1e-5 and c <= 0:
        tx = np.sqrt(max((R[0, 0] + 1) * 0.5, 0.0))
        ty = np.sqrt(max((R[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        tz = np.sqrt(max((R[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(tx) < abs(ty) and abs(tx) < abs(tz) and ((R[1, 2] > 0) != (ty * tz > 0)):
            tz = -tz
        v = np.array([tx, ty, tz])
        return v * np.arccos(c) / np.linalg.norm(v)
    return rv * (0.5 / s * np.arctan2(s, c))


def _distort_jac(k, x, y):
    """(xd, yd) and d(xd, yd)/d(x, y) (N, 2, 2) of OpenCV's model at normalised points x, y (N,)"""
    r2 = x * x + y * y
    num = 1 + k[0] * r2 + k[1] * r2 ** 2 + k[4] * r2 ** 3
    den = 1 + k[5] * r2 + k[6] * r2 ** 2 + k[7] * r2 ** 3
    g = num / den
    dg = ((k[0] + 2 * k[1] * r2 + 3 * k[4] * r2 ** 2) * den - num * (k[5] + 2 * k[6] * r2 + 3 * k[7] * r2 ** 2)) / den ** 2
    xd = x * g + 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x)
    yd = y * g + k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y
    D = np.empty((len(x), 2, 2))
    D[:, 0, 0] = g + 2 * x * x * dg + 2 * k[2] * y + 6 * k[3] * x
    D[:, 0, 1] = D[:, 1, 0] = 2 * x * y * dg + 2 * k[2] * x + 2 * k[3] * y
    D[:, 1, 1] = g + 2 * y * y * dg + 6 * k[2] * y + 2 * k[3] * x
    return xd, yd, D


def project(P, R, t, K, k=None):
    """pixels (N, 2) of object points P (N, 3) under (R, t), optionally distorted"""
    c = np.asarray(P, np.float64) @ np.asarray(R).T + np.asarray(t).reshape(3)
    x, y = c[:, 0] / c[:, 2], c[:, 1] / c[:, 2]
    if k is not None:
        x, y, _D = _distort_jac(np.asarray(k, np.float64), x, y)
    return np.stack([K[0, 0] * x + K[0, 2], K[1, 1] * y + K[1, 2]], 1)


def pose_jacobian(P, R, t, K, k=None):
    """J (2N, 6), rows u0, v0, u1, ...: d pixel / d(dth, dt_) under the left perturbation; None when a point is at depth <= 0"""
    a = np.asarray(P, np.float64) @ np.asarray(R, np.float64).T
    c = a + np.asarray(t, np.float64).reshape(3)
    if not (c[:, 2] > 0).all():
        return None
    n = len(c)
    dc = np.zeros((n, 3, 6))
    dc[:, :, :3] = -np.stack([skew(ai) for ai in a])
    dc[:, :, 3:] = np.eye(3)
    z = c[:, 2:3]
    dn = np.stack([(dc[:, 0] - c[:, 0:1] / z * dc[:, 2]) / z, (dc[:, 1] - c[:, 1:2] / z * dc[:, 2]) / z], 1)     # (N, 2, 6)
    if k is not None:
        _xd, _yd, D = _distort_jac(np.asarray(k, np.float64), c[:, 0] / c[:, 2], c[:, 1] / c[:, 2])
        dn = D @ dn
    return (np.diag([K[0, 0], K[1, 1]]) @ dn).reshape(2 * n, 6)


def chol_ok(A):
    """the core's pivot rule: every Cholesky pivot > PIVOT x the largest diagonal entry"""
    A = np.asarray(A, np.float64)
    n = len(A)
    L = np.zeros_like(A)
    dmax = max(np.diag(A).max(), 0.0)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        if not d > PIVOT * dmax:
            return False
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return True


def pose_covariance(P, R, t, K, sigma, k=None):
    """-> (Sigma (6, 6), status): sigma^2 (J^T J)^-1, zeros with status DEPTH or SINGULAR when it is unusable"""
    J = pose_jacobian(P, R, t, K, k)
    if J is None:
        return np.zeros((6, 6)), DEPTH
    A = J.T @ J
    if not chol_ok(A):
        return np.zeros((6, 6)), SINGULAR
    S = sigma * sigma * np.linalg.inv(A)
    return 0.5 * (S + S.T), 0


def transition(dt):
    F = np.eye(12)
    F[:6, 6:] = dt * np.eye(6)
    return F


def process_noise(dt, accel_sigma):
    Q = np.zeros((12, 12))
    for a in range(6):
        q = accel_sigma[0 if a < 3 else 1] ** 2
        Q[a, a], Q[a, a + 6], Q[a + 6, a], Q[a + 6, a + 6] = q * dt ** 3 / 3, q * dt ** 2 / 2, q * dt ** 2 / 2, q * dt
    return Q


class FilterRef:
    """one track slot's filter"""

    def __init__(self, accel_sigma, init_velocity_sigma, gate=22.46):
        self.accel_sigma, self.v0, self.gate = accel_sigma, init_velocity_sigma, gate
        self.valid = False
        self.R, self.t, self.w, self.v, self.P = np.eye(3), np.zeros(3), np.zeros(3), np.zeros(3), np.zeros((12, 12))

    def init(self, R, t, S, usable=True):
        self.R, self.t = np.array(R, np.float64), np.array(t, np.float64).reshape(3)
        self.w, self.v = np.zeros(3), np.zeros(3)
        self.P = np.zeros((12, 12))
        if usable:
            self.P[:6, :6] = S
        self.P[6:9, 6:9] = self.v0[0] ** 2 * np.eye(3)
        self.P[9:, 9:] = self.v0[1] ** 2 * np.eye(3)
        self.valid = bool(usable)

    def predict(self, dt):
        self.R = so3_exp(self.w * dt) @ self.R
        self.t = self.t + self.v * dt
        F = transition(dt)
        P = F @ self.P @ F.T + process_noise(dt, self.accel_sigma)
        self.P = 0.5 * (P + P.T)

    def update(self, R, t, S, usable=True):
        """-> True when the measurement was folded in, False when it re-initialised the filter"""
        if not usable or not self.valid:
            self.init(R, t, S, usable)
            return False
        y = np.concatenate([so3_log(np.asarray(R) @ self.R.T), np.asarray(t).reshape(3) - self.t])
        Sy = self.P[:6, :6] + S
        if not chol_ok(Sy) or not y @ np.linalg.solve(Sy, y) <= self.gate:
            self.init(R, t, S, usable)
            return False
        H = np.zeros((6, 12))
        H[:, :6] = np.eye(6)
        Kg = self.P @ H.T @ np.linalg.inv(Sy)
        dx = Kg @ y
        self.R = so3_exp(dx[:3]) @ self.R
        self.t, self.w, self.v = self.t + dx[3:6], self.w + dx[6:9], self.v + dx[9:]
        A = np.eye(12) - Kg @ H
        P = A @ self.P @ A.T + Kg @ S @ Kg.T
        self.P = 0.5 * (P + P.T)
        return True
