"""Oracle of the multi-view fusion (singleshotpose_b200/csrc/multiview_core.h) in numpy, written from the rule's text with whole
arrays per view.  It starts from the per-view poses of step 1 (the PnP of pnp_core.h, which tests/test_pnp_*.py check against
cv2) and restates steps 2-5 for one (capture, slot).

A world pose (R, t) is seen by camera c as (R_c R, R_c t + t_c).  Hypothesis v: (R_v^T R_(v), R_v^T (t_(v) - t_v)).  View w
agrees at thr when all its points lie at depth > 0 and their mean squared reprojection error is <= thr^2.  Stage one fits the
views that agree at the gate, stage two the views that agree with that fit at reproj_thresh when they differ, and while a view
of the set leaves reproj_thresh of the fit it is dropped and the rest refitted; the winner's own final pose is the fused pose.  A
fit of one view
is its hypothesis, of more views the LM: J = pose_jacobian at the camera pose times diag(R_c, R_c), (A + lambda diag A) delta =
-g, lambda from 1e-3, / 10 on a lower cost, x 10 otherwise, at most max_iter steps, stop at |delta| < 1e-12, R <- exp(dth) R,
t <- t + dt_.  The winner has the most final views, then the lower cost (by more than COST_TIE relative), then the lower index."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import chol_ok, pose_jacobian, project, so3_exp

NO_VALID, NO_VIEW, SINGULAR = 1, 2, 4
COST_TIE = 1e-9             # a cost counts as lower only below (1 - COST_TIE) x the best so far


class Rig:
    """K (C, 3, 3) fp32 values, dist (C, 8) or None, R (C, 3, 3), t (C, 3)"""

    def __init__(self, K, dist, R, t):
        self.K = np.asarray(K, np.float32).astype(np.float64)
        self.dist = None if dist is None else np.asarray(dist, np.float64)
        self.R, self.t = np.asarray(R, np.float64), np.asarray(t, np.float64)
        self.C = len(self.K)

    def k(self, c):
        return None if self.dist is None or not self.dist[c].any() else self.dist[c]

    def pose(self, c, R, t):
        return self.R[c] @ R, self.R[c] @ t + self.t[c]


def view_mse(rig, c, R, t, P, uv):
    """(all points in front, mean squared reprojection error) of view c under the world pose"""
    Rw, tw = rig.pose(c, R, t)
    z = (P @ Rw.T + tw)[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        e = project(P, Rw, tw, rig.K[c], rig.k(c)) - uv
    return bool((z > 0).all()), float((e * e).sum() / len(P))


def agree(rig, valid, R, t, P, uv, thr):
    out = set()
    for c in np.flatnonzero(valid):
        front, mse = view_mse(rig, c, R, t, P[c], uv[c])
        if front and mse <= thr * thr:
            out.add(int(c))
    return frozenset(out)


def residuals(rig, views, R, t, P, uv):
    """r (2N,) and J (2N, 6) over the views, or None when a point lies at depth <= 0"""
    rs, Js = [], []
    for c in sorted(views):
        Rw, tw = rig.pose(c, R, t)
        J = pose_jacobian(P[c], Rw, tw, rig.K[c], rig.k(c))
        if J is None:
            return None
        rs.append((project(P[c], Rw, tw, rig.K[c], rig.k(c)) - uv[c]).reshape(-1))
        Js.append(J @ np.kron(np.eye(2), rig.R[c]))
    return np.concatenate(rs), np.concatenate(Js)


def lm(rig, views, R, t, P, uv, max_iter=20):
    r, J = residuals(rig, views, R, t, P, uv)
    cost, lam = r @ r, 1e-3
    for _ in range(max_iter):
        A, g = J.T @ J, J.T @ r
        M = A + lam * np.diag(np.diag(A))
        try:
            np.linalg.cholesky(M)
        except np.linalg.LinAlgError:
            lam *= 10
            continue
        d = -np.linalg.solve(M, g)
        if np.linalg.norm(d) < 1e-12:
            break
        Rn, tn = so3_exp(d[:3]) @ R, t + d[3:]
        out = residuals(rig, views, Rn, tn, P, uv)
        if out is not None and out[0] @ out[0] < cost:
            R, t, (r, J), cost = Rn, tn, out, out[0] @ out[0]
            lam /= 10
        else:
            lam *= 10
    return R, t


def hypothesis(rig, h, R_rows, t_rows):
    return rig.R[h].T @ R_rows[h], rig.R[h].T @ (t_rows[h] - rig.t[h])


def fit(rig, views, R, t, R_rows, t_rows, P, uv, max_iter):
    if len(views) == 1:
        return hypothesis(rig, next(iter(views)), R_rows, t_rows)
    return lm(rig, views, R, t, P, uv, max_iter)


def fuse_ref(rig, P, uv, valid, R_rows, t_rows, gate=40.0, reproj_thresh=8.0, sigma=2.0, max_iter=20):
    """one (capture, slot): P (C, N, 3), uv (C, N, 2), valid (C,) bool, R_rows (C, 3, 3), t_rows (C, 3) the per-view poses ->
    dict(R, t, cov, views (C,) bool, view_err (C,), hyp, status)"""
    P = np.asarray(P, np.float32).astype(np.float64)
    uv = np.asarray(uv, np.float32).astype(np.float64)
    valid = np.asarray(valid, bool)
    C = rig.C
    zero = dict(R=np.zeros((3, 3)), t=np.zeros(3), cov=np.zeros((6, 6)), views=np.zeros(C, bool), view_err=-np.ones(C), hyp=-1)
    if not valid.any():
        return dict(zero, status=NO_VALID)
    best = None
    for h in np.flatnonzero(valid):
        R, t = hypothesis(rig, h, R_rows, t_rows)
        A = agree(rig, valid, R, t, P, uv, gate)
        if not A:
            continue
        R, t = fit(rig, A, R, t, R_rows, t_rows, P, uv, max_iter)
        A2 = agree(rig, valid, R, t, P, uv, reproj_thresh)
        if not A2:
            continue
        if A2 != A:
            R, t = fit(rig, A2, R, t, R_rows, t_rows, P, uv, max_iter)
        while A2:                                       # the check: fused views beyond reproj_thresh leave, the rest is refitted
            A3 = agree(rig, np.isin(np.arange(C), list(A2)), R, t, P, uv, reproj_thresh)
            if A3 == A2:
                break
            A2 = A3
            if A2:
                R, t = fit(rig, A2, R, t, R_rows, t_rows, P, uv, max_iter)
        if not A2:
            continue
        r, _J = residuals(rig, A2, R, t, P, uv)
        cost = r @ r
        if best is None or len(A2) > len(best[3]) or (len(A2) == len(best[3]) and cost < best[1] * (1 - COST_TIE)):
            best = (h, cost, (R, t), A2)
    if best is None:
        return dict(zero, status=NO_VIEW)
    h, _cost, (R, t), views = best
    _r, J = residuals(rig, views, R, t, P, uv)
    A = J.T @ J
    status = 0 if chol_ok(A) else SINGULAR
    cov = sigma * sigma * np.linalg.inv(A) if status == 0 else np.zeros((6, 6))
    err = np.array([np.sqrt(view_mse(rig, c, R, t, P[c], uv[c])[1]) if valid[c] else -1.0 for c in range(C)])
    return dict(R=R, t=t, cov=cov, views=np.isin(np.arange(C), list(views)), view_err=err, hyp=int(h), status=status)
