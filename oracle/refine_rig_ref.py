"""Oracle of the rig refinement (singleshotpose_b200/csrc/refine_rig_core.h) in numpy, written from the rule's text: whole arrays
per camera and iteration, numpy's summation order where the core sums per virtual thread, by a halving tree and in camera order.

The rule per iteration k (gate tau_k as refine_depth_ref): camera c's pose is (R_c R, R_c t + t_c); its pairs are refine_depth_ref's
pairs with its depth frame, fp64 K_c and coefficients; each pair's terms are taken in world axes, a_w = R x, m_w = R n,
p_w = a_w + t, q_w = R_c^T (q - t_c); the normal equations of every camera are added and solved once for the world pose (left
perturbation: R <- exp([dth]x) R, t <- t + dt_).  Fewer than 50 pairs in all (status 1) or a Cholesky pivot <= 1e-12 x the largest
diagonal (status 2) stops with the input pose; a pose that is not finite, or a fusion status with NO_VALID or NO_VIEW, is status 4."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import chol_ok, so3_exp
from .refine_depth_ref import BAD_POSE, FEW_POINTS, MIN_POINTS, SINGULAR, pairs, terms

FUSE_NONE = 1 | 2                                                      # SSP_FUSE_NO_VALID | SSP_FUSE_NO_VIEW


def world_terms(depth, X, N, R, t, K, k, Rc, tc, tau, depth_scale):
    """r (n,) and J (n, 6) in world axes of one camera's pairs under the world pose (R, t)"""
    a, m, p, q = pairs(depth, X, N, Rc @ R, Rc @ t + tc, K, tau, depth_scale, k)
    aw, mw = a @ Rc, m @ Rc                                            # R_c^T (R_c R x) = R x
    pw = aw + t
    qw = (q - tc) @ Rc
    return terms(aw, mw, pw, qw)


def refine_rig_ref(depths, X, N, Ks, dists, Rr, tr, R, t, diam, depth_scale=0.001, iters=10, gate=(0.5, 0.02), fuse_status=0):
    """one problem: depths (C, H, W), Ks (C, 3, 3), dists None or (C, 8) (a zero row: pinhole), Rr (C, 3, 3), tr (C, 3) ->
    (R, t, points, rmse, status, view_points (C,), view_rmse (C,))"""
    Cn = len(Ks)
    R0, t0 = np.asarray(R, np.float64), np.asarray(t, np.float64).reshape(3)
    vp, vr = np.zeros(Cn, np.int64), np.zeros(Cn)
    if not (np.isfinite(R0).all() and np.isfinite(t0).all()) or fuse_status & FUSE_NONE:
        return R0, t0, 0, 0.0, BAD_POSE, vp, vr
    ks = [None if dists is None or not np.any(dists[c]) else np.asarray(dists[c], np.float64) for c in range(Cn)]
    s, e = gate
    R, t = R0.copy(), t0.copy()
    for it in range(iters):
        tau = diam * (s if iters == 1 else s * (e / s) ** (it / (iters - 1)))
        rs, Js = [], []
        for c in range(Cn):
            r, J = world_terms(depths[c], X, N, R, t, np.asarray(Ks[c], np.float64), ks[c], Rr[c], tr[c], tau, depth_scale)
            rs.append(r)
            Js.append(J)
            vp[c], vr[c] = len(r), (np.sqrt((r @ r) / len(r)) if len(r) else 0.0)
        r, J = np.concatenate(rs), np.concatenate(Js)
        n = len(r)
        rmse = float(np.sqrt((r @ r) / n)) if n else 0.0
        if n < MIN_POINTS:
            return R0, t0, n, rmse, FEW_POINTS, vp, vr
        A = J.T @ J
        if not chol_ok(A):
            return R0, t0, n, rmse, SINGULAR, vp, vr
        delta = -np.linalg.solve(A, J.T @ r)
        R, t = so3_exp(delta[:3]) @ R, t + delta[3:]
    return R, t, n, rmse, 0, vp, vr
