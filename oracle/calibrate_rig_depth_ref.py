"""Oracle of the depth calibration of a rig (singleshotpose_b200/csrc/calibrate_rig_depth_core.h) in numpy, written from the rule's
text: whole arrays per view and iteration, one dense solve of the joint normal equations where the core takes the Schur complement
over the free cameras, and numpy's summation order where the core sums by virtual threads, lanes and trees.

The rule per iteration k (gate tau_k as refine_depth_ref): every active view (linked observation that has not stopped, a view of
its set, a connected camera) pairs the mesh with camera c's depth at the camera pose (R_c R_o, R_c t_o + t_c), as refine_rig_ref;
r = m_c . (p_c - q_c); J_obs = refine_rig_ref's world-axis terms; for a free camera (connected, not the reference) J_cam =
[a x m_c + m_c x (p_c - q_c); m_c] with a = R_c (R_o x + t_o).  An observation with fewer than 50 pairs over its views (1) or whose
J_obs^T J_obs fails chol_ok (2) stops with its input pose.  A free camera with fewer than 50 pairs over the remaining views is held.
The joint normal equations over the solved cameras and the remaining observations give (dc, do); a Schur complement that is not
positive definite stops everything with every pose its input (global status 4).  R <- exp([dth]x) R, t <- t + dt_ for both."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import chol_ok, so3_exp
from .refine_depth_ref import FEW_POINTS, MIN_POINTS, SINGULAR, pairs, terms

UNCONNECTED, CAM_FEW_POINTS, CAM_SINGULAR = 1, 2, 4


def view_terms(depth, X, N, Ro, to, K, k, Rc, tc, tau, depth_scale):
    """r (n,), J_obs (n, 6) and J_cam (n, 6) of one view's pairs"""
    a, m, p, q = pairs(depth, X, N, Rc @ Ro, Rc @ to + tc, K, tau, depth_scale, k)
    aw, mw = a @ Rc, m @ Rc
    pw = aw + to
    _rw, Jo = terms(aw, mw, pw, (q - tc) @ Rc)
    r, Jc = terms(pw @ Rc.T, m, p, q)
    return r, Jo, Jc


def calibrate_depth_ref(depths, X, N, Ks, dists, reference, cam_status, R_cam, t_cam, R_world, t_world, views, linked, diam,
                        depth_scale=0.001, iters=10, gate=(0.5, 0.02)):
    """depths (G, C, H, W); Ks (C, 3, 3); dists None or (C, 8); R_cam (C, 3, 3), t_cam (C, 3); R_world (O, 3, 3), t_world (O, 3)
    with O = G S; views (O, C), linked (O,) -> dict of the outputs"""
    Cn, O, G = len(Ks), len(R_world), len(depths)
    S = O // G
    conn = (np.asarray(cam_status) & UNCONNECTED) == 0
    free = conn & (np.arange(Cn) != reference)
    ks = [None if dists is None or not np.any(dists[c]) else np.asarray(dists[c], np.float64) for c in range(Cn)]
    Rc, tc = np.array(R_cam, np.float64), np.array(t_cam, np.float64)
    Ro, to = np.array(R_world, np.float64), np.array(t_world, np.float64)
    stop = np.zeros(O, np.int32)
    out = dict(cam_cov=np.zeros((Cn, 6, 6)), cam_points=np.zeros(Cn, np.int64), cam_rmse=np.zeros(Cn), cam_status=np.where(conn, 0, UNCONNECTED),
               obs_points=np.zeros(O, np.int64), obs_rmse=np.zeros(O), obs_status=np.zeros(O, np.int32), status=0, iter_rmse=np.zeros(iters))
    s, e = gate
    for it in range(iters):
        tau = diam * (s if iters == 1 else s * (e / s) ** (it / (iters - 1)))
        T = {}
        for o in range(O):
            if not linked[o] or stop[o]:
                continue
            for c in range(Cn):
                if views[o, c] and conn[c]:
                    T[o, c] = view_terms(depths[o // S, c], X, N, Ro[o], to[o], np.asarray(Ks[c], np.float64), ks[c], Rc[c], tc[c], tau,
                                         depth_scale)
            rs = [T[o, c][0] for c in range(Cn) if (o, c) in T]
            r = np.concatenate(rs) if rs else np.zeros(0)
            Jo = np.concatenate([T[o, c][1] for c in range(Cn) if (o, c) in T]) if rs else np.zeros((0, 6))
            n = len(r)
            out["obs_points"][o], out["obs_rmse"][o] = n, (np.sqrt((r @ r) / n) if n else 0.0)
            if n < MIN_POINTS:
                stop[o] = FEW_POINTS
            elif not chol_ok(Jo.T @ Jo):
                stop[o] = SINGULAR
            out["obs_status"][o] = stop[o]
        live = [o for o in range(O) if linked[o] and not stop[o]]
        n_c, r2_c = np.zeros(Cn), np.zeros(Cn)
        for (o, c), (r, _Jo, _Jc) in T.items():
            if not stop[o]:
                n_c[c] += len(r)
                r2_c[c] += r @ r
        held = free & (n_c < MIN_POINTS)
        cams = [c for c in range(Cn) if free[c] and not held[c]]
        out["iter_rmse"][it] = np.sqrt(r2_c[conn].sum() / n_c[conn].sum()) if n_c[conn].sum() else 0.0
        out["cam_points"] = np.where(conn, n_c, 0).astype(np.int64)
        out["cam_rmse"] = np.where(conn & (n_c > 0), np.sqrt(r2_c / np.maximum(n_c, 1)), 0.0)
        # the joint normal equations: cameras first, then the live observations
        nc, nx = 6 * len(cams), 6 * (len(cams) + len(live))
        Hm, g = np.zeros((nx, nx)), np.zeros(nx)
        for i, o in enumerate(live):
            oi = nc + 6 * i
            for c in range(Cn):
                if (o, c) not in T:
                    continue
                r, Jo, Jc = T[o, c]
                J = np.zeros((len(r), nx))
                J[:, oi:oi + 6] = Jo
                if c in cams:
                    ci = 6 * cams.index(c)
                    J[:, ci:ci + 6] = Jc
                Hm += J.T @ J
                g += J.T @ r
        Hcc, Hco, Hoo = Hm[:nc, :nc], Hm[:nc, nc:], Hm[nc:, nc:]
        Sc = Hcc - Hco @ np.linalg.solve(Hoo, Hco.T) if live else Hcc
        try:
            np.linalg.cholesky(Sc) if nc else None
        except np.linalg.LinAlgError:
            out["status"] = CAM_SINGULAR
            out["cam_status"] = np.where(conn, 0, UNCONNECTED) | np.where(held, CAM_FEW_POINTS, 0) | np.where(free, CAM_SINGULAR, 0)
            out.update(R=np.array(R_cam, np.float64), t=np.array(t_cam, np.float64), R_world=np.array(R_world, np.float64),
                       t_world=np.array(t_world, np.float64))
            return out
        out["cam_status"] = np.where(conn, 0, UNCONNECTED) | np.where(held, CAM_FEW_POINTS, 0)
        if it == iters - 1 and nc:
            cov = out["iter_rmse"][it] ** 2 * np.linalg.inv(Sc)
            for i, c in enumerate(cams):
                out["cam_cov"][c] = cov[6 * i:6 * i + 6, 6 * i:6 * i + 6]
        delta = -np.linalg.solve(Hm, g) if nx else np.zeros(0)
        for i, c in enumerate(cams):
            d = delta[6 * i:6 * i + 6]
            Rc[c], tc[c] = so3_exp(d[:3]) @ Rc[c], tc[c] + d[3:]
        for i, o in enumerate(live):
            d = delta[nc + 6 * i:nc + 6 * i + 6]
            Ro[o], to[o] = so3_exp(d[:3]) @ Ro[o], to[o] + d[3:]
    keep = (~np.asarray(linked, bool)) | (stop != 0)
    out.update(R=Rc, t=tc, R_world=np.where(keep[:, None, None], R_world, Ro), t_world=np.where(keep[:, None], t_world, to))
    return out
