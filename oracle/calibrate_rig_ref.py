"""Oracle of the rig calibration (singleshotpose_b200/csrc/calibrate_rig_core.h) in numpy, written from the rule's text with whole
arrays.  It starts from the per-view poses of step 1 (the PnP of pnp_core.h) and restates steps 2-6; the fusion of step 4 is
oracle/multiview_ref.py's.

Pair a < b: each co-observation o gives T_ba = T_b,o T_a,o^-1 (the ones at floor(i n / 256) past 256); it agrees with o' when
view a's pose carried into camera b and view b's pose carried into camera a both lie in front within gate px (mean squared
error); the winner has the most agreements, then the lower summed error (COST_TIE), then the lower index.  Prim's maximum spanning
tree from the reference over edges with >= 3 agreements gives the initial rig.  Then rounds of: fuse every observation under the
rig; stop when no linked set changed; LM over the free cameras (left perturbation in the camera frame) and the linked
observations' world poses, solved here on the full normal equations (the Schur complement is the same system)."""
from __future__ import annotations

import numpy as np

from .multiview_ref import COST_TIE, Rig, fuse_ref, view_mse
from .pose_filter_ref import pose_jacobian, project, so3_exp

MAX_PAIR_HYP, MIN_AGREE, ROUNDS = 256, 3, 4
UNCONNECTED, SINGULAR = 1, 2


def _mse(K, d, R, t, P, uv):
    rig = Rig(K[None], None if d is None else d[None], np.eye(3)[None], np.zeros((1, 3)))
    return view_mse(rig, 0, R, t, P, uv)


def pair_scores(K, dist, P, uv, valid, R_rows, t_rows, a, b, gate):
    """-> [(R_ba, t_ba, agreements, cost)] of pair (a, b); P (O, C, N, 3), uv (O, C, N, 2), valid (O, C), R_rows (O, C, 3, 3)"""
    co = np.flatnonzero(valid[:, a] & valid[:, b])
    n = len(co)
    idx = co if n <= MAX_PAIR_HYP else co[(np.arange(MAX_PAIR_HYP) * n) // MAX_PAIR_HYP]
    da, db = (None if dist is None or not dist[c].any() else dist[c] for c in (a, b))
    out = []
    for o in idx:
        Rba = R_rows[o, b] @ R_rows[o, a].T
        tba = t_rows[o, b] - Rba @ t_rows[o, a]
        agree, cost = 0, 0.0
        for q in co:
            fb, mb = _mse(K[b], db, Rba @ R_rows[q, a], Rba @ t_rows[q, a] + tba, P[q, b], uv[q, b])
            fa, ma = _mse(K[a], da, Rba.T @ R_rows[q, b], Rba.T @ (t_rows[q, b] - tba), P[q, a], uv[q, a])
            if fa and fb and ma <= gate * gate and mb <= gate * gate:
                agree, cost = agree + 1, cost + mb + ma
        out.append((Rba, tba, agree, cost))
    return out


def winner(scores):
    best = None
    for i, (_R, _t, n, c) in enumerate(scores):
        if best is None or n > scores[best][2] or (n == scores[best][2] and c < scores[best][3] * (1 - COST_TIE)):
            best = i
    return best


def initial_rig(C, reference, wins):
    """wins {(a, b): (R_ba, t_ba, agreements)} -> R (C, 3, 3), t (C, 3), parent (C,), edge_agree (C,), connected (C,) bool"""
    R, t = np.zeros((C, 3, 3)), np.zeros((C, 3))
    R[reference] = np.eye(3)
    parent, agree = -np.ones(C, int), np.zeros(C, int)
    inn = np.zeros(C, bool)
    inn[reference] = True
    pairs = [(a, b) for a in range(C) for b in range(a + 1, C)]
    while True:
        best = None
        for p, (a, b) in enumerate(pairs):
            if inn[a] == inn[b] or (a, b) not in wins or wins[(a, b)][2] < MIN_AGREE:
                continue
            if best is None or wins[(a, b)][2] > wins[pairs[best]][2]:
                best = p
        if best is None:
            break
        a, b = pairs[best]
        Rba, tba, n = wins[(a, b)]
        if inn[a]:
            R[b], t[b], parent[b], agree[b], inn[b] = Rba @ R[a], Rba @ t[a] + tba, a, n, True
        else:
            R[a], t[a], parent[a], agree[a], inn[a] = Rba.T @ R[b], Rba.T @ (t[b] - tba), b, n, True
    return R, t, parent, agree, inn


def _residuals(K, dist, Rc, tc, P, uv, obs, sets, poses, free):
    """r and J over the linked observations: columns 6 per free camera, then 6 per observation; None when a point is behind"""
    nf = len(free)
    rs, rows = [], []
    ncol = 6 * nf + 6 * len(obs)
    for j, o in enumerate(obs):
        R, t = poses[j]
        for c in sorted(sets[o]):
            k = None if dist is None or not dist[c].any() else dist[c]
            Rw, tw = Rc[c] @ R, Rc[c] @ t + tc[c]
            Jo = pose_jacobian(P[o, c], Rw, tw, K[c], k)
            if Jo is None:
                return None
            Xw = P[o, c] @ R.T + t
            J = np.zeros((2 * len(Xw), ncol))
            J[:, 6 * nf + 6 * j:6 * nf + 6 * j + 6] = Jo @ np.kron(np.eye(2), Rc[c])
            if c in free:
                i = free.index(c)
                J[:, 6 * i:6 * i + 6] = pose_jacobian(Xw, Rc[c], tc[c], K[c], k)
            rs.append((project(P[o, c], Rw, tw, K[c], k) - uv[o, c]).reshape(-1))
            rows.append(J)
    if not rows:
        return np.zeros(0), np.zeros((0, ncol))
    return np.concatenate(rs), np.concatenate(rows)


def bundle_adjust(K, dist, Rc, tc, P, uv, obs, sets, poses, free, max_iter):
    """LM of step 5 -> (Rc, tc, poses, cost, steps, J at the end)"""
    Rc, tc, poses = Rc.copy(), tc.copy(), list(poses)
    out = _residuals(K, dist, Rc, tc, P, uv, obs, sets, poses, free)
    if out is None:
        return Rc, tc, poses, np.inf, 0, None
    r, J = out
    cost, lam, steps = r @ r, 1e-3, 0
    nf = len(free)
    for _ in range(max_iter):
        steps += 1
        A, g = J.T @ J, J.T @ r
        M = A + lam * np.diag(np.diag(A))
        try:
            np.linalg.cholesky(M)
        except np.linalg.LinAlgError:
            lam *= 10
            continue
        d = -np.linalg.solve(M, g) if len(g) else np.zeros(0)
        if np.linalg.norm(d) < 1e-12:
            break
        Rn, tn = Rc.copy(), tc.copy()
        for i, c in enumerate(free):
            Rn[c], tn[c] = so3_exp(d[6 * i:6 * i + 3]) @ Rc[c], tc[c] + d[6 * i + 3:6 * i + 6]
        pn = [(so3_exp(d[6 * nf + 6 * j:6 * nf + 6 * j + 3]) @ R, t + d[6 * nf + 6 * j + 3:6 * nf + 6 * j + 6]) for j, (R, t) in enumerate(poses)]
        new = _residuals(K, dist, Rn, tn, P, uv, obs, sets, pn, free)
        if new is not None and new[0] @ new[0] < cost:
            Rc, tc, poses, (r, J), cost = Rn, tn, pn, new, new[0] @ new[0]
            lam /= 10
        else:
            lam *= 10
    return Rc, tc, poses, cost, steps, J


def calibrate_ref(K, dist, P, uv, valid, R_rows, t_rows, reference=0, gate=40.0, reproj_thresh=8.0, sigma=2.0, max_iter=30):
    """K (C, 3, 3) fp32 values, dist (C, 8) or None; per observation o and camera c: P (O, C, N, 3), uv (O, C, N, 2), valid (O, C),
    R_rows (O, C, 3, 3), t_rows (O, C, 3) the per-view poses -> dict of the outputs"""
    K = np.asarray(K, np.float32).astype(np.float64)
    P = np.asarray(P, np.float32).astype(np.float64)
    uv = np.asarray(uv, np.float32).astype(np.float64)
    valid = np.asarray(valid, bool)
    O, C = valid.shape
    wins = {}
    for a in range(C):
        for b in range(a + 1, C):
            sc = pair_scores(K, dist, P, uv, valid, R_rows, t_rows, a, b, gate)
            if sc:
                w = sc[winner(sc)]
                wins[(a, b)] = (w[0], w[1], w[2])
    Rc, tc, parent, edge, conn = initial_rig(C, reference, wins)
    R_tree, t_tree = Rc.copy(), tc.copy()
    free = [c for c in range(C) if conn[c] and c != reference]
    keys, rounds, iters, cost, cov, singular = None, 0, 0, 0.0, np.zeros((C, 6, 6)), False
    while True:
        rig = Rig(K, dist, Rc, tc)
        fused = [fuse_ref(rig, P[o], uv[o], valid[o] & conn, R_rows[o], t_rows[o], gate, reproj_thresh, sigma, max_iter) for o in range(O)]
        sets = [frozenset(np.flatnonzero(f["views"])) for f in fused]
        new = [s if len(s) >= 2 else frozenset() for s in sets]
        if (keys is not None and new == keys) or rounds == ROUNDS:
            break
        keys = new
        obs = [o for o in range(O) if new[o]]
        Rc, tc, poses, cost, steps, J = bundle_adjust(K, dist, Rc, tc, P, uv, obs, new, [(fused[o]["R"], fused[o]["t"]) for o in obs],
                                                      free, max_iter)
        rounds, iters = rounds + 1, iters + steps
        cov, singular = np.zeros((C, 6, 6)), False
        if free:
            _r, J = _residuals(K, dist, Rc, tc, P, uv, obs, new, poses, free)
            A = J.T @ J
            try:
                np.linalg.cholesky(A)
                Ai = np.linalg.inv(A)
                for i, c in enumerate(free):
                    cov[c] = sigma * sigma * Ai[6 * i:6 * i + 6, 6 * i:6 * i + 6]
            except np.linalg.LinAlgError:
                singular = True
    linked = np.array([len(s) >= 2 for s in sets])
    views = np.array([f["views"] for f in fused])
    view_err = np.array([f["view_err"] for f in fused])
    cam_obs = np.array([(linked & views[:, c]).sum() for c in range(C)])
    cam_rmse = np.array([np.sqrt((view_err[linked & views[:, c], c] ** 2).mean()) if cam_obs[c] else -1.0 for c in range(C)])
    status = np.array([(0 if conn[c] else UNCONNECTED) | (SINGULAR if singular and c in free else 0) for c in range(C)])
    return dict(R=Rc, t=tc, cam_cov=cov, cam_obs=cam_obs, cam_rmse=cam_rmse, tree_parent=parent, edge_agree=edge, cam_status=status,
                R_world=np.array([f["R"] for f in fused]), t_world=np.array([f["t"] for f in fused]), views=views, view_err=view_err,
                linked=linked, rounds=rounds, iterations=iters, cost=cost, R_tree=R_tree, t_tree=t_tree)
