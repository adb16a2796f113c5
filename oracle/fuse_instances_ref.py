"""Oracle of the instance fusion (singleshotpose_b200/csrc/multiview_instances_core.h) in numpy, written from the rule's text with
whole arrays per view and multiview_ref's agreement, LM and residuals.  It starts from the per-row poses of step 1 and restates
the association for one capture, rescoring every available hypothesis in every round.

A detection (c, m) exists when m < count[c]; hypothesis h = c M + m is its pose in the world frame.  assign(R, t, k, thr, U)
takes, per view, the available class-k detection with every point in front and the lowest mean squared reprojection error
(ties: the lower slot) and keeps it when that error is <= thr^2.  A hypothesis is fitted on assign(gate), refitted on
assign(reproj_thresh) of that fit when the choice changed, and members beyond reproj_thresh leave while any do.  Each class's
candidate is the best of its hypotheses (most views, then a cost lower by COST_TIE relative, then the lower index, scanned in
index order); the winner is the best candidate by the same scan.  It becomes a world instance, its detections leave, and the
rounds repeat until no hypothesis keeps a view or M instances are out."""
from __future__ import annotations

import numpy as np

from .multiview_ref import COST_TIE, SINGULAR, lm, residuals, view_mse
from .pose_filter_ref import chol_ok


def _assign(rig, R, t, k, thr, avail, cls, P, uv):
    """-> {view: chosen slot} of the views that join"""
    C, M = cls.shape
    out = {}
    for c in range(C):
        cands = [m for m in range(M) if avail[c, m] and cls[c, m] == k]
        errs = [view_mse(rig, c, R, t, P[k], uv[c, m]) for m in cands]
        front = [(e, m) for (f, e), m in zip(errs, cands) if f]
        if front:
            e, m = min(front, key=lambda x: (x[0], x[1]))
            if e <= thr * thr:
                out[c] = m
    return out


def _fit(rig, sel, R, t, k, P, uv, R_rows, t_rows, max_iter):
    """a fit of the chosen detections {view: slot}"""
    Pv, uvv = _views(rig, sel, k, P, uv)
    if len(sel) == 1:
        (c, m), = sel.items()
        return rig.R[c].T @ R_rows[c, m], rig.R[c].T @ (t_rows[c, m] - rig.t[c])
    return lm(rig, frozenset(sel), R, t, Pv, uvv, max_iter)


def _views(rig, sel, k, P, uv):
    """(C, N, 3) and (C, N, 2) arrays holding the chosen detections in their views' rows"""
    Pv = np.repeat(P[k][None], rig.C, 0)
    uvv = np.zeros((rig.C,) + uv.shape[2:])
    for c, m in sel.items():
        uvv[c] = uv[c, m]
    return Pv, uvv


def _score(rig, h, avail, cls, P, uv, R_rows, t_rows, gate, thr, max_iter):
    """-> (views, cost, R, t, {view: slot}) of hypothesis h"""
    C, M = cls.shape
    c0, m0 = divmod(h, M)
    k = cls[c0, m0]
    R, t = rig.R[c0].T @ R_rows[c0, m0], rig.R[c0].T @ (t_rows[c0, m0] - rig.t[c0])
    A = _assign(rig, R, t, k, gate, avail, cls, P, uv)
    if not A:
        return 0, np.inf, R, t, {}
    R, t = _fit(rig, A, R, t, k, P, uv, R_rows, t_rows, max_iter)
    A2 = _assign(rig, R, t, k, thr, avail, cls, P, uv)
    if A2 != A and A2:
        R, t = _fit(rig, A2, R, t, k, P, uv, R_rows, t_rows, max_iter)
    while A2:                                           # the check, the chosen detections held fixed
        A3 = {c: m for c, m in A2.items() if (lambda f, e: f and e <= thr * thr)(*view_mse(rig, c, R, t, P[k], uv[c, m]))}
        if A3 == A2:
            break
        A2 = A3
        if A2:
            R, t = _fit(rig, A2, R, t, k, P, uv, R_rows, t_rows, max_iter)
    if not A2:
        return 0, np.inf, R, t, {}
    Pv, uvv = _views(rig, A2, k, P, uv)
    out = residuals(rig, frozenset(A2), R, t, Pv, uvv)
    cost = np.inf if out is None else float(out[0] @ out[0])
    return len(A2), cost, R, t, A2


def _scan(hyps, scores):
    best, bn, bc = -1, 0, 0.0
    for h in hyps:
        n, cost = scores[h][0], scores[h][1]
        if n > bn or (n == bn and n > 0 and cost < bc * (1 - COST_TIE)):
            best, bn, bc = h, n, cost
    return best


def fuse_instances_ref(rig, P, uv, cls, count, R_rows, t_rows, gate=40.0, reproj_thresh=8.0, sigma=2.0, max_iter=20):
    """one capture: P (num_classes, N, 3) class points, uv (C, M, N, 2), cls (C, M), count (C,), R_rows (C, M, 3, 3), t_rows
    (C, M, 3) -> list of world instances dict(cls, R, t, cov, members (C,) slot or -1, hyp, status), and the unfused count"""
    P = np.asarray(P, np.float32).astype(np.float64)
    uv = np.asarray(uv, np.float32).astype(np.float64)
    cls = np.asarray(cls)
    C, M = cls.shape
    nC = len(P)
    avail = (np.arange(M)[None] < np.asarray(count)[:, None]) & (cls >= 0) & (cls < nC)
    out = []
    while len(out) < M:
        scores = {h: _score(rig, h, avail, cls, P, uv, R_rows, t_rows, gate, reproj_thresh, max_iter)
                  for h in range(C * M) if avail.flat[h]}
        cands = sorted(w for w in (_scan([h for h in scores if cls.flat[h] == k], scores) for k in range(nC)) if w >= 0)
        win = _scan(cands, scores)
        if win < 0:
            break
        n, _cost, R, t, sel = scores[win]
        k = int(cls.flat[win])
        Pv, uvv = _views(rig, sel, k, P, uv)
        _r, J = residuals(rig, frozenset(sel), R, t, Pv, uvv)
        A = J.T @ J
        ok = chol_ok(A)
        members = -np.ones(C, int)
        for c, m in sel.items():
            members[c] = m
            avail[c, m] = False
        out.append(dict(cls=k, R=R, t=t, cov=sigma * sigma * np.linalg.inv(A) if ok else np.zeros((6, 6)), members=members, hyp=int(win),
                        status=0 if ok else SINGULAR))
    return out, int(avail.sum())
