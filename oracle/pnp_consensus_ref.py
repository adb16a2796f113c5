"""Oracle: the consensus PnP rule of singleshotpose_b200/csrc/pnp_consensus_core.h restated in numpy fp64, on top of the cold solve
of oracle/pnp_ref.py (cv2.solvePnP ITERATIVE) and the warm solve of oracle/track_ref.py (useExtrinsicGuess=True).

Hypothesis 0 is the cold solve on all points, hypothesis h >= 1 the cold solve on the 6 points of subsets[h-1] in ascending order.
Each is scored on all points with its final LM vector: no inliers if any camera depth is <= 0, else the points whose squared
reprojection error ((fx*x)*iz + cx - u)^2 + (...)^2 is <= thr^2.  The most inliers win, the lower index on a tie; hyp = -1 when no
hypothesis has an inlier.  The winner is refined by a warm LM on its inliers when they differ from its own points and number >= 6.
TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np

from oracle.pnp_ref import rodrigues_vec2mat, solve_pnp_iterative
from oracle.track_ref import solve_pnp_guess


def subset_indices(mask):
    return [i for i in range(16) if (int(mask) >> i) & 1]


def score(R, t, P3, uv, K, thr):
    """-> (inlier mask, squared errors (np,) or None when a point has z <= 0), in the header's order of operations"""
    P = np.asarray(P3, np.float64)
    q = np.asarray(uv, np.float64)
    fx, fy, cx, cy = (np.float64(np.float32(v)) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    x = ((R[0, 0] * P[:, 0] + R[0, 1] * P[:, 1]) + R[0, 2] * P[:, 2]) + t[0]
    y = ((R[1, 0] * P[:, 0] + R[1, 1] * P[:, 1]) + R[1, 2] * P[:, 2]) + t[1]
    z = ((R[2, 0] * P[:, 0] + R[2, 1] * P[:, 1]) + R[2, 2] * P[:, 2]) + t[2]
    if not (z > 0).all():
        return 0, None
    iz = 1.0 / z
    du = ((fx * x) * iz + cx) - q[:, 0]
    dv = ((fy * y) * iz + cy) - q[:, 1]
    e2 = du * du + dv * dv
    thr2 = np.float64(thr) * np.float64(thr)
    return int(sum(1 << i for i in np.nonzero(e2 <= thr2)[0])), e2


def hypotheses(P3, uv, K, subsets, max_iter=20, solve=solve_pnp_iterative):
    """-> list of (rvec, t) of hypothesis 0..H; `solve(P, uv, K)` -> (rvec, t) is the cold solve (cv2.solvePnP for the goldens)"""
    P3 = np.asarray(P3, np.float32)
    uv = np.asarray(uv, np.float32)
    out = [solve(P3, uv, K, max_iter)]
    for m in subsets:
        idx = subset_indices(m)
        out.append(solve(P3[idx], uv[idx], K, max_iter))
    return out


def consensus_ref(P3, uv, K, thr, subsets, max_iter=20, solve=solve_pnp_iterative, refine=solve_pnp_guess, rodrigues=rodrigues_vec2mat):
    """-> dict(R (3,3), t (3,), params (6,), mask int, hyp int, gap): gap = the smallest |e2 - thr^2| over the chosen hypothesis's
    points (over every hypothesis with positive depths when hyp = -1): how far the result is from a threshold flip"""
    P3 = np.asarray(P3, np.float32)
    uv = np.asarray(uv, np.float32)
    npts = len(P3)
    hyps = hypotheses(P3, uv, K, subsets, max_iter, solve)
    masks, errs = [], []
    for r, t in hyps:
        m, e2 = score(rodrigues(r), t, P3, uv, K, thr)
        masks.append(m)
        errs.append(e2)
    counts = [bin(m).count("1") for m in masks]
    hyp = int(np.argmax(counts)) if max(counts) > 0 else -1
    thr2 = float(thr) * float(thr)
    gaps = [np.abs(e - thr2).min() for e in (errs if hyp < 0 else [errs[hyp]]) if e is not None]
    gap = min(gaps) if gaps else np.inf
    r, t = hyps[max(hyp, 0)]
    mask = masks[hyp] if hyp >= 0 else 0
    own = (1 << npts) - 1 if hyp <= 0 else int(subsets[hyp - 1])
    if hyp >= 0 and mask != own and bin(mask).count("1") >= 6:
        idx = subset_indices(mask)
        r, t = refine(P3[idx], uv[idx], K, r, t, max_iter)
    r, t = np.asarray(r, np.float64).reshape(3), np.asarray(t, np.float64).reshape(3)
    return dict(R=rodrigues(r), t=t, params=np.concatenate([r, t]), mask=mask, hyp=hyp, gap=gap)
