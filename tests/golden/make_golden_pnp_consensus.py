#!/usr/bin/env python
"""Goldens of the consensus PnP (singleshotpose_b200/csrc/pnp_consensus_core.h) computed with cv2 itself: every hypothesis is
cv2.solvePnP(..., SOLVEPNP_ITERATIVE) on all points or on a 6-point subset, the scoring uses cv2.Rodrigues of its rvec, and the
refinement is cv2.solvePnP(..., useExtrinsicGuess=True) on the inliers.  Problems: the 9 box points (centroid + corners) and the
8 corners; keypoint noise sigma = 0, 1, 3 px; k = 0..3 keypoints moved by 40-150 px in a random direction; threshold 8 px.  Plus
uniform garbage keypoints at a 2 px threshold, for the no-inlier and the fewer-than-6-inliers branches.  Per problem: cv2's pose,
the chosen hypothesis, its inlier mask and `gap`, the smallest |e2 - thr^2| over the chosen hypothesis's points (over every
hypothesis in front of the camera when none has an inlier), so that tests can leave threshold-borderline problems out.  A
problem where cv2's LM runs away (|t| > 10 m) is left out, as in make_golden_pnp_guess.py.  Needs cv2 only; writes
tests/golden/pnp_consensus.npz.

    python tests/golden/make_golden_pnp_consensus.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.pnp_consensus_ref import consensus_ref            # noqa: E402
from singleshotpose_b200 import synth                         # noqa: E402
from singleshotpose_b200.utils import consensus_subsets       # noqa: E402

SIGMAS = (0, 1, 3)
OUTLIERS = (0, 1, 2, 3)
N = 8                # problems per (points, sigma, k)
N_GARBAGE = 12       # per point count


def _cv2_solve(P, uv, K, max_iter):
    import cv2
    ok, r, t = cv2.solvePnP(np.ascontiguousarray(P, np.float32), np.ascontiguousarray(uv, np.float32), np.asarray(K, np.float32), None,
                            flags=cv2.SOLVEPNP_ITERATIVE)
    assert ok
    return r.reshape(3), t.reshape(3)


def _cv2_refine(P, uv, K, r, t, max_iter):
    import cv2
    r_in, t_in = np.asarray(r, np.float64).reshape(3, 1).copy(), np.asarray(t, np.float64).reshape(3, 1).copy()
    ok, r, t = cv2.solvePnP(np.ascontiguousarray(P, np.float32), np.ascontiguousarray(uv, np.float32), np.asarray(K, np.float32), None,
                            r_in, t_in, useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
    assert ok
    return r.reshape(3), t.reshape(3)


def _cv2_rodrigues(r):
    import cv2
    return cv2.Rodrigues(np.asarray(r, np.float64).reshape(3, 1))[0]


def _problem(P3, K, rng, sigma, k):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    R = _cv2_rodrigues(ax * rng.uniform(0, np.pi))
    t = np.array([rng.uniform(-.2, .2), rng.uniform(-.15, .15), rng.uniform(.6, 1.2)])
    Pc = P3.astype(np.float64) @ R.T + t
    uv = np.stack([K[0, 0] * Pc[:, 0] / Pc[:, 2] + K[0, 2], K[1, 1] * Pc[:, 1] / Pc[:, 2] + K[1, 2]], -1)
    uv = uv + rng.normal(size=uv.shape) * sigma
    bad = rng.choice(len(P3), k, replace=False)
    ang, rad = rng.uniform(0, 2 * np.pi, k), rng.uniform(40, 150, k)
    uv[bad] += np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
    return uv.astype(np.float32), sum(1 << int(i) for i in bad)


def main():
    import cv2
    K = synth.intrinsics().astype(np.float32)
    res = {}
    for npts in (9, 8):
        P3 = synth.box_points(with_center=npts == 9).astype(np.float32)
        subsets = consensus_subsets(P3)
        rows = {k: [] for k in ("uv", "thr", "sigma", "outliers", "bad", "R", "t", "params", "hyp", "mask", "gap")}
        dropped = 0
        cases = [(s, k, 8.0) for s in SIGMAS for k in OUTLIERS for _ in range(N)] + [(-1, 0, 2.0)] * N_GARBAGE
        rng = np.random.default_rng(77 + npts)
        for sigma, k, thr in cases:
            if sigma < 0:
                uv, bad = np.stack([rng.uniform(0, 640, npts), rng.uniform(0, 480, npts)], 1).astype(np.float32), (1 << npts) - 1
            else:
                uv, bad = _problem(P3, K, rng, sigma, k)
            o = consensus_ref(P3, uv, K, thr, subsets, solve=_cv2_solve, refine=_cv2_refine, rodrigues=_cv2_rodrigues)
            if not np.abs(o["t"]).max() < 10.0:
                dropped += 1
                continue
            for key, v in (("uv", uv), ("thr", thr), ("sigma", sigma), ("outliers", k), ("bad", bad)):
                rows[key].append(v)
            for key in ("R", "t", "params", "hyp", "mask", "gap"):
                rows[key].append(o[key])
        for key, v in rows.items():
            res["%s_p%d" % (key, npts)] = np.array(v)
        res["P3_p%d" % npts] = P3
        res["subsets_p%d" % npts] = subsets
        h = np.array(rows["hyp"])
        print("p%d: %d problems (%d left out: |t| > 10 m), cv2 %s; hyp -1: %d, 0: %d, refined or subset: %d; gap < 1e-6: %d"
              % (npts, len(h), dropped, cv2.__version__, (h < 0).sum(), (h == 0).sum(), (h > 0).sum(), (np.array(rows["gap"]) < 1e-6).sum()))
    np.savez_compressed(os.path.join(HERE, "pnp_consensus.npz"), K=K, **res)


if __name__ == "__main__":
    main()
