#!/usr/bin/env python
"""Goldens of PnP and projection with lens distortion, from cv2 itself: cv2.solvePnP(P3, uv, K, dist, SOLVEPNP_ITERATIVE), cold and
warm (useExtrinsicGuess=True), cv2.projectPoints and cv2.undistortPoints.

  calibrations (OpenCV's order k1, k2, p1, p2[, k3[, k4, k5, k6]]): barrel (a typical webcam), pincushion, 4, 5 and 8 coefficients
  (the rational model); LINEMOD's K (float32, as valid.py passes it);
  point sets: the 9 box points (centroid + 8 corners) and the 8 corners;
  poses 0.6-1.0 m away, the object at the image centre or 60-140 px from a corner of the 640 x 480 frame (where distortion is
  largest), keypoint noise sigma = 0, 1, 5, 20 px;
  warm starts as tests/golden/make_golden_pnp_guess.py: 'prev' = cv2's cold solution of the previous frame of the moving box,
  'pert' = the frame's true pose perturbed by about 0.05 rad and 1 cm.
A solve where cv2's LM runs away is left out, as its digits are noise rather than a pose: |t| > 10 m, t_z < 0.1 m (the box
stands 0.6-1 m away; behind or at the lens the solve is lost), or an RMS reprojection error above 1000 px (a start that puts the
box a few cm from the camera evaluates the distortion polynomial far outside the frame, where the errors reach 1e9 px and 20 LM
steps end anywhere).  The numpy restatement
(oracle/pnp_dist_ref.py) is pinned to cv2 here: the script prints its worst deviation.  Needs cv2; writes tests/golden/pnp_dist.npz.

    python tests/golden/make_golden_pnp_dist.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.pnp_dist_ref import dist8, project_points, solve_pnp_dist, undistort_points       # noqa: E402
from singleshotpose_b200 import synth                                                          # noqa: E402

CALIBRATIONS = {
    "barrel": (-0.3, 0.12, 1e-3, -5e-4, -0.02),
    "pincushion": (0.22, -0.1, -8e-4, 6e-4, 0.03),
    "four": (-0.18, 0.04, 5e-4, 1e-3),
    "five": (-0.08, 0.3, -2e-3, 1.5e-3, -0.5),
    "rational": (0.6, -0.4, 1e-3, -1e-3, 0.1, 0.9, -0.3, 0.15),
}
SIGMAS = (0, 1, 5, 20)
N = 6                            # poses per (calibration, point set, region, sigma)
W, H = 640, 480


def _rodrigues(r):
    import cv2
    return cv2.Rodrigues(np.asarray(r, np.float64).reshape(3, 1))[0]


def _pose(rng, K, corner):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    rv = ax * rng.uniform(0, np.pi)
    z = rng.uniform(0.6, 1.0)
    if corner:
        du, dv = rng.uniform(60, 140, size=2)
        u = du if rng.random() < 0.5 else W - du
        v = dv if rng.random() < 0.5 else H - dv
    else:
        u, v = W / 2 + rng.uniform(-20, 20), H / 2 + rng.uniform(-20, 20)
    t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0])
    return rv, t


def _runaway(P3, uv, K, dist, r, t):
    import cv2
    if not (np.abs(t).max() < 10.0 and t.reshape(3)[2] > 0.1):
        return True
    px = cv2.projectPoints(P3.astype(np.float64), r.reshape(3, 1), t.reshape(3, 1), K.astype(np.float64), dist)[0].reshape(-1, 2)
    return not np.sqrt(((px - uv) ** 2).sum(1).mean()) < 1000.0


def main():
    import cv2
    K = synth.intrinsics().astype(np.float32)
    res = dict(K=K)
    worst = 0.0
    grid = np.stack(np.meshgrid(np.arange(0, W + 1, 40.0), np.arange(0, H + 1, 40.0)), -1).reshape(-1, 2)
    res["und_uv"] = grid
    for name, coefs in CALIBRATIONS.items():
        dist = np.array(coefs, np.float64)
        res["dist_" + name] = dist
        und = cv2.undistortPoints(res["und_uv"].reshape(-1, 1, 2), K, dist).reshape(-1, 2)
        res["und_" + name] = und
        dev_und = np.abs(undistort_points(res["und_uv"], K, dist) - und).max()
        for npts in (9, 8):
            P3 = synth.box_points(with_center=npts == 9).astype(np.float32)
            res["P3_%d" % npts] = P3
            cold = {k: [] for k in ("uv", "sigma", "corner", "rvec", "tvec", "rvec_true", "tvec_true", "proj_true")}
            warm = {k: [] for k in ("uv", "guess", "perturbed", "rvec", "tvec")}
            dev, dropped = [], 0
            seed = sum(map(ord, name)) * 100 + npts
            rng = np.random.default_rng(seed)
            for corner in (False, True):
                for sigma in SIGMAS:
                    for _ in range(N):
                        rv0, t0 = _pose(rng, K, corner)
                        rv1, t1 = rv0 + rng.normal(size=3) * 0.03, t0 + rng.normal(size=3) * 0.01
                        uv_true0 = cv2.projectPoints(P3, rv0, t0, K, dist)[0].reshape(-1, 2)
                        uv_true1 = cv2.projectPoints(P3, rv1, t1, K, dist)[0].reshape(-1, 2)
                        uv0 = (uv_true0 + rng.normal(size=uv_true0.shape) * sigma).astype(np.float32)
                        uv1 = (uv_true1 + rng.normal(size=uv_true1.shape) * sigma).astype(np.float32)
                        ok, r0, tt0 = cv2.solvePnP(P3, uv0, K, dist, flags=cv2.SOLVEPNP_ITERATIVE)
                        ok1, r1, tt1 = cv2.solvePnP(P3, uv1, K, dist, flags=cv2.SOLVEPNP_ITERATIVE)
                        assert ok and ok1
                        if not _runaway(P3, uv1, K, dist, r1, tt1):
                            ro, to = solve_pnp_dist(P3, uv1, K, dist)
                            dev.append(max(np.abs(ro - r1.reshape(3)).max(), np.abs(to - tt1.reshape(3)).max()))
                            for k, v in (("uv", uv1), ("sigma", sigma), ("corner", corner), ("rvec", r1.reshape(3)), ("tvec", tt1.reshape(3)),
                                         ("rvec_true", rv1), ("tvec_true", t1), ("proj_true", uv_true1)):
                                cold[k].append(v)
                        else:
                            dropped += 1
                        pert = (rv1 + rng.normal(size=3) * 0.05 / np.sqrt(3), t1 + rng.normal(size=3) * 0.01 / np.sqrt(3))
                        for kind, (rg, tg) in (("prev", (r0.reshape(3), tt0.reshape(3))), ("pert", pert)):
                            r_in, t_in = rg.reshape(3, 1).astype(np.float64).copy(), tg.reshape(3, 1).astype(np.float64).copy()
                            ok, rw, tw = cv2.solvePnP(P3, uv1, K, dist, r_in, t_in, useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
                            assert ok
                            if _runaway(P3, uv1, K, dist, rw, tw):
                                dropped += 1
                                continue
                            ro, to = solve_pnp_dist(P3, uv1, K, dist, rg, tg)
                            dev.append(max(np.abs(ro - rw.reshape(3)).max(), np.abs(to - tw.reshape(3)).max()))
                            for k, v in (("uv", uv1), ("guess", np.concatenate([rg, tg])), ("perturbed", kind == "pert"),
                                         ("rvec", rw.reshape(3)), ("tvec", tw.reshape(3))):
                                warm[k].append(v)
            tag = "%s_p%d" % (name, npts)
            for k, v in cold.items():
                res["%s_%s" % (k, tag)] = np.array(v, np.float32 if k == "uv" else None)
            res["R_" + tag] = np.array([_rodrigues(r) for r in cold["rvec"]])
            for k, v in warm.items():
                res["warm_%s_%s" % (k, tag)] = np.array(v, np.float32 if k == "uv" else None)
            res["warm_R_" + tag] = np.array([_rodrigues(r) for r in warm["rvec"]])
            dev_proj = max(np.abs(project_points(P3, rv, tv, K, dist) - pj).max()
                           for rv, tv, pj in zip(cold["rvec_true"], cold["tvec_true"], cold["proj_true"]))
            dev = np.array(dev)
            worst = max(worst, dev.max())
            print("%s: %d cold + %d warm solves (%d left out: runaway), cv2 %s; oracle vs cv2: solve %.1e, projectPoints %.1e px, "
                  "undistortPoints %.1e" % (tag, len(cold["uv"]), len(warm["uv"]), dropped, cv2.__version__, dev.max(), dev_proj, dev_und))
    print("worst solve deviation of oracle/pnp_dist_ref.py from cv2: %.1e" % worst)
    assert dist8(CALIBRATIONS["four"]).shape == (8,)
    np.savez_compressed(os.path.join(HERE, "pnp_dist.npz"), **res)


if __name__ == "__main__":
    main()
