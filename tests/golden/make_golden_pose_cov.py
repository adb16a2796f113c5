#!/usr/bin/env python
"""Golden of the covariance of a PnP pose, from cv2 itself: per pose, cv2.solvePnP(P3, uv + noise, K, dist, SOLVEPNP_ITERATIVE) over
DRAWS seeded draws of sigma = 1 px Gaussian keypoint noise, and the empirical covariance of the errors (log(R_i R0^T), t_i - t0)
under the left perturbation x_cam = exp([dth]x) R X + t + dt_ that csrc/pose_filter_core.h uses.  Each solve starts LM from the
true pose (useExtrinsicGuess): the covariance is that of the solution near the truth; a cold solve's DLT start lands on a mirrored
solution in a share of the draws of some poses, and those draws would dominate the empirical covariance.

  LINEMOD's K (float32, as valid.py passes it); the 9 box points (centroid + 8 corners) of an ape-sized box; poses 0.5-1 m away
  with a random rotation; no distortion (the object near the image centre) and the barrel calibration of pnp_dist.npz (the object
  60-140 px from a frame corner, where the distortion is largest).
The relative sampling error of a variance from DRAWS draws is sqrt(2 / DRAWS), about 3 %.  Needs cv2; writes tests/golden/pose_cov.npz.

    python tests/golden/make_golden_pose_cov.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.pnp_dist_ref import dist8                             # noqa: E402
from oracle.pose_filter_ref import so3_log                        # noqa: E402
from singleshotpose_b200 import synth                             # noqa: E402

BARREL = (-0.3, 0.12, 1e-3, -5e-4, -0.02)                          # pnp_dist.npz's "barrel"
DRAWS, POSES, SIGMA = 2000, 4, 1.0
W, H = 640, 480


def _pose(rng, K, corner):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    rv = ax * rng.uniform(0, np.pi)
    z = rng.uniform(0.5, 1.0)
    if corner:
        du, dv = rng.uniform(60, 140, size=2)
        u = du if rng.random() < 0.5 else W - du
        v = dv if rng.random() < 0.5 else H - dv
    else:
        u, v = W / 2 + rng.uniform(-60, 60), H / 2 + rng.uniform(-60, 60)
    return rv, z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0])


def main():
    import cv2
    K = synth.intrinsics().astype(np.float32)
    P3 = synth.box_points((0.038, 0.039, 0.046), with_center=True).astype(np.float32)        # (9, 3), centroid first
    out = dict(K=K, P3=P3, sigma=np.float64(SIGMA), draws=np.int64(DRAWS), dist_barrel=dist8(BARREL))
    for tag, dist in (("plain", None), ("barrel", np.asarray(BARREL, np.float64))):
        rng = np.random.default_rng(11 if dist is None else 12)
        Rs, ts, covs = [], [], []
        for _ in range(POSES):
            rv, t = _pose(rng, K, dist is not None)
            R0 = cv2.Rodrigues(rv.reshape(3, 1))[0]
            uv0 = cv2.projectPoints(P3.astype(np.float64), rv, t, K.astype(np.float64), dist)[0].reshape(-1, 2)
            err = np.empty((DRAWS, 6))
            for i in range(DRAWS):
                uv = (uv0 + rng.normal(0, SIGMA, uv0.shape)).astype(np.float32)
                ok, r, tt = cv2.solvePnP(P3, uv, K, dist, rv.reshape(3, 1).copy(), t.reshape(3, 1).copy(), useExtrinsicGuess=True,
                                         flags=cv2.SOLVEPNP_ITERATIVE)
                assert ok
                err[i, :3] = so3_log(cv2.Rodrigues(r)[0] @ R0.T)
                err[i, 3:] = tt.reshape(3) - t
            Rs.append(R0); ts.append(t); covs.append(np.cov(err.T))
        out["R_" + tag], out["t_" + tag], out["cov_" + tag] = np.array(Rs), np.array(ts), np.array(covs)
    np.savez_compressed(os.path.join(HERE, "pose_cov.npz"), **out)
    print("wrote pose_cov.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
