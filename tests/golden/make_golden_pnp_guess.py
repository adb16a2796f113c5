#!/usr/bin/env python
"""Goldens of the warm-started PnP: cv2.solvePnP(..., flags=SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) itself, on pairs of frames of
a moving box (the 9 box-plus-centroid points, or the 8 corners) at keypoint noise sigma = 0, 1, 5, 20, 80 px.  Two guesses per
problem: 'prev' = cv2's cold solution of the previous frame (what a tracker stores), 'pert' = the frame's true pose perturbed by
about 0.05 rad and 1 cm.  A solve where cv2's LM runs away (|t| > 10 m: at sigma = 80 px the previous frame's cold solution can be
garbage) is left out, as its digits are overflow noise rather than a pose.  Needs cv2 only; writes tests/golden/pnp_guess.npz.

    python tests/golden/make_golden_pnp_guess.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.track_ref import solve_pnp_guess                 # noqa: E402
from singleshotpose_b200 import synth                         # noqa: E402

SIGMAS = (0, 1, 5, 20, 80)
N = 32


def _rodrigues(r):
    import cv2
    return cv2.Rodrigues(np.asarray(r, np.float64).reshape(3, 1))[0]


def _uv(P3, K, rv, t, rng, sigma):
    Pc = P3.astype(np.float64) @ _rodrigues(rv).T + t
    uv = np.stack([K[0, 0] * Pc[:, 0] / Pc[:, 2] + K[0, 2], K[1, 1] * Pc[:, 1] / Pc[:, 2] + K[1, 2]], -1)
    return (uv + rng.normal(size=uv.shape) * sigma).astype(np.float32)


def main():
    import cv2
    res = {}
    K = synth.intrinsics().astype(np.float32)
    for npts in (9, 8):
        P3 = synth.box_points(with_center=npts == 9).astype(np.float32)
        res["P3_%d" % npts] = P3
        for sigma in SIGMAS:
            rng = np.random.default_rng(1000 * npts + sigma)
            uvs, guesses, rvecs, tvecs, kinds, dev, dropped = [], [], [], [], [], [], 0
            for i in range(N):
                ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
                rv0 = ax * rng.uniform(0, np.pi)
                t0 = np.array([rng.uniform(-.2, .2), rng.uniform(-.15, .15), rng.uniform(.6, 1.2)])
                rv1 = rv0 + rng.normal(size=3) * 0.03                        # the object moves between the two frames
                t1 = t0 + rng.normal(size=3) * 0.01
                uv0, uv1 = _uv(P3, K, rv0, t0, rng, sigma), _uv(P3, K, rv1, t1, rng, sigma)
                ok0, r_prev, t_prev = cv2.solvePnP(P3, uv0, K, None, flags=cv2.SOLVEPNP_ITERATIVE)
                assert ok0
                pert = (rv1 + rng.normal(size=3) * 0.05 / np.sqrt(3), t1 + rng.normal(size=3) * 0.01 / np.sqrt(3))
                for kind, (rg, tg) in (("prev", (r_prev.reshape(3), t_prev.reshape(3))), ("pert", pert)):
                    r_in, t_in = rg.reshape(3, 1).astype(np.float64).copy(), tg.reshape(3, 1).astype(np.float64).copy()
                    ok, rw, tw = cv2.solvePnP(P3, uv1, K, None, r_in, t_in, useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
                    assert ok
                    if not np.abs(tw).max() < 10.0:                      # cv2's LM ran away from a garbage guess: no pose to compare
                        dropped += 1
                        continue
                    ro, to = solve_pnp_guess(P3, uv1, K, rg, tg)
                    dev.append(max(np.abs(ro - rw.reshape(3)).max(), np.abs(to - tw.reshape(3)).max()))
                    uvs.append(uv1); guesses.append(np.concatenate([rg, tg])); kinds.append(kind == "pert")
                    rvecs.append(rw.reshape(3)); tvecs.append(tw.reshape(3))
            tag = "p%d_s%d" % (npts, sigma)
            res["uv_" + tag] = np.array(uvs, np.float32)
            res["guess_" + tag] = np.array(guesses, np.float64)
            res["perturbed_" + tag] = np.array(kinds)
            res["rvec_" + tag] = np.array(rvecs)
            res["tvec_" + tag] = np.array(tvecs)
            res["R_" + tag] = np.array([_rodrigues(r) for r in rvecs])
            dev = np.array(dev)
            print("%s: %d warm solves (%d left out: |t| > 10 m), cv2 %s; numpy restatement (oracle/track_ref.py) vs cv2: %d above 1e-6, worst %.1e"
                  % (tag, len(uvs), dropped, cv2.__version__, (dev > 1e-6).sum(), dev.max()))
    np.savez_compressed(os.path.join(HERE, "pnp_guess.npz"), K=K, **res)


if __name__ == "__main__":
    main()
