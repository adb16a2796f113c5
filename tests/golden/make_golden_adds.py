"""Generate tests/golden/adds.npz from the REFERENCE ITSELF: utils.py's adi, calc_pts_diameter, compute_transformation,
compute_projection and calcAngularDistance on seeded synthetic data, and valid.py's summary (the running sums of valid.py:179-183
and the statistics of valid.py:202-229), executed from the reference's own source text.

Run where the reference checkout is available (path in REF below):
    python tests/golden/make_golden_adds.py

Data:
  * mesh_a: about 6000 vertices of an object-sized box, rounded to 6 decimals as a .ply stores them;
  * mesh_s: a mesh with a 2-fold symmetry about z, the union of P and R_z(pi) P (R_z(pi) negates x and y, so the union is
    exactly symmetric);
  * pose pairs on both meshes at several error levels (rotation noise about a random axis, translation noise);
  * symmetric pairs on mesh_s, R_est = R_gt R_z(pi) and t_est = t_gt, whose ADD is large and whose ADD-S is about 0, then the
    same pairs perturbed by 1 degree and 2 mm.
Stored per pair: Rt_est, Rt_gt (3, 4), the reference's adi(pts_est, pts_gt) and its ADD (valid.py:173-177); per mesh the
reference's calc_pts_diameter.  For the summary, over the pairs of mesh_s at summary_idx as one evaluation run: the per-image
errors in the reference's dtypes (pixel and corner errors float32, the others float64, valid.py:146-177), every summary figure
valid.py computes, its printed lines, and acc_adds10 with the same formula on adi.  The exact symmetric pairs are left out
of the summary: at exactly 180 degrees the reference's calcAngularDistance returns NaN (arccos of a value rounded below -1),
and so would the mean angle.  No noise level is 0, so no other angle is NaN either (see utils.pose_accuracy).

A separate script, not a flag of make_golden.py: that generator and the fixtures it writes are left exactly as they are.
"""
import contextlib
import io
import os
import re
import sys
import textwrap

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REPO)

from singleshotpose_b200 import synth          # noqa: E402

HALF = np.array([0.038, 0.039, 0.046])
# (rotation noise deg, translation noise m, pairs) per error level
LEVELS = [(0.5, 0.002, 4), (2.0, 0.005, 4), (5.0, 0.01, 4), (15.0, 0.03, 4)]
N_SYM = 4


def poses(rng, n):
    ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    R = synth._rodrigues(ax * rng.uniform(0.2, 2.5, size=(n, 1)))
    t = np.stack([rng.uniform(-.1, .1, n), rng.uniform(-.07, .07, n), rng.uniform(.6, 1.1, n)], 1)
    return R, t


def perturb(rng, R, t, deg, sigma_t):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    dR = synth._rodrigues((ax * np.deg2rad(deg))[None])[0]
    return dR @ R, t + rng.normal(0, sigma_t, size=3)


def pairs(rng, symmetric):
    est, gt = [], []
    n = sum(k for *_, k in LEVELS)
    R, t = poses(rng, n + (N_SYM if symmetric else 0))
    i = 0
    for deg, st, k in LEVELS:
        for _ in range(k):
            Re, te = perturb(rng, R[i], t[i], deg, st)
            est.append(np.c_[Re, te]); gt.append(np.c_[R[i], t[i]])
            i += 1
    if symmetric:
        Rz = np.diag([-1.0, -1.0, 1.0])
        for j in range(2 * N_SYM):                      # exact, then perturbed by 1 degree and 2 mm
            Re, te = R[i + j % N_SYM] @ Rz, t[i + j % N_SYM]
            if j >= N_SYM:
                Re, te = perturb(rng, Re, te, 1.0, 0.002)
            est.append(np.c_[Re, te]); gt.append(np.c_[R[i + j % N_SYM], t[i + j % N_SYM]])
    return np.stack(est), np.stack(gt)


def source_block(src, first, last):
    """the reference's lines from the one containing `first` through the one containing `last`, dedented"""
    lines = src.splitlines()
    a = next(i for i, s in enumerate(lines) if first in s)
    b = next(i for i in range(a, len(lines)) if last in lines[i])
    return textwrap.dedent("\n".join(lines[a:b + 1]))


def main():
    rng = np.random.default_rng(20261016)
    for d in (REF,):
        sys.path.insert(0, d)
    with contextlib.redirect_stdout(io.StringIO()):
        import utils as RU
    mesh_a = np.round(rng.uniform(-1, 1, size=(6000, 3)) * HALF, 6)
    P = np.round(rng.uniform(-1, 1, size=(3000, 3)) * HALF, 6)
    mesh_s = np.concatenate([P, P * np.array([-1.0, -1.0, 1.0])])
    Kc = synth.intrinsics()
    out = dict(mesh_a=mesh_a, mesh_s=mesh_s, K=Kc)
    for name, mesh, sym in (("a", mesh_a, False), ("s", mesh_s, True)):
        est, gt = pairs(rng, sym)
        vertices = np.c_[mesh, np.ones((len(mesh), 1))].transpose()          # valid.py:67
        adds, add = [], []
        for Re, Rg in zip(est, gt):
            tf_pr, tf_gt = RU.compute_transformation(vertices, Re), RU.compute_transformation(vertices, Rg)
            adds.append(RU.adi(tf_pr.T, tf_gt.T))
            add.append(np.mean(np.linalg.norm(tf_gt - tf_pr, axis=0)))
        out.update({"Rt_est_" + name: est, "Rt_gt_" + name: gt, "adds_" + name: np.array(adds), "add_" + name: np.array(add),
                    "diam_" + name: np.array(RU.calc_pts_diameter(mesh))})
    # valid.py's per-image errors for the pairs of mesh_s, then its summary, from its own source text
    src = open(os.path.join(REF, "valid.py")).read()
    sums = compile(source_block(src, "testing_error_trans  +=", "testing_samples      +="), "valid.py", "exec")
    summary = compile(source_block(src, "px_threshold = 5", "nts = float(testing_samples)"), "valid.py", "exec")
    printed = compile(source_block(src, "logging('Results of", "logging('   Translation error"), "valid.py", "exec")
    vertices = np.c_[mesh_s, np.ones((len(mesh_s), 1))].transpose()
    corners = RU.get_3D_corners(vertices)
    P9 = np.concatenate([np.zeros((3, 1)), corners[:3]], 1)                     # [0; corners3D], valid.py:152
    ns = dict(np=np, diam=float(out["diam_s"]), name="synthetic", testing_error_trans=0.0, testing_error_angle=0.0,
              testing_error_pixel=0.0, testing_samples=0.0, errs_2d=[], errs_3d=[], errs_trans=[], errs_angle=[], errs_corner2D=[])
    n_rand = sum(k for *_, k in LEVELS)
    summary_idx = np.r_[np.arange(n_rand), n_rand + N_SYM + np.arange(N_SYM)]
    for Re, Rg in zip(out["Rt_est_s"][summary_idx], out["Rt_gt_s"][summary_idx]):
        c_gt = RU.compute_projection(np.r_[P9, np.ones((1, 9))], Rg, Kc).T        # float32 (9, 2) pixels, as valid.py:137-142
        c_pr = RU.compute_projection(np.r_[P9, np.ones((1, 9))], Re, Kc).T
        corner_dist = np.mean(np.linalg.norm(c_gt - c_pr, axis=1))
        trans_dist = np.sqrt(np.sum(np.square(Rg[:, 3:] - Re[:, 3:])))
        angle_dist = RU.calcAngularDistance(Rg[:, :3], Re[:, :3])
        pixel_dist = np.mean(np.linalg.norm(RU.compute_projection(vertices, Rg, Kc) - RU.compute_projection(vertices, Re, Kc), axis=0))
        vertex_dist = np.mean(np.linalg.norm(RU.compute_transformation(vertices, Rg) - RU.compute_transformation(vertices, Re), axis=0))
        for k, v in (("errs_corner2D", corner_dist), ("errs_trans", trans_dist), ("errs_angle", angle_dist), ("errs_2d", pixel_dist),
                     ("errs_3d", vertex_dist)):
            ns[k].append(v)
        ns.update(trans_dist=trans_dist, angle_dist=angle_dist, pixel_dist=pixel_dist, count=0)
        exec(sums, ns)
    exec(summary, ns)
    log = []
    ns["logging"] = log.append
    exec(printed, ns)
    assert not np.isnan(ns["errs_angle"]).any()
    eps = 1e-5
    adds_sum = out["adds_s"][summary_idx]
    acc_adds10 = len(np.where(np.array(adds_sum) <= ns["diam"] * 0.1)[0]) * 100. / (len(adds_sum) + eps)
    out.update(summary_idx=summary_idx, errs_2d=np.array(ns["errs_2d"]), errs_3d=np.array(ns["errs_3d"]), errs_trans=np.array(ns["errs_trans"]),
               errs_angle=np.array(ns["errs_angle"]), errs_corner2D=np.array(ns["errs_corner2D"]),
               acc=np.array(ns["acc"]), acc3d10=np.array(ns["acc3d10"]), acc5cm5deg=np.array(ns["acc5cm5deg"]),
               corner_acc=np.array(ns["corner_acc"]), mean_err_2d=np.array(ns["mean_err_2d"]), mean_vertex_err=np.array(np.mean(ns["errs_3d"])),
               mean_corner_err_2d=np.array(ns["mean_corner_err_2d"]), mean_trans_err=np.array(ns["testing_error_trans"] / ns["nts"]),
               mean_angle_err=np.array(ns["testing_error_angle"] / ns["nts"]), mean_pixel_err=np.array(ns["testing_error_pixel"] / ns["nts"]),
               acc_adds10=np.array(acc_adds10), printed=np.array(log))
    assert out["errs_2d"].dtype == np.float32 and out["errs_corner2D"].dtype == np.float32
    assert out["acc_adds10"] > out["acc3d10"]
    np.savez_compressed(os.path.join(HERE, "adds.npz"), **out)
    print("adds golden: diameters %.9f %.9f; ADD-S a %s; ADD-S s %s" % (out["diam_a"], out["diam_s"], np.round(out["adds_a"], 5).tolist(),
                                                                        np.round(out["adds_s"], 5).tolist()))
    print("\n".join(log))


if __name__ == "__main__":
    main()
