"""Calibrate a camera rig from the object it sees: python -m singleshotpose_b200.calibrate_rig --datacfg c0.data c1.data ...
--poses p0.npz p1.npz ... --out rig.npz.  Each --poses file is one camera's `predict --out` file of the same recording (row i of
every file is capture i); each --datacfg file is that camera's .data file (K and the optional dist entry, read as predict reads
them).  The 3-D points are the 9 points PosePredictor solves with, from the first .data file's mesh.  A view takes part when its
conf > --conf-thresh.  The rig (utils_host.write_rig) feeds `predict --rig`; it is not written when a camera stays unconnected.

With --depth-dir D0 D1 ... (one directory per camera, in the --poses order) the keypoint rig is then calibrated against depth
(utils.calibrate_rig_depth_batched): capture i of camera c is D_c/<stem of row i of camera c's `paths`>.png, a 16-bit depth PNG
registered to that camera, and the mesh is the first .data file's.  The depth-calibrated rig is written."""
from __future__ import annotations

import argparse
import os

import numpy as np

from ._lib import SspError

POSE_KEYS = ("keypoints_px", "conf")
CONF_THRESH = 0.1                       # yolo-pose.cfg's conf_thresh


def read_poses(paths, need_paths=False):
    """-> (keypoints (C, N, 9, 2) float32, conf (C, N), image paths (C, N) or None) of the --poses files; SspError naming the file
    for a missing file or key (`paths` only with need_paths), or a row count that differs from the first file's"""
    kps, confs, names = [], [], []
    for p in paths:
        if not os.path.isfile(p):
            raise SspError("poses file %s does not exist" % p)
        with np.load(p) as z:
            missing = [k for k in POSE_KEYS if k not in z.files]
            if missing:
                raise SspError("poses file %s has no %s (a `predict --out` file has both)" % (p, ", ".join(missing)))
            if need_paths and "paths" not in z.files:
                raise SspError("poses file %s has no paths (the image of each row): --depth-dir names each depth file after it" % p)
            kp, conf = np.asarray(z["keypoints_px"], np.float32), np.asarray(z["conf"], np.float64).reshape(-1)
            names.append([str(x) for x in np.asarray(z["paths"]).reshape(-1)] if need_paths else None)
        if kp.ndim != 3 or kp.shape[1:] != (9, 2) or len(conf) != len(kp):
            raise SspError("poses file %s: keypoints_px must be (N, 9, 2) with one conf per row, got %s and %s" % (p, kp.shape, conf.shape))
        if kps and len(kp) != len(kps[0]):
            raise SspError("poses file %s has %d rows, %s has %d: row i of every file must be capture i" % (p, len(kp), paths[0], len(kps[0])))
        if need_paths and len(names[-1]) != len(kp):
            raise SspError("poses file %s has %d paths for %d rows" % (p, len(names[-1]), len(kp)))
        kps.append(kp)
        confs.append(conf)
    return np.stack(kps), np.stack(confs), (names if need_paths else None)


def depth_files(dirs, names):
    """-> [camera][capture] depth file paths, D_c/<image stem>.png; SspError naming the first one that does not exist"""
    files = [[os.path.join(d, os.path.splitext(os.path.basename(n))[0] + ".png") for n in ns] for d, ns in zip(dirs, names)]
    for f in (f for row in files for f in row):
        if not os.path.isfile(f):
            raise SspError("depth file %s does not exist" % f)
    return files


def read_depths(files):
    """-> (N C, H, W) uint16, row i C + c capture i of camera c; SspError naming a file that cannot be read or whose size differs
    from the first file's"""
    from PIL import Image
    from .predict import read_depth_png
    with Image.open(files[0][0]) as im:
        size = im.size
    C, N = len(files), len(files[0])
    return np.stack([read_depth_png(files[c][i], size) for i in range(N) for c in range(C)])


def read_cameras(datacfgs):
    """-> (K (C, 3, 3), dist list (C,) of (8,) or None, mesh path of the first file) from the .data files"""
    from .predict import SIZE_KEYS, camera_dist, read_camera
    Ks, dists, mesh = [], [], None
    for i, d in enumerate(datacfgs):
        if not os.path.isfile(d):
            raise SspError(".data file %s does not exist" % d)
        m, K, _size = read_camera(d, SIZE_KEYS)
        if i == 0:
            if m is None:
                raise SspError("%s has no mesh entry: the object's 3-D points come from the first .data file's mesh" % d)
            mesh = m
        Ks.append(K)
        dists.append(camera_dist(argparse.Namespace(dist=None, datacfg=d)))
    return np.stack(Ks), dists, mesh


def object_points(mesh):
    """the 9 PnP points [0; corners3D[:3]] of PosePredictor for the mesh"""
    from .predict import mesh_corners
    C3 = np.asarray(mesh_corners(mesh), np.float64)[:3]
    return np.concatenate([np.zeros((1, 3)), C3.T]).astype(np.float32)


def check_args(a):
    """SspError, before any file is read, for a count of --datacfg other than that of --poses or a camera count outside 2..16"""
    if len(a.datacfg) != len(a.poses):
        raise SspError("%d --datacfg files for %d --poses files: give one .data file per camera" % (len(a.datacfg), len(a.poses)))
    if not 2 <= len(a.poses) <= 16:
        raise SspError("a rig to calibrate has 2..16 cameras, got %d" % len(a.poses))
    if not 0 <= a.reference < len(a.poses):
        raise SspError("--reference must be one of 0..%d, got %d" % (len(a.poses) - 1, a.reference))
    if a.depth_dir is not None:
        if len(a.depth_dir) != len(a.poses):
            raise SspError("%d --depth-dir directories for %d cameras: give one per camera, in the --poses order" % (len(a.depth_dir), len(a.poses)))
        from .utils import check_refine_args
        check_refine_args(a.depth_scale, a.refine_iters, (0.5, 0.02))


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.calibrate_rig",
                                 description="the extrinsics of a camera rig from each camera's predict --out file of one recording")
    ap.add_argument("--datacfg", nargs="+", required=True, help="one .data file per camera: fx fy u0 v0 [dist]; the first one's mesh")
    ap.add_argument("--poses", nargs="+", required=True, help="one `predict --out` .npz per camera, in the --datacfg order")
    ap.add_argument("--out", required=True, help="the rig .npz (utils_host.read_rig; predict --rig)")
    ap.add_argument("--conf-thresh", type=float, default=CONF_THRESH, help="a view takes part when its conf > this (default %(default)s)")
    ap.add_argument("--reference", type=int, default=0, help="the camera whose frame is the world frame (default 0)")
    ap.add_argument("--depth-dir", nargs="+", metavar="DIR",
                    help="calibrate against depth too: one directory per camera, in the --poses order, holding <image stem>.png, a "
                         "16-bit depth PNG registered to the camera, for each row of its --poses file's paths")
    ap.add_argument("--depth-scale", type=float, default=0.001, help="--depth-dir: mesh units per depth unit (default %(default)s)")
    ap.add_argument("--refine-iters", type=int, default=10, help="--depth-dir: iterations of the depth stage (default %(default)s)")
    a = ap.parse_args(argv)
    check_args(a)
    kp, conf, names = read_poses(a.poses, need_paths=a.depth_dir is not None)
    depth = read_depths(depth_files(a.depth_dir, names)) if a.depth_dir is not None else None
    K, dists, mesh = read_cameras(a.datacfg)
    P9 = object_points(mesh)
    if depth is not None:
        from .predict import read_mesh
        V, F = read_mesh(mesh)
    from .utils import calibrate_rig_batched
    from .utils_host import write_rig
    C, N = kp.shape[:2]
    uv = np.ascontiguousarray(kp.transpose(1, 0, 2, 3).reshape(N * C, 9, 2))              # row g C + c: camera c of capture g
    valid = (conf.T > a.conf_thresh).reshape(N * C)
    dist = dists if any(d is not None for d in dists) else None
    o = calibrate_rig_batched(P9, uv, K, dist=dist, valid=valid, reference=a.reference)
    status, rmse, nobs = (o[k].cpu().numpy() for k in ("cam_status", "cam_rmse", "cam_obs"))
    sd = np.sqrt(np.maximum(np.diagonal(o["cam_cov"].cpu().numpy(), axis1=1, axis2=2), 0.0))
    names = {1: "UNCONNECTED", 2: "SINGULAR", 3: "UNCONNECTED|SINGULAR"}
    for c in range(C):
        print("camera %d (%s): %s, cam_rmse %.3f px over %d observations, sd rot %s rad, sd t %s"
              % (c, a.poses[c], names.get(int(status[c]), "ok"), rmse[c], nobs[c], np.array2string(sd[c, :3], precision=3),
                 np.array2string(sd[c, 3:], precision=4)))
    print("%d rounds, %d LM steps, cost %.6g" % (o["rounds"], o["iterations"], o["cost"]))
    if o["rig"] is None:
        bad = [("%d (%s)" % (c, a.poses[c])) for c in range(C) if status[c] & 1]
        raise SspError("camera %s shares too few agreeing captures with the others: no rig is written; record more captures in "
                       "their shared field of view" % ", ".join(bad))
    if depth is not None:
        o = calibrate_depth(a, depth, V, F, K, dist, o)
    write_rig(a.out, o["rig"])
    print("rig of %d cameras -> %s" % (C, a.out))


def calibrate_depth(a, depth, V, F, K, dist, calib):
    """the depth stage after the keypoint calibration: prints per camera its status, pairs, RMS and standard deviations -> the
    stage's dict; SspError, writing nothing, when its global status is set"""
    from .utils import calibrate_rig_depth_batched
    o = calibrate_rig_depth_batched(depth, V, F, K, calib, dist=dist, reference=a.reference, depth_scale=a.depth_scale,
                                    iters=a.refine_iters)
    status, pts, rmse = (o[k].cpu().numpy() for k in ("cam_status", "cam_points", "cam_rmse"))
    sd = np.sqrt(np.maximum(np.diagonal(o["cam_cov"].cpu().numpy(), axis1=1, axis2=2), 0.0))
    names = {0: "ok", 1: "UNCONNECTED", 2: "FEW_POINTS", 4: "SINGULAR", 6: "FEW_POINTS|SINGULAR"}
    for c in range(len(K)):
        print("depth camera %d (%s): %s, %d pairs, rmse %.3g mesh units, sd rot %s rad, sd t %s"
              % (c, a.poses[c], names.get(int(status[c]), str(int(status[c]))), pts[c], rmse[c], np.array2string(sd[c, :3], precision=3),
                 np.array2string(sd[c, 3:], precision=4)))
    print("depth stage: RMS residual per iteration %s" % np.array2string(o["iter_rmse"].cpu().numpy(), precision=4))
    if o["status"]:
        raise SspError("the depth stage's reduced system could not be factored: no rig is written; the run without --depth-dir "
                       "writes the keypoint rig")
    return o


if __name__ == "__main__":
    main()
