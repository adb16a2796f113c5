"""Decode and pose utilities -- drop-in for the hot-path subset of reference utils.py.

get_region_boxes (utils.py:216-296) and pnp (utils.py:86-100) run on the GPU kernels; the small numpy helpers
(compute_projection, compute_transformation, calcAngularDistance, get_3D_corners, get_camera_intrinsic,
convert2cpu) keep the reference's names and conventions.  Batched entry points (region_boxes_batched,
pnp_batched, project_points_batched) expose the same kernels without the per-image Python loop.
"""
from __future__ import annotations

import collections

import numpy as np
import torch

from ._lib import CONSTANTS, call, load, ptr, stream_ptr, SspError
from .utils_host import (makedirs, get_all_files, calc_pts_diameter, adi, get_2d_bb, compute_2d_bb, compute_2d_bb_from_orig_pix,  # noqa: F401
                         corner_confidences, corner_confidence, sigmoid, softmax, fix_corner_order, read_truths, read_truths_args,
                         read_pose, load_class_names, image2torch, read_data_cfg, scale_bboxes, file_lines, get_image_size, logging,
                         label_rows_from_projection)


def _dev():
    if not torch.cuda.is_available():
        raise SspError("singleshotpose_b200 needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


# ------------------------------------------------------------------------------------------ host helpers
def get_camera_intrinsic(u0, v0, fx, fy):
    return np.array([[fx, 0.0, u0], [0.0, fy, v0], [0.0, 0.0, 1.0]])


def compute_projection(points_3D, transformation, internal_calibration):
    """K [R|t] X, perspective divide; float32 (2, N) like utils.py:40-45."""
    cam = internal_calibration.dot(transformation).dot(points_3D)
    out = np.zeros((2, points_3D.shape[1]), dtype="float32")
    out[0, :] = cam[0, :] / cam[2, :]
    out[1, :] = cam[1, :] / cam[2, :]
    return out


def compute_transformation(points_3D, transformation):
    return transformation.dot(points_3D)


def calcAngularDistance(gt_rot, pr_rot):
    trace = np.trace(np.dot(gt_rot, np.transpose(pr_rot)))
    return np.rad2deg(np.arccos((trace - 1.0) / 2.0))


def get_3D_corners(vertices):
    """(4, 8): min/max box corners, x outermost, z fastest (utils.py:66-84), homogeneous."""
    mn, mx = vertices[:3].min(axis=1), vertices[:3].max(axis=1)
    c = np.array([[x, y, z] for x in (mn[0], mx[0]) for y in (mn[1], mx[1]) for z in (mn[2], mx[2])])
    return np.concatenate((c.T, np.ones((1, 8))), axis=0)


def convert2cpu(gpu_matrix):
    return torch.FloatTensor(gpu_matrix.size()).copy_(gpu_matrix)


def convert2cpu_long(gpu_matrix):
    return torch.LongTensor(gpu_matrix.size()).copy_(gpu_matrix)


# ------------------------------------------------------------------------------------------ decode
def region_boxes_batched(output, num_classes, num_keypoints, only_objectness=1):
    """-> (boxes (B, 2K+3) per image, best_conf (B,), box_global (2K+3,)) as CUDA tensors."""
    if output.dim() == 3:
        output = output.unsqueeze(0)
    if not output.is_cuda:
        raise SspError("get_region_boxes runs on CUDA tensors only")
    out = output.detach().contiguous().float()
    B, C, H, W = out.shape
    assert C == 2 * num_keypoints + 1 + num_classes
    nv = 2 * num_keypoints + 3
    boxes = torch.empty(B, nv, dtype=torch.float32, device=out.device)
    best = torch.empty(B, dtype=torch.float32, device=out.device)
    glob = torch.empty(nv, dtype=torch.float32, device=out.device)
    call("ssp_region_decode_argmax", ptr(out), B, num_keypoints, num_classes, H, W, int(bool(only_objectness)),
         ptr(boxes), ptr(best), ptr(glob), stream_ptr())
    return boxes, best, glob


def get_region_boxes(output, num_classes, num_keypoints, only_objectness=1, validation=True):
    """Reference semantics: ONE box, the best cell over the whole batch -> list of 2K+3 scalars."""
    _, _, glob = region_boxes_batched(output, num_classes, num_keypoints, only_objectness)
    v = glob.cpu()
    box = [v[j] for j in range(2 * num_keypoints + 2)]
    box.append(v[2 * num_keypoints + 2].long())
    return box


# ------------------------------------------------------------------------------------------ pose
def _pnp_inputs(points_3D, points_2D, cameraMatrix):
    """-> P3 (P,3) or (n,P,3), uv (n,P,2), K (3,3): contiguous float32 CUDA tensors"""
    dev = _dev()
    P3, uv, K = (torch.as_tensor(np.asarray(a, dtype=np.float32) if not torch.is_tensor(a) else a).to(dev, torch.float32).contiguous()
                 for a in (points_3D, points_2D, cameraMatrix))
    return P3, uv.unsqueeze(0) if uv.dim() == 2 else uv, K


def camera_distortion(d):
    """OpenCV distortion coefficients (k1, k2, p1, p2[, k3[, k4, k5, k6]]), as cv2.calibrateCamera returns them -> (8,) float64
    numpy array, zero-padded; None for None, an empty input or all zeros (the zero-distortion solve).  Any shape that flattens to
    4, 5 or 8 values; float32 input keeps its float32 values, as cv2 does.  SspError for 12 or 14 coefficients (the thin-prism and
    tilted models), any other count, or a value that is not finite."""
    if d is None:
        return None
    a = d.detach().cpu().numpy() if torch.is_tensor(d) else np.asarray(d)
    a = a.reshape(-1)
    if a.size == 0:
        return None
    if a.size in (12, 14):
        raise SspError("%d distortion coefficients: the thin-prism / tilted models are not supported (4, 5 or 8)" % a.size)
    if a.size not in (4, 5, 8):
        raise SspError("distortion coefficients are (k1, k2, p1, p2[, k3[, k4, k5, k6]]): 4, 5 or 8 values, got %d" % a.size)
    try:
        a = a.astype(np.float64)
    except (TypeError, ValueError):
        raise SspError("distortion coefficients must be numbers, got %r" % (d,))
    if not np.isfinite(a).all():
        raise SspError("distortion coefficients must be finite, got %s" % (a,))
    if not a.any():
        return None
    return np.concatenate([a, np.zeros(8 - a.size)])


def distortion_tensor(k, dev):
    """camera_distortion's (8,) array -> the DEVICE double[8] the *_dist entry points read"""
    return torch.from_numpy(np.ascontiguousarray(k, np.float64)).to(dev)


def pnp_batched(points_3D, points_2D, cameraMatrix, max_iter=20, return_iters=False, dist_coeffs=None):
    """points_3D (P,3) shared or (n,P,3); points_2D (n,P,2); K (3,3) -> R (n,3,3) f64, t (n,3) f64 CUDA tensors.
    dist_coeffs: OpenCV distortion coefficients (camera_distortion), cv2.solvePnP's distCoeffs (ssp_pnp_dist); None or all zeros
    is the zero-distortion solve (ssp_pnp_batched)."""
    k = camera_distortion(dist_coeffs)
    P3, uv, K = _pnp_inputs(points_3D, points_2D, cameraMatrix)
    dev = uv.device
    n, npts = uv.shape[0], uv.shape[1]
    shared = P3.dim() == 2
    assert P3.shape[-2] == npts and P3.shape[-1] == 3 and uv.shape[-1] == 2
    R = torch.empty(n, 3, 3, dtype=torch.float64, device=dev)
    t = torch.empty(n, 3, dtype=torch.float64, device=dev)
    if k is not None:
        work = torch.empty(n, 3, dtype=torch.int32, device=dev) if return_iters else None
        call("ssp_pnp_dist", ptr(P3), 1 if shared else 0, ptr(uv), ptr(K), ptr(distortion_tensor(k, dev)), npts, n, 1, None, None, None,
             max_iter, ptr(R), ptr(t), None, ptr(work), stream_ptr())
        return (R, t, work[:, 1]) if return_iters else (R, t)
    iters = torch.empty(n, dtype=torch.int32, device=dev) if return_iters else None
    call("ssp_pnp_batched", ptr(P3), 1 if shared else 0, ptr(uv), ptr(K), npts, n, max_iter, ptr(R), ptr(t), ptr(iters), stream_ptr())
    return (R, t, iters) if return_iters else (R, t)


def check_sigma(name, value):
    """-> float(value); SspError unless it is > 0 and finite"""
    try:
        v = float(value)
    except (TypeError, ValueError):
        raise SspError("%s must be a number, got %r" % (name, value))
    if not (v > 0.0 and np.isfinite(v)):
        raise SspError("%s must be > 0 and finite, got %r" % (name, value))
    return v


def pose_covariance_batched(points_3D, cameraMatrix, R, t, keypoint_sigma, dist_coeffs=None):
    """Covariance of PnP poses (ssp_pose_covariance, rules: csrc/pose_filter_core.h): points_3D (P,3) shared or (n,P,3); K (3,3);
    R (n,3,3), t (n,3) the solved poses (pnp_batched's outputs); keypoint_sigma: the keypoint noise in pixels (> 0).
    -> (cov (n,6,6) fp64, status (n,) int32) CUDA tensors.  cov = keypoint_sigma^2 (J^T J)^-1 over (dth, dt_), the pose perturbed
    on the left (x_cam = exp([dth]x) R X + t + dt_), J the keypoints' pixel Jacobian at the pose: the covariance of the pose to
    first order when the keypoints carry independent Gaussian noise of keypoint_sigma px.  It depends on the points, the camera and
    the pose, not on the keypoints.  status: 0, or SSP_POSE_COV_SINGULAR (1: J^T J is singular to 1e-12 of its largest diagonal
    entry) | SSP_POSE_COV_DEPTH (2: a point at depth <= 0); such a cov is zero.  dist_coeffs: as pnp_batched (the distorted
    projection's Jacobian)."""
    sigma = check_sigma("keypoint_sigma", keypoint_sigma)
    k = camera_distortion(dist_coeffs)
    dev = _dev()
    P3, K = (torch.as_tensor(np.asarray(a, dtype=np.float32) if not torch.is_tensor(a) else a).to(dev, torch.float32).contiguous()
             for a in (points_3D, cameraMatrix))
    R, t = (torch.as_tensor(a).to(dev, torch.float64).contiguous() for a in (R, t))
    R, t = R.reshape(-1, 3, 3), t.reshape(-1, 3)
    n, npts = R.shape[0], P3.shape[-2]
    shared = P3.dim() == 2
    if t.shape[0] != n or P3.shape[-1] != 3 or (not shared and P3.shape[0] != n):
        raise SspError("pose_covariance_batched: R (n,3,3), t (n,3) and points_3D (P,3) or (n,P,3) disagree: %s, %s, %s"
                       % (tuple(R.shape), tuple(t.shape), tuple(P3.shape)))
    cov = torch.empty(n, 6, 6, dtype=torch.float64, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    call("ssp_pose_covariance", ptr(P3), 1 if shared else 0, ptr(K), None if k is None else ptr(distortion_tensor(k, dev)), npts, n, 1,
         None, ptr(R), ptr(t), sigma, ptr(cov), ptr(status), stream_ptr())
    return cov, status


def object_table(objects, num_classes, K):
    """The constants of a pose head, checked: objects {class id in [0, num_classes): (3|4, 8) box corners}, K (3, 3).
    -> (classes (Q,) int64 sorted ids, points (num_classes, 9, 3) float64 PnP points [0; corners3D_c[:3]] of each requested class
    by class id (valid.py:146, valid_multi.py:135; zeros for the others), K as (3, 3) float64)"""
    if not isinstance(objects, dict) or not objects:
        raise SspError("objects must be a non-empty {class id: corners3D} dict")
    nC = int(num_classes)
    classes = sorted(objects)
    points = np.zeros((nC, 9, 3))
    for c in classes:
        if isinstance(c, bool) or not isinstance(c, (int, np.integer)) or not 0 <= c < nC:
            raise SspError("class id %r is not in [0, %d)" % (c, nC))
        corners = np.asarray(objects[c], dtype=np.float64)
        if corners.ndim != 2 or corners.shape[0] not in (3, 4) or corners.shape[1] != 8:
            raise SspError("corners3D must be (3|4, 8), got %s" % (corners.shape,))
        points[c, 1:] = corners[:3].T
    Km = np.asarray(K, dtype=np.float64)
    if Km.shape != (3, 3):
        raise SspError("K must be (3, 3), got %s" % (Km.shape,))
    return np.array(classes, dtype=np.int64), points, Km


def pnp_one(points_3D, points_2D, cameraMatrix, distCoeffs=None):
    """one problem of pnp_batched: numpy in, R (3,3) float64 and t (3,1) float64 out"""
    assert points_3D.shape[0] == points_2D.shape[0], "points 3D and points 2D must have same number of vertices"
    R, t = pnp_batched(points_3D, np.ascontiguousarray(points_2D[:, :2]), cameraMatrix, dist_coeffs=distCoeffs)
    return R[0].cpu().numpy(), t[0].cpu().numpy().reshape(3, 1)


def pnp(points_3D, points_2D, cameraMatrix):
    """Same contract as utils.py:86-100: numpy in, R (3,3) float64 and t (3,1) float64 out.  Like the reference, the distortion
    coefficients are the function attribute pnp.distCoeffs (cv2's 4, 5 or 8 values, camera_distortion); unset or all zeros is the
    zero-distortion solve."""
    return pnp_one(points_3D, points_2D, cameraMatrix, getattr(pnp, "distCoeffs", None))


# ------------------------------------------------------------------------------------------ consensus pose (csrc/pnp_consensus_core.h)
PNP_MODES = ("plain", "consensus")


def check_pnp_args(pnp, reproj_thresh):
    """-> (pnp, reproj_thresh as float); SspError for an unknown mode or a threshold that is not > 0 and finite"""
    if pnp not in PNP_MODES:
        raise SspError("pnp must be one of %s, got %r" % (", ".join(PNP_MODES), pnp))
    thr = float(reproj_thresh)
    if not (np.isfinite(thr) and thr > 0):
        raise SspError("reproj_thresh must be > 0 and finite (pixels), got %r" % (reproj_thresh,))
    return pnp, thr


def consensus_subsets(point_sets, size=6):
    """(H,) uint16 bitmasks of the `size`-subsets of the P points, in lexicographic order, without those in which 5 points are
    coplanar for any of the given point sets: the DLT of cv2.solvePnP's ITERATIVE solve is degenerate there.  Coplanar means the
    smallest singular value of the centred 5 x 3 matrix is below 1e-6 times the set's largest extent (largest coordinate range).
    point_sets: one (P, 3) array or a sequence of them, all with the same P.  For the 9 box points (centroid + 8 corners) 60 of 84
    subsets are kept: each of the six diagonal planes through two opposite edges holds 4 corners and the centroid."""
    import itertools
    sets = np.asarray(point_sets, np.float64)
    sets = sets[None] if sets.ndim == 2 else sets
    if sets.ndim != 3 or sets.shape[2] != 3:
        raise SspError("point_sets must be (P, 3) or (S, P, 3), got %s" % (sets.shape,))
    P = sets.shape[1]
    if size != 6 or not 7 <= P <= 10:
        raise SspError("consensus subsets are 6 of 7..10 points, got %d of %d" % (size, P))
    extent = np.ptp(sets, axis=1).max(axis=1)                       # (S,)
    coplanar = set()
    for five in itertools.combinations(range(P), 5):
        X = sets[:, list(five)]
        X = X - X.mean(axis=1, keepdims=True)
        smin = np.linalg.svd(X, compute_uv=False)[:, -1]
        if (smin < 1e-6 * extent).any():
            coplanar.add(five)
    out = [sum(1 << i for i in S) for S in itertools.combinations(range(P), size)
           if not any(f in coplanar for f in itertools.combinations(S, 5))]
    return np.array(out, np.uint16)


def pnp_consensus_batched(points_3D, points_2D, cameraMatrix, reproj_thresh=8.0, max_iter=20, subsets=None, dist_coeffs=None):
    """Consensus PnP of n problems on the GPU (ssp_pnp_consensus, rule: csrc/pnp_consensus_core.h): the plain all-point solve and
    one cold solve per 6-point subset, each scored by its inliers (squared reprojection error <= reproj_thresh^2 px^2, none if a
    point lies behind the camera); the best is refined on its inliers.  A pose that survives one or two wrong keypoints; where
    the all-point solve already has every point as an inlier the result is bit-identical to pnp_batched.
    points_3D (P,3) shared or (n,P,3), 7 <= P <= 10; points_2D (n,P,2); K (3,3); reproj_thresh in pixels (8, cv2.solvePnPRansac's
    default); subsets: (H,) uint16 masks, default consensus_subsets(points_3D).
    -> R (n,3,3) f64, t (n,3) f64, params (n,6) f64 (rvec, t), inliers (n,P) bool, hyp (n,) int32 (the chosen hypothesis: 0 the
    all-point solve, h the subset subsets[h-1], -1 none had an inlier), CUDA tensors.
    dist_coeffs: OpenCV distortion coefficients (camera_distortion): every solve is cv2.solvePnP(..., distCoeffs) and the inliers
    are scored on the distorted reprojection (ssp_pnp_consensus_dist); None or all zeros is ssp_pnp_consensus."""
    _, thr = check_pnp_args("consensus", reproj_thresh)
    k = camera_distortion(dist_coeffs)
    P3, uv, K = _pnp_inputs(points_3D, points_2D, cameraMatrix)
    dev = uv.device
    n, npts = uv.shape[0], uv.shape[1]
    shared = P3.dim() == 2
    if P3.shape[-2] != npts or P3.shape[-1] != 3 or uv.shape[-1] != 2 or (not shared and P3.shape[0] != n):
        raise SspError("points_3D %s does not match points_2D %s" % (tuple(P3.shape), tuple(uv.shape)))
    if subsets is None:
        subsets = consensus_subsets(P3.cpu().numpy())
    tab = np.ascontiguousarray(subsets, np.uint16).reshape(-1)
    R = torch.empty(n, 3, 3, dtype=torch.float64, device=dev)
    t = torch.empty(n, 3, dtype=torch.float64, device=dev)
    params = torch.empty(n, 6, dtype=torch.float64, device=dev)
    inl = torch.empty(n, dtype=torch.int32, device=dev)
    hyp = torch.empty(n, dtype=torch.int32, device=dev)
    wb = consensus_work_bytes(npts, len(tab), n)
    work = torch.empty(max(wb, 8) // 8, dtype=torch.float64, device=dev)
    if k is None:
        call("ssp_pnp_consensus", ptr(P3), 1 if shared else 0, ptr(uv), ptr(K), npts, n, 1, None, tab.ctypes.data, len(tab), thr, max_iter,
             ptr(R), ptr(t), ptr(params), ptr(inl), ptr(hyp), ptr(work), work.numel() * 8, stream_ptr())
    else:
        call("ssp_pnp_consensus_dist", ptr(P3), 1 if shared else 0, ptr(uv), ptr(K), ptr(distortion_tensor(k, dev)), npts, n, 1, None,
             tab.ctypes.data, len(tab), thr, max_iter, ptr(R), ptr(t), ptr(params), ptr(inl), ptr(hyp), ptr(work), work.numel() * 8,
             stream_ptr())
    return R, t, params, inlier_bits(inl, keypoint_bits(npts, dev)), hyp


def consensus_work_bytes(npts, n_subsets, n):
    """bytes of device workspace ssp_pnp_consensus needs for n problems of npts points and n_subsets subsets"""
    import ctypes
    out = ctypes.c_longlong(0)
    call("ssp_pnp_consensus_work_bytes", int(npts), int(n_subsets), int(n), ctypes.byref(out))
    return out.value


def keypoint_bits(npts, device):
    """(npts,) int32 1 << i: the bit of keypoint i in an inlier mask of ssp_pnp_consensus"""
    return torch.tensor([1 << i for i in range(npts)], dtype=torch.int32, device=device)


def inlier_bits(mask, bits, out=None):
    """(...,) int32 inlier masks -> (..., npts) bool, with bits = keypoint_bits(npts, mask.device); out: the (..., npts) bool
    tensor to write"""
    return torch.ne(torch.bitwise_and(mask.unsqueeze(-1), bits), 0, out=out)


def pnp_consensus(points_3D, points_2D, cameraMatrix, reproj_thresh=8.0, dist_coeffs=None):
    """pnp's contract (numpy in, R (3,3) and t (3,1) float64 out) with the consensus solve of pnp_consensus_batched, plus the
    indices of the inlier keypoints (int64, ascending).  dist_coeffs: as pnp_consensus_batched."""
    assert points_3D.shape[0] == points_2D.shape[0], "points 3D and points 2D must have same number of vertices"
    R, t, _p, inl, _h = pnp_consensus_batched(points_3D, np.ascontiguousarray(points_2D[:, :2]), cameraMatrix, reproj_thresh,
                                              dist_coeffs=dist_coeffs)
    return R[0].cpu().numpy(), t[0].cpu().numpy().reshape(3, 1), np.nonzero(inl[0].cpu().numpy())[0]


def project_points_batched(points_3D, Rt, internal_calibration, dist_coeffs=None):
    """points_3D (3|4, Nv); Rt (n,3,4) -> (n, 2, Nv) float32 CUDA tensor (compute_projection for n poses).  dist_coeffs: OpenCV
    distortion coefficients (camera_distortion): cv2.projectPoints with them (ssp_project_points_dist), the pixels of the raw,
    distorted frame; None or all zeros is compute_projection."""
    k = camera_distortion(dist_coeffs)
    dev = _dev()
    X = torch.as_tensor(points_3D).to(dev, torch.float32).contiguous()
    T = torch.as_tensor(Rt).to(dev, torch.float64).contiguous()
    K = torch.as_tensor(internal_calibration).to(dev, torch.float64).contiguous()
    if T.dim() == 2:
        T = T.unsqueeze(0)
    n, nv = T.shape[0], X.shape[1]
    out = torch.empty(n, 2, nv, dtype=torch.float32, device=dev)
    if k is None:
        call("ssp_project_points", ptr(X), X.shape[0], nv, ptr(T), ptr(K), n, ptr(out), stream_ptr())
    else:
        call("ssp_project_points_dist", ptr(X), X.shape[0], nv, ptr(T), ptr(K), ptr(distortion_tensor(k, dev)), n, ptr(out), stream_ptr())
    return out


# ------------------------------------------------------------------------------------------ pose errors over the mesh
def _mesh_rows(vertices, dev):
    """(3|4, Nv) or (Nv, 3), any float dtype -> (Nv, 3) fp64 contiguous on `dev` (converted there).  An array with 3 or 4 rows
    is read as (3|4, Nv), the layout of valid.py's `vertices`."""
    V = vertices if torch.is_tensor(vertices) else torch.as_tensor(np.asarray(vertices))
    if V.dim() != 2 or not (V.shape[0] in (3, 4) or V.shape[1] == 3):
        raise SspError("vertices must be (3|4, Nv) or (Nv, 3), got %s" % (tuple(V.shape),))
    V = V.to(dev)
    V = V[:3].t() if V.shape[0] in (3, 4) else V
    return V.double().contiguous()


def _pose_stack(Rt, dev):
    T = (Rt if torch.is_tensor(Rt) else torch.as_tensor(np.asarray(Rt))).to(dev, torch.float64)
    T = T.unsqueeze(0) if T.dim() == 2 else T
    if T.dim() != 3 or tuple(T.shape[1:]) != (3, 4):
        raise SspError("poses must be (n, 3, 4), got %s" % (tuple(T.shape),))
    return T.contiguous()


def adi_batched(vertices, Rt_est, Rt_gt, with_add=False):
    """adi(pts_est, pts_gt) of utils.py:60-64 for n pose pairs: for each vertex under Rt_gt[p], the distance to the nearest
    vertex under Rt_est[p], averaged over the mesh (ADD-S, the LINEMOD error of the symmetric eggbox and glue).
    vertices (3|4, Nv) or (Nv, 3), any float dtype (converted to fp64 on the device); Rt_est, Rt_gt (n, 3, 4).
    -> (n,) fp64 CUDA tensor; with with_add=True (adds, add), add[p] = mean_i |Rt_gt[p] x_i - Rt_est[p] x_i| (ADD) from the
    same launch.  Brute force on the GPU (n * Nv^2 fp64 pair distances, ssp_adds_batched) where the reference builds a k-d
    tree; each pose's value is computed in a fixed order, the same in any batch."""
    dev = _dev()
    X = _mesh_rows(vertices, dev)
    E, G = _pose_stack(Rt_est, dev), _pose_stack(Rt_gt, dev)
    if E.shape[0] != G.shape[0]:
        raise SspError("Rt_est and Rt_gt hold %d and %d poses" % (E.shape[0], G.shape[0]))
    n, nv = E.shape[0], X.shape[0]
    adds = torch.empty(n, dtype=torch.float64, device=dev)
    add = torch.empty(n, dtype=torch.float64, device=dev) if with_add else None
    if n:
        wb = int(load().ssp_adds_work_bytes(nv, n))
        if wb < 0:
            raise SspError("ssp_adds_work_bytes: bad size (Nv = %d, n = %d)" % (nv, n))
        work = torch.empty(wb // 8, dtype=torch.float64, device=dev)
        call("ssp_adds_batched", ptr(X), nv, ptr(E), ptr(G), n, ptr(adds), ptr(add), ptr(work), wb, stream_ptr())
    return (adds, add) if with_add else adds


def mesh_diameter(pts):
    """calc_pts_diameter (utils.py:50-58) on the GPU: the largest distance between two of the (Nv, 3) points -> Python float,
    bit-identical to calc_pts_diameter on float64 points.  Waits for the result."""
    dev = _dev()
    P = pts if torch.is_tensor(pts) else torch.as_tensor(np.asarray(pts))
    if P.dim() != 2 or P.shape[1] != 3:
        raise SspError("mesh_diameter takes (Nv, 3) points, got %s" % (tuple(P.shape),))
    P = P.to(dev).double().contiguous()
    out = torch.empty(1, dtype=torch.float64, device=dev)
    call("ssp_mesh_diameter", ptr(P), P.shape[0], ptr(out), stream_ptr())
    return float(out.item())


# ------------------------------------------------------------------------------------------ refinement against depth frames
REFINE_STATUS = {"few_points": 1, "singular": 2, "bad_pose": 4}         # ssp_refine_depth's status bits (SSP_REFINE_*)


def vertex_normals(vertices, faces):
    """Unit outward normals (Nv, 3) float64 of a triangle mesh: each vertex sums the unnormalised cross products (b - a) x (c - a)
    of its faces (normals weighted by area), the sum is normalised, and every normal is flipped when the mesh's signed volume is
    negative, so a closed mesh of either winding gets outward normals.  A vertex whose sum is zero gets a zero normal (the
    refinement never pairs it).  vertices (Nv, 3); faces (Nf, 3) indices in [0, Nv)."""
    V = np.asarray(vertices, np.float64)
    F = np.asarray(faces)
    if V.ndim != 2 or V.shape[1] != 3:
        raise SspError("vertices must be (Nv, 3), got %s" % (V.shape,))
    if F.ndim != 2 or F.shape[1] != 3 or not np.issubdtype(F.dtype, np.integer):
        raise SspError("faces must be (Nf, 3) integers, got %s %s" % (F.shape, F.dtype))
    if F.size and (F.min() < 0 or F.max() >= len(V)):
        raise SspError("a face index lies outside [0, %d)" % len(V))
    a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    cr = np.cross(b - a, c - a)
    N = np.zeros_like(V)
    for k in range(3):
        np.add.at(N, F[:, k], cr)
    if (a * np.cross(b, c)).sum() < 0:                  # 6 x the signed volume
        N = -N
    norm = np.linalg.norm(N, axis=1, keepdims=True)
    return np.divide(N, norm, out=np.zeros_like(N), where=norm > 0)


def check_refine_args(depth_scale, iters, gate):
    """-> (depth_scale, iters, (gate_start, gate_end)); SspError for a depth_scale not > 0 and finite, iters outside [1, 100] or a
    gate range that is not 0 < gate_end <= gate_start < inf (fractions of the object's diameter)"""
    depth_scale = check_sigma("depth_scale", depth_scale)
    maxit = CONSTANTS["SSP_REFINE_MAX_ITERS"]
    if isinstance(iters, bool) or not isinstance(iters, (int, np.integer)) or not 1 <= iters <= maxit:
        raise SspError("refine iters must be an integer in [1, %d], got %r" % (maxit, iters))
    try:
        s, e = (float(g) for g in gate)
    except (TypeError, ValueError):
        raise SspError("the refine gate is (start, end) as fractions of the diameter, got %r" % (gate,))
    if not (0.0 < e <= s < np.inf):
        raise SspError("the refine gate needs 0 < end <= start < inf, got %r" % (gate,))
    return depth_scale, int(iters), (s, e)


def refine_model_table(meshes, num_classes, dev):
    """{class id: (vertices, faces)} -> device (model [total][6] fp64 points and outward normals, offsets [num_classes + 1] int32,
    diam [num_classes] fp64): the tables ssp_refine_depth reads, class c's rows at offsets[c] .. offsets[c + 1] - 1 (no rows for the
    classes not given).  The diameter is mesh_diameter of the vertices."""
    if not isinstance(meshes, dict) or not meshes:
        raise SspError("meshes must be a non-empty {class id: (vertices, faces)} dict")
    rows, counts, diam = [], np.zeros(num_classes, np.int64), np.zeros(num_classes)
    for c in sorted(meshes):
        if isinstance(c, bool) or not isinstance(c, (int, np.integer)) or not 0 <= c < num_classes:
            raise SspError("class id %r is not in [0, %d)" % (c, num_classes))
        try:
            V, F = meshes[c]
        except (TypeError, ValueError):
            raise SspError("the mesh of class %d must be (vertices, faces)" % c)
        V = np.asarray(V, np.float64)
        N = vertex_normals(V, F)
        rows.append(np.concatenate([V, N], 1))
        counts[c], diam[c] = len(V), mesh_diameter(V)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    model = np.concatenate(rows) if rows else np.zeros((0, 6))
    return (torch.from_numpy(np.ascontiguousarray(model)).to(dev), torch.from_numpy(offsets).to(dev), torch.from_numpy(diam).to(dev))


def _depth_tensor(depth, dev):
    """(n, H, W) uint16 numpy array or CUDA tensor -> the device int16 tensor of its bits; SspError for another type or shape"""
    if torch.is_tensor(depth):
        if not depth.is_cuda or depth.dtype != torch.uint16:
            raise SspError("depth given as a torch tensor must be a CUDA uint16 tensor, got %s %s" % (depth.device, depth.dtype))
        D = depth.to(dev).view(torch.int16).contiguous()
    else:
        D = np.asarray(depth)
        if D.dtype != np.uint16:
            raise SspError("depth must be uint16, got %s" % D.dtype)
        D = torch.from_numpy(np.ascontiguousarray(D).view(np.int16)).to(dev)
    if D.dim() != 3:
        raise SspError("depth must be (n, H, W), got %s" % (tuple(D.shape),))
    return D


def refine_depth_batched(depth, vertices, faces, K, R, t, depth_scale=0.001, iters=10, gate=(0.5, 0.02), dist_coeffs=None):
    """Refine n poses of one mesh against n registered depth frames on the GPU (ssp_refine_depth, rule: csrc/refine_depth_core.h):
    projective point-to-plane ICP of the mesh's vertices, with the outward normals of vertex_normals, against the depth pixel
    each front-facing vertex projects to, over `iters` fixed iterations whose pair gate |p_z - q_z| shrinks geometrically from
    gate[0] to gate[1] times the mesh's diameter (mesh_diameter).
    depth (n, H, W) uint16 numpy array or CUDA tensor (0: no measurement), registered to the camera K (3, 3) with dist_coeffs
    (camera_distortion); depth_scale: mesh units per depth unit (0.001 for millimetre depth and metre meshes); R (n, 3, 3), t (n, 3)
    camera from model.  -> (R (n, 3, 3) fp64, t (n, 3) fp64, points (n,) int32 pairs of the last iteration, rmse (n,) fp64 its RMS
    point-to-plane residual before the update, status (n,) int32: 0, or REFINE_STATUS bits, with which the pose is the input
    pose), CUDA tensors."""
    depth_scale, iters, (s, e) = check_refine_args(depth_scale, iters, gate)
    k = camera_distortion(dist_coeffs)
    dev = _dev()
    D = _depth_tensor(depth, dev)
    n, H, W = D.shape
    R, t = (torch.as_tensor(a).to(dev, torch.float64).contiguous() for a in (R, t))
    R, t = R.reshape(-1, 3, 3), t.reshape(-1, 3)
    if R.shape[0] != n or t.shape[0] != n:
        raise SspError("refine_depth_batched: %d depth frames but R %s, t %s" % (n, tuple(R.shape), tuple(t.shape)))
    model, offsets, diam = refine_model_table({0: (vertices, faces)}, 1, dev)
    if n == 0:
        return R.clone(), t.clone(), *(torch.zeros(0, dtype=d, device=dev) for d in (torch.int32, torch.float64, torch.int32))
    Kd = torch.as_tensor(np.asarray(K, np.float64)).to(dev).contiguous()
    cls = torch.zeros(n, dtype=torch.int32, device=dev)
    R_out, t_out = torch.empty_like(R), torch.empty_like(t)
    points, status = torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev)
    rmse = torch.empty(n, dtype=torch.float64, device=dev)
    call("ssp_refine_depth", ptr(D), W, H, depth_scale, ptr(Kd), None if k is None else ptr(distortion_tensor(k, dev)), ptr(model),
         ptr(offsets), ptr(diam), 1, ptr(cls), n, 1, None, ptr(R), ptr(t), iters, s, e, ptr(R_out), ptr(t_out), ptr(points), ptr(rmse),
         ptr(status), stream_ptr())
    return R_out, t_out, points, rmse, status


# ------------------------------------------------------------------------------------------ several calibrated cameras
FUSE_STATUS = {"no_valid": 1, "no_view": 2, "singular": 4}              # ssp_fuse_views' status bits (SSP_FUSE_*)
CameraRig = collections.namedtuple("CameraRig", "K R t dist")


def camera_rig(K, R, t, dist=None):
    """A rig of C calibrated cameras (1 <= C <= 16), checked -> CameraRig(K (C, 3, 3), R (C, 3, 3), t (C, 3) float64, dist (C, 8)
    float64 or None).  K: each camera's intrinsics; R, t: its extrinsics camera-from-world, x_c = R_c x_w + t_c, in the mesh's
    units; dist: None, or one set of OpenCV coefficients per camera (4, 5 or 8 values each, camera_distortion; None or zeros for a
    pinhole camera).  SspError for a value that is not finite, fx or fy <= 0, an R_c that is not a rotation (|R^T R - I| > 1e-6 or
    det < 0), C outside 1..16 or shapes that disagree.  cv2.stereoCalibrate's (K1, d1, K2, d2, R, T) is camera_rig([K1, K2],
    [I, R], [0, T], [d1, d2]): the world frame is camera 0's."""
    try:
        K, R, t = (np.asarray(a, np.float64) for a in (K, R, t))
    except (TypeError, ValueError):
        raise SspError("the rig's K, R and t must be numeric arrays")
    C = len(K) if K.ndim == 3 else -1
    maxv = CONSTANTS["SSP_RIG_MAX_VIEWS"]
    if not 1 <= C <= maxv:
        raise SspError("a rig has 1..%d cameras: K must be (C, 3, 3), got %s" % (maxv, K.shape))
    if K.shape != (C, 3, 3) or R.shape != (C, 3, 3) or t.shape != (C, 3):
        raise SspError("the rig's shapes disagree: K %s, R %s, t %s for (C, 3, 3), (C, 3, 3), (C, 3)" % (K.shape, R.shape, t.shape))
    if not (np.isfinite(K).all() and np.isfinite(R).all() and np.isfinite(t).all()):
        raise SspError("the rig's K, R and t must be finite")
    if not ((K[:, 0, 0] > 0).all() and (K[:, 1, 1] > 0).all()):
        raise SspError("every camera needs fx > 0 and fy > 0")
    for c in range(C):
        if np.abs(R[c].T @ R[c] - np.eye(3)).max() > 1e-6 or np.linalg.det(R[c]) < 0:
            raise SspError("R of camera %d is not a rotation" % c)
    D = None
    if dist is not None:
        if len(dist) != C:
            raise SspError("dist must hold one set of coefficients per camera: %d for %d cameras" % (len(dist), C))
        rows = [camera_distortion(d) for d in dist]
        if any(r is not None for r in rows):
            D = np.stack([np.zeros(8) if r is None else r for r in rows])
    return CameraRig(K, R, t, D)


def rig_tensors(rig, dev):
    """the device tables ssp_fuse_views reads: K (C, 3, 3) fp32 and fp64, dist (C, 8) or None, R (C, 3, 3), t (C, 3)"""
    to = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    return (to(rig.K, np.float32), to(rig.K, np.float64), None if rig.dist is None else to(rig.dist, np.float64), to(rig.R, np.float64),
            to(rig.t, np.float64))


def check_fuse_args(gate, reproj_thresh, keypoint_sigma):
    """-> the three as floats; SspError for a value not > 0 and finite or gate < reproj_thresh"""
    gate, thr, sigma = (check_sigma(n, v) for n, v in (("gate", gate), ("reproj_thresh", reproj_thresh), ("keypoint_sigma", keypoint_sigma)))
    if gate < thr:
        raise SspError("the gate (%g px) must be >= reproj_thresh (%g px)" % (gate, thr))
    return gate, thr, sigma


def fuse_work_bytes(groups, views, slots):
    """bytes of device workspace ssp_fuse_views needs"""
    import ctypes
    out = ctypes.c_longlong(0)
    call("ssp_fuse_views_work_bytes", int(groups), int(views), int(slots), ctypes.byref(out))
    return out.value


def fuse_views_batched(points_3D, keypoints_px, rig, valid=None, gate=40.0, reproj_thresh=8.0, keypoint_sigma=2.0, max_iter=20):
    """Fuse the poses of several calibrated cameras on the GPU (ssp_fuse_views, rule: csrc/multiview_core.h).  rig: camera_rig's
    CameraRig of C cameras.  keypoints_px (B, P, 2) or (B, S, P, 2) raw pixels, 7 <= P <= 10: row b = g C + c is camera c's view of
    capture g (B a multiple of C), S objects per row; points_3D (P, 3) shared, or one set per row (and slot); valid (B,) or (B, S)
    bool, default all: the views that take part.  Every row gets its own cold PnP with its camera; each valid view's pose in the
    world frame is a hypothesis; the views that agree with it within `gate` px (mean squared reprojection error) are fused by LM,
    then the views within `reproj_thresh` px of that fit; the hypothesis with the most views wins.
    -> dict of CUDA tensors: per row R (B[, S], 3, 3), t, corners_px (B[, S], P, 2) (the per-view solve); per capture R_world (G[, S],
    3, 3), t_world (G[, S], 3) world-from-object, world_cov (G[, S], 6, 6) (keypoint_sigma^2 (J^T J)^-1, left perturbation, world
    axes), views (G[, S], C) bool, view_err (G[, S], C) (RMS px of each valid view under the fused pose, -1 for the others),
    fuse_hyp (G[, S]) int32 (the winning view, -1 for none), fuse_status (G[, S]) int32 (FUSE_STATUS bits); per row
    corners_world_px (B[, S], P, 2), the fused pose in each row's camera."""
    gate, thr, sigma = check_fuse_args(gate, reproj_thresh, keypoint_sigma)
    if not isinstance(rig, CameraRig):
        raise SspError("rig must be a CameraRig (utils.camera_rig)")
    dev = _dev()
    uv = torch.as_tensor(np.asarray(keypoints_px, np.float32) if not torch.is_tensor(keypoints_px) else keypoints_px).to(dev, torch.float32)
    slotted = uv.dim() == 4
    uv = (uv if slotted else uv.unsqueeze(1)).contiguous()
    if uv.dim() != 4 or uv.shape[-1] != 2:
        raise SspError("keypoints_px must be (B, P, 2) or (B, S, P, 2), got %s" % (tuple(uv.shape),))
    B, S, npts = uv.shape[:3]
    C = len(rig.K)
    if B % C:
        raise SspError("%d rows are not whole captures of the rig's %d cameras" % (B, C))
    P3 = torch.as_tensor(np.asarray(points_3D, np.float32) if not torch.is_tensor(points_3D) else points_3D).to(dev, torch.float32).contiguous()
    shared = P3.dim() == 2
    if P3.shape[-2:] != (npts, 3) or (not shared and P3.numel() != B * S * npts * 3):
        raise SspError("points_3D %s does not match keypoints_px %s" % (tuple(P3.shape), tuple(uv.shape)))
    ok = torch.ones(B, S, dtype=torch.bool, device=dev) if valid is None else torch.as_tensor(valid).to(dev, torch.bool).reshape(B, S).contiguous()
    K32, K64, D, Rr, tr = rig_tensors(rig, dev)
    G = B // C
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device=dev)
    o = dict(R=f64(B, S, 3, 3), t=f64(B, S, 3), corners_px=torch.empty(B, S, npts, 2, dtype=torch.float32, device=dev), R_world=f64(G, S, 3, 3),
             t_world=f64(G, S, 3), world_cov=f64(G, S, 6, 6), views=torch.empty(G, S, C, dtype=torch.bool, device=dev), view_err=f64(G, S, C),
             fuse_hyp=torch.empty(G, S, dtype=torch.int32, device=dev), fuse_status=torch.empty(G, S, dtype=torch.int32, device=dev),
             corners_world_px=torch.empty(B, S, npts, 2, dtype=torch.float32, device=dev))
    work = f64(max(fuse_work_bytes(G, C, S), 8) // 8)
    call("ssp_fuse_views", ptr(P3), 1 if shared else 0, ptr(uv), ptr(ok), npts, G, C, S, ptr(K32), ptr(K64), ptr(D), ptr(Rr), ptr(tr), gate,
         thr, sigma, max_iter, ptr(o["R"]), ptr(o["t"]), ptr(o["corners_px"]), ptr(o["R_world"]), ptr(o["t_world"]), ptr(o["world_cov"]),
         ptr(o["views"]), ptr(o["view_err"]), ptr(o["fuse_hyp"]), ptr(o["fuse_status"]), ptr(o["corners_world_px"]), ptr(work),
         work.numel() * 8, stream_ptr())
    return o if slotted else {k: v[:, 0] for k, v in o.items()}


def refine_depth_rig_batched(depth, vertices, faces, rig, R_world, t_world, depth_scale=0.001, iters=10, gate=(0.5, 0.02), fuse_status=None):
    """Refine world poses of one mesh against the depth frames of every camera of a rig at once on the GPU (ssp_refine_depth_rig,
    rule: csrc/refine_rig_core.h): each camera pairs the mesh's vertices with its own depth frame as refine_depth_batched does,
    and one point-to-plane ICP over the pairs of all cameras solves for the world pose.  rig: camera_rig's CameraRig of C cameras;
    depth (G C, H, W) uint16 numpy array or CUDA tensor, row g C + c registered to camera c (its K and coefficients); R_world
    (G[, S], 3, 3), t_world (G[, S], 3) world from model (fuse_views_batched's); fuse_status (G[, S]) int or None: a pose whose
    status has FUSE_STATUS no_valid or no_view is left as it is (bad_pose).  depth_scale, iters and gate as refine_depth_batched.
    -> (R (G[, S], 3, 3), t (G[, S], 3), points (G[, S]) int32 pairs of the last iteration over all cameras, rmse (G[, S]) its RMS
    point-to-plane residual, status (G[, S]) int32 REFINE_STATUS bits (with a bit set the pose is the input pose), view_points
    (G[, S], C) int32 and view_rmse (G[, S], C) each camera's pairs and RMS residual of the last iteration), CUDA tensors."""
    depth_scale, iters, (s, e) = check_refine_args(depth_scale, iters, gate)
    if not isinstance(rig, CameraRig):
        raise SspError("rig must be a CameraRig (utils.camera_rig)")
    dev = _dev()
    D = _depth_tensor(depth, dev)
    B, H, W = D.shape
    C = len(rig.K)
    if B % C:
        raise SspError("%d depth frames are not whole captures of the rig's %d cameras" % (B, C))
    G = B // C
    R, t = (torch.as_tensor(a).to(dev, torch.float64).contiguous() for a in (R_world, t_world))
    if R.dim() < 3 or R.shape[-2:] != (3, 3) or R.shape[0] != G or t.shape != R.shape[:-1]:
        raise SspError("refine_depth_rig_batched: %d captures but R_world %s, t_world %s: (G[, S], 3, 3) and (G[, S], 3)"
                       % (G, tuple(R.shape), tuple(t.shape)))
    lead = tuple(R.shape[:-2])
    S = int(np.prod(lead[1:], dtype=np.int64)) if len(lead) > 1 else 1
    fs = None
    if fuse_status is not None:
        fs = torch.as_tensor(fuse_status).to(dev, torch.int32).contiguous()
        if tuple(fs.shape) != lead:
            raise SspError("fuse_status must be %s, got %s" % (lead, tuple(fs.shape)))
    model, offsets, diam = refine_model_table({0: (vertices, faces)}, 1, dev)
    i32 = lambda *sh: torch.empty(*sh, dtype=torch.int32, device=dev)
    f64 = lambda *sh: torch.empty(*sh, dtype=torch.float64, device=dev)
    out = (torch.empty_like(R), torch.empty_like(t), i32(*lead), f64(*lead), i32(*lead), i32(*lead, C), f64(*lead, C))
    if G == 0 or S == 0:
        return out
    _K32, K64, Dd, Rr, tr = rig_tensors(rig, dev)
    V = np.asarray(vertices, np.float64)
    box = np.concatenate([V.mean(0, keepdims=True), get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)[:3].T])    # the drawn points
    table = torch.from_numpy(box.astype(np.float32)).to(dev)
    corners = torch.empty(B, S, 9, 2, dtype=torch.float32, device=dev)
    cls = torch.zeros(G, S, dtype=torch.int32, device=dev)
    call("ssp_refine_depth_rig", ptr(D), W, H, depth_scale, C, ptr(K64), ptr(Dd), ptr(Rr), ptr(tr), ptr(model), ptr(offsets), ptr(diam),
         ptr(table), 9, 1, ptr(cls), G, S, None, ptr(fs), ptr(R), ptr(t), iters, s, e, *(ptr(o) for o in out), ptr(corners), stream_ptr())
    return out


def fuse_instances_work_bytes(groups, views, slots):
    """bytes of device workspace ssp_fuse_instances needs"""
    import ctypes
    out = ctypes.c_longlong(0)
    call("ssp_fuse_instances_work_bytes", int(groups), int(views), int(slots), ctypes.byref(out))
    return out.value


def fuse_instances_outputs(B, C, M, npts, dev):
    """the device outputs of ssp_fuse_instances for B rows of a C-camera rig with M slots, in its argument order"""
    G = B // C
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device=dev)
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=dev)
    return dict(R=f64(B, M, 3, 3), t=f64(B, M, 3), corners_px=torch.empty(B, M, npts, 2, dtype=torch.float32, device=dev), world_count=i32(G),
                unfused=i32(G), world_cls=i32(G, M), R_world=f64(G, M, 3, 3), t_world=f64(G, M, 3), world_cov=f64(G, M, 6, 6),
                members=i32(G, M, C), view_err=f64(G, M, C), fuse_hyp=i32(G, M), fuse_status=i32(G, M), world_index=i32(B, M),
                corners_world_px=torch.empty(B, M, npts, 2, dtype=torch.float32, device=dev))


def fuse_instances_batched(points3D_table, keypoints_px, cls, count, rig, gate=40.0, reproj_thresh=8.0, keypoint_sigma=2.0, max_iter=20):
    """Fuse every detected instance across the cameras of a rig on the GPU (ssp_fuse_instances, rule:
    csrc/multiview_instances_core.h).  points3D_table (num_classes, P, 3): the PnP points of each class id, 7 <= P <= 10;
    keypoints_px (B, M, P, 2) raw pixels, cls (B, M) int class ids and count (B,) int: row b = g C + c is camera c's detections of
    capture g (B a multiple of C), slot m < count[b] a detection (InstancePosePredictor's count, cls and keypoints_px).  Every
    detection gets its own cold PnP with its camera; each detection's pose in the world frame is a hypothesis; in each view the
    closest detection of its class within `gate` px joins, the set is fused by LM, then again with the detections within
    `reproj_thresh` px of that fit; the best-supported hypothesis becomes a world instance, its detections leave, and so on.
    -> dict of CUDA tensors: per row R (B, M, 3, 3), t (B, M, 3), corners_px (B, M, P, 2) (the per-row solve, zeros in empty slots),
    world_index (B, M) (the world slot each detection joined, -1 for none), corners_world_px (B, M, P, 2) (world instance m of the
    row's capture in the row's camera, zeros past world_count); per capture world_count (G,), unfused (G,) (detections in no world
    instance), world_cls (G, M) (-1 for an empty slot), R_world (G, M, 3, 3), t_world (G, M, 3) world-from-object, world_cov
    (G, M, 6, 6), members (G, M, C) (view c's fused slot, -1 for none), view_err (G, M, C) (RMS px of the members, -1 for the
    others), fuse_hyp (G, M) (the winning detection c M + m, -1 for an empty slot), fuse_status (G, M) (FUSE_STATUS bits)."""
    gate, thr, sigma = check_fuse_args(gate, reproj_thresh, keypoint_sigma)
    if not isinstance(rig, CameraRig):
        raise SspError("rig must be a CameraRig (utils.camera_rig)")
    dev = _dev()
    t32 = lambda a, dt: (a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))).to(dev, dt).contiguous()
    uv, table = t32(keypoints_px, torch.float32), t32(points3D_table, torch.float32)
    cls, count = t32(cls, torch.int32), t32(count, torch.int32)
    if uv.dim() != 4 or uv.shape[-1] != 2:
        raise SspError("keypoints_px must be (B, M, P, 2), got %s" % (tuple(uv.shape),))
    B, M, npts = uv.shape[:3]
    if table.dim() != 3 or table.shape[1:] != (npts, 3):
        raise SspError("points3D_table %s does not match keypoints_px %s: (num_classes, P, 3)" % (tuple(table.shape), tuple(uv.shape)))
    if tuple(cls.shape) != (B, M) or tuple(count.shape) != (B,):
        raise SspError("cls must be (B, M) and count (B,) for keypoints_px %s, got %s and %s" % (tuple(uv.shape), tuple(cls.shape), tuple(count.shape)))
    C = len(rig.K)
    if B % C:
        raise SspError("%d rows are not whole captures of the rig's %d cameras" % (B, C))
    K32, K64, D, Rr, tr = rig_tensors(rig, dev)
    o = fuse_instances_outputs(B, C, M, npts, dev)
    work = torch.empty(max(fuse_instances_work_bytes(B // C, C, M), 8) // 8, dtype=torch.float64, device=dev)
    call("ssp_fuse_instances", ptr(table), table.shape[0], ptr(uv), ptr(cls), ptr(count), npts, B // C, C, M, ptr(K32), ptr(K64), ptr(D), ptr(Rr),
         ptr(tr), gate, thr, sigma, max_iter, *(ptr(v) for v in o.values()), ptr(work), work.numel() * 8, stream_ptr())
    return o


CALIB_STATUS = {"unconnected": 1, "singular": 2}                       # ssp_calibrate_rig's camera status bits (SSP_CALIB_*)


def calibrate_work_bytes(groups, views, slots):
    """bytes of device workspace ssp_calibrate_rig needs"""
    import ctypes
    out = ctypes.c_longlong(0)
    call("ssp_calibrate_rig_work_bytes", int(groups), int(views), int(slots), ctypes.byref(out))
    return out.value


def check_calibrate_args(K, dist, reference, gate, reproj_thresh, keypoint_sigma, max_iter):
    """-> (K (C, 3, 3) float64, dist (C, 8) float64 or None, reference, gate, reproj_thresh, keypoint_sigma, max_iter), checked as
    camera_rig checks the intrinsics and as ssp_calibrate_rig checks the rest; SspError otherwise"""
    K = np.asarray(K, np.float64)
    if K.ndim != 3:
        raise SspError("K must be (C, 3, 3), one per camera, got %s" % (K.shape,))
    C = len(K)
    rig = camera_rig(K, np.repeat(np.eye(3)[None], max(C, 0), 0), np.zeros((C, 3)), dist)      # the intrinsics' and dist's checks
    gate, thr, sigma = check_fuse_args(gate, reproj_thresh, keypoint_sigma)
    if not isinstance(reference, (int, np.integer)) or not 0 <= reference < C:
        raise SspError("the reference camera must be one of 0..%d, got %r" % (C - 1, reference))
    if not isinstance(max_iter, (int, np.integer)) or max_iter < 1:
        raise SspError("max_iter must be an integer >= 1, got %r" % (max_iter,))
    return rig.K, rig.dist, int(reference), gate, thr, sigma, int(max_iter)


def calibrate_rig_batched(points_3D, keypoints_px, K, dist=None, valid=None, reference=0, gate=40.0, reproj_thresh=8.0, keypoint_sigma=2.0,
                          max_iter=30):
    """Calibrate the extrinsics of a rig of C cameras from the object they see, on the GPU (ssp_calibrate_rig, rule:
    csrc/calibrate_rig_core.h).  K (C, 3, 3) each camera's intrinsics, dist as camera_rig takes it; keypoints_px (B, P, 2) or
    (B, S, P, 2) raw pixels, row b = g C + c camera c's view of capture g; points_3D (P, 3) shared or one set per row (and slot);
    valid (B,) or (B, S) bool, default all.  Each camera pair's relative pose comes from the consensus of its co-observations, a
    maximum spanning tree rooted at camera `reference` gives the initial rig (its world frame is the reference camera's: R = I,
    t = 0), and rounds of ssp_fuse_views' fusion and a bundle adjustment of the extrinsics and the fused world poses refine it.
    -> dict: per camera R (C, 3, 3), t (C, 3) camera-from-world, cam_cov (C, 6, 6) (keypoint_sigma^2 times the marginal covariance
    of (dth, dt_), the left perturbation in the camera frame), cam_obs (C,) (fused observations the camera is in), cam_rmse (C,)
    (RMS px of those views), tree_parent (C,), edge_agree (C,), cam_status (C,) (CALIB_STATUS bits); per observation R_world
    (G[, S], 3, 3), t_world (G[, S], 3), views (G[, S], C) bool, view_err (G[, S], C), linked (G[, S]) bool; per row R_rows, t_rows (the
    per-view solve); rounds, iterations, cost; and rig, a CameraRig for PosePredictor(rig=...), or None when a camera is
    unconnected.  Arrays are CUDA tensors, rig numpy."""
    K, D, reference, gate, thr, sigma, max_iter = check_calibrate_args(K, dist, reference, gate, reproj_thresh, keypoint_sigma, max_iter)
    dev = _dev()
    uv = torch.as_tensor(np.asarray(keypoints_px, np.float32) if not torch.is_tensor(keypoints_px) else keypoints_px).to(dev, torch.float32)
    slotted = uv.dim() == 4
    uv = (uv if slotted else uv.unsqueeze(1)).contiguous()
    if uv.dim() != 4 or uv.shape[-1] != 2:
        raise SspError("keypoints_px must be (B, P, 2) or (B, S, P, 2), got %s" % (tuple(uv.shape),))
    B, S, npts = uv.shape[:3]
    C = len(K)
    if B % C:
        raise SspError("%d rows are not whole captures of the rig's %d cameras" % (B, C))
    P3 = torch.as_tensor(np.asarray(points_3D, np.float32) if not torch.is_tensor(points_3D) else points_3D).to(dev, torch.float32).contiguous()
    shared = P3.dim() == 2
    if P3.shape[-2:] != (npts, 3) or (not shared and P3.numel() != B * S * npts * 3):
        raise SspError("points_3D %s does not match keypoints_px %s" % (tuple(P3.shape), tuple(uv.shape)))
    ok = torch.ones(B, S, dtype=torch.bool, device=dev) if valid is None else torch.as_tensor(valid).to(dev, torch.bool).reshape(B, S).contiguous()
    to = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    K32, K64, Dt = to(K, np.float32), to(K, np.float64), None if D is None else to(D, np.float64)
    G = B // C
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device=dev)
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=dev)
    o = dict(R_rows=f64(B, S, 3, 3), t_rows=f64(B, S, 3), R=f64(C, 3, 3), t=f64(C, 3), cam_cov=f64(C, 6, 6), cam_obs=i32(C), cam_rmse=f64(C),
             tree_parent=i32(C), edge_agree=i32(C), cam_status=i32(C), R_world=f64(G, S, 3, 3), t_world=f64(G, S, 3),
             views=torch.empty(G, S, C, dtype=torch.bool, device=dev), view_err=f64(G, S, C),
             linked=torch.empty(G, S, dtype=torch.bool, device=dev), rounds=i32(1), iterations=i32(1), cost=f64(1))
    work = f64(max(calibrate_work_bytes(G, C, S), 8) // 8)
    call("ssp_calibrate_rig", ptr(P3), 1 if shared else 0, ptr(uv), ptr(ok), npts, G, C, S, ptr(K32), ptr(K64), ptr(Dt), reference, gate, thr,
         sigma, max_iter, *(ptr(v) for v in o.values()), ptr(work), work.numel() * 8, stream_ptr())
    if not slotted:
        for k in ("R_rows", "t_rows", "R_world", "t_world", "views", "view_err", "linked"):
            o[k] = o[k][:, 0]
    for k in ("rounds", "iterations"):
        o[k] = int(o[k][0])
    o["cost"] = float(o["cost"][0])
    status = o["cam_status"].cpu().numpy()
    o["rig"] = None if (status & CALIB_STATUS["unconnected"]).any() else camera_rig(K, o["R"].cpu().numpy(), o["t"].cpu().numpy(), D)
    return o


# ------------------------------------------------------------------------------------------ training-set creation
RENDER_CHUNK_BYTES = 1 << 30           # device scratch of one ssp_render_masks launch; larger batches go in chunks


def render_masks(vertices, faces, Rt, K, width, height):
    """Silhouette masks of a mesh under n poses, as LINEMOD's mask/*.png: (n, H, W) uint8 CUDA tensor, 255 where the pixel
    centre (x, y) lies inside the projected mesh, and (n,) int32 status (bit 0 a vertex behind the camera, bit 1 a projected
    coordinate outside +-2^20 px, bit 2 a bad face index; such a pose's mask is all zeros).  The vertices are projected by
    ssp_project_points, the kernel of project_points_batched, so masks and label rows agree.  The exact rule is in
    csrc/render_core.h.  vertices (Nv, 3) or (3|4, Nv); faces (Nf, 3) int; Rt (n, 3, 4); K (3, 3)."""
    dev = _dev()
    V = torch.as_tensor(np.asarray(vertices) if not torch.is_tensor(vertices) else vertices)
    if V.dim() != 2 or not (V.shape[0] in (3, 4) or V.shape[1] == 3):
        raise SspError("vertices must be (3|4, Nv) or (Nv, 3), got %s" % (tuple(V.shape),))
    X = (V if V.shape[0] in (3, 4) else V.t()).to(dev, torch.float32).contiguous()
    F = torch.as_tensor(np.asarray(faces) if not torch.is_tensor(faces) else faces).to(dev, torch.int32).contiguous()
    if F.dim() != 2 or F.shape[1] != 3:
        raise SspError("faces must be (Nf, 3), got %s" % (tuple(F.shape),))
    T = _pose_stack(Rt, dev)
    Kd = torch.as_tensor(np.asarray(K) if not torch.is_tensor(K) else K).to(dev, torch.float64).contiguous()
    n, nv, nf, W, H = T.shape[0], X.shape[1], F.shape[0], int(width), int(height)
    masks = torch.empty(n, H, W, dtype=torch.uint8, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    lib = load()
    per_pose = int(lib.ssp_render_work_bytes(nv, nf, 1, W, H))
    if per_pose < 0:
        raise SspError("ssp_render_work_bytes: bad size (Nv = %d, Nf = %d, %d x %d)" % (nv, nf, W, H))
    chunk = max(1, RENDER_CHUNK_BYTES // per_pose)
    work = None
    for p0 in range(0, n, chunk):
        m = min(chunk, n - p0)
        wb = int(lib.ssp_render_work_bytes(nv, nf, m, W, H))
        if work is None:
            work = torch.empty(wb, dtype=torch.uint8, device=dev)
        call("ssp_render_masks", ptr(X), X.shape[0], nv, ptr(F), nf, ptr(T[p0:p0 + m]), ptr(Kd), m, W, H, ptr(masks[p0:p0 + m]),
             ptr(status[p0:p0 + m]), ptr(work), work.numel(), stream_ptr())
    return masks, status


def pose_label_rows(corners3D, Rt, K, width, height, class_id=0):
    """(n, 21) float64 label rows of label_file_creation.md for n poses: the class, the projected model origin [0, 0, 0] and
    the 8 corners (corners3D (3|4, 8), get_3D_corners' order) over the image size, then the x and y ranges of the 8 projected
    corners over the image size.  The projection is project_points_batched's; the row rule is label_rows_from_projection."""
    C3 = np.asarray(corners3D, dtype=np.float64)[:3]
    if C3.shape != (3, 8):
        raise SspError("corners3D must be (3|4, 8), got %s" % (C3.shape,))
    P9 = np.concatenate([np.zeros((3, 1)), C3], 1)
    px = project_points_batched(P9, Rt, K).cpu().numpy()
    return label_rows_from_projection(px, width, height, class_id)


# ------------------------------------------------------------------------------------------ batched evaluation tail
def pnp_truth_and_prediction(P3, uv, K, pnp, reproj_thresh, dist_coeffs=None):
    """The poses of n ground truths uv[:n] and n predictions uv[n:] (uv (2n, P, 2)) -> R (2n, 3, 3), t (2n, 3) fp64 and the
    predictions' inliers (n, P) and hyp (n,) for pnp="consensus" ({} for "plain").  The ground truth is always the plain solve;
    "plain" solves all 2n problems in one launch.  dist_coeffs: both solves with these distortion coefficients (pnp_batched)."""
    dev, n = uv.device, len(uv) // 2
    if n == 0:                                  # nothing to launch: the PnP entry points take no empty (null) buffers
        R, t = torch.zeros(0, 3, 3, dtype=torch.float64, device=dev), torch.zeros(0, 3, dtype=torch.float64, device=dev)
        if pnp != "consensus":
            return R, t, {}
        return R, t, dict(inliers=torch.zeros(0, uv.shape[1], dtype=torch.bool, device=dev), hyp=torch.zeros(0, dtype=torch.int32, device=dev))
    if pnp != "consensus":
        R, t = pnp_batched(P3, uv, K, dist_coeffs=dist_coeffs)
        return R, t, {}
    R_gt, t_gt = pnp_batched(P3, uv[:n], K, dist_coeffs=dist_coeffs)
    R_pr, t_pr, _p, inl, hyp = pnp_consensus_batched(P3, uv[n:], K, reproj_thresh, dist_coeffs=dist_coeffs)
    return torch.cat([R_gt, R_pr]), torch.cat([t_gt, t_pr]), dict(inliers=inl, hyp=hyp)


def evaluate_poses_batched(output, target, vertices, points_3D, internal_calibration, num_classes=1, num_keypoints=9,
                           im_width=640, im_height=480, adds=False, pnp="plain", reproj_thresh=8.0, dist_coeffs=None):
    """GPU-resident version of the per-image evaluation loop of reference valid.py:123-183 (SURVEY 8f.1): per-image decode
    (arg-max cell of EACH image, not the whole batch), PnP of the ground-truth and the predicted keypoints, reprojection of
    all mesh vertices, pixel / 3-D / angular / translation errors -- no Python loop over images.

    output (B, 2K+1+C, h, w) CUDA; target (B, >= 2K+1) rows [cls, x0, y0, ..., x8, y8, ...] (first object);
    vertices (3|4, Nv); points_3D (K, 3); internal_calibration (3, 3).  Returns a dict of CUDA tensors with leading dim B.
    adds=True adds `adds_dist` (B,) fp64, adi(pts_pr, pts_gt) over the mesh as given in fp64 (adi_batched): the error that
    replaces vertex_dist for the symmetric objects (eggbox, glue).  The angle error is arccos of the trace clamped to [-1, 1],
    so an exact pose gives 0 where the reference's calcAngularDistance can give NaN.
    pnp="consensus" solves the predicted pose with the consensus PnP (pnp_consensus_batched, inliers within reproj_thresh pixels of
    the im_width x im_height image) and adds `inliers` (B, K) bool and `hyp` (B,) int32; the ground-truth pose stays the plain
    solve.  Passing the results of both modes of one network output to pose_accuracy compares the two solves.
    dist_coeffs: OpenCV distortion coefficients of the camera (camera_distortion): the ground-truth and the predicted poses are both
    solved with them, as valid.py does when pnp.distCoeffs is set; the pixel and vertex errors stay the undistorted projection
    (compute_projection), which is also what valid.py computes then."""
    pnp, reproj_thresh = check_pnp_args(pnp, reproj_thresh)
    camera_distortion(dist_coeffs)
    dev = output.device
    K = num_keypoints
    boxes, best, _ = region_boxes_batched(output, num_classes, K)
    B = boxes.shape[0]
    scale = torch.tensor([im_width, im_height], dtype=torch.float32, device=dev)
    pr2d = boxes[:, :2 * K].reshape(B, K, 2) * scale
    gt2d = torch.as_tensor(target)[:, 1:1 + 2 * K].to(dev, torch.float32).reshape(B, K, 2) * scale
    Kc = torch.as_tensor(np.asarray(internal_calibration, dtype=np.float32)).to(dev)
    P3 = torch.as_tensor(np.asarray(points_3D, dtype=np.float32)).to(dev)
    R, t, extra = pnp_truth_and_prediction(P3, torch.cat([gt2d, pr2d], 0), Kc, pnp, reproj_thresh, dist_coeffs)
    R_gt, R_pr, t_gt, t_pr = R[:B], R[B:], t[:B], t[B:]
    Rt_gt = torch.cat([R_gt, t_gt.unsqueeze(2)], 2)
    Rt_pr = torch.cat([R_pr, t_pr.unsqueeze(2)], 2)
    V = torch.as_tensor(np.asarray(vertices, dtype=np.float32)).to(dev)
    if V.shape[0] == 3:
        V = torch.cat([V, torch.ones(1, V.shape[1], device=dev)], 0)
    Kd = Kc.double()
    proj = project_points_batched(V, torch.cat([Rt_gt, Rt_pr], 0), Kd)  # (2B, 2, Nv)
    pixel_err = (proj[:B] - proj[B:]).norm(dim=1).mean(dim=1)           # valid.py:169-171 mean 2-D vertex reprojection distance
    Vd = V.double()
    tf_gt, tf_pr = Rt_gt @ Vd, Rt_pr @ Vd                               # compute_transformation
    vertex_dist = (tf_gt - tf_pr).norm(dim=1).mean(dim=1)               # valid.py:176-178
    tr = torch.einsum("bij,bij->b", R_gt, R_pr)                         # trace(R_gt R_pr^T)
    angle = torch.rad2deg(torch.arccos(((tr - 1.0) / 2.0).clamp(-1.0, 1.0)))
    res = dict(boxes=boxes, conf=best, corner_err_px=(pr2d - gt2d).norm(dim=2).mean(dim=1), R_gt=R_gt, t_gt=t_gt, R_pr=R_pr, t_pr=t_pr,
               pixel_err=pixel_err, vertex_dist=vertex_dist, angle_err_deg=angle, trans_err=(t_gt - t_pr).norm(dim=1), **extra)
    if adds:
        res["adds_dist"] = adi_batched(vertices, Rt_pr, Rt_gt)
    return res


def _host_array(results, key):
    v = [r[key] for r in results]
    v = [x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x) for x in v]
    return np.concatenate([x.reshape(-1) for x in v]) if v else np.zeros(0)


def pose_accuracy(results, diam, px_threshold=5):
    """The summary of valid.py:202-229 from one result dict of evaluate_poses_batched or a list of them (accumulated in order),
    with the reference's formulas: a rate is len(where(err <= threshold)) * 100 / (n + 1e-5), a mean error is np.mean over the
    per-image values, and the translation / angle / pixel errors are the running sums over the images divided by n.
    -> dict: acc (2-D projection error <= px_threshold px), acc3d10 (vertex_dist, ADD, <= 10 % of diam), acc5cm5deg,
    corner_acc (mean corner error <= px_threshold px), mean_err_2d, mean_vertex_err, mean_corner_err_2d, mean_trans_err,
    mean_angle_err, mean_pixel_err, and acc_adds10 (adds_dist <= 10 % of diam) when the results hold adds_dist.

    diam is the object's diameter in the mesh's units: valid.py takes it from calc_pts_diameter of the mesh (mesh_diameter
    gives the same value on the GPU), train.py:296 from the `diam` entry of the .data file.  The batched tail clamps the
    angle's cosine to [-1, 1], so an exact pose counts as 0 degrees; the reference's calcAngularDistance can return NaN there,
    which fails the 5 degree test."""
    if isinstance(results, dict):
        results = [results]
    eps = 1e-5
    e2d, e3d, ecorner = (_host_array(results, k) for k in ("pixel_err", "vertex_dist", "corner_err_px"))
    etrans, eangle = _host_array(results, "trans_err"), _host_array(results, "angle_err_deg")
    n = len(e2d)
    rate = lambda ok: len(np.where(ok)[0]) * 100. / (n + eps)
    total = lambda errs: sum(errs, 0.0)                   # valid.py:180-182: += per image, in order, from 0.0
    out = dict(acc=rate(e2d <= px_threshold), acc3d10=rate(e3d <= diam * 0.1), acc5cm5deg=rate((etrans <= 0.05) & (eangle <= 5)),
               corner_acc=rate(ecorner <= px_threshold), mean_err_2d=np.mean(e2d), mean_vertex_err=np.mean(e3d),
               mean_corner_err_2d=np.mean(ecorner), mean_trans_err=total(etrans) / float(n), mean_angle_err=total(eangle) / float(n),
               mean_pixel_err=total(e2d) / float(n))
    if all("adds_dist" in r for r in results):
        out["acc_adds10"] = rate(_host_array(results, "adds_dist") <= diam * 0.1)
    return out
