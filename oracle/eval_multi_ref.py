"""Oracle: one batch-1 iteration of the reference's multi-object evaluation loop, multi_obj_pose_estimation/valid_multi.py:97-149,
restated on the CPU.

TEST INFRASTRUCTURE ONLY (checker for utils_multi.evaluate_multi_poses_batched, SURVEY 8f.6).  Built on the reference-pinned
oracles: `get_multi_region_boxes_ref` (utils_multi.py:266-382, tests/golden/decode_multi.npz) for the box list, `pnp_ref`
(cv2.solvePnP, tests/golden/pnp*.npz) for the poses and the numpy `compute_projection` of oracle/eval_ref.py.  The loop itself is
pinned by tests/golden/eval_multi.npz, made by running valid_multi.valid() unmodified.  Kept as the reference has it: the
selection `boxes[j][2K] > best_conf_est and boxes[j][2K+2] == int(truths[k][0])` starting from -sys.maxsize (the first maximum
wins), and `box_pr` carried over from the previous ground truth when no box has the class.
"""
from __future__ import annotations

import sys

import numpy as np
import torch

from .decode_multi_ref import get_multi_region_boxes_ref
from .eval_ref import compute_projection
from .pnp_ref import pnp_ref

_FIX = (0, 1, 3, 5, 7, 2, 4, 6, 8)


def fix_corner_order(c):
    """utils_multi.py:244-255"""
    out = np.zeros((9, 2), dtype="float32")
    for dst, src in enumerate(_FIX):
        out[dst, :] = c[src, :]
    return out


def truths_length(truths):
    """valid_multi.py:20-23 (returns None when all 50 rows are filled, as the reference does)"""
    for i in range(50):
        if truths[i][1] == 0:
            return i


def select_ref(boxes, truths, num_keypoints):
    """valid_multi.py:110-123 on one image's box list -> per ground truth (list position j, carried over?).  `boxes` as
    get_multi_region_boxes returns them; truths (rows, 2K+3)."""
    K2 = 2 * num_keypoints
    picks = []
    j_pr = None
    for k in range(truths_length(truths)):
        best_conf_est = -sys.maxsize
        carried = True
        for j in range(len(boxes)):
            if (boxes[j][K2] > best_conf_est) and (boxes[j][K2 + 2] == int(truths[k][0])):
                best_conf_est = boxes[j][K2]
                j_pr = j
                carried = False
        picks.append((j_pr, carried))
    return picks


def evaluate_image_multi_ref(output_1, target_1, conf_thresh, num_classes, num_keypoints, anchors, num_anchors, vertices, corners3D,
                             intrinsic_calibration, im_width=640, im_height=480, with_pose=True):
    """One iteration of valid_multi.py:97-149 with batch size 1: output_1 (1, (2K+1+C)*A, H, W) CPU tensor, target_1 the image's
    (50*(2K+3),) label -> list (per ground truth) of dicts: pos (index in the box list), carried, fallback (the box is the
    appended fallback box), box (2K+3 fp32), uv_gt / uv_pr (the fp32 points passed to pnp) and, with_pose, R_gt, t_gt, R_pr,
    t_pr, pixel_err; plus the box list itself."""
    K = num_keypoints
    nl = 2 * K + 3
    truths = target_1.reshape(-1, nl)
    boxes = get_multi_region_boxes_ref(output_1, conf_thresh, num_classes, K, anchors, num_anchors, int(truths[0][0]),
                                       only_objectness=0)[0]
    n_listed = _count_listed(output_1, conf_thresh, num_classes, K, num_anchors)
    if with_pose:
        objpoints3D = np.array(np.transpose(np.concatenate((np.zeros((3, 1)), np.asarray(corners3D)[:3, :]), axis=1)), dtype="float32")
        Kf = np.array(intrinsic_calibration, dtype="float32")
    res = []
    for k, (j, carried) in enumerate(select_ref(boxes, truths, K)):
        box_gt = [truths[k][i] for i in range(1, nl)]
        box_pr = boxes[j]
        c_gt = np.array(np.reshape([float(v) for v in box_gt[:2 * K]], [-1, 2]), dtype="float32")
        c_pr = np.array(np.reshape([float(v) for v in box_pr[:2 * K]], [-1, 2]), dtype="float32")
        c_gt[:, 0] = c_gt[:, 0] * im_width
        c_gt[:, 1] = c_gt[:, 1] * im_height
        c_pr[:, 0] = c_pr[:, 0] * im_width
        c_pr[:, 1] = c_pr[:, 1] * im_height
        c_gt = fix_corner_order(c_gt)
        r = dict(pos=j, carried=carried, fallback=j >= n_listed, box=np.array([float(v) for v in box_pr], np.float32),
                 uv_gt=c_gt, uv_pr=c_pr)
        if with_pose:
            R_gt, t_gt = pnp_ref(objpoints3D, c_gt, Kf)
            R_pr, t_pr = pnp_ref(objpoints3D, c_pr, Kf)
            r.update(R_gt=R_gt, t_gt=t_gt, R_pr=R_pr, t_pr=t_pr, pixel_err=pixel_error(vertices, R_gt, t_gt, R_pr, t_pr, intrinsic_calibration))
        res.append(r)
    return res, boxes


def _count_listed(output_1, conf_thresh, num_classes, num_keypoints, num_anchors):
    """the boxes get_multi_region_boxes lists before its fallback: det_conf * cls_max_conf > conf_thresh (utils_multi.py:293-332)"""
    h, w, K = output_1.size(2), output_1.size(3), num_keypoints
    out = output_1.reshape(num_anchors, 2 * K + 1 + num_classes, h * w).transpose(0, 1).reshape(2 * K + 1 + num_classes, -1)
    det = torch.sigmoid(out[2 * K])
    cls_max = torch.softmax(out[2 * K + 1:].transpose(0, 1), dim=1).max(1)[0]
    return int((det * cls_max > conf_thresh).sum())


def pixel_error(vertices, R_gt, t_gt, R_pr, t_pr, intrinsic_calibration):
    """valid_multi.py:141-148"""
    Rt_gt = np.concatenate((R_gt, t_gt), axis=1)
    Rt_pr = np.concatenate((R_pr, t_pr), axis=1)
    Kd = np.asarray(intrinsic_calibration, np.float64)
    proj_2d_gt = compute_projection(vertices, Rt_gt, Kd)
    proj_2d_pred = compute_projection(vertices, Rt_pr, Kd)
    return np.mean(np.linalg.norm(proj_2d_gt - proj_2d_pred, axis=0))


def projection_accuracy_ref(errs_2d, thresholds=(5, 10, 15, 20, 25, 30, 35, 40, 45, 50)):
    """valid_multi.py:154-156"""
    eps = 1e-5
    return [len(np.where(np.array(errs_2d) <= px)[0]) * 100. / (len(errs_2d) + eps) for px in thresholds]
