"""Multi-object decode -- drop-in for ``get_multi_region_boxes`` of reference multi_obj_pose_estimation/utils_multi.py:266-382.
The dense per-(cell, anchor) arithmetic and the reference's sequential fallback maxima run on the GPU; the host only
applies the confidence mask (one device->host copy).  The pose helpers are shared with utils.py."""
from __future__ import annotations

import ctypes as _ctypes

import numpy as np
import torch

from ._lib import call, ptr, stream_ptr, SspError
from .utils import (pnp, pnp_batched, compute_projection, compute_transformation, calcAngularDistance, get_3D_corners,  # noqa: F401
                    get_camera_intrinsic, convert2cpu, convert2cpu_long, project_points_batched, adi_batched, mesh_diameter)
from .utils_host import (makedirs, get_all_files, calc_pts_diameter, adi, get_2d_bb, corner_confidences, corner_confidence,  # noqa: F401
                         sigmoid, softmax, read_truths, read_truths_args, read_pose, load_class_names, image2torch, scale_bboxes,
                         file_lines, get_image_size, logging)
from . import utils_host as _host


def read_data_cfg(datacfg):
    """utils_multi.py:428-443: as utils.read_data_cfg, but 'gpus' defaults to '0,1,2,3'"""
    options = _host.read_data_cfg(datacfg)
    with open(datacfg, 'r') as fp:
        if not any(line.split('=')[0].strip() == 'gpus' for line in fp if '=' in line):
            options['gpus'] = '0,1,2,3'
    return options


def bbox_iou(box1, box2, x1y1x2y2=False):
    """utils_multi.py:125-156: IoU of two boxes given as corners (x1y1x2y2) or as centre + size; 0.0 when they do not overlap"""
    if x1y1x2y2:
        l1, t1, r1, b1 = box1[0], box1[1], box1[2], box1[3]
        l2, t2, r2, b2 = box2[0], box2[1], box2[2], box2[3]
        w1, h1, w2, h2 = r1 - l1, b1 - t1, r2 - l2, b2 - t2
    else:
        w1, h1, w2, h2 = box1[2], box1[3], box2[2], box2[3]
        l1, r1, t1, b1 = box1[0] - w1 / 2.0, box1[0] + w1 / 2.0, box1[1] - h1 / 2.0, box1[1] + h1 / 2.0
        l2, r2, t2, b2 = box2[0] - w2 / 2.0, box2[0] + w2 / 2.0, box2[1] - h2 / 2.0, box2[1] + h2 / 2.0
    cw = w1 + w2 - (max(r1, r2) - min(l1, l2))          # overlap = sum of the sizes minus the extent of the union box
    ch = h1 + h2 - (max(b1, b2) - min(t1, t2))
    if cw <= 0 or ch <= 0:
        return 0.0
    carea = cw * ch
    return carea / (w1 * h1 + w2 * h2 - carea)


def nms(boxes, nms_thresh):
    """utils_multi.py:223-241: greedy suppression in decreasing box[4] order; suppressed boxes get box[4] = 0 IN PLACE (like the
    reference) and are left out of the returned list"""
    if len(boxes) == 0:
        return boxes
    keys = torch.zeros(len(boxes))
    for i in range(len(boxes)):
        keys[i] = 1 - boxes[i][4]
    _, order = torch.sort(keys)
    kept = []
    for i in range(len(boxes)):
        bi = boxes[order[i]]
        if bi[4] > 0:
            kept.append(bi)
            for j in range(i + 1, len(boxes)):
                bj = boxes[order[j]]
                if bbox_iou(bi, bj, x1y1x2y2=False) > nms_thresh:
                    bj[4] = 0
    return kept


def fix_corner_order(corners2D_gt):
    """utils_multi.py:244-255"""
    import numpy as np
    out = np.zeros((9, 2), dtype="float32")
    for dst, src in enumerate((0, 1, 3, 5, 7, 2, 4, 6, 8)):
        out[dst, :] = corners2D_gt[src, :]
    return out


def multi_region_dense(output, num_classes, num_keypoints, num_anchors, correspondingclass, only_objectness=1):
    """-> dict of CUDA tensors in the reference's visiting order (cell-major, anchor fastest):
    boxes (B, HW*A, 2K+3), conf (B, HW*A), max_ind (B,), max_conf (B,), max_cls (B,)."""
    if output.dim() == 3:
        output = output.unsqueeze(0)
    if not output.is_cuda:
        raise SspError("get_multi_region_boxes runs on CUDA tensors only")
    out = output.detach().contiguous().float()
    B, C, H, W = out.shape
    K, nC, nA = num_keypoints, num_classes, num_anchors
    assert C == (2 * K + 1 + nC) * nA
    n = H * W * nA
    dev = out.device
    boxes = torch.empty(B, n, 2 * K + 3, dtype=torch.float32, device=dev)
    conf = torch.empty(B, n, dtype=torch.float32, device=dev)
    det = torch.empty(B, n, dtype=torch.float32, device=dev)
    clsc = torch.empty(B, n, dtype=torch.float32, device=dev)
    max_ind = torch.empty(B, dtype=torch.int64, device=dev)
    max_conf = torch.empty(B, dtype=torch.float32, device=dev)
    max_cls = torch.empty(B, dtype=torch.float32, device=dev)
    call("ssp_region_decode_multi", ptr(out), B, K, nC, nA, H, W, int(bool(only_objectness)), int(correspondingclass), ptr(boxes),
         ptr(conf), ptr(det), ptr(clsc), ptr(max_ind), ptr(max_conf), ptr(max_cls), stream_ptr())
    return dict(boxes=boxes, conf=conf, max_ind=max_ind, max_conf=max_conf, max_cls=max_cls)


def get_multi_region_boxes(output, conf_thresh, num_classes, num_keypoints, anchors, num_anchors, correspondingclass,
                           only_objectness=1, validation=False):
    """Reference contract: list (per image) of lists of boxes [x0/w, y0/h, ..., det_conf, cls_max_conf, cls_max_id]."""
    if validation and not only_objectness:
        raise NotImplementedError("validation=True appends per-class extras; valid_multi.py does not use it")
    d = multi_region_dense(output, num_classes, num_keypoints, num_anchors, correspondingclass, only_objectness)
    K = num_keypoints
    boxes, conf = d["boxes"].cpu(), d["conf"].cpu()
    max_ind, max_conf, max_cls = d["max_ind"].cpu(), d["max_conf"].cpu(), d["max_cls"].cpu()
    flat = boxes.view(-1, 2 * K + 3)
    all_boxes = []
    for b in range(boxes.size(0)):
        sel = boxes[b][conf[b] > conf_thresh]
        cur = [[float(v) for v in row[:2 * K + 2]] + [int(row[2 * K + 2])] for row in sel]
        if len(cur) == 0 or correspondingclass not in [bx[2 * K + 2] for bx in cur]:
            src = flat[int(max_ind[b])]
            cur.append([float(v) for v in src[:2 * K]] + [float(max_conf[b]), float(max_cls[b]), int(correspondingclass)])
        all_boxes.append(cur)
    return all_boxes


def detect_instances(output, conf_thresh, nms_thresh, num_classes, num_keypoints, num_anchors, frame_size, classes=None,
                     max_instances=32):
    """Every instance of the requested classes in each image of a CUDA network output (B, (2K+1+C)*A, H, W): one
    ssp_detect_instances launch (rules: csrc/detect_core.h).  Candidates are the boxes get_multi_region_boxes(...,
    only_objectness=0) lists (det_conf * cls_max_conf > conf_thresh, never its fallback box) whose arg-max class is in `classes`
    (default: all); they are ranked by det_conf (the earlier box on ties) and a candidate is dropped when the rectangle of its 8
    corner keypoints in frame pixels has IoU > nms_thresh with a kept box of its own class.  The reference's nms, written for YOLO
    boxes, is not reproduced.  frame_size = (width, height) the keypoints are scaled to.

    Returns padded device tensors: count (B,) int32 = min(kept, max_instances), kept (B,) = boxes kept before the truncation,
    cls (B, M) int32 (-1 in empty slots), conf (B, M) det_conf, cls_conf (B, M), keypoints_px (B, M, K, 2); empty slots are zero."""
    if output.dim() == 3:
        output = output.unsqueeze(0)
    if not output.is_cuda:
        raise SspError("detect_instances runs on CUDA tensors only")
    out = output.detach().contiguous().float()
    B, C, H, W = out.shape
    K, nC, nA, M = int(num_keypoints), int(num_classes), int(num_anchors), int(max_instances)
    if C != (2 * K + 1 + nC) * nA:
        raise SspError("output has %d channels, expected (2K+1+C)*A = %d" % (C, (2 * K + 1 + nC) * nA))
    cls_host = np.ascontiguousarray(range(nC) if classes is None else [int(c) for c in classes], dtype=np.int32)
    dev = out.device
    boxes = torch.empty(B, M, 2 * K + 3, dtype=torch.float32, device=dev)
    cls = torch.empty(B, M, dtype=torch.int32, device=dev)
    uv = torch.empty(B, M, K, 2, dtype=torch.float32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    kept = torch.empty(B, dtype=torch.int32, device=dev)
    call("ssp_detect_instances", ptr(out), B, K, nC, nA, H, W, _ctypes.c_void_p(cls_host.ctypes.data), len(cls_host), float(conf_thresh),
         float(nms_thresh), M, float(frame_size[0]), float(frame_size[1]), ptr(boxes), ptr(cls), ptr(uv), ptr(count), ptr(kept),
         stream_ptr())
    return dict(count=count, kept=kept, cls=cls, conf=boxes[..., 2 * K], cls_conf=boxes[..., 2 * K + 1], keypoints_px=uv)


# ------------------------------------------------------------------------------------------ batched evaluation tail
ACCURACY_THRESHOLDS = (5, 10, 15, 20, 25, 30, 35, 40, 45, 50)


def truths_lengths(target, num_keypoints=9, max_num_gt=50):
    """valid_multi.py:20-23 per image of a (B, rows*(2K+3)) label: the rows before the first with x0 == 0 -> int64 numpy (B,).
    A label whose max_num_gt rows are all filled counts them all (the reference's truths_length returns None there)."""
    nl = 2 * num_keypoints + 3
    t = (target.detach().cpu().float().numpy() if torch.is_tensor(target) else np.asarray(target, np.float32))
    t = t.reshape(t.shape[0], -1, nl)[:, :max_num_gt]
    empty = t[:, :, 1] == 0
    return np.where(empty.any(1), empty.argmax(1), t.shape[1]).astype(np.int64)


def projection_accuracy(pixel_err, thresholds=ACCURACY_THRESHOLDS):
    """valid_multi.py:154-158 over the accumulated per-object 2-D projection errors: [% of errors <= px for px in thresholds],
    computed as the reference does, len(where(err <= px)) * 100 / (n + 1e-5)."""
    if torch.is_tensor(pixel_err):
        pixel_err = pixel_err.detach().cpu().numpy()
    err = np.asarray(pixel_err, dtype=np.float64).reshape(-1)
    return [len(np.where(err <= px)[0]) * 100. / (len(err) + 1e-5) for px in thresholds]


def evaluate_multi_poses_batched(output, target, conf_thresh, num_classes, num_keypoints, num_anchors, vertices, corners3D,
                                 internal_calibration, im_width=640, im_height=480, adds=False):
    """GPU version of the multi-object evaluation loop (valid_multi.py:97-149, train_multi.py:196-240) for a whole batch.

    output (B, (2K+1+C)*A, H, W) CUDA network output; target (B, 50*(2K+3)) label of dataset_multi.listDataset in test mode, host
    or device; vertices (3|4, Nv) mesh; corners3D (3|4, 8) from get_3D_corners; internal_calibration (3, 3).

    Per image, exactly as one iteration of the reference's batch-1 loop: the box list of get_multi_region_boxes(output, conf_thresh,
    ..., int(target[0]), only_objectness=0); for each ground truth the first box of its class with the largest det_conf, else the
    previous ground truth's box; PnP of the fix_corner_order'ed ground truth and of the prediction against [0; corners3D]; the
    mean 2-D distance of all vertices projected with both poses.  One launch selects (ssp_eval_multi_select), one PnP launch
    solves all 2G problems, one projects all vertices for the 2G poses.  The object counts come from a host copy of the target
    (one device->host copy when it lives on the device), so nothing waits on the GPU.

    Returns a dict of CUDA tensors with leading dimension G (all ground truths of the batch, image-major): image, gt_index, cls,
    box (the chosen box [x0/w, y0/h, ..., det_conf, cls_conf, cls_id]), fallback and carried (bool), R_gt, t_gt, R_pr, t_pr (fp64),
    pixel_err.  Accumulate pixel_err over batches and pass it to projection_accuracy.  adds=True adds the 3-D errors over the
    mesh as given, in fp64, from one more launch (utils.adi_batched): vertex_dist (ADD, as valid.py:173-177 computes it) and
    adds_dist (ADD-S, adi(pts_pr, pts_gt), for the symmetric eggbox and glue), both (G,) fp64.

    Deliberate departures: with B > 1 every image is evaluated as the reference's own batch-1 call (the reference takes
    correspondingclass from image 0 and keeps its fallback maxima across the batch); a label with all 50 rows filled is evaluated
    in full, where the reference raises TypeError from range(None).  The reference's per-object corner_confidence and projected
    corners are never used by it and are not computed."""
    if output.dim() == 3:
        output = output.unsqueeze(0)
    if not output.is_cuda:
        raise SspError("evaluate_multi_poses_batched runs on CUDA tensors only")
    out = output.detach().contiguous().float()
    dev = out.device
    B, C, H, W = out.shape
    K, nC, nA = num_keypoints, num_classes, num_anchors
    assert C == (2 * K + 1 + nC) * nA
    nl = 2 * K + 3
    tgt = target.detach() if torch.is_tensor(target) else torch.as_tensor(np.asarray(target))
    tgt = tgt.reshape(B, -1)
    if tgt.shape[1] < nl:
        raise SspError("target rows hold %d values, need at least 2K+3 = %d" % (tgt.shape[1], nl))
    counts = truths_lengths(tgt, K)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    G = int(offsets[-1])
    image = torch.from_numpy(np.repeat(np.arange(B), counts)).to(dev)
    gt_index = torch.from_numpy(np.arange(G) - np.repeat(offsets[:-1].astype(np.int64), counts)).to(dev)
    tgt_d = tgt.to(dev, torch.float32).contiguous()
    off_d = torch.from_numpy(offsets).to(dev)
    box = torch.empty(G, nl, dtype=torch.float32, device=dev)
    flags = torch.empty(G, dtype=torch.int32, device=dev)
    uv = torch.empty(2 * G, K, 2, dtype=torch.float32, device=dev)
    if G:
        call("ssp_eval_multi_select", ptr(out), B, K, nC, nA, H, W, ptr(tgt_d), tgt_d.shape[1], ptr(off_d), float(conf_thresh),
             float(im_width), float(im_height), ptr(box), ptr(flags), ptr(uv), stream_ptr())
    rows = tgt_d.shape[1] // nl
    cls = tgt_d[:, :rows * nl].reshape(B, rows, nl)[image, gt_index, 0].long()
    res = dict(image=image, gt_index=gt_index, cls=cls, box=box, fallback=(flags & 1) != 0, carried=(flags & 2) != 0)
    if G == 0:                                                  # nothing to solve: empty poses and errors
        R0 = torch.zeros(0, 3, 3, dtype=torch.float64, device=dev)
        t0 = torch.zeros(0, 3, dtype=torch.float64, device=dev)
        res = dict(res, R_gt=R0, t_gt=t0, R_pr=R0.clone(), t_pr=t0.clone(), pixel_err=torch.zeros(0, dtype=torch.float32, device=dev))
        if adds:
            res.update(vertex_dist=torch.zeros(0, dtype=torch.float64, device=dev), adds_dist=torch.zeros(0, dtype=torch.float64, device=dev))
        return res
    c3 = np.asarray(corners3D, dtype=np.float64)[:3]
    P3 = np.array(np.transpose(np.concatenate((np.zeros((3, 1)), c3), axis=1)), dtype="float32")          # valid_multi.py:135
    Kc = torch.as_tensor(np.asarray(internal_calibration, dtype=np.float32)).to(dev)
    R, t = pnp_batched(torch.from_numpy(P3).to(dev), uv, Kc)                                                 # 2G problems, one launch
    Rt = torch.cat([R, t.unsqueeze(2)], 2)
    V = torch.as_tensor(np.asarray(vertices, dtype=np.float32)).to(dev)
    if V.shape[0] == 3:
        V = torch.cat([V, torch.ones(1, V.shape[1], device=dev)], 0)
    proj = project_points_batched(V, Rt, torch.as_tensor(np.asarray(internal_calibration, dtype=np.float64)).to(dev))   # (2G, 2, Nv)
    d = proj[:G] - proj[G:]
    # valid_multi.py:143-149.  Elementwise distances, then an fp64 mean: the result of one object does not depend on how many
    # objects the batch holds (a batched fp32 reduction may change its summation order with the shape)
    pixel_err = torch.hypot(d[:, 0], d[:, 1]).double().mean(dim=1).float()
    res = dict(res, R_gt=R[:G], t_gt=t[:G], R_pr=R[G:], t_pr=t[G:], pixel_err=pixel_err)
    if adds:
        res["adds_dist"], res["vertex_dist"] = adi_batched(vertices, Rt[G:], Rt[:G], with_add=True)
    return res
