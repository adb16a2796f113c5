"""Oracle of every-instance detection (singleshotpose_b200/csrc/detect_core.h) in numpy.  TEST INFRASTRUCTURE ONLY.

The candidates are the box list of the reference's get_multi_region_boxes(..., only_objectness=0) without its fallback box,
restricted to the requested classes; they are ranked by descending det_conf, the earlier box on ties; greedy suppression within
each class drops a candidate whose corner rectangle (keypoints 1..8 in frame pixels) has IoU > nms_thresh with a kept box of its
class.  The IoU is fp32, each operation rounded on its own, in the order detect_core.h states.  The reference's own nms reads YOLO
boxes and is not used."""
from __future__ import annotations

import numpy as np

from .decode_multi_ref import get_multi_region_boxes_ref

F32 = np.float32


def listing_ref(output, conf_thresh, num_classes, num_keypoints, anchors, num_anchors):
    """per image, the boxes get_multi_region_boxes_ref(..., only_objectness=0) lists before its fallback box.  With
    correspondingclass = -1, which no box has, the fallback is always appended last, so it is the last box of each list."""
    return [boxes[:-1] for boxes in get_multi_region_boxes_ref(output, conf_thresh, num_classes, num_keypoints, anchors, num_anchors, -1,
                                                               only_objectness=0)]


def corner_rects(uv):
    """(m, 9, 2) fp32 pixel keypoints -> (m, 4) fp32 [x0, y0, x1, y1] of keypoints 1..8"""
    c = np.asarray(uv, F32)[:, 1:9]
    return np.stack([c[..., 0].min(1), c[..., 1].min(1), c[..., 0].max(1), c[..., 1].max(1)], 1).astype(F32)


def iou_ref(a, b):
    """IoU of rectangle a (4,) against rectangles b (k, 4), fp32: inter = (min x1 - max x0) * (min y1 - max y0) when both sides
    are positive, union = (area a + area b) - inter, inter / union (0 when union <= 0)"""
    a = np.asarray(a, F32)
    b = np.asarray(b, F32).reshape(-1, 4)
    iw = np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0])
    ih = np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1])
    ok = (iw > 0) & (ih > 0)
    inter = np.where(ok, iw * ih, F32(0))
    area_a = (a[2] - a[0]) * (a[3] - a[1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    uni = (area_a + area_b) - inter
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(ok & (uni > 0), inter / np.where(uni > 0, uni, F32(1)), F32(0))
    return r.astype(F32)


def nms_ref(det, cls, uv, nms_thresh, max_instances):
    """greedy class-wise suppression of m candidates given in visiting order: det (m,) fp32, cls (m,), uv (m, 9, 2) fp32 ->
    (positions of the first max_instances kept candidates in key order, number kept before truncation)"""
    det = np.asarray(det, F32)
    m = len(det)
    order = sorted(range(m), key=lambda j: (-float(det[j]), j))
    rects = corner_rects(uv) if m else np.zeros((0, 4), F32)
    kept_of = {}
    out, nk = [], 0
    thr = F32(nms_thresh)
    for j in order:
        k = kept_of.setdefault(int(cls[j]), [])
        if k and (iou_ref(rects[j], rects[k]) > thr).any():
            continue
        k.append(j)
        if nk < max_instances:
            out.append(j)
        nk += 1
    return out, nk


def detect_ref(det, cmax, cls_id, uv, conf_thresh, nms_thresh, classes, max_instances):
    """one frame from its decoded entries in visiting order (det, cmax, cls_id (n,), uv (n, 9, 2) fp32 pixels): candidates
    det * cmax > conf_thresh in fp32 whose class is in `classes`, then nms_ref -> (kept entry indices in key order, kept)"""
    det, cmax = np.asarray(det, F32), np.asarray(cmax, F32)
    cls_id = np.asarray(cls_id).astype(np.int64)
    cand = np.nonzero((det * cmax > F32(conf_thresh)) & np.isin(cls_id, np.asarray(list(classes))))[0]
    pos, nk = nms_ref(det[cand], cls_id[cand], np.asarray(uv, F32)[cand], nms_thresh, max_instances)
    return [int(cand[j]) for j in pos], nk
