"""Multi-object decode -- drop-in for ``get_multi_region_boxes`` of reference multi_obj_pose_estimation/utils_multi.py:266-382.
The dense per-(cell, anchor) arithmetic and the reference's sequential fallback maxima run on the GPU; the host only
applies the confidence mask (one device->host copy).  The pose helpers are shared with utils.py."""
from __future__ import annotations

import ctypes as _ctypes

import numpy as np
import torch

from ._lib import CONSTANTS, call, ptr, stream_ptr, SspError
from .utils import (pnp_batched, compute_projection, compute_transformation, calcAngularDistance, get_3D_corners,  # noqa: F401
                    get_camera_intrinsic, convert2cpu, convert2cpu_long, project_points_batched, adi_batched, mesh_diameter,
                    check_pnp_args, object_table, pnp_truth_and_prediction, pnp_one, camera_distortion, distortion_tensor, check_sigma)
from .utils_host import (makedirs, get_all_files, calc_pts_diameter, adi, get_2d_bb, corner_confidences, corner_confidence,  # noqa: F401
                         sigmoid, softmax, read_truths, read_truths_args, read_pose, load_class_names, image2torch, scale_bboxes,
                         file_lines, get_image_size, logging)
from . import utils_host as _host


def pnp(points_3D, points_2D, cameraMatrix):
    """utils.pnp for valid_multi.py (utils_multi.py:95-109).  A function of its own, as in the reference: its distortion coefficients
    are ITS attribute pnp.distCoeffs, independent of utils.pnp.distCoeffs; unset or all zeros is the zero-distortion solve."""
    return pnp_one(points_3D, points_2D, cameraMatrix, getattr(pnp, "distCoeffs", None))


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


def detect_buffers(c, batch, max_instances, device):
    """the device buffers detect_slots writes for batch x max_instances slots, as attributes of c (c.kp is the caller's)"""
    B, M, K = batch, max_instances, 9
    c.boxes = torch.empty(B, M, 2 * K + 3, dtype=torch.float32, device=device)
    c.cls = torch.empty(B, M, dtype=torch.int32, device=device)
    c.cls0 = torch.empty(B, M, dtype=torch.int32, device=device)
    c.count = torch.empty(B, dtype=torch.int32, device=device)
    c.kept = torch.empty(B, dtype=torch.int32, device=device)
    c.P3 = torch.empty(B * M, K, 3, dtype=torch.float32, device=device)


def detect_slots(c, logits, classes, points, num_classes, num_anchors, conf_thresh, nms_thresh, frame_size, stream):
    """detect_instances into the buffers of detect_buffers and c.kp (B, M, 9, 2), then each slot's PnP points c.P3 (B*M, 9, 3)
    gathered from points (num_classes, 9, 3) by class.  logits: the contiguous fp32 network output; classes: the requested
    class ids, a HOST int32 array copied into the launch."""
    B, M = c.cls.shape
    h, w = logits.shape[2:]
    call("ssp_detect_instances", ptr(logits), B, 9, num_classes, num_anchors, h, w, _ctypes.c_void_p(classes.ctypes.data), len(classes),
         conf_thresh, nms_thresh, M, float(frame_size[0]), float(frame_size[1]), ptr(c.boxes), ptr(c.cls), ptr(c.kp), ptr(c.count),
         ptr(c.kept), stream)
    torch.clamp(c.cls, min=0, out=c.cls0)                  # empty slots hold -1: any in-range index will do, PnP skips them
    torch.index_select(points, 0, c.cls0.view(-1), out=c.P3)


# ------------------------------------------------------------------------------------------ tracking across frames
MAX_TRACKS = 256            # largest max_tracks (track_core.h kMaxTracks)
FILTER_DOUBLES = CONSTANTS["SSP_FILTER_DOUBLES"]            # one track's pose filter (pose_filter_core.h kFilterDoubles)


def check_track_args(max_tracks, match_iou, max_misses):
    """-> (max_tracks, match_iou, max_misses) as int, float, int; SspError for max_tracks outside [1, 256], match_iou outside [0, 1]
    or max_misses < 0"""
    if isinstance(max_tracks, bool) or not isinstance(max_tracks, (int, np.integer)) or not 1 <= max_tracks <= MAX_TRACKS:
        raise SspError("max_tracks must be an integer in [1, %d], got %r" % (MAX_TRACKS, max_tracks))
    match_iou = float(match_iou)
    if not 0.0 <= match_iou <= 1.0:
        raise SspError("match_iou must be in [0, 1], got %r" % match_iou)
    if isinstance(max_misses, bool) or not isinstance(max_misses, (int, np.integer)) or max_misses < 0:
        raise SspError("max_misses must be an integer >= 0, got %r" % (max_misses,))
    return int(max_tracks), match_iou, int(max_misses)


MOTIONS = (None, "constant_velocity")


def check_motion_args(motion, keypoint_sigma, accel_sigma, init_velocity_sigma, gate, frame_dt):
    """-> (motion, keypoint_sigma, accel_sigma (rot, trans), init_velocity_sigma (rot, trans), gate, frame_dt) checked: motion None or
    'constant_velocity', every sigma, the gate and frame_dt > 0 and finite; SspError otherwise"""
    if not any(motion is m or motion == m for m in MOTIONS):
        raise SspError("motion must be None or 'constant_velocity', got %r" % (motion,))

    def pair(name, v):
        if isinstance(v, (str, bytes)) or np.ndim(v) != 1 or len(v) != 2:
            raise SspError("%s must be a pair (rotation, translation), got %r" % (name, v))
        return tuple(check_sigma("%s[%d]" % (name, i), x) for i, x in enumerate(v))
    return (motion, check_sigma("keypoint_sigma", keypoint_sigma), pair("accel_sigma", accel_sigma),
            pair("init_velocity_sigma", init_velocity_sigma), check_sigma("gate", gate), check_sigma("frame_dt", frame_dt))


def rodrigues_batched(r):
    """(n, 3) fp64 rotation vectors -> (n, 3, 3) rotation matrices (cv2.Rodrigues' formula; the identity below machine epsilon)"""
    th = torch.linalg.vector_norm(r, dim=1)
    small = th < np.finfo(np.float64).eps
    u = r / torch.where(small, torch.ones_like(th), th).unsqueeze(1)
    c, s = torch.cos(th)[:, None, None], torch.sin(th)[:, None, None]
    z = torch.zeros_like(th)
    ux = torch.stack([z, -u[:, 2], u[:, 1], u[:, 2], z, -u[:, 0], -u[:, 1], u[:, 0], z], 1).view(-1, 3, 3)
    eye = torch.eye(3, dtype=r.dtype, device=r.device).expand(len(r), 3, 3)
    R = c * eye + (1 - c) * u.unsqueeze(2) * u.unsqueeze(1) + s * ux
    return torch.where(small[:, None, None], eye, R)


class InstanceTracker:
    """Stable track ids across the frames of B camera streams, and PnP warm-started from each track's last pose (rules:
    csrc/track_core.h).  Per frame: the instances of detect_instances; ssp_track_associate matches each to an alive track of its
    class (highest IoU of the corner rectangles > match_iou, in det_conf order), ages the unmatched tracks (a track dies after
    max_misses + 1 missed frames in a row) and gives the other detections the lowest free slot and the stream's next id;
    ssp_pnp_batched_guess starts Levenberg-Marquardt from the matched track's pose (no DLT) and solves the others cold;
    ssp_track_commit stores each track's rectangle and final LM vector.  With motion=None (the default) there is no motion model: a
    track is matched against its last rectangle and the guess is its last pose (motion="constant_velocity": see below).  update(logits) is the eager, logits-level surface; predict_instances.
    TrackingPosePredictor issues the same launches inside its graph replay.

    objects: {class id: (3|4, 8) box corners}; K (3, 3); frame_size (width, height); batch = streams; max_tracks in [1, 256] slots
    per stream, match_iou in [0, 1], max_misses >= 0; dist_coeffs: the camera's OpenCV distortion coefficients (utils.camera_distortion),
    for the warm and the cold solves (ssp_pnp_dist); the association compares the raw keypoints' rectangles.  The state lives in four device arrays allocated once (graphs bake their
    addresses in): tracks (B, T, 5) int32 = alive, id, cls, misses, hits; rects (B, T, 4) fp32; poses (B, T, 6) fp64 = (rvec, t);
    next_id (B,) int32.  reset() zeroes them in place.

    motion="constant_velocity" adds a pose filter per track (rules: csrc/pose_filter_core.h): an error-state Kalman filter of the
    pose, the angular velocity and the linear velocity, fed by each frame's PnP with its covariance (utils.pose_covariance_batched
    with keypoint_sigma px).  Each frame, ssp_track_predict moves every alive track's filter to the frame's time first, and the
    association then compares each detection with the track's PREDICTED corner rectangle and warm-starts its PnP from the
    predicted pose, so an object that moves more than about half its width per frame keeps its id.  After the PnP,
    ssp_track_filter_update starts the filter of a new track and gates and updates a matched one: a measurement with
    y^T S^-1 y > gate (default 22.46, chi^2 with 6 degrees of freedom at 99.9 %) restarts the filter instead, as a mirrored PnP
    solution would.  accel_sigma = (rad/s^2, mesh units/s^2): the white-noise acceleration; init_velocity_sigma = (rad/s, mesh
    units/s): the velocity prior of a new track; frame_dt: the frame interval in seconds when update() is given no timestamps.
    These defaults are not tuned on real data: set keypoint_sigma to the network's keypoint error in pixels and the
    accelerations to how fast the objects can change their motion.  The filter state is one more device array, filter (B, T, 163)
    fp64 (csrc/pose_filter_core.h's layout), and each stream's last timestamp stays on the host.
    meshes= (the predictors' depth refinement) is refused: how a refined pose should feed the tracks and the filter is not defined."""

    def __init__(self, objects, K, num_classes, num_anchors, frame_size, batch=1, conf_thresh=0.05, nms_thresh=0.4, max_instances=32,
                 max_tracks=64, match_iou=0.3, max_misses=5, num_keypoints=9, device=None, dist_coeffs=None, motion=None,
                 keypoint_sigma=2.0, accel_sigma=(2.0, 1.0), init_velocity_sigma=(1.0, 0.5), gate=22.46, frame_dt=1 / 30, meshes=None):
        if meshes is not None:
            raise SspError("InstanceTracker does not refine against depth (meshes=): how a refined pose should feed the tracks and the "
                           "pose filter is not defined yet")
        self.max_tracks, self.match_iou, self.max_misses = check_track_args(max_tracks, match_iou, max_misses)
        (self.motion, self.keypoint_sigma, self.accel_sigma, self.init_velocity_sigma, self.gate,
         self.frame_dt) = check_motion_args(motion, keypoint_sigma, accel_sigma, init_velocity_sigma, gate, frame_dt)
        classes, points, Km = object_table(objects if isinstance(objects, dict) else {0: objects}, num_classes, K)
        if int(num_keypoints) != 9:
            raise SspError("tracking solves PnP on the centroid + 8 box corners: 9 keypoints, not %d" % int(num_keypoints))
        self.batch, self.max_instances = int(batch), int(max_instances)
        if self.batch < 1:
            raise SspError("batch must be >= 1")
        self.num_classes, self.num_anchors, self.num_keypoints = int(num_classes), int(num_anchors), 9
        self.frame_size = (float(frame_size[0]), float(frame_size[1]))
        self.conf_thresh, self.nms_thresh = float(conf_thresh), float(nms_thresh)
        self.classes = classes.astype(np.int32)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self._P3_table = torch.from_numpy(points.astype(np.float32)).to(dev)
        self._K32 = torch.from_numpy(np.ascontiguousarray(Km, dtype=np.float32)).to(dev)
        self._K64 = torch.from_numpy(np.ascontiguousarray(Km, dtype=np.float64)).to(dev)
        dist = camera_distortion(dist_coeffs)
        self._dist = None if dist is None else distortion_tensor(dist, dev)
        B, T = self.batch, self.max_tracks
        self.state_tracks = torch.zeros(B, T, 5, dtype=torch.int32, device=dev)
        self.state_rects = torch.zeros(B, T, 4, dtype=torch.float32, device=dev)
        self.state_poses = torch.zeros(B, T, 6, dtype=torch.float64, device=dev)
        self.state_next_id = torch.zeros(B, dtype=torch.int32, device=dev)
        if self.motion:
            self.state_filter = torch.zeros(B, T, FILTER_DOUBLES, dtype=torch.float64, device=dev)
            self._dt = torch.zeros(B, dtype=torch.float64, device=dev)        # this frame's interval per stream, read by the replay
            self._dt_pin = torch.zeros(B, dtype=torch.float64).pin_memory()
            self._dt_copied = torch.cuda.Event()      # the launches that last read _dt_pin have been enqueued before this
            self._last_time = np.full(B, np.nan)      # each stream's last timestamp (NaN: none since the start or a reset)
        self._bufs = None

    # ------------------------------------------------------------------ state
    def _state(self):
        base = (self.state_tracks, self.state_rects, self.state_poses, self.state_next_id)
        return base + (self.state_filter,) if self.motion else base

    def reset(self, streams=None):
        """forget every track of the given streams (default: all), in place: ids start again from 0; with motion, their filters
        and last timestamps too (the next frame of such a stream has dt = 0)"""
        sel = slice(None) if streams is None else np.asarray(streams, np.int64).reshape(-1)
        idx = sel if streams is None else torch.as_tensor(sel, device=self.device)
        for t in self._state():
            t[idx] = 0
        if self.motion:
            self._last_time[sel] = np.nan

    def snapshot(self):
        saved = tuple(t.clone() for t in self._state())
        return saved + (self._last_time.copy(),) if self.motion else saved

    def restore(self, saved):
        for t, s in zip(self._state(), saved):
            t.copy_(s)
        if self.motion:
            self._last_time[:] = saved[-1]

    def stage_times(self, timestamps=None):
        """with motion: this frame's interval per stream into the pinned buffer the next launches copy from.  timestamps: (B,)
        seconds, or None for each stream's last timestamp + frame_dt (a stream's first frame is at 0); dt = 0 for a stream's first
        frame.  SspError, before anything changes, for a timestamp that is not finite or not after the stream's last one."""
        if not self.motion:
            return
        last = self._last_time
        if timestamps is None:
            now = np.where(np.isnan(last), 0.0, last + self.frame_dt)
        else:
            try:
                now = np.asarray(timestamps, np.float64).reshape(-1)
            except (TypeError, ValueError):
                raise SspError("timestamps must be %d numbers (seconds), got %r" % (self.batch, timestamps))
            if now.shape != (self.batch,) or not np.isfinite(now).all():
                raise SspError("timestamps must be %d finite numbers (seconds), one per stream, got %r" % (self.batch, timestamps))
            bad = ~np.isnan(last) & ~(now > last)
            if bad.any():
                b = int(np.nonzero(bad)[0][0])
                raise SspError("stream %d: timestamp %r is not after the stream's last one, %r" % (b, float(now[b]), float(last[b])))
        # the last frame's copy out of the pinned buffer has run.  The event is recorded after ALL of that frame's launches (the copy
        # is a node inside the captured graph, where no host-visible event can follow it alone), so this waits until the previous
        # frame has finished.  Host frames already wait for their own staging buffer this way; for device and JPEG frames it is a
        # host synchronisation per frame that motion=None does not have.
        self._dt_copied.synchronize()
        self._dt_pin.numpy()[:] = np.where(np.isnan(last), 0.0, now - last)
        self._last_time = now

    def staged(self):
        """after the launches of a frame are enqueued: the pinned interval buffer may be rewritten once they have run"""
        if self.motion:
            self._dt_copied.record()

    def tracks(self, to_host=False):
        """the alive tracks of every stream, ordered by (stream, slot): stream, slot, id, cls, misses, hits (n,) int32; rvec (n, 3),
        R (n, 3, 3) (Rodrigues of rvec), t (n, 3) fp64 = the track's last pose; rect (n, 4) fp32 = its last corner rectangle.
        With motion also the filter's R_filt (n, 3, 3), t_filt (n, 3), velocity (n, 6) = (w, v) and pose_cov (n, 6, 6) at the last
        frame's time (a track that missed the frame reports its prediction) and filter_valid (n,) bool (False while the track has
        had no measurement with a usable covariance)."""
        st = self.state_tracks
        b, s = torch.nonzero(st[..., 0] != 0, as_tuple=True)
        f, pose = st[b, s], self.state_poses[b, s]
        out = dict(stream=b.int(), slot=s.int(), id=f[:, 1], cls=f[:, 2], misses=f[:, 3], hits=f[:, 4], rvec=pose[:, :3],
                   R=rodrigues_batched(pose[:, :3]), t=pose[:, 3:], rect=self.state_rects[b, s])
        if self.motion:             # the filter: this frame's estimate, or its prediction for a track that missed the frame
            fs = self.state_filter[b, s]
            P = fs[:, 18:162].reshape(-1, 12, 12)
            out.update(R_filt=fs[:, :9].reshape(-1, 3, 3), t_filt=fs[:, 9:12], velocity=fs[:, 12:18], pose_cov=P[:, :6, :6].contiguous(),
                       filter_valid=fs[:, 162] == 1.0)
        if to_host:
            return {k: v.cpu().numpy() for k, v in out.items()}
        return out

    # ------------------------------------------------------------------ launches
    def buffers(self, c):
        """the per-frame device buffers of the tracking launches, as attributes of c (B streams x M detection slots)"""
        dev, B, M = self.device, self.batch, self.max_instances
        c.slot = torch.empty(B, M, dtype=torch.int32, device=dev)
        c.track_id = torch.empty(B, M, dtype=torch.int32, device=dev)
        c.guess = torch.empty(B, M, 6, dtype=torch.float64, device=dev)
        c.use_guess = torch.empty(B, M, dtype=torch.int32, device=dev)
        c.params = torch.empty(B, M, 6, dtype=torch.float64, device=dev)
        c.warm = torch.empty(B, M, dtype=torch.bool, device=dev)
        if self.motion:
            T = self.max_tracks
            c.pred_poses = torch.empty(B, T, 6, dtype=torch.float64, device=dev)
            c.pred_rects = torch.empty(B, T, 4, dtype=torch.float32, device=dev)
            c.cov_m = torch.empty(B, M, 6, 6, dtype=torch.float64, device=dev)
            c.cov_status = torch.empty(B, M, dtype=torch.int32, device=dev)
            c.R_filt = torch.empty(B, M, 3, 3, dtype=torch.float64, device=dev)
            c.t_filt = torch.empty(B, M, 3, dtype=torch.float64, device=dev)
            c.pose_cov = torch.empty(B, M, 6, 6, dtype=torch.float64, device=dev)
            c.velocity = torch.empty(B, M, 6, dtype=torch.float64, device=dev)
            c.reinit_i = torch.empty(B, M, dtype=torch.int32, device=dev)
            c.reinit = torch.empty(B, M, dtype=torch.bool, device=dev)

    def outputs(self, c):
        """the filter's outputs per detection slot (empty with motion None)"""
        if not self.motion:
            return {}
        return dict(R_filt=c.R_filt, t_filt=c.t_filt, pose_cov=c.pose_cov, velocity=c.velocity, reinit=c.reinit)

    def solve(self, c, s, P3, K32):
        """associate, warm-started PnP, commit: reads c.count, c.cls, c.kp (ssp_detect_instances' outputs) and P3 (B*M, 9, 3) the
        slots' PnP points; writes c.R, c.t, c.params, c.slot, c.track_id, c.guess, c.use_guess, c.warm.  With motion the tracks are
        predicted first and associated on the predictions, and the filters are updated last (outputs())."""
        B, T, M = self.batch, self.max_tracks, self.max_instances
        rects, poses = self.state_rects, self.state_poses
        dist = None if self._dist is None else ptr(self._dist)
        if self.motion:
            self._dt.copy_(self._dt_pin, non_blocking=True)
            call("ssp_track_predict", B, T, ptr(self.state_tracks), ptr(rects), ptr(poses), ptr(self.state_filter), ptr(self._dt),
                 ptr(self._P3_table), self.num_classes, ptr(self._K64), dist, self.accel_sigma[0], self.accel_sigma[1], ptr(c.pred_poses),
                 ptr(c.pred_rects), s)
            rects, poses = c.pred_rects, c.pred_poses
        call("ssp_track_associate", B, T, M, ptr(c.count), ptr(c.cls), ptr(c.kp), self.match_iou, self.max_misses, ptr(self.state_tracks),
             ptr(rects), ptr(poses), ptr(self.state_next_id), ptr(c.slot), ptr(c.track_id), ptr(c.guess), ptr(c.use_guess), s)
        if self._dist is None:
            call("ssp_pnp_batched_guess", ptr(P3), ptr(c.kp), ptr(K32), 9, B, M, ptr(c.count), ptr(c.guess), ptr(c.use_guess), 20, ptr(c.R),
                 ptr(c.t), ptr(c.params), None, s)
        else:
            call("ssp_pnp_dist", ptr(P3), 0, ptr(c.kp), ptr(K32), ptr(self._dist), 9, B, M, ptr(c.count), ptr(c.guess), ptr(c.use_guess), 20,
                 ptr(c.R), ptr(c.t), ptr(c.params), None, s)
        call("ssp_track_commit", B, T, M, ptr(c.count), ptr(c.kp), ptr(c.slot), ptr(c.params), ptr(self.state_tracks), ptr(self.state_rects),
             ptr(self.state_poses), s)
        torch.ne(c.use_guess, 0, out=c.warm)
        if self.motion:
            call("ssp_pose_covariance", ptr(P3), 0, ptr(K32), dist, 9, B, M, ptr(c.count), ptr(c.R), ptr(c.t), self.keypoint_sigma, ptr(c.cov_m),
                 ptr(c.cov_status), s)
            call("ssp_track_filter_update", B, T, M, ptr(c.count), ptr(c.slot), ptr(c.use_guess), ptr(c.R), ptr(c.t), ptr(c.cov_m),
                 ptr(c.cov_status), ptr(self.state_filter), self.init_velocity_sigma[0], self.init_velocity_sigma[1], self.gate,
                 ptr(c.R_filt), ptr(c.t_filt), ptr(c.pose_cov), ptr(c.velocity), ptr(c.reinit_i), s)
            torch.ne(c.reinit_i, 0, out=c.reinit)

    def update(self, logits, timestamps=None):
        """one frame of every stream from the network output (B, (2K+1+C)*A, H, W) -> dict of device tensors: count, kept (B,);
        cls, track_id (B, M) int32 (-1 in empty and untracked slots); warm (B, M) bool; conf, cls_conf (B, M); keypoints_px
        (B, M, 9, 2); R (B, M, 3, 3), t (B, M, 3), params (B, M, 6) fp64 (zero in empty slots).  Returned tensors are reused.
        With motion: timestamps (B,) seconds of this frame per stream (stage_times), and the outputs add, per detection slot with a
        track, the filtered pose R_filt (B, M, 3, 3), t_filt (B, M, 3), its covariance pose_cov (B, M, 6, 6) over (dth, dt_), the
        velocity (B, M, 6) = (w rad/s, v mesh units/s) and reinit (B, M) bool (the filter was started from this frame's PnP: a new
        track, a measurement outside the gate or one without a usable covariance); zeros elsewhere.  R, t stay this frame's PnP."""
        if not logits.is_cuda:
            raise SspError("InstanceTracker.update runs on CUDA tensors only")
        out = logits.detach().contiguous().float()
        B, Cn, H, W = out.shape
        K, nC, nA, M = 9, self.num_classes, self.num_anchors, self.max_instances
        if B != self.batch:
            raise SspError("this tracker follows %d streams, got a batch of %d" % (self.batch, B))
        if Cn != (2 * K + 1 + nC) * nA:
            raise SspError("output has %d channels, expected (2K+1+C)*A = %d" % (Cn, (2 * K + 1 + nC) * nA))
        self.stage_times(timestamps)
        c = self._bufs
        if c is None:
            import types
            c = self._bufs = types.SimpleNamespace()
            detect_buffers(c, B, M, self.device)
            c.kp = torch.empty(B, M, K, 2, dtype=torch.float32, device=self.device)
            c.R = torch.empty(B, M, 3, 3, dtype=torch.float64, device=self.device)
            c.t = torch.empty(B, M, 3, dtype=torch.float64, device=self.device)
            self.buffers(c)
        s = stream_ptr()
        detect_slots(c, out, self.classes, self._P3_table, nC, nA, self.conf_thresh, self.nms_thresh, self.frame_size, s)
        self.solve(c, s, c.P3, self._K32)
        self.staged()
        return dict(count=c.count, kept=c.kept, cls=c.cls, track_id=c.track_id, warm=c.warm, conf=c.boxes[..., 2 * K],
                    cls_conf=c.boxes[..., 2 * K + 1], keypoints_px=c.kp, R=c.R, t=c.t, params=c.params, **self.outputs(c))


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
                                 internal_calibration, im_width=640, im_height=480, adds=False, pnp="plain", reproj_thresh=8.0,
                                 dist_coeffs=None):
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
    corners are never used by it and are not computed.

    pnp="consensus" solves the G predicted poses with the consensus PnP (utils.pnp_consensus_batched, inliers within reproj_thresh
    pixels) and adds `inliers` (G, K) bool and `hyp` (G,) int32; the ground-truth poses stay the plain solve.  projection_accuracy
    of the pixel_err of both modes on one network output compares the two solves.

    dist_coeffs: OpenCV distortion coefficients of the camera (utils.camera_distortion): the ground-truth and the predicted poses are
    both solved with them, as valid_multi.py does when pnp.distCoeffs is set; pixel_err stays the undistorted projection
    (compute_projection), which is also what valid_multi.py computes then."""
    pnp, reproj_thresh = check_pnp_args(pnp, reproj_thresh)
    camera_distortion(dist_coeffs)
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
    c3 = np.asarray(corners3D, dtype=np.float64)[:3]
    P3 = np.array(np.transpose(np.concatenate((np.zeros((3, 1)), c3), axis=1)), dtype="float32")          # valid_multi.py:135
    Kc = torch.as_tensor(np.asarray(internal_calibration, dtype=np.float32)).to(dev)
    R, t, extra = pnp_truth_and_prediction(torch.from_numpy(P3).to(dev), uv, Kc, pnp, reproj_thresh, dist_coeffs)       # 2G problems
    if G == 0:                                                  # nothing to project: empty errors
        res = dict(res, R_gt=R, t_gt=t, R_pr=R.clone(), t_pr=t.clone(), pixel_err=torch.zeros(0, dtype=torch.float32, device=dev), **extra)
        if adds:
            res.update(vertex_dist=torch.zeros(0, dtype=torch.float64, device=dev), adds_dist=torch.zeros(0, dtype=torch.float64, device=dev))
        return res
    Rt = torch.cat([R, t.unsqueeze(2)], 2)
    V = torch.as_tensor(np.asarray(vertices, dtype=np.float32)).to(dev)
    if V.shape[0] == 3:
        V = torch.cat([V, torch.ones(1, V.shape[1], device=dev)], 0)
    proj = project_points_batched(V, Rt, torch.as_tensor(np.asarray(internal_calibration, dtype=np.float64)).to(dev))   # (2G, 2, Nv)
    d = proj[:G] - proj[G:]
    # valid_multi.py:143-149.  Elementwise distances, then an fp64 mean: the result of one object does not depend on how many
    # objects the batch holds (a batched fp32 reduction may change its summation order with the shape)
    pixel_err = torch.hypot(d[:, 0], d[:, 1]).double().mean(dim=1).float()
    res = dict(res, R_gt=R[:G], t_gt=t[:G], R_pr=R[G:], t_pr=t[G:], pixel_err=pixel_err, **extra)
    if adds:
        res["adds_dist"], res["vertex_dist"] = adi_batched(vertices, Rt[G:], Rt[:G], with_add=True)
    return res
