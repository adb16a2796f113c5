"""Camera frames -> the 6-D pose of every detected instance of the requested objects, in one CUDA graph replay.

    pred = InstancePosePredictor(model, {0: corners_ape, 4: corners_can}, K, frame_size=(640, 480), batch=1)
    r = pred(frames)            # (B, H, W, 3) uint8 numpy array / CUDA tensor, or a list of B JPEG files' bytes
    for m in range(r["count"][b]): r["cls"][b, m], r["R"][b, m], r["t"][b, m], ...

Frames go through the chain the other predictors run (predict.py: resize + ToTensor, the split-K eval forward, the graph LRU, the
weight re-pack); only the head differs.  PosePredictor and MultiPosePredictor return one pose per (frame, class); this head
returns every instance (rules: csrc/detect_core.h):
  * candidates: the boxes get_multi_region_boxes(..., only_objectness=0) lists -- det_conf * cls_max_conf > conf_thresh, never the
    fallback box -- whose arg-max class is requested; with one anchor and one class that is det_conf > conf_thresh;
  * ranked by det_conf, the earlier (cell, anchor) on ties, so instance 0 of class c is MultiPosePredictor's slot c whenever that
    slot is detected;
  * greedy suppression within each class: a candidate is dropped when the rectangle of its 8 corner keypoints in frame pixels
    has IoU > nms_thresh with a kept box of its class (the reference's nms reads YOLO boxes and cannot run on pose boxes);
  * the first max_instances kept boxes; count = min(kept, max_instances), kept = the number before the truncation.
Then per slot: PnP of the 9 points [0; corners3D_c[:3]] of the slot's class with the fp32 K, and the projection of the centroid
and the 8 corners under that pose.  Slots >= count are zero (cls -1).

The head is one ssp_detect_instances launch (one CTA per frame), a device gather of each slot's PnP points by cls.clamp(min=0)
(empty slots hold cls = -1), one ssp_pnp_batched_counted over the B x M slots (empty slots are skipped on the device: no host
read-back), one ssp_project_points of every requested class's points under every slot's pose, of which each slot keeps its own
class's columns, masked to zero in the empty slots.

Returned device tensors are the predictor's static outputs: the next call overwrites them.

TrackingPosePredictor adds stable track ids across calls (each batch row is a camera stream) and PnP warm-started from each
track's last pose (utils_multi.InstanceTracker, rules: csrc/track_core.h).  WorldTrackingPosePredictor tracks the fused world
instances of a rig instead: each capture is a stream, and every world instance is matched to the nearest track of its class in
the world frame (utils_multi.WorldInstanceTracker, rules: csrc/world_track_core.h), after ssp_fuse_instances in the same graph
replay.

Command line: python -m singleshotpose_b200.predict_instances --datacfg cfg/occlusion.data --modelcfg cfg/yolo-pose-multi.cfg
              --weightfile w.weights --object 0=../LINEMOD/ape/ape.ply --object 4=../LINEMOD/can/can.ply --out det.npz img...
              [--track [--match-iou 0.3 --max-misses 5 --max-tracks 64]]: the images, in the order given, as one stream, with a
              track_id column
              [--track --motion cv [--keypoint-sigma 2 --fps 30]]: with the constant-velocity pose filter, adding the columns
              R_filt, t_filt, velocity and pose_cov
              [--pnp consensus [--reproj-thresh 8]]: the consensus PnP, with inliers and hyp columns (not with --track)
              [--depth-dir DIR [--depth-scale 0.001 --refine-iters 10]]: refine against 16-bit depth PNGs, as predict's command line
              (not with --track)
              [--rig rig.npz]: the images come in groups of C calibrated cameras (image i is camera i % C; utils_host.read_rig)
              and each capture's detections are associated into world instances, adding the per-detection column world_index and
              the per-world-instance rows capture world_cls R_world t_world world_cov members view_err fuse_hyp fuse_status
              (not with --dist, --depth-dir or --pnp consensus)
              [--rig rig.npz --track [--match-dist 0.5 --max-misses 5 --max-tracks 64] [--motion cv --keypoint-sigma 2 --fps 30]]:
              the captures, in order, as one stream of tracked world instances, adding the per-detection column track_id, the
              per-world-instance column world_track_id and, with --motion, the per-world-instance columns R_filt t_filt velocity
              pose_cov (--keypoint-sigma is then the fusion's keypoint noise, which sets world_cov)
"""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from . import predict, predict_multi
from ._lib import SspError
from .predict import (CONSENSUS_KEYS, REFINE_KEYS, _FramePredictor, add_depth_args, add_dist_arg, add_pnp_args, camera_dist, check_depth_args,
                      check_rig_args, mesh_corners, predict_files, read_camera, read_mesh, refine_kwargs)
from .predict_multi import cfg_conf_thresh, check_grid, parse_objects
from .utils import CameraRig, camera_distortion, check_pnp_args, check_sigma
from .utils_multi import InstanceTracker, WorldInstanceTracker, check_motion_args, check_track_args, detect_buffers, detect_slots

MAX_INSTANCES = 256         # largest max_instances (detect_core.h kMaxInstances)
OUTPUT_KEYS = ("count", "kept", "cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px")
ROW_KEYS = ("cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px")
MOTION_KEYS = ("R_filt", "t_filt", "velocity", "pose_cov")          # the --motion columns
WORLD_KEYS = ("world_cls", "R_world", "t_world", "world_cov", "members", "view_err", "fuse_hyp", "fuse_status")   # --rig: per world instance


class InstancePosePredictor(_FramePredictor):
    """model: a singleshotpose_b200.Darknet (single-object head) or darknet_multi.Darknet (multi-object head), 9 keypoints.
    objects: {class id: (3|4, 8) box corners of that class's mesh (utils.get_3D_corners)}; a bare corners array means {0: corners}.
    K: (3, 3) camera matrix; frame_size: (width, height) of the camera frames (other sizes are accepted and captured separately);
    shape: network input (width, height), default the cfg's test size for one anchor (as PosePredictor) and its training size for
    several (as MultiPosePredictor); batch: frames per call; conf_thresh: default the cfg net block's conf_thresh; nms_thresh in
    [0, 1]; max_instances in [1, 256] slots per frame.  graph=False runs the same launches eagerly (no capture).

    Returns dict(count (B,) int32, kept (B,) int32, cls (B, M) int32, R (B, M, 3, 3) fp64, t (B, M, 3) fp64, conf (B, M) det_conf,
    cls_conf (B, M), keypoints_px (B, M, 9, 2), corners_px (B, M, 9, 2)): device tensors, or numpy with to_host=True.
    pnp="consensus" solves each slot with the consensus PnP (utils.pnp_consensus_batched, inliers within reproj_thresh frame
    pixels) and adds inliers (B, M, 9) bool and hyp (B, M) int32 (empty slots: False and 0); pnp="plain" (default) is the all-point
    solve.  dist_coeffs: the camera's OpenCV distortion coefficients, as predict.PosePredictor takes them (the suppression still
    compares the raw keypoints' rectangles).
    meshes={class id: (vertices, faces)}, one for every requested class: refine every instance's pose against the call's
    depth=(B, H, W) uint16 frames, as predict.PosePredictor's mesh= does, adding R_ref (B, M, 3, 3), t_ref (B, M, 3),
    corners_ref_px (B, M, 9, 2), refine_points, refine_rmse and refine_status (B, M) (empty slots: zeros).
    rig=utils.camera_rig(...) of C calibrated cameras (K=None; no dist_coeffs, each camera brings its own): batch is a multiple of
    C and frame g C + c is camera c of capture g.  Every per-frame output is what a one-camera predictor with that camera's K and
    distortion gives; the detections are then associated across the views into world instances (utils.fuse_instances_batched,
    fuse = (gate, reproj_thresh, keypoint_sigma)), adding per capture world_count (G,), unfused (G,), world_cls (G, M), R_world
    (G, M, 3, 3), t_world (G, M, 3), world_cov (G, M, 6, 6), members (G, M, C), view_err (G, M, C), fuse_hyp (G, M), fuse_status
    (G, M), and per frame world_index (B, M) and corners_world_px (B, M, 9, 2).  Not with pnp="consensus" or meshes."""

    def __init__(self, model, objects, K, frame_size=(640, 480), shape=None, batch=1, conf_thresh=None, nms_thresh=0.4, max_instances=32,
                 graph=True, max_graphs=4, pnp="plain", reproj_thresh=8.0, dist_coeffs=None, meshes=None, depth_scale=0.001, refine_iters=10,
                 refine_gate=(0.5, 0.02), rig=None, fuse=(40.0, 8.0, 2.0)):
        self.num_anchors = int(getattr(model, "num_anchors", 0))
        if self.num_anchors < 1:
            raise SspError("InstancePosePredictor needs a model with a region head")
        self.nms_thresh, self.max_instances = check_detect_args(nms_thresh, max_instances)
        self.conf_thresh = cfg_conf_thresh(model, conf_thresh)
        if shape is None:
            shape = (model.test_width, model.test_height) if self.num_anchors == 1 else (model.width, model.height)
        super().__init__(model, objects if isinstance(objects, dict) else {0: objects}, K, frame_size, shape, batch, graph, max_graphs,
                         pnp, reproj_thresh, slots=self.max_instances, dist_coeffs=dist_coeffs, meshes=meshes, depth_scale=depth_scale,
                         refine_iters=refine_iters, refine_gate=refine_gate, rig=rig, fuse=fuse)
        check_grid(self, "detect")

    def _head_buffers(self, c):
        detect_buffers(c, self.batch, self.max_instances, self.device)

    def _head(self, c, s):
        detect_slots(c, c.logits, self._cls_host, self._P3_table, self.num_classes, self.num_anchors, self.conf_thresh, self.nms_thresh,
                     c.frame, s)
        self._tail(c, s)

    def _outputs(self, c):
        K = self.num_keypoints
        return dict(count=c.count, kept=c.kept, cls=c.cls, R=c.R, t=c.t, conf=c.boxes[..., 2 * K], cls_conf=c.boxes[..., 2 * K + 1],
                    keypoints_px=c.kp, corners_px=c.corners, **self._consensus_outputs(c), **self._refine_outputs(c), **self._fuse_outputs(c))


class _TrackedCalls:
    """What a tracking predictor adds around InstancePosePredictor's call, for its tracker self._tracker (utils_multi.InstanceTracker
    or WorldInstanceTracker): with motion, each stream's timestamp staged before the launches (checked before any launch, after the
    frames); reset and tracks; and the track state put back after the warm-up runs of a graph capture, which advance it."""

    def __call__(self, frames, to_host=False, events=None, timestamps=None):
        """InstancePosePredictor's call; timestamps: one per stream, seconds, for the motion model (ignored without it)"""
        if not self.motion:
            return super().__call__(frames, to_host, events)
        self._check(frames)                        # the frames' errors before the timestamps change anything
        with torch.cuda.device(self.device):
            self._tracker.stage_times(timestamps)
        out = super().__call__(frames, to_host, events)
        with torch.cuda.device(self.device):
            self._tracker.staged()
        return out

    def reset(self, streams=None):
        """forget the tracks of the given streams (default: all); their ids start again from 0"""
        with torch.cuda.device(self.device):
            self._tracker.reset(streams)

    def tracks(self, to_host=False):
        """the alive tracks (the tracker's tracks())"""
        with torch.cuda.device(self.device):
            return self._tracker.tracks(to_host)

    def _capture(self, c, warmup=2):
        saved = self._tracker.snapshot()          # the warm-up runs advance the tracks: put them back before the first replay
        super()._capture(c, warmup)
        self._tracker.restore(saved)


class TrackingPosePredictor(_TrackedCalls, InstancePosePredictor):
    """InstancePosePredictor whose instances keep their identity across calls: each row b of a batch is its own camera stream, and
    each instance is matched to a track of its class (utils_multi.InstanceTracker, rules: csrc/track_core.h).  A matched instance's
    PnP starts Levenberg-Marquardt from its track's last pose (cv2.solvePnP's useExtrinsicGuess), the others are solved cold.
    With motion=None (the default) there is no motion model: a track is matched against its last corner rectangle, and the guess
    is its last pose; motion="constant_velocity" matches and warm-starts on predictions (below).

    max_tracks in [1, 256] track slots per stream, match_iou in [0, 1] (a match needs IoU > match_iou), max_misses >= 0 (a track
    dies after max_misses + 1 frames in a row without a match); the other arguments are InstancePosePredictor's.

    Returns InstancePosePredictor's dict plus track_id (B, M) int32 (-1 in empty and untracked slots) and warm (B, M) bool (the
    slot's solve started from its track's pose).  The track state is shared by every frame size and source (one set of device
    arrays, zeroed in place by reset); the warm-up runs before a graph capture do not advance it.
    Only pnp="plain": the consensus solve has no rule yet for how a track's warm guess competes with its subset hypotheses.
    dist_coeffs: the camera's OpenCV distortion coefficients; the warm and the cold solves both use them, the association compares
    the raw keypoints' rectangles.

    motion="constant_velocity" smooths and predicts each track's pose with a constant-velocity pose filter
    (utils_multi.InstanceTracker, rules: csrc/pose_filter_core.h): the association compares each detection with its track's
    predicted rectangle, the warm start is the predicted pose, and the outputs add R_filt (B, M, 3, 3), t_filt (B, M, 3),
    pose_cov (B, M, 6, 6), velocity (B, M, 6) and reinit (B, M) bool; R and t stay this frame's PnP.  keypoint_sigma (px),
    accel_sigma, init_velocity_sigma, gate and frame_dt (s) are InstanceTracker's, and their defaults are not tuned on real data.
    __call__ then takes timestamps= (B,) seconds per stream (default: the stream's last + frame_dt), checked before any launch.
    reset(streams) forgets the tracks of some streams; tracks() lists the alive ones (utils_multi.InstanceTracker.tracks).
    meshes= (the depth refinement) is refused: how a refined pose should feed the tracks and the pose filter is not defined yet."""

    def __init__(self, model, objects, K, frame_size=(640, 480), shape=None, batch=1, conf_thresh=None, nms_thresh=0.4, max_instances=32,
                 max_tracks=64, match_iou=0.3, max_misses=5, graph=True, max_graphs=4, pnp="plain", dist_coeffs=None, motion=None,
                 keypoint_sigma=2.0, accel_sigma=(2.0, 1.0), init_velocity_sigma=(1.0, 0.5), gate=22.46, frame_dt=1 / 30, meshes=None):
        check_tracking_pnp(pnp)
        check_tracking_meshes(meshes)
        check_track_args(max_tracks, match_iou, max_misses)
        check_motion_args(motion, keypoint_sigma, accel_sigma, init_velocity_sigma, gate, frame_dt)
        super().__init__(model, objects, K, frame_size, shape, batch, conf_thresh, nms_thresh, max_instances, graph, max_graphs,
                         dist_coeffs=dist_coeffs)
        self._tracker = InstanceTracker(objects, K, self.num_classes, self.num_anchors, self.frame_size, self.batch, self.conf_thresh,
                                        self.nms_thresh, self.max_instances, max_tracks, match_iou, max_misses, device=self.device,
                                        dist_coeffs=dist_coeffs, motion=motion, keypoint_sigma=keypoint_sigma, accel_sigma=accel_sigma,
                                        init_velocity_sigma=init_velocity_sigma, gate=gate, frame_dt=frame_dt)
        self.max_tracks, self.match_iou, self.max_misses = self._tracker.max_tracks, self._tracker.match_iou, self._tracker.max_misses
        self.motion = self._tracker.motion

    def _head_buffers(self, c):
        super()._head_buffers(c)
        self._tracker.buffers(c)

    def _solve(self, c, s):
        self._tracker.solve(c, s, c.P3, self._K32)

    def _outputs(self, c):
        return dict(super()._outputs(c), track_id=c.track_id, warm=c.warm, **self._tracker.outputs(c))


class WorldTrackingPosePredictor(_TrackedCalls, InstancePosePredictor):
    """InstancePosePredictor(rig=...) whose world instances keep their identity across calls (utils_multi.WorldInstanceTracker,
    rules: csrc/world_track_core.h).  rig: utils.camera_rig(...) of C cameras; batch (default C) a multiple of C, frame g C + c
    being camera c of capture g, and each capture g its own stream.  After ssp_fuse_instances, in the same graph replay, each
    world instance (in the fusion's emission order) takes the alive track of its class whose position lies nearest, strictly within
    match_dist x the class's box diagonal (the largest distance between two of its 8 corners); unmatched tracks die after
    max_misses + 1 captures in a row without a match, and unmatched instances take the lowest free slot of max_tracks and the
    stream's next id.  The other arguments are InstancePosePredictor's with a rig (fuse = (gate, reproj_thresh, keypoint_sigma)).

    Returns every output of InstancePosePredictor(rig=...), with its bits, plus track_id (B, M) int32 (each detection's world
    instance's track, -1 for none) and world_track_id (G, M) int32 (-1 in empty and untracked world slots).  The per-row PnP and
    the fusion stay cold: a track's prediction does not feed them.  The track state is one set of device arrays shared by every
    frame size and source; reset(streams) zeroes some streams in place; the warm-up runs before a graph capture do not advance it.

    motion="constant_velocity" runs TrackingPosePredictor's constant-velocity pose filter per track in world axes (a rig is static,
    so the velocity is the object's own), fed by each instance's fused pose and world_cov; the match then compares each instance
    with the track's predicted position.  The outputs add, per world slot, R_filt (G, M, 3, 3), t_filt (G, M, 3), pose_cov (G, M,
    6, 6), velocity (G, M, 6) = (w rad/s, v mesh units/s) and reinit (G, M) bool; __call__ takes timestamps= (G,) seconds, one per
    capture.  accel_sigma, init_velocity_sigma, gate and frame_dt are TrackingPosePredictor's, and not tuned on real data."""

    def __init__(self, model, objects, rig, frame_size=(640, 480), shape=None, batch=None, conf_thresh=None, nms_thresh=0.4,
                 max_instances=32, max_tracks=64, match_dist=0.5, max_misses=5, graph=True, max_graphs=4, motion=None,
                 accel_sigma=(2.0, 1.0), init_velocity_sigma=(1.0, 0.5), gate=22.46, frame_dt=1 / 30, fuse=(40.0, 8.0, 2.0)):
        if not isinstance(rig, CameraRig):
            raise SspError("WorldTrackingPosePredictor tracks the world instances of a rig: rig must be a CameraRig (utils.camera_rig)")
        check_track_args(max_tracks, 0.0, max_misses)
        check_sigma("match_dist", match_dist)
        check_motion_args(motion, 1.0, accel_sigma, init_velocity_sigma, gate, frame_dt)
        super().__init__(model, objects, None, frame_size, shape, len(rig.K) if batch is None else batch, conf_thresh, nms_thresh,
                         max_instances, graph, max_graphs, rig=rig, fuse=fuse)
        self._tracker = WorldInstanceTracker(objects, rig, self.num_classes, self.batch // len(rig.K), max_tracks, match_dist, max_misses,
                                             motion=motion, accel_sigma=accel_sigma, init_velocity_sigma=init_velocity_sigma, gate=gate,
                                             frame_dt=frame_dt, device=self.device)
        self.max_tracks, self.match_dist, self.max_misses = self._tracker.max_tracks, self._tracker.match_dist, self._tracker.max_misses
        self.motion = self._tracker.motion

    def _head_buffers(self, c):
        super()._head_buffers(c)
        self._tracker.buffers(c, self.max_instances)

    def _tail(self, c, s, valid=None):
        super()._tail(c, s, valid)
        self._tracker.solve(c, s, c.fi)            # the world instances of ssp_fuse_instances, in the same stream

    def _outputs(self, c):
        return dict(super()._outputs(c), **self._tracker.outputs(c))


def check_detect_args(nms_thresh, max_instances):
    """-> (nms_thresh, max_instances) as float, int; SspError for nms_thresh outside [0, 1] or max_instances outside [1, 256]"""
    nms_thresh = float(nms_thresh)
    if not 0.0 <= nms_thresh <= 1.0:
        raise SspError("nms_thresh must be in [0, 1], got %r" % nms_thresh)
    if isinstance(max_instances, bool) or not isinstance(max_instances, (int, np.integer)) or not 1 <= max_instances <= MAX_INSTANCES:
        raise SspError("max_instances must be an integer in [1, %d], got %r" % (MAX_INSTANCES, max_instances))
    return nms_thresh, int(max_instances)


def check_tracking_meshes(meshes):
    if meshes is not None:
        raise SspError("tracking does not refine against depth (meshes=): how a refined pose should feed the tracks and the pose "
                       "filter is not defined yet")


def check_tracking_pnp(pnp):
    if pnp != "plain":
        raise SspError("tracking solves with pnp='plain' only, got %r: the consensus solve has no rule for how a track's warm guess "
                       "competes with its subset hypotheses" % (pnp,))


# ---------------------------------------------------------------------------------------------- command line
SIZE_KEYS = predict_multi.SIZE_KEYS + predict.SIZE_KEYS      # a multi-object .data file's frame size, else a single-object one's


def parse_args(argv=None):
    """the command line, checked before any model is built: raises SspError for a bad --object, --nms-thresh, --max-instances,
    --match-iou, --max-misses, --max-tracks, --match-dist, --reproj-thresh, --dist, --keypoint-sigma, --fps, --depth-scale or
    --refine-iters, for --track with --pnp consensus or --depth-dir, for --motion without --track, for --match-dist without --rig,
    and for --rig with --dist, --depth-dir, --pnp consensus or an image count that is not whole captures (a.rig_cams is then the
    rig's CameraRig, else None)"""
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.predict_instances",
                                 description="6-D pose of every detected instance of the requested objects in each image")
    ap.add_argument("--datacfg", required=True, help=".data file: fx fy u0 v0 and width height (or im_width im_height); mesh")
    ap.add_argument("--modelcfg", required=True)
    ap.add_argument("--weightfile", required=True)
    ap.add_argument("--object", action="append", metavar="CLASS=MESH.ply",
                    help="a class id of the model and the mesh of its object; repeat per object (default: the .data file's mesh as class 0)")
    ap.add_argument("--nms-thresh", type=float, default=0.4)
    ap.add_argument("--max-instances", type=int, default=32)
    ap.add_argument("--out", default="instances.npz")
    ap.add_argument("--track", action="store_true",
                    help="treat the images, in the order given, as one camera stream: add a track_id column (TrackingPosePredictor)")
    ap.add_argument("--match-iou", type=float, default=0.3)
    ap.add_argument("--max-misses", type=int, default=5)
    ap.add_argument("--max-tracks", type=int, default=64)
    ap.add_argument("--motion", choices=("cv",), default=None,
                    help="with --track: smooth each track's pose with the constant-velocity pose filter, adding the columns R_filt, "
                         "t_filt, velocity and pose_cov")
    ap.add_argument("--keypoint-sigma", type=float, default=2.0, help="--motion: the keypoint noise in pixels")
    ap.add_argument("--fps", type=float, default=30.0, help="--motion: the frame rate of the image sequence")
    add_pnp_args(ap)
    add_dist_arg(ap)
    add_depth_args(ap)
    ap.add_argument("--rig", metavar="RIG.npz",
                    help="associate the detections of several calibrated cameras (utils_host.read_rig: K, R, t[, dist] per camera) into "
                         "world instances: the images come in groups of C, image i is camera i %% C; adds the column world_index and the "
                         "per-world-instance rows capture " + " ".join(WORLD_KEYS))
    ap.add_argument("--match-dist", type=float, default=None,
                    help="--rig --track: a world instance matches a track of its class within this many box diagonals (default 0.5)")
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    if a.match_dist is not None:
        if a.rig is None:
            raise SspError("--match-dist is the radius of the world tracks: it needs --rig (one camera's tracks match by --match-iou)")
        check_sigma("--match-dist", a.match_dist)
    check_pnp_args(a.pnp, a.reproj_thresh)
    check_depth_args(a)
    if a.track:
        check_tracking_pnp(a.pnp)
        if a.depth_dir is not None:
            raise SspError("--depth-dir does not combine with --track: how a refined pose should feed the tracks is not defined yet")
    check_detect_args(a.nms_thresh, a.max_instances)
    check_track_args(a.max_tracks, a.match_iou, a.max_misses)
    if a.motion and not a.track:
        raise SspError("--motion filters tracks: it needs --track")
    check_sigma("--keypoint-sigma", a.keypoint_sigma)
    check_sigma("--fps", a.fps)
    a.objects = parse_objects(a.object) if a.object else None
    if a.dist is not None:
        camera_distortion(a.dist)
    a.rig_cams = check_rig_args(a, refines=False)
    return a


def _region_anchors(modelcfg):
    from .cfg import parse_cfg
    for b in parse_cfg(modelcfg):
        if b["type"] == "region":
            return int(b.get("num", 1))
    raise SspError("%s has no [region] block" % modelcfg)


def check_inputs(a):
    """SspError, before any model is built, for a --datacfg, --modelcfg, --weightfile or image that is not a file"""
    for name, path in [("--datacfg", a.datacfg), ("--modelcfg", a.modelcfg), ("--weightfile", a.weightfile)] + [("image", p) for p in a.images]:
        if not os.path.isfile(path):
            raise SspError("%s %s: no such file" % (name, path))


def main(argv=None):
    a = parse_args(argv)
    check_inputs(a)
    mesh, K, size = read_camera(a.datacfg, SIZE_KEYS)
    dist = camera_dist(a) if a.rig_cams is None else None
    meshes = a.objects
    if meshes is None:
        if not mesh:
            raise SspError("%s has no mesh entry: give --object CLASS=MESH.ply" % a.datacfg)
        meshes = {0: mesh}
    objects = {c: mesh_corners(path) for c, path in meshes.items()}
    refine = dict(meshes={c: read_mesh(p) for c, p in meshes.items()}, **refine_kwargs(a)) if a.depth_dir is not None else {}
    if _region_anchors(a.modelcfg) > 1:
        from .darknet_multi import Darknet
    else:
        from .darknet import Darknet
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    motion = "constant_velocity" if a.motion else None
    rig = a.rig_cams
    if rig is not None:
        return _main_rig(a, model, objects, size, rig)
    if a.track:
        pred = TrackingPosePredictor(model, objects, K, frame_size=size, nms_thresh=a.nms_thresh, max_instances=a.max_instances,
                                     max_tracks=a.max_tracks, match_iou=a.match_iou, max_misses=a.max_misses, dist_coeffs=dist,
                                     motion=motion, keypoint_sigma=a.keypoint_sigma, frame_dt=1.0 / a.fps)
    else:
        pred = InstancePosePredictor(model, objects, K, frame_size=size, nms_thresh=a.nms_thresh, max_instances=a.max_instances,
                                     pnp=a.pnp, reproj_thresh=a.reproj_thresh, dist_coeffs=dist, **refine)
    rows = {k: [] for k in ROW_KEYS + (("track_id",) if a.track else ()) + (MOTION_KEYS if motion else ()) + CONSENSUS_KEYS[a.pnp]
            + (REFINE_KEYS if refine else ())}
    image = []
    for i, r in enumerate(predict_files(pred, a.images, a.depth_dir)):
        n = int(r["count"][0])
        image += [i] * n
        for k in rows:
            rows[k].append(r[k][0, :n])
    np.savez(a.out, paths=np.array(a.images), image=np.array(image, dtype=np.int64), **{k: np.concatenate(v) for k, v in rows.items()})
    print("%d images -> %d detections -> %s" % (len(a.images), len(image), a.out))


def _main_rig(a, model, objects, size, rig):
    """the --rig command line: one call per capture of C images"""
    Cn = len(rig.K)
    kw = dict(frame_size=size, batch=Cn, nms_thresh=a.nms_thresh, max_instances=a.max_instances, rig=rig)
    motion = "constant_velocity" if a.motion else None
    if a.track:
        pred = WorldTrackingPosePredictor(model, objects, max_tracks=a.max_tracks, max_misses=a.max_misses,
                                          match_dist=0.5 if a.match_dist is None else a.match_dist, motion=motion,
                                          fuse=(40.0, 8.0, a.keypoint_sigma), frame_dt=1.0 / a.fps, **kw)
    else:
        pred = InstancePosePredictor(model, objects, None, **kw)
    rows = {k: [] for k in ROW_KEYS + ("world_index",) + (("track_id",) if a.track else ())}
    world = {k: [] for k in WORLD_KEYS + (("world_track_id",) if a.track else ()) + (MOTION_KEYS if motion else ())}
    image, capture = [], []
    for g, r in enumerate(predict_files(pred, a.images, None, Cn)):
        for b in range(Cn):
            n = int(r["count"][b])
            image += [g * Cn + b] * n
            for k in rows:
                rows[k].append(r[k][b, :n])
        n = int(r["world_count"][0])
        capture += [g] * n
        for k in world:
            world[k].append(r[k][0, :n])
    np.savez(a.out, paths=np.array(a.images), image=np.array(image, dtype=np.int64), capture=np.array(capture, dtype=np.int64),
             **{k: np.concatenate(v) for k, v in rows.items()}, **{k: np.concatenate(v) for k, v in world.items()})
    print("%d images -> %d detections -> %d world instances -> %s" % (len(a.images), len(image), len(capture), a.out))


if __name__ == "__main__":
    main()
