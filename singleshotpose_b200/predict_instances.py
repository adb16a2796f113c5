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
track's last pose (utils_multi.InstanceTracker, rules: csrc/track_core.h).

Command line: python -m singleshotpose_b200.predict_instances --datacfg cfg/occlusion.data --modelcfg cfg/yolo-pose-multi.cfg
              --weightfile w.weights --object 0=../LINEMOD/ape/ape.ply --object 4=../LINEMOD/can/can.ply --out det.npz img...
              [--track [--match-iou 0.3 --max-misses 5 --max-tracks 64]]: the images, in the order given, as one stream, with a
              track_id column
"""
from __future__ import annotations

import argparse
import ctypes as C

import numpy as np
import torch

from ._lib import SspError, call, ptr
from .predict import _FramePredictor
from .predict_multi import MAX_ENTRIES, parse_objects
from .utils_multi import MAX_TRACKS, InstanceTracker, check_track_args

MAX_INSTANCES = 256         # largest max_instances (detect_core.h kMaxInstances)
OUTPUT_KEYS = ("count", "kept", "cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px")
ROW_KEYS = ("cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px")


class InstancePosePredictor(_FramePredictor):
    """model: a singleshotpose_b200.Darknet (single-object head) or darknet_multi.Darknet (multi-object head), 9 keypoints.
    objects: {class id: (3|4, 8) box corners of that class's mesh (utils.get_3D_corners)}; a bare corners array means {0: corners}.
    K: (3, 3) camera matrix; frame_size: (width, height) of the camera frames (other sizes are accepted and captured separately);
    shape: network input (width, height), default the cfg's test size for one anchor (as PosePredictor) and its training size for
    several (as MultiPosePredictor); batch: frames per call; conf_thresh: default the cfg net block's conf_thresh; nms_thresh in
    [0, 1]; max_instances in [1, 256] slots per frame.  graph=False runs the same launches eagerly (no capture).

    Returns dict(count (B,) int32, kept (B,) int32, cls (B, M) int32, R (B, M, 3, 3) fp64, t (B, M, 3) fp64, conf (B, M) det_conf,
    cls_conf (B, M), keypoints_px (B, M, 9, 2), corners_px (B, M, 9, 2)): device tensors, or numpy with to_host=True."""

    def __init__(self, model, objects, K, frame_size=(640, 480), shape=None, batch=1, conf_thresh=None, nms_thresh=0.4, max_instances=32,
                 graph=True, max_graphs=4):
        self.num_anchors = int(getattr(model, "num_anchors", 0))
        if self.num_anchors < 1:
            raise SspError("InstancePosePredictor needs a model with a region head")
        nC = int(model.num_classes)
        if not isinstance(objects, dict):
            objects = {0: objects}
        if not objects:
            raise SspError("objects must be a non-empty {class id: corners3D} dict")
        ids = sorted(objects)
        for c in ids:
            if isinstance(c, bool) or not isinstance(c, (int, np.integer)) or not 0 <= c < nC:
                raise SspError("class id %r is not in [0, %d)" % (c, nC))
        pts = [self._box_points(objects[c]) for c in ids]
        nms_thresh = float(nms_thresh)
        if not 0.0 <= nms_thresh <= 1.0:
            raise SspError("nms_thresh must be in [0, 1], got %r" % nms_thresh)
        if isinstance(max_instances, bool) or not isinstance(max_instances, (int, np.integer)) or not 1 <= max_instances <= MAX_INSTANCES:
            raise SspError("max_instances must be an integer in [1, %d], got %r" % (MAX_INSTANCES, max_instances))
        if conf_thresh is None:
            if "conf_thresh" not in model.blocks[0]:
                raise SspError("the model's cfg has no conf_thresh in its [net] block: pass conf_thresh")
            conf_thresh = float(model.blocks[0]["conf_thresh"])
        self.conf_thresh, self.nms_thresh, self.max_instances = float(conf_thresh), nms_thresh, int(max_instances)
        if shape is None:
            shape = (model.test_width, model.test_height) if self.num_anchors == 1 else (model.width, model.height)
        super().__init__(model, K, frame_size, shape, batch, graph, max_graphs)
        h, w = self.out_hw
        if h * w * self.num_anchors > MAX_ENTRIES:
            raise SspError("network shape %dx%d gives a %dx%d grid of %d anchors: more than the %d entries the detect kernel holds"
                           % (self.shape[0], self.shape[1], h, w, self.num_anchors, MAX_ENTRIES))
        dev, Q = self.device, len(ids)
        self.classes = np.array(ids, dtype=np.int64)
        self._cls_host = np.array(ids, dtype=np.int32)                            # copied into the detect kernel's launch
        table = np.zeros((nC, 9, 3), np.float32)                                  # PnP points by class id (unrequested: zeros)
        slot_of = np.zeros(nC, np.int64)                                          # class id -> its column block in the projection
        for q, (c, P) in enumerate(zip(ids, pts)):
            table[c] = P.T
            slot_of[c] = q
        self._P3_table = torch.from_numpy(table).to(dev)
        self._slot_of = torch.from_numpy(slot_of).to(dev)
        X = np.concatenate([np.concatenate([P, np.ones((1, 9))], 0) for P in pts], 1)                     # (4, 9Q)
        self._X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
        self._slots = torch.arange(self.max_instances, device=dev)
        self._rows = torch.arange(self.batch * self.max_instances, device=dev)
        self._zero = torch.zeros((), dtype=torch.float32, device=dev)
        self._Q = Q

    def _head_buffers(self, c):
        dev, B, K, M, Q = self.device, self.batch, self.num_keypoints, self.max_instances, self._Q
        c.boxes = torch.empty(B, M, 2 * K + 3, dtype=torch.float32, device=dev)
        c.cls = torch.empty(B, M, dtype=torch.int32, device=dev)
        c.cls0 = torch.empty(B, M, dtype=torch.int32, device=dev)
        c.count = torch.empty(B, dtype=torch.int32, device=dev)
        c.kept = torch.empty(B, dtype=torch.int32, device=dev)
        c.valid = torch.empty(B, M, dtype=torch.bool, device=dev)
        c.kp = torch.empty(B, M, K, 2, dtype=torch.float32, device=dev)
        c.P3 = torch.empty(B * M, K, 3, dtype=torch.float32, device=dev)
        c.R = torch.empty(B, M, 3, 3, dtype=torch.float64, device=dev)
        c.t = torch.empty(B, M, 3, dtype=torch.float64, device=dev)
        c.Rt = torch.empty(B, M, 3, 4, dtype=torch.float64, device=dev)
        c.proj = torch.empty(B * M, 2, Q * K, dtype=torch.float32, device=dev)
        c.corners = torch.empty(B, M, K, 2, dtype=torch.float32, device=dev)

    def _head(self, c, s):
        self._detect(c, s)
        self._solve(c, s)
        self._project(c, s)

    def _detect(self, c, s):
        B, K, M, Q = self.batch, self.num_keypoints, self.max_instances, self._Q
        Wf, Hf = c.frame
        h, w = c.logits.shape[2:]
        call("ssp_detect_instances", ptr(c.logits), B, K, self.num_classes, self.num_anchors, h, w, C.c_void_p(self._cls_host.ctypes.data),
             Q, self.conf_thresh, self.nms_thresh, M, float(Wf), float(Hf), ptr(c.boxes), ptr(c.cls), ptr(c.kp), ptr(c.count), ptr(c.kept), s)
        torch.clamp(c.cls, min=0, out=c.cls0)                  # empty slots hold -1: any in-range index will do, PnP skips them
        torch.index_select(self._P3_table, 0, c.cls0.view(-1), out=c.P3)

    def _solve(self, c, s):
        call("ssp_pnp_batched_counted", ptr(c.P3), ptr(c.kp), ptr(self._K32), self.num_keypoints, self.batch, self.max_instances,
             ptr(c.count), 20, ptr(c.R), ptr(c.t), s)

    def _project(self, c, s):
        B, K, M, Q = self.batch, self.num_keypoints, self.max_instances, self._Q
        c.Rt[..., :3].copy_(c.R)
        c.Rt[..., 3].copy_(c.t)
        # every requested class's points under every slot's pose (each point is projected on its own, so a slot's own columns are
        # what ssp_project_points gives for its class's (4, 9) points alone); slot (b, m) keeps the columns of its class
        call("ssp_project_points", ptr(self._X), 4, Q * K, ptr(c.Rt), ptr(self._K64), B * M, ptr(c.proj), s)
        own = c.proj.view(B * M, 2, Q, K)[self._rows, :, self._slot_of[c.cls0.view(-1)]]          # (B*M, 2, K)
        torch.lt(self._slots, c.count.unsqueeze(1), out=c.valid)
        torch.where(c.valid.view(B, M, 1, 1), own.view(B, M, 2, K).transpose(2, 3), self._zero, out=c.corners)

    def _outputs(self, c):
        K = self.num_keypoints
        return dict(count=c.count, kept=c.kept, cls=c.cls, R=c.R, t=c.t, conf=c.boxes[..., 2 * K], cls_conf=c.boxes[..., 2 * K + 1],
                    keypoints_px=c.kp, corners_px=c.corners)


class TrackingPosePredictor(InstancePosePredictor):
    """InstancePosePredictor whose instances keep their identity across calls: each row b of a batch is its own camera stream, and
    each instance is matched to a track of its class (utils_multi.InstanceTracker, rules: csrc/track_core.h).  A matched instance's
    PnP starts Levenberg-Marquardt from its track's last pose (cv2.solvePnP's useExtrinsicGuess), the others are solved cold.
    No motion model: a track is matched against its last corner rectangle, and the guess is its last pose.

    max_tracks in [1, 256] track slots per stream, match_iou in [0, 1] (a match needs IoU > match_iou), max_misses >= 0 (a track
    dies after max_misses + 1 frames in a row without a match); the other arguments are InstancePosePredictor's.

    Returns InstancePosePredictor's dict plus track_id (B, M) int32 (-1 in empty and untracked slots) and warm (B, M) bool (the
    slot's solve started from its track's pose).  The track state is shared by every frame size and source (one set of device
    arrays, zeroed in place by reset); the warm-up runs before a graph capture do not advance it."""

    def __init__(self, model, objects, K, frame_size=(640, 480), shape=None, batch=1, conf_thresh=None, nms_thresh=0.4, max_instances=32,
                 max_tracks=64, match_iou=0.3, max_misses=5, graph=True, max_graphs=4):
        check_track_args(max_tracks, match_iou, max_misses)
        super().__init__(model, objects, K, frame_size, shape, batch, conf_thresh, nms_thresh, max_instances, graph, max_graphs)
        if not isinstance(objects, dict):
            objects = {0: objects}
        self._tracker = InstanceTracker(objects, K, self.num_classes, self.num_anchors, self.frame_size, self.batch, self.conf_thresh,
                                        self.nms_thresh, self.max_instances, max_tracks, match_iou, max_misses, device=self.device)
        self.max_tracks, self.match_iou, self.max_misses = self._tracker.max_tracks, self._tracker.match_iou, self._tracker.max_misses

    def reset(self, streams=None):
        """forget the tracks of the given streams (default: all); their ids start again from 0"""
        with torch.cuda.device(self.device):
            self._tracker.reset(streams)

    def tracks(self, to_host=False):
        """the alive tracks (utils_multi.InstanceTracker.tracks): stream, slot, id, cls, misses, hits, rvec, R, t, rect"""
        with torch.cuda.device(self.device):
            return self._tracker.tracks(to_host)

    def _head_buffers(self, c):
        super()._head_buffers(c)
        self._tracker.buffers(c)

    def _solve(self, c, s):
        self._tracker.solve(c, s, c.P3, self._K32)

    def _capture(self, c, warmup=2):
        saved = self._tracker.snapshot()          # the warm-up runs advance the tracks: put them back before the first replay
        super()._capture(c, warmup)
        self._tracker.restore(saved)

    def _outputs(self, c):
        return dict(super()._outputs(c), track_id=c.track_id, warm=c.warm)


# ---------------------------------------------------------------------------------------------- command line
def camera_from_any_data_cfg(datacfg):
    """-> (mesh path or None, K (3, 3) float64, (width, height)) from a single-object .data file (mesh, width, height) or a
    multi-object one (im_width, im_height); fx, fy, u0, v0 in both"""
    from .utils_host import read_data_cfg
    o = read_data_cfg(datacfg)
    try:
        fx, fy, u0, v0 = (float(o[k]) for k in ("fx", "fy", "u0", "v0"))
        if "im_width" in o or "im_height" in o:
            size = (int(o["im_width"]), int(o["im_height"]))
        else:
            size = (int(o["width"]), int(o["height"]))
    except KeyError as e:
        raise SspError("%s has no %s entry" % (datacfg, e))
    K = np.array([[fx, 0.0, u0], [0.0, fy, v0], [0.0, 0.0, 1.0]])
    return o.get("mesh"), K, size


def parse_args(argv=None):
    """the command line, checked before any model is built: raises SspError for a bad --object, --nms-thresh, --max-instances,
    --match-iou, --max-misses or --max-tracks"""
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
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    if not 0.0 <= a.nms_thresh <= 1.0:
        raise SspError("--nms-thresh must be in [0, 1], got %r" % a.nms_thresh)
    if not 1 <= a.max_instances <= MAX_INSTANCES:
        raise SspError("--max-instances must be in [1, %d], got %d" % (MAX_INSTANCES, a.max_instances))
    if not 0.0 <= a.match_iou <= 1.0:
        raise SspError("--match-iou must be in [0, 1], got %r" % a.match_iou)
    if a.max_misses < 0:
        raise SspError("--max-misses must be >= 0, got %d" % a.max_misses)
    if not 1 <= a.max_tracks <= MAX_TRACKS:
        raise SspError("--max-tracks must be in [1, %d], got %d" % (MAX_TRACKS, a.max_tracks))
    a.objects = parse_objects(a.object) if a.object else None
    return a


def _region_anchors(modelcfg):
    from .cfg import parse_cfg
    for b in parse_cfg(modelcfg):
        if b["type"] == "region":
            return int(b.get("num", 1))
    raise SspError("%s has no [region] block" % modelcfg)


def main(argv=None):
    a = parse_args(argv)
    from .utils import get_3D_corners
    from .utils_host import read_ply_vertices
    mesh, K, size = camera_from_any_data_cfg(a.datacfg)
    meshes = a.objects
    if meshes is None:
        if not mesh:
            raise SspError("%s has no mesh entry: give --object CLASS=MESH.ply" % a.datacfg)
        meshes = {0: mesh}
    objects = {}
    for c, path in meshes.items():
        V = read_ply_vertices(path)
        objects[c] = get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    if _region_anchors(a.modelcfg) > 1:
        from .darknet_multi import Darknet
    else:
        from .darknet import Darknet
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    if a.track:
        pred = TrackingPosePredictor(model, objects, K, frame_size=size, nms_thresh=a.nms_thresh, max_instances=a.max_instances,
                                     max_tracks=a.max_tracks, match_iou=a.match_iou, max_misses=a.max_misses)
    else:
        pred = InstancePosePredictor(model, objects, K, frame_size=size, nms_thresh=a.nms_thresh, max_instances=a.max_instances)
    rows = {k: [] for k in ROW_KEYS + (("track_id",) if a.track else ())}
    image = []
    for i, path in enumerate(a.images):
        with open(path, "rb") as f:
            data = f.read()
        if data[:2] == b"\xff\xd8":
            r = pred([data], to_host=True)
        else:
            from PIL import Image
            r = pred(np.asarray(Image.open(path).convert("RGB"))[None], to_host=True)
        n = int(r["count"][0])
        image += [i] * n
        for k in rows:
            rows[k].append(r[k][0, :n])
    np.savez(a.out, paths=np.array(a.images), image=np.array(image, dtype=np.int64), **{k: np.concatenate(v) for k, v in rows.items()})
    print("%d images -> %d detections -> %s" % (len(a.images), len(image), a.out))


if __name__ == "__main__":
    main()
