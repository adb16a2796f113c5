"""Camera frames -> 6-D object poses in one CUDA graph replay (the per-image chain of reference valid.py:95-153, what valid.ipynb
draws).

    pred = PosePredictor(model, corners3D, K, frame_size=(640, 480), shape=(model.test_width, model.test_height), batch=1)
    r = pred(frames)            # (B, H, W, 3) uint8 numpy array / CUDA tensor, or a list of B JPEG files' bytes
    r["R"], r["t"], r["conf"], r["keypoints_px"], r["corners_px"]       # device tensors; pred(frames, to_host=True) -> numpy

Per frame: Image.resize(shape) (BICUBIC, byte-identical to Pillow, ssp_aug_resize_u8) and ToTensor; the eval-mode forward
(running-statistics BN) with split-K for the layers that have few output tiles (Engine.forward(split_k=True)); the arg-max
decode of the frame's own best cell (ssp_region_decode_argmax, only_objectness=1); keypoints x frame size; PnP of the 9 points
[0; corners3D[:3]] (ssp_pnp_batched, cv2.solvePnP's ITERATIVE solve); projection of the centroid and the 8 box corners under
the predicted pose (ssp_project_points).

The chain is captured once per (frame size, frame source) as one CUDA graph (a small LRU keeps the last few), after eager
warm-up calls that make every first-use allocation.  Constants (3-D points, K) live on the device; host frames go through one
pinned staging buffer whose copy to the device is part of the replay; CUDA frames are copied device-to-device into the static
input; JPEG bytes are decoded by jpeg.GpuJpegDecoder before the replay (its status read-back synchronises, so it stays
outside the graph).  The graph reads the engine's packed weight planes and the BN running statistics in place: a replay sees
load_weights / optimiser updates (the planes are re-packed before the replay when the weights changed), and the chain is
re-captured if the parameters were moved to new memory.  The predictor owns its activation buffers, so model(x) or a training
step between two replays cannot write into memory the graph replays.

Returned device tensors are the predictor's static outputs: the next call overwrites them.  Everything but the head's selection
lives in _FramePredictor, which predict_multi.MultiPosePredictor and predict_instances.InstancePosePredictor share.

Command line: python -m singleshotpose_b200.predict --datacfg cfg/ape.data --modelcfg cfg/yolo-pose.cfg --weightfile w.weights
              --out poses.npz img1.jpg img2.jpg ...
"""
from __future__ import annotations

import argparse
import collections

import numpy as np
import torch

from ._lib import SspError, call, load, ptr, stream_ptr
from .engine import Buffers
from .image import BICUBIC
from .utils import (camera_distortion, check_pnp_args, consensus_subsets, consensus_work_bytes, distortion_tensor, inlier_bits,
                    keypoint_bits, object_table)


class _Chain:
    """static buffers (and the graph) of one (frame size, frame source); the head's buffers come from pred._slot_buffers and
    pred._head_buffers"""

    def __init__(self, pred, Wf, Hf, src):
        dev, B = pred.device, pred.batch
        W, H = pred.shape
        self.frame, self.src, self.graph = (Wf, Hf), src, None
        self.u8 = torch.zeros(B, Hf, Wf, 3, dtype=torch.uint8, device=dev)
        self.pin = torch.zeros(B, Hf, Wf, 3, dtype=torch.uint8).pin_memory() if src == "host" else None
        self.copied = torch.cuda.Event()          # the replay that last read `pin` has been enqueued after this
        self.rs = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
        self.x = torch.empty(B, 3, H, W, dtype=torch.float32, device=dev)
        nb = int(load().ssp_aug_resize_work_bytes(Wf, Hf, W, H, BICUBIC))
        if nb < 0:
            raise SspError("frame size %dx%d cannot be resized to %dx%d" % (Wf, Hf, W, H))
        self.work = torch.empty(nb + 16, dtype=torch.uint8, device=dev)
        self.scale = torch.tensor([Wf, Hf], dtype=torch.float32, device=dev)
        self.logits = None
        pred._slot_buffers(self)
        pred._head_buffers(self)


class _FramePredictor:
    """What every pose predictor shares: input checks and the pinned staging buffer; JPEG, host and device frame sources; resize
    and ToTensor; the split-K eval forward on private Buffers; the per-(frame size, source) LRU of captured graphs; the re-pack
    and re-capture after the weights change; and the pose tail of the head.

    Each frame's head selects into S slots.  With slots=None there is one slot per requested class and slot q holds the q-th
    (PosePredictor: S = 1; MultiPosePredictor: S = Q).  With slots=M the selection detects: it fills c.cls, a device c.count and
    each slot's PnP points c.P3 (utils_multi.detect_slots), and slots >= count[b] of frame b are empty.  The tail is _solve (PnP
    of every slot: plain, counted or consensus) and _project (each slot's class's centroid and corners under its pose).  With lens
    distortion coefficients (dist_coeffs, utils.camera_distortion) both are cv2's distorted model: the PnP fits the raw keypoints
    (ssp_pnp_dist / ssp_pnp_consensus_dist) and the corners land on the raw frame (ssp_project_points_dist).  The coefficients are
    a device constant read by the replay; the selection (NMS, track association) works on the raw keypoints either way.
    A subclass supplies the rest: _head_buffers(chain) allocates its selection's static buffers, _head(chain, stream) launches
    the selection after the forward and then the tail, and _outputs(chain) names the returned tensors."""

    def __init__(self, model, objects, K, frame_size, shape, batch, graph, max_graphs, pnp, reproj_thresh, slots=None, dist_coeffs=None):
        name = type(self).__name__
        if not torch.cuda.is_available():
            raise SspError("%s needs a CUDA device (no CPU fallback)" % name)
        self.model, self.eng = model, model._engine
        self.num_keypoints, self.num_classes = int(model.num_keypoints), int(model.num_classes)
        if self.num_keypoints != 9:
            raise SspError("%s solves PnP on the centroid + 8 box corners: the model must have 9 keypoints, not %d" % (name, self.num_keypoints))
        self.shape = (int(shape[0]), int(shape[1]))
        self.batch = int(batch)
        if self.batch < 1:
            raise SspError("batch must be >= 1")
        self.frame_size = (int(frame_size[0]), int(frame_size[1]))
        self.use_graph, self.max_graphs = bool(graph), int(max_graphs)
        dev = self.eng.device if self.eng.device is not None else torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.eng.materialize(dev)
        self.classes, points, Km = object_table(objects, self.num_classes, K)
        dist = camera_distortion(dist_coeffs)
        self.dist_coeffs = dist                                                  # (8,) float64, or None: no distortion
        self._dist = None if dist is None else distortion_tensor(dist, dev)
        self._cls_host = self.classes.astype(np.int32)                          # copied into the selection's launch
        self._K32 = torch.from_numpy(np.ascontiguousarray(Km, dtype=np.float32)).to(dev)       # PnP takes float32 K (valid.py:147)
        self._K64 = torch.from_numpy(np.ascontiguousarray(Km)).to(dev)
        P3 = points[self.classes]                                                # (Q, 9, 3) PnP points of the requested classes
        Q, B = len(P3), self.batch
        # row-major copies: the kernels read raw pointers, and numpy keeps a transposed input's column-major order through
        # concatenate / astype
        X = np.concatenate([P3.reshape(-1, 3).T, np.ones((1, 9 * Q))], 0)
        self._X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)                 # (4, 9Q)
        self.pnp, self.reproj_thresh = check_pnp_args(pnp, reproj_thresh)
        self._subsets = consensus_subsets(P3) if self.pnp == "consensus" else None
        self._bits = keypoint_bits(self.num_keypoints, dev)
        self.num_slots, self._detects = (Q if slots is None else int(slots)), slots is not None
        if self._detects:
            slot_of = np.zeros(self.num_classes, np.int64)                       # class id -> its column block in the projection
            slot_of[self.classes] = np.arange(Q)
            self._P3_table = torch.from_numpy(points.astype(np.float32)).to(dev)         # PnP points by class id
            self._slot_of = torch.from_numpy(slot_of).to(dev)
            self._slot_index = torch.arange(self.num_slots, device=dev)
            self._rows = torch.arange(B * self.num_slots, device=dev)
            self._zero = torch.zeros((), dtype=torch.float32, device=dev)
        else:
            self._P3 = torch.from_numpy(np.repeat(P3[None], B, 0).astype(np.float32)).to(dev)   # (B, Q, 9, 3): one per slot
        W, H = self.shape
        self.out_hw = self.eng.spatial(self.eng.layers[-1], H, W)               # raises for a shape off the pooling pyramid
        self._bufs = Buffers(self.eng, self.batch, H, W, False, split_k=True)
        self._chains = collections.OrderedDict()
        self._sig = None
        self._jpeg = None
        self._last = None

    # ------------------------------------------------------------------ the pose tail: slots -> PnP -> projection
    def _slot_buffers(self, c):
        dev, B, S, K, Q = self.device, self.batch, self.num_slots, self.num_keypoints, len(self.classes)
        c.kp = torch.empty(B, S, K, 2, dtype=torch.float32, device=dev)
        c.R = torch.empty(B, S, 3, 3, dtype=torch.float64, device=dev)
        c.t = torch.empty(B, S, 3, dtype=torch.float64, device=dev)
        c.Rt = torch.empty(B, S, 3, 4, dtype=torch.float64, device=dev)
        c.proj = torch.empty(B * S, 2, Q * K, dtype=torch.float32, device=dev)
        c.corners = torch.empty(B, S, K, 2, dtype=torch.float32, device=dev)
        if self._detects:
            c.valid = torch.empty(B, S, dtype=torch.bool, device=dev)
        else:
            c.P3, c.count = self._P3, None
        if self.pnp == "consensus":
            c.params = torch.empty(B, S, 6, dtype=torch.float64, device=dev)
            c.inl_mask = torch.empty(B, S, dtype=torch.int32, device=dev)
            c.hyp = torch.empty(B, S, dtype=torch.int32, device=dev)
            c.inliers = torch.empty(B, S, K, dtype=torch.bool, device=dev)
            wb = consensus_work_bytes(K, len(self._subsets), B * S)
            c.pnp_work = torch.empty(max(wb, 8) // 8, dtype=torch.float64, device=dev)

    def _solve(self, c, s):
        """PnP of every slot's keypoints c.kp against its points c.P3 with the fp32 K into c.R, c.t (the consensus solve: also
        c.params, c.inliers, c.hyp); with a device c.count, frame b solves its first count[b] slots and the others get zeros"""
        B, S, K = self.batch, self.num_slots, self.num_keypoints
        if self.pnp == "consensus":
            if self._dist is None:
                call("ssp_pnp_consensus", ptr(c.P3), 0, ptr(c.kp), ptr(self._K32), K, B, S, ptr(c.count), self._subsets.ctypes.data,
                     len(self._subsets), self.reproj_thresh, 20, ptr(c.R), ptr(c.t), ptr(c.params), ptr(c.inl_mask), ptr(c.hyp),
                     ptr(c.pnp_work), c.pnp_work.numel() * 8, s)
            else:
                call("ssp_pnp_consensus_dist", ptr(c.P3), 0, ptr(c.kp), ptr(self._K32), ptr(self._dist), K, B, S, ptr(c.count),
                     self._subsets.ctypes.data, len(self._subsets), self.reproj_thresh, 20, ptr(c.R), ptr(c.t), ptr(c.params),
                     ptr(c.inl_mask), ptr(c.hyp), ptr(c.pnp_work), c.pnp_work.numel() * 8, s)
            inlier_bits(c.inl_mask, self._bits, out=c.inliers)
        elif self._dist is not None:                # plain or counted (c.count None: every slot)
            call("ssp_pnp_dist", ptr(c.P3), 0, ptr(c.kp), ptr(self._K32), ptr(self._dist), K, B, S, ptr(c.count), None, None, 20, ptr(c.R),
                 ptr(c.t), None, None, s)
        elif c.count is None:
            call("ssp_pnp_batched", ptr(c.P3), 0, ptr(c.kp), ptr(self._K32), K, B * S, 20, ptr(c.R), ptr(c.t), None, s)
        else:
            call("ssp_pnp_batched_counted", ptr(c.P3), ptr(c.kp), ptr(self._K32), K, B, S, ptr(c.count), 20, ptr(c.R), ptr(c.t), s)

    def _project(self, c, s):
        """c.corners: each slot's class's 9 points projected under the slot's pose (zero in empty slots)"""
        B, S, K, Q = self.batch, self.num_slots, self.num_keypoints, len(self.classes)
        c.Rt[..., :3].copy_(c.R)
        c.Rt[..., 3].copy_(c.t)
        # every requested class's points under every slot's pose (each point is projected on its own, so a slot's own columns are
        # what ssp_project_points gives for its class's (4, 9) points alone); each slot keeps the columns of its class
        if self._dist is None:
            call("ssp_project_points", ptr(self._X), 4, Q * K, ptr(c.Rt), ptr(self._K64), B * S, ptr(c.proj), s)
        else:
            call("ssp_project_points_dist", ptr(self._X), 4, Q * K, ptr(c.Rt), ptr(self._K64), ptr(self._dist), B * S, ptr(c.proj), s)
        if not self._detects:                      # slot q: class q
            c.corners.copy_(torch.diagonal(c.proj.view(B, S, 2, Q, K), dim1=1, dim2=3).permute(0, 3, 2, 1))
            return
        own = c.proj.view(B * S, 2, Q, K)[self._rows, :, self._slot_of[c.cls0.view(-1)]]          # (B*S, 2, K)
        torch.lt(self._slot_index, c.count.unsqueeze(1), out=c.valid)
        torch.where(c.valid.view(B, S, 1, 1), own.view(B, S, 2, K).transpose(2, 3), self._zero, out=c.corners)

    def _consensus_outputs(self, c):
        return dict(inliers=c.inliers, hyp=c.hyp) if self.pnp == "consensus" else {}

    # ------------------------------------------------------------------ inputs
    def _check(self, frames):
        """-> (source kind, array / tensor); raises SspError before anything is launched"""
        B = self.batch
        if isinstance(frames, (list, tuple)):
            if len(frames) != B or not all(isinstance(f, (bytes, bytearray, memoryview)) for f in frames):
                raise SspError("a list of frames must hold %d JPEG files' bytes" % B)
            from .jpeg import read_jpeg_size
            blobs = [bytes(f) for f in frames]
            sizes = [read_jpeg_size(b) for b in blobs]
            if any(s is None for s in sizes):
                raise SspError("frame %d is not a JPEG file" % [s is None for s in sizes].index(True))
            if len(set(sizes)) != 1:
                raise SspError("the frames of one call must have one size, got %s" % sorted(set(sizes)))
            return "jpeg", blobs
        if isinstance(frames, np.ndarray):
            kind = "host"
        elif torch.is_tensor(frames):
            if not frames.is_cuda:
                raise SspError("frames given as a torch tensor must be on the GPU (pass host frames as a numpy array)")
            kind = "device"
        else:
            raise SspError("frames must be a (B, H, W, 3) uint8 numpy array or CUDA tensor, or a list of JPEG bytes; got %s" % type(frames).__name__)
        if frames.dtype != (np.uint8 if kind == "host" else torch.uint8):
            raise SspError("frames must be uint8, got %s" % frames.dtype)
        if frames.ndim != 4 or frames.shape[3] != 3:
            raise SspError("frames must be (B, H, W, 3) RGB, got %s" % (tuple(frames.shape),))
        if frames.shape[0] != B:
            raise SspError("this predictor takes batches of %d frames, got %d" % (B, frames.shape[0]))
        if frames.shape[1] < 1 or frames.shape[2] < 1:
            raise SspError("empty frames %s" % (tuple(frames.shape),))
        return kind, frames

    # ------------------------------------------------------------------ the chain
    def _body(self, c, events=None):
        """every launch of one prediction, in stream order; events (4 CUDA events, eager runs only) bracket image / forward / head"""
        s = stream_ptr()
        B = self.batch
        W, H = self.shape
        Wf, Hf = c.frame
        if events:
            events[0].record()
        if c.src == "host":
            c.u8.copy_(c.pin, non_blocking=True)
        for i in range(B):
            call("ssp_aug_resize_u8", ptr(c.u8[i]), Wf, Hf, 0, 0, Wf, Hf, ptr(c.rs[i]), W, H, BICUBIC, ptr(c.work), c.work.numel(), s)
            call("ssp_aug_to_tensor_u8", ptr(c.rs[i]), H * W, ptr(c.x[i]), s)
        if events:
            events[1].record()
        c.logits, _b, _g = self.eng.forward(c.x, False, False, split_k=True, buffers=self._bufs)
        if events:
            events[2].record()
        self._head(c, s)
        if events:
            events[3].record()

    def _capture(self, c, warmup=2):
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):               # first-use allocations, cudaFuncSetAttribute, tensor maps: all before capture
                self._body(c)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._body(c)
        c.graph = g

    def _weights_sig(self):
        eng = self.eng
        stats = tuple(t.data_ptr() for _c, bn in eng.conv_modules() if bn is not None for t in (bn.running_mean, bn.running_var))
        return (eng.flat_params.data_ptr(), tuple(t.data_ptr() for t in eng.w_hi + eng.w_lo if t is not None)) + stats

    def _ensure_current(self):
        eng = self.eng
        eng.materialize(self.device)              # no-op unless the parameters were replaced
        eng.pack_weights()                        # no-op unless the weights changed since the last pack
        sig = self._weights_sig()
        if sig != self._sig:                      # parameters or running statistics moved: the captured addresses are stale
            self._chains.clear()
            self._sig = sig

    def _chain(self, Wf, Hf, src):
        key = (Wf, Hf, src)
        c = self._chains.get(key)
        if c is None:
            c = _Chain(self, Wf, Hf, src)
            self._chains[key] = c
            while len(self._chains) > self.max_graphs:
                self._chains.popitem(last=False)
        self._chains.move_to_end(key)
        return c

    def __call__(self, frames, to_host=False, events=None):
        kind, arr = self._check(frames)
        with torch.cuda.device(self.device):
            if kind == "jpeg":
                if self._jpeg is None:
                    from .jpeg import GpuJpegDecoder
                    self._jpeg = GpuJpegDecoder(self.device)
                arr, kind = torch.stack(self._jpeg(arr)), "device"
            Hf, Wf = int(arr.shape[1]), int(arr.shape[2])
            self._ensure_current()
            c = self._chain(Wf, Hf, kind)
            if kind == "host":
                c.copied.synchronize()            # the previous replay's copy out of the staging buffer has run
                np.copyto(c.pin.numpy(), arr, casting="no")
            else:
                c.u8.copy_(arr)
            if self.use_graph and not events:
                if c.graph is None:
                    self._capture(c)
                c.graph.replay()
            else:
                self._body(c, events)
            if kind == "host":
                c.copied.record()
            self._last = c
        out = self._outputs(c)
        if to_host:
            return {k: v.cpu().numpy() for k, v in out.items()}
        return out

    @property
    def logits(self):
        """raw network output (B, 2K+1+C, h, w) of the last call"""
        return None if self._last is None else self._last.logits

    @property
    def input(self):
        """(B, 3, H, W) float32 network input of the last call (resized + ToTensor)"""
        return None if self._last is None else self._last.x


class PosePredictor(_FramePredictor):
    """model: a singleshotpose_b200.Darknet (single-object yolo-pose head, 9 keypoints).  corners3D: (3|4, 8) box corners of the
    mesh (utils.get_3D_corners); K: (3, 3) camera matrix; frame_size: (width, height) of the camera frames (other sizes are
    accepted and captured separately); shape: network input (width, height), default the cfg's test size; batch: frames per call.
    graph=False runs the same launches eagerly (no capture).
    pnp="consensus" solves each pose with the consensus PnP (utils.pnp_consensus_batched): a pose that survives one or two wrong
    keypoints, with inlier keypoints within reproj_thresh frame pixels; the outputs then add inliers (B, 9) bool and hyp (B,) int32.
    pnp="plain" (default) is the all-point solve.
    dist_coeffs: the camera's OpenCV distortion coefficients (k1, k2, p1, p2[, k3[, k4, k5, k6]]): the pose is cv2.solvePnP(...,
    distCoeffs) of the raw keypoints and corners_px is cv2.projectPoints with them, on the raw frame; None or all zeros: no distortion."""

    def __init__(self, model, corners3D, K, frame_size=(640, 480), shape=None, batch=1, graph=True, max_graphs=4, pnp="plain",
                 reproj_thresh=8.0, dist_coeffs=None):
        super().__init__(model, {0: corners3D}, K, frame_size, shape if shape is not None else (model.test_width, model.test_height),
                         batch, graph, max_graphs, pnp, reproj_thresh, dist_coeffs=dist_coeffs)

    def _head_buffers(self, c):
        dev, B, K = self.device, self.batch, self.num_keypoints
        c.boxes = torch.empty(B, 2 * K + 3, dtype=torch.float32, device=dev)
        c.conf = torch.empty(B, dtype=torch.float32, device=dev)

    def _head(self, c, s):
        B, K = self.batch, self.num_keypoints
        h, w = c.logits.shape[2:]
        call("ssp_region_decode_argmax", ptr(c.logits), B, K, self.num_classes, h, w, 1, ptr(c.boxes), ptr(c.conf), None, s)
        torch.mul(c.boxes[:, :2 * K].view(B, 1, K, 2), c.scale, out=c.kp)
        self._solve(c, s)
        self._project(c, s)

    def _outputs(self, c):
        one = {k: v[:, 0] for k, v in self._consensus_outputs(c).items()}          # the one slot of each frame
        return dict(R=c.R[:, 0], t=c.t[:, 0], conf=c.conf, keypoints_px=c.kp[:, 0], corners_px=c.corners[:, 0], **one)


# ---------------------------------------------------------------------------------------------- command line
CONSENSUS_KEYS = {"plain": (), "consensus": ("inliers", "hyp")}          # the .npz columns each --pnp adds
SIZE_KEYS = (("width", "height"),)                                      # the frame size entries of a single-object .data file


def add_pnp_args(ap):
    ap.add_argument("--pnp", choices=("plain", "consensus"), default="plain",
                    help="consensus: a pose that survives wrong keypoints (PnP over keypoint subsets); adds inliers and hyp columns")
    ap.add_argument("--reproj-thresh", type=float, default=8.0, help="inlier threshold of --pnp consensus, frame pixels")


def add_dist_arg(ap):
    ap.add_argument("--dist", type=float, nargs="+", metavar="K",
                    help="the camera's OpenCV distortion coefficients k1 k2 p1 p2 [k3 [k4 k5 k6]] (cv2.calibrateCamera's distCoeffs); "
                         "overrides the .data file's dist entry.  End the list with -- when the images follow it")


def camera_dist(args):
    """the distortion coefficients of a command line: --dist if given, else the .data file's optional `dist = k1 k2 p1 p2 [k3 [k4 k5
    k6]]` entry (the flag's values, separated by spaces or commas) -> utils.camera_distortion's (8,) float64 array, or None for
    neither (or all zeros).  SspError for a count other than 4, 5 or 8 or a value that is not a finite number."""
    if args.dist is not None:
        return camera_distortion(args.dist)
    from .utils_host import read_data_cfg
    text = read_data_cfg(args.datacfg).get("dist")
    if text is None:
        return None
    try:
        values = [float(v) for v in text.replace(",", " ").split()]
    except ValueError:
        raise SspError("%s: dist must be numbers k1 k2 p1 p2 [k3 [k4 k5 k6]], got %r" % (args.datacfg, text))
    return camera_distortion(values)


def read_camera(datacfg, size_keys):
    """-> (mesh path or None, K (3, 3) float64, (width, height)) from a .data file (utils.py read_data_cfg; valid.py:26-35,
    valid_multi.py:30-35): fx, fy, u0, v0, and the size from the first (width key, height key) pair of size_keys of which the
    file has either key (else the last pair)"""
    from .utils_host import read_data_cfg
    o = read_data_cfg(datacfg)
    wk, hk = next((p for p in size_keys if p[0] in o or p[1] in o), size_keys[-1])
    try:
        fx, fy, u0, v0 = (float(o[k]) for k in ("fx", "fy", "u0", "v0"))
        size = (int(o[wk]), int(o[hk]))
    except KeyError as e:
        raise SspError("%s has no %s entry" % (datacfg, e))
    K = np.array([[fx, 0.0, u0], [0.0, fy, v0], [0.0, 0.0, 1.0]])
    return o.get("mesh"), K, size


def mesh_corners(path):
    """(4, 8) box corners (utils.get_3D_corners) of the vertices of a PLY mesh"""
    from .utils import get_3D_corners
    from .utils_host import read_ply_vertices
    V = read_ply_vertices(path)
    return get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)


def predict_files(pred, paths):
    """yields pred's host result for each image file, one frame per call: JPEG files go to the GPU decoder, others through Pillow"""
    for path in paths:
        with open(path, "rb") as f:
            data = f.read()
        if data[:2] == b"\xff\xd8":
            yield pred([data], to_host=True)
        else:
            from PIL import Image
            yield pred(np.asarray(Image.open(path).convert("RGB"))[None], to_host=True)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.predict",
                                 description="6-D pose of the object of a trained single-object model in each image")
    ap.add_argument("--datacfg", required=True, help=".data file: mesh, fx fy u0 v0, width height")
    ap.add_argument("--modelcfg", required=True)
    ap.add_argument("--weightfile", required=True)
    ap.add_argument("--out", default="poses.npz")
    add_pnp_args(ap)
    add_dist_arg(ap)
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    check_pnp_args(a.pnp, a.reproj_thresh)
    dist = camera_dist(a)
    from .darknet import Darknet
    mesh, K, size = read_camera(a.datacfg, SIZE_KEYS)
    if mesh is None:
        raise SspError("%s has no mesh entry" % a.datacfg)
    corners3D = mesh_corners(mesh)
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    pred = PosePredictor(model, corners3D, K, frame_size=size, pnp=a.pnp, reproj_thresh=a.reproj_thresh, dist_coeffs=dist)
    res = {k: [] for k in ("R", "t", "conf", "keypoints_px", "corners_px") + CONSENSUS_KEYS[a.pnp]}
    for r in predict_files(pred, a.images):
        for k in res:
            res[k].append(r[k][0])
    np.savez(a.out, paths=np.array(a.images), **{k: np.stack(v) for k, v in res.items()})
    print("%d poses -> %s" % (len(a.images), a.out))


if __name__ == "__main__":
    main()
