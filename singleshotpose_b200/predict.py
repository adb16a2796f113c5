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

Returned device tensors are the predictor's static outputs: the next call overwrites them.  Everything but the head lives in
_FramePredictor, which predict_multi.MultiPosePredictor shares.

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
from .utils import check_pnp_args, consensus_subsets, consensus_work_bytes


class _Chain:
    """static buffers (and the graph) of one (frame size, frame source); the head's buffers come from pred._head_buffers"""

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
        pred._head_buffers(self)


class _FramePredictor:
    """What every pose predictor shares: input checks and the pinned staging buffer; JPEG, host and device frame sources; resize
    and ToTensor; the split-K eval forward on private Buffers; the per-(frame size, source) LRU of captured graphs; the re-pack
    and re-capture after the weights change.  A subclass supplies the head: _head_buffers(chain) allocates its static buffers,
    _head(chain, stream) launches it after the forward and _outputs(chain) names the returned tensors."""

    def __init__(self, model, K, frame_size, shape, batch, graph, max_graphs):
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
        Km = np.asarray(K, dtype=np.float64)
        if Km.shape != (3, 3):
            raise SspError("K must be (3, 3), got %s" % (Km.shape,))
        self._K32 = torch.from_numpy(np.ascontiguousarray(Km, dtype=np.float32)).to(dev)       # PnP takes float32 K (valid.py:147)
        self._K64 = torch.from_numpy(np.ascontiguousarray(Km)).to(dev)
        W, H = self.shape
        self.out_hw = self.eng.spatial(self.eng.layers[-1], H, W)               # raises for a shape off the pooling pyramid
        self._bufs = Buffers(self.eng, self.batch, H, W, False, split_k=True)
        self._chains = collections.OrderedDict()
        self._sig = None
        self._jpeg = None
        self._last = None

    # ------------------------------------------------------------------ PnP: plain (ssp_pnp_batched*) or consensus (ssp_pnp_consensus)
    def _init_pnp(self, pnp, reproj_thresh, point_sets):
        """point_sets: the (9, 3) PnP points of every class; all give the subset table (box points share their structure)"""
        self.pnp, self.reproj_thresh = check_pnp_args(pnp, reproj_thresh)
        self._subsets = consensus_subsets(np.stack(point_sets)) if self.pnp == "consensus" else None
        self._bits = torch.tensor([1 << i for i in range(self.num_keypoints)], dtype=torch.int32, device=self.device)

    def _consensus_buffers(self, c, lead):
        """the consensus solve's outputs and workspace for the problems of shape `lead` (nothing for the plain solve)"""
        if self.pnp != "consensus":
            return
        dev, K, n = self.device, self.num_keypoints, int(np.prod(lead))
        c.params = torch.empty(*lead, 6, dtype=torch.float64, device=dev)
        c.inl_mask = torch.empty(*lead, dtype=torch.int32, device=dev)
        c.hyp = torch.empty(*lead, dtype=torch.int32, device=dev)
        c.inliers = torch.empty(*lead, K, dtype=torch.bool, device=dev)
        wb = consensus_work_bytes(K, len(self._subsets), n)
        c.pnp_work = torch.empty(max(wb, 8) // 8, dtype=torch.float64, device=dev)

    def _consensus(self, c, s, P3, shared, groups, per_group, count):
        """the consensus solve of groups x per_group problems into c.R, c.t, c.params, c.inliers, c.hyp (count: device int [groups] or None)"""
        call("ssp_pnp_consensus", ptr(P3), shared, ptr(c.kp), ptr(self._K32), self.num_keypoints, groups, per_group, ptr(count),
             self._subsets.ctypes.data, len(self._subsets), self.reproj_thresh, 20, ptr(c.R), ptr(c.t), ptr(c.params), ptr(c.inl_mask),
             ptr(c.hyp), ptr(c.pnp_work), c.pnp_work.numel() * 8, s)
        torch.ne(torch.bitwise_and(c.inl_mask.unsqueeze(-1), self._bits), 0, out=c.inliers)

    def _consensus_outputs(self, c):
        return dict(inliers=c.inliers, hyp=c.hyp) if self.pnp == "consensus" else {}

    @staticmethod
    def _box_points(corners3D):
        """(3|4, 8) box corners -> (3, 9) float64 [0; corners3D[:3]] as columns (valid.py:146, valid_multi.py:135)"""
        c = np.asarray(corners3D, dtype=np.float64)
        if c.ndim != 2 or c.shape[0] not in (3, 4) or c.shape[1] != 8:
            raise SspError("corners3D must be (3|4, 8), got %s" % (c.shape,))
        return np.concatenate([np.zeros((3, 1)), c[:3]], axis=1)

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
    pnp="plain" (default) is the all-point solve."""

    def __init__(self, model, corners3D, K, frame_size=(640, 480), shape=None, batch=1, graph=True, max_graphs=4, pnp="plain",
                 reproj_thresh=8.0):
        P = self._box_points(corners3D)
        super().__init__(model, K, frame_size, shape if shape is not None else (model.test_width, model.test_height), batch, graph,
                         max_graphs)
        self._init_pnp(pnp, reproj_thresh, [P.T])
        dev = self.device
        self._P3 = torch.from_numpy(np.ascontiguousarray(P.T, dtype=np.float32)).to(dev)           # (9, 3) PnP points
        # row-major copies: the kernels read raw pointers, and numpy keeps a transposed input's column-major order through
        # concatenate / astype
        self._X = torch.from_numpy(np.ascontiguousarray(np.concatenate([P, np.ones((1, 9))], 0), dtype=np.float32)).to(dev)   # (4, 9)

    def _head_buffers(self, c):
        dev, B, K = self.device, self.batch, self.num_keypoints
        c.boxes = torch.empty(B, 2 * K + 3, dtype=torch.float32, device=dev)
        c.conf = torch.empty(B, dtype=torch.float32, device=dev)
        c.kp = torch.empty(B, K, 2, dtype=torch.float32, device=dev)
        c.R = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
        c.t = torch.empty(B, 3, dtype=torch.float64, device=dev)
        c.Rt = torch.empty(B, 3, 4, dtype=torch.float64, device=dev)
        c.proj = torch.empty(B, 2, K, dtype=torch.float32, device=dev)
        c.corners = torch.empty(B, K, 2, dtype=torch.float32, device=dev)
        self._consensus_buffers(c, (B,))

    def _head(self, c, s):
        B, K = self.batch, self.num_keypoints
        h, w = c.logits.shape[2:]
        call("ssp_region_decode_argmax", ptr(c.logits), B, K, self.num_classes, h, w, 1, ptr(c.boxes), ptr(c.conf), None, s)
        torch.mul(c.boxes[:, :2 * K].view(B, K, 2), c.scale, out=c.kp)
        if self.pnp == "consensus":
            self._consensus(c, s, self._P3, 1, B, 1, None)
        else:
            call("ssp_pnp_batched", ptr(self._P3), 1, ptr(c.kp), ptr(self._K32), K, B, 20, ptr(c.R), ptr(c.t), None, s)
        c.Rt[:, :, :3].copy_(c.R)
        c.Rt[:, :, 3].copy_(c.t)
        call("ssp_project_points", ptr(self._X), 4, K, ptr(c.Rt), ptr(self._K64), B, ptr(c.proj), s)
        c.corners.copy_(c.proj.transpose(1, 2))

    def _outputs(self, c):
        return dict(R=c.R, t=c.t, conf=c.conf, keypoints_px=c.kp, corners_px=c.corners, **self._consensus_outputs(c))


# ---------------------------------------------------------------------------------------------- command line
CONSENSUS_KEYS = {"plain": (), "consensus": ("inliers", "hyp")}          # the .npz columns each --pnp adds


def add_pnp_args(ap):
    ap.add_argument("--pnp", choices=("plain", "consensus"), default="plain",
                    help="consensus: a pose that survives wrong keypoints (PnP over keypoint subsets); adds inliers and hyp columns")
    ap.add_argument("--reproj-thresh", type=float, default=8.0, help="inlier threshold of --pnp consensus, frame pixels")


def camera_from_data_cfg(datacfg):
    """-> (mesh path, K (3, 3) float64, (width, height)) from a .data file (utils.py read_data_cfg keys mesh, fx, fy, u0, v0, width,
    height; valid.py:26-35)"""
    from .utils_host import read_data_cfg
    o = read_data_cfg(datacfg)
    try:
        fx, fy, u0, v0 = (float(o[k]) for k in ("fx", "fy", "u0", "v0"))
        size = (int(o["width"]), int(o["height"]))
        mesh = o["mesh"]
    except KeyError as e:
        raise SspError("%s has no %s entry" % (datacfg, e))
    K = np.array([[fx, 0.0, u0], [0.0, fy, v0], [0.0, 0.0, 1.0]])
    return mesh, K, size


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.predict",
                                 description="6-D pose of the object of a trained single-object model in each image")
    ap.add_argument("--datacfg", required=True, help=".data file: mesh, fx fy u0 v0, width height")
    ap.add_argument("--modelcfg", required=True)
    ap.add_argument("--weightfile", required=True)
    ap.add_argument("--out", default="poses.npz")
    add_pnp_args(ap)
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    check_pnp_args(a.pnp, a.reproj_thresh)
    from .darknet import Darknet
    from .utils_host import read_ply_vertices
    from .utils import get_3D_corners
    mesh, K, size = camera_from_data_cfg(a.datacfg)
    V = read_ply_vertices(mesh)
    corners3D = get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    pred = PosePredictor(model, corners3D, K, frame_size=size, pnp=a.pnp, reproj_thresh=a.reproj_thresh)
    res = {k: [] for k in ("R", "t", "conf", "keypoints_px", "corners_px") + CONSENSUS_KEYS[a.pnp]}
    for path in a.images:
        with open(path, "rb") as f:
            data = f.read()
        if data[:2] == b"\xff\xd8":
            r = pred([data], to_host=True)
        else:
            from PIL import Image
            r = pred(np.asarray(Image.open(path).convert("RGB"))[None], to_host=True)
        for k in res:
            res[k].append(r[k][0])
    np.savez(a.out, paths=np.array(a.images), **{k: np.stack(v) for k, v in res.items()})
    print("%d poses -> %s" % (len(a.images), a.out))


if __name__ == "__main__":
    main()
