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
              [--depth-dir DIR [--depth-scale 0.001 --refine-iters 10]]: refine each pose against DIR/<image stem>.png, a 16-bit
              depth PNG registered to the image, adding the columns R_ref t_ref corners_ref_px refine_points refine_rmse refine_status
              [--rig rig.npz]: the images come in groups of C calibrated cameras (image i is camera i % C; utils_host.read_rig), adding
              the per-capture columns R_world t_world world_cov views view_err fuse_hyp fuse_status and the per-image corners_world_px;
              with --depth-dir too, the fused poses are refined against every camera's depth, adding the columns RIG_REFINE_KEYS
"""
from __future__ import annotations

import argparse
import collections
import os

import numpy as np
import torch

from ._lib import SspError, call, load, ptr, stream_ptr
from .engine import Buffers
from .image import BICUBIC
from .utils import (CameraRig, camera_distortion, check_fuse_args, check_instance_meshes, check_pnp_args, check_refine_args, consensus_subsets,
                    consensus_work_bytes, distortion_tensor, fuse_instances_outputs, fuse_instances_work_bytes, fuse_work_bytes, inlier_bits,
                    keypoint_bits, object_table, refine_face_table, refine_instances_work_bytes, refine_model_table, rig_tensors)


class _Chain:
    """static buffers (and the graph) of one (frame size, frame source, depth source); the head's buffers come from
    pred._slot_buffers and pred._head_buffers"""

    def __init__(self, pred, Wf, Hf, src, dsrc=None):
        dev, B = pred.device, pred.batch
        W, H = pred.shape
        self.frame, self.src, self.dsrc, self.graph = (Wf, Hf), src, dsrc, None
        self.u8 = torch.zeros(B, Hf, Wf, 3, dtype=torch.uint8, device=dev)
        self.pin = torch.zeros(B, Hf, Wf, 3, dtype=torch.uint8).pin_memory() if src == "host" else None
        # depth frames (uint16 bits in int16 storage), staged like the frames when they come from the host
        self.depth = torch.zeros(B, Hf, Wf, dtype=torch.int16, device=dev) if dsrc else None
        self.dpin = torch.zeros(B, Hf, Wf, dtype=torch.int16).pin_memory() if dsrc == "host" else None
        self.copied = torch.cuda.Event()          # the replay that last read `pin` / `dpin` has been enqueued after this
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
    With meshes ({class id: (vertices, faces)}, one for every requested class) the tail ends with _refine: one ssp_refine_depth
    launch refines every slot's pose against the call's registered depth frames (rule: csrc/refine_depth_core.h) into c.R_ref,
    c.t_ref, and a second _project of the refined poses gives c.corners_ref.  With a rig (utils.camera_rig of C cameras;
    row b = g C + c is camera c of capture g) the tail is _fuse instead: one ssp_fuse_views (rule: csrc/multiview_core.h) solves
    every row with its own camera into c.R, c.t, c.corners and fuses each capture's valid views (the head's flags) into one world
    pose per slot; a detecting head's slots are instead associated across the views by one ssp_fuse_instances (rule:
    csrc/multiview_instances_core.h), which solves every row likewise and fuses each capture's detections into world instances.
    With a rig and meshes _fuse is followed by _refine_rig: one ssp_refine_depth_rig (rule: csrc/refine_rig_core.h) refines each
    capture's fused world poses against the depth frames of all its cameras; a detecting head's world instances are refined
    together by _refine_instances instead: one ssp_refine_instances_rig (rule: csrc/refine_instances_core.h), in which each depth
    pixel belongs to the instance drawn in front of it.
    _tail runs the whole tail; every head calls it.
    A subclass supplies the rest: _head_buffers(chain) allocates its selection's static buffers, _head(chain, stream) launches
    the selection after the forward and then the tail, and _outputs(chain) names the returned tensors."""

    def __init__(self, model, objects, K, frame_size, shape, batch, graph, max_graphs, pnp, reproj_thresh, slots=None, dist_coeffs=None,
                 meshes=None, depth_scale=0.001, refine_iters=10, refine_gate=(0.5, 0.02), rig=None, fuse=(40.0, 8.0, 2.0)):
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
        self.rig = rig
        if rig is not None:
            check_rig_predictor(name, rig, K, dist_coeffs, pnp, meshes, self.batch, detects=slots is not None, num_classes=self.num_classes)
            self.fuse_gate, self.fuse_thresh, self.keypoint_sigma = check_fuse_args(*fuse)
            K = rig.K[0]                        # object_table's check only: each row is solved and projected with its camera's K
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
        if rig is not None:
            self._rig = rig_tensors(rig, dev)
        self._refines = meshes is not None
        if self._refines:
            self.depth_scale, self.refine_iters, self.refine_gate = check_refine_args(depth_scale, refine_iters, refine_gate)
            if not isinstance(meshes, dict) or sorted(meshes) != self.classes.tolist():
                raise SspError("meshes must hold one (vertices, faces) mesh for every requested class %s, got %s"
                               % (self.classes.tolist(), sorted(meshes) if isinstance(meshes, dict) else type(meshes).__name__))
            self._model, self._offsets, self._diam = refine_model_table(meshes, self.num_classes, dev)
            if not self._detects:                  # slot q: class classes[q]
                self._slot_cls = torch.from_numpy(np.tile(self.classes.astype(np.int32), (B, 1))).to(dev)
            if rig is not None:                    # the drawn points of corners_world_ref, by class id
                self._P3_table = torch.from_numpy(points.astype(np.float32)).to(dev)
            if rig is not None and self._detects:  # the faces the world instances are drawn with
                self._faces, self._face_offsets, self._max_faces = refine_face_table(check_instance_meshes(meshes, self.num_classes),
                                                                                     self.num_classes, dev)
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
        if self._refines and self.rig is not None:
            G, Cn = B // len(self.rig.K), len(self.rig.K)
            c.R_world_ref = torch.empty(G, S, 3, 3, dtype=torch.float64, device=dev)
            c.t_world_ref = torch.empty(G, S, 3, dtype=torch.float64, device=dev)
            c.ref_points = torch.empty(G, S, dtype=torch.int32, device=dev)
            c.ref_rmse = torch.empty(G, S, dtype=torch.float64, device=dev)
            c.ref_status = torch.empty(G, S, dtype=torch.int32, device=dev)
            c.ref_view_points = torch.empty(G, S, Cn, dtype=torch.int32, device=dev)
            c.ref_view_rmse = torch.empty(G, S, Cn, dtype=torch.float64, device=dev)
            c.corners_world_ref = torch.empty(B, S, K, 2, dtype=torch.float32, device=dev)
            if self._detects:
                Wf, Hf = c.frame
                c.ref_view_hidden = torch.empty(G, S, Cn, dtype=torch.int32, device=dev)
                c.instance_map = torch.empty(B, Hf, Wf, dtype=torch.int16, device=dev)
                c.ref_work = torch.empty(max(refine_instances_work_bytes(G, Cn, S, Wf, Hf), 8) // 8, dtype=torch.float64, device=dev)
        elif self._refines:
            c.R_ref = torch.empty(B, S, 3, 3, dtype=torch.float64, device=dev)
            c.t_ref = torch.empty(B, S, 3, dtype=torch.float64, device=dev)
            c.corners_ref = torch.empty(B, S, K, 2, dtype=torch.float32, device=dev)
            c.ref_points = torch.empty(B, S, dtype=torch.int32, device=dev)
            c.ref_rmse = torch.empty(B, S, dtype=torch.float64, device=dev)
            c.ref_status = torch.empty(B, S, dtype=torch.int32, device=dev)
        if self.rig is not None and self._detects:
            Cn = len(self.rig.K)
            c.fi = {k: v for k, v in fuse_instances_outputs(B, Cn, S, K, dev).items() if k not in ("R", "t", "corners_px")}
            c.fuse_work = torch.empty(max(fuse_instances_work_bytes(B // Cn, Cn, S), 8) // 8, dtype=torch.float64, device=dev)
        elif self.rig is not None:
            G, Cn = B // len(self.rig.K), len(self.rig.K)
            c.R_world = torch.empty(G, S, 3, 3, dtype=torch.float64, device=dev)
            c.t_world = torch.empty(G, S, 3, dtype=torch.float64, device=dev)
            c.world_cov = torch.empty(G, S, 6, 6, dtype=torch.float64, device=dev)
            c.views = torch.empty(G, S, Cn, dtype=torch.bool, device=dev)
            c.view_err = torch.empty(G, S, Cn, dtype=torch.float64, device=dev)
            c.fuse_hyp = torch.empty(G, S, dtype=torch.int32, device=dev)
            c.fuse_status = torch.empty(G, S, dtype=torch.int32, device=dev)
            c.corners_world = torch.empty(B, S, K, 2, dtype=torch.float32, device=dev)
            c.row_valid = torch.empty(B, S, dtype=torch.bool, device=dev)
            c.fuse_work = torch.empty(max(fuse_work_bytes(G, Cn, S), 8) // 8, dtype=torch.float64, device=dev)

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

    def _project(self, c, s, R=None, t=None, corners=None):
        """corners (default c.corners): each slot's class's 9 points projected under the slot's pose R, t (default c.R, c.t), zero
        in empty slots"""
        B, S, K, Q = self.batch, self.num_slots, self.num_keypoints, len(self.classes)
        R, t, corners = (c.R, c.t, c.corners) if R is None else (R, t, corners)
        c.Rt[..., :3].copy_(R)
        c.Rt[..., 3].copy_(t)
        # every requested class's points under every slot's pose (each point is projected on its own, so a slot's own columns are
        # what ssp_project_points gives for its class's (4, 9) points alone); each slot keeps the columns of its class
        if self._dist is None:
            call("ssp_project_points", ptr(self._X), 4, Q * K, ptr(c.Rt), ptr(self._K64), B * S, ptr(c.proj), s)
        else:
            call("ssp_project_points_dist", ptr(self._X), 4, Q * K, ptr(c.Rt), ptr(self._K64), ptr(self._dist), B * S, ptr(c.proj), s)
        if not self._detects:                      # slot q: class q
            corners.copy_(torch.diagonal(c.proj.view(B, S, 2, Q, K), dim1=1, dim2=3).permute(0, 3, 2, 1))
            return
        own = c.proj.view(B * S, 2, Q, K)[self._rows, :, self._slot_of[c.cls0.view(-1)]]          # (B*S, 2, K)
        torch.lt(self._slot_index, c.count.unsqueeze(1), out=c.valid)
        torch.where(c.valid.view(B, S, 1, 1), own.view(B, S, 2, K).transpose(2, 3), self._zero, out=corners)

    def _refine(self, c, s):
        """c.R_ref, c.t_ref, c.ref_points, c.ref_rmse, c.ref_status: every slot's pose refined against its frame's depth c.depth;
        c.corners_ref its projection (empty slots: zeros)"""
        Wf, Hf = c.frame
        cls = self._slot_cls if not self._detects else c.cls
        call("ssp_refine_depth", ptr(c.depth), Wf, Hf, self.depth_scale, ptr(self._K64), ptr(self._dist), ptr(self._model), ptr(self._offsets),
             ptr(self._diam), self.num_classes, ptr(cls), self.batch, self.num_slots, ptr(c.count), ptr(c.R), ptr(c.t), self.refine_iters,
             self.refine_gate[0], self.refine_gate[1], ptr(c.R_ref), ptr(c.t_ref), ptr(c.ref_points), ptr(c.ref_rmse), ptr(c.ref_status), s)
        self._project(c, s, c.R_ref, c.t_ref, c.corners_ref)

    def _refine_rig(self, c, s):
        """with a rig and meshes: each capture's fused world poses c.R_world, c.t_world refined against the depth frames of all
        its cameras at once (ssp_refine_depth_rig; row b of c.depth is camera b % C) into c.R_world_ref, c.t_world_ref, ...;
        c.corners_world_ref the refined pose in each frame's camera"""
        Wf, Hf = c.frame
        _K32, K64, D, Rr, tr = self._rig
        Cn = len(self.rig.K)
        call("ssp_refine_depth_rig", ptr(c.depth), Wf, Hf, self.depth_scale, Cn, ptr(K64), ptr(D), ptr(Rr), ptr(tr), ptr(self._model),
             ptr(self._offsets), ptr(self._diam), ptr(self._P3_table), self.num_keypoints, self.num_classes, ptr(self._slot_cls),
             self.batch // Cn, self.num_slots, None, ptr(c.fuse_status), ptr(c.R_world), ptr(c.t_world), self.refine_iters,
             self.refine_gate[0], self.refine_gate[1], ptr(c.R_world_ref), ptr(c.t_world_ref), ptr(c.ref_points), ptr(c.ref_rmse),
             ptr(c.ref_status), ptr(c.ref_view_points), ptr(c.ref_view_rmse), ptr(c.corners_world_ref), s)

    def _refine_instances(self, c, s):
        """with a rig, meshes and a detecting head: every world instance of each capture (c.fi) refined against the depth frames
        of all its cameras, each depth pixel owned by the instance drawn in front of it (ssp_refine_instances_rig), into
        c.R_world_ref, c.t_world_ref, ..., c.ref_view_hidden and c.instance_map"""
        Wf, Hf = c.frame
        _K32, K64, D, Rr, tr = self._rig
        Cn = len(self.rig.K)
        fi = c.fi
        call("ssp_refine_instances_rig", ptr(c.depth), Wf, Hf, self.depth_scale, Cn, ptr(K64), ptr(D), ptr(Rr), ptr(tr), ptr(self._model),
             ptr(self._offsets), ptr(self._diam), ptr(self._faces), ptr(self._face_offsets), self._max_faces, ptr(self._P3_table),
             self.num_keypoints, self.num_classes, ptr(fi["world_cls"]), self.batch // Cn, self.num_slots, ptr(fi["world_count"]),
             ptr(fi["fuse_status"]), ptr(fi["R_world"]), ptr(fi["t_world"]), self.refine_iters, self.refine_gate[0], self.refine_gate[1],
             ptr(c.R_world_ref), ptr(c.t_world_ref), ptr(c.ref_points), ptr(c.ref_rmse), ptr(c.ref_status), ptr(c.ref_view_points),
             ptr(c.ref_view_rmse), ptr(c.ref_view_hidden), ptr(c.corners_world_ref), ptr(c.instance_map), ptr(c.ref_work),
             c.ref_work.numel() * 8, s)

    def _fuse(self, c, s, valid):
        """with a rig: every row's PnP and projection with its camera into c.R, c.t, c.corners, and each capture's valid views
        (valid (B, S) bool) fused into c.R_world, c.t_world, ... (ssp_fuse_views)"""
        K32, K64, D, Rr, tr = self._rig
        Cn = len(self.rig.K)
        call("ssp_fuse_views", ptr(c.P3), 0, ptr(c.kp), ptr(valid), self.num_keypoints, self.batch // Cn, Cn, self.num_slots, ptr(K32), ptr(K64),
             ptr(D), ptr(Rr), ptr(tr), self.fuse_gate, self.fuse_thresh, self.keypoint_sigma, 20, ptr(c.R), ptr(c.t), ptr(c.corners),
             ptr(c.R_world), ptr(c.t_world), ptr(c.world_cov), ptr(c.views), ptr(c.view_err), ptr(c.fuse_hyp), ptr(c.fuse_status),
             ptr(c.corners_world), ptr(c.fuse_work), c.fuse_work.numel() * 8, s)

    def _fuse_instances(self, c, s):
        """with a rig and a detecting head: every row's PnP and projection with its camera into c.R, c.t, c.corners (zeros in empty
        slots), and each capture's detections (c.cls, c.count, c.kp) associated across the views into world instances
        (ssp_fuse_instances) in c.fi"""
        K32, K64, D, Rr, tr = self._rig
        Cn = len(self.rig.K)
        call("ssp_fuse_instances", ptr(self._P3_table), self.num_classes, ptr(c.kp), ptr(c.cls), ptr(c.count), self.num_keypoints, self.batch // Cn,
             Cn, self.num_slots, ptr(K32), ptr(K64), ptr(D), ptr(Rr), ptr(tr), self.fuse_gate, self.fuse_thresh, self.keypoint_sigma, 20,
             ptr(c.R), ptr(c.t), ptr(c.corners), *(ptr(v) for v in c.fi.values()), ptr(c.fuse_work), c.fuse_work.numel() * 8, s)

    def _tail(self, c, s, valid=None):
        """the pose tail every head runs after its selection: PnP, projection and, with meshes, the depth refinement; with a rig
        the fusion of the views whose slots are valid (B, S) bool"""
        if self.rig is not None and self._detects:
            self._fuse_instances(c, s)
            if self._refines:
                self._refine_instances(c, s)
            return
        if self.rig is not None:
            self._fuse(c, s, valid)
            if self._refines:
                self._refine_rig(c, s)
            return
        self._solve(c, s)
        self._project(c, s)
        if self._refines:
            self._refine(c, s)

    def _consensus_outputs(self, c):
        return dict(inliers=c.inliers, hyp=c.hyp) if self.pnp == "consensus" else {}

    def _fuse_outputs(self, c):
        if self.rig is None:
            return {}
        if self._detects:
            return dict(c.fi)
        return dict(R_world=c.R_world, t_world=c.t_world, world_cov=c.world_cov, views=c.views, view_err=c.view_err, fuse_hyp=c.fuse_hyp,
                    fuse_status=c.fuse_status, corners_world_px=c.corners_world)

    def _refine_outputs(self, c):
        if not self._refines:
            return {}
        if self.rig is not None:
            out = dict(R_world_ref=c.R_world_ref, t_world_ref=c.t_world_ref, refine_points=c.ref_points, refine_rmse=c.ref_rmse,
                       refine_status=c.ref_status, refine_view_points=c.ref_view_points, refine_view_rmse=c.ref_view_rmse,
                       corners_world_ref_px=c.corners_world_ref)
            if self._detects:
                out.update(refine_view_hidden=c.ref_view_hidden, instance_map=c.instance_map)
            return out
        return dict(R_ref=c.R_ref, t_ref=c.t_ref, corners_ref_px=c.corners_ref, refine_points=c.ref_points, refine_rmse=c.ref_rmse,
                    refine_status=c.ref_status)

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

    def _check_depth(self, depth, kind, frames):
        """-> (depth source kind or None, array / tensor) for the frames checked by _check; raises SspError before anything is
        launched: depth without meshes, no depth with meshes, or depth that is not (B, H, W) uint16 at the frames' own size"""
        if not self._refines:
            if depth is not None:
                raise SspError("depth= is read by the refinement only: build the predictor with a mesh (mesh= / meshes=)")
            return None, None
        if depth is None:
            raise SspError("this predictor refines its poses against depth: pass depth=(B, H, W) uint16 frames registered to the frames")
        if kind == "jpeg":
            from .jpeg import read_jpeg_size
            Wf, Hf = read_jpeg_size(frames[0])
        else:
            Hf, Wf = int(frames.shape[1]), int(frames.shape[2])
        if isinstance(depth, np.ndarray):
            dkind, ok = "host", depth.dtype == np.uint16
        elif torch.is_tensor(depth):
            if not depth.is_cuda:
                raise SspError("depth given as a torch tensor must be on the GPU (pass host depth as a numpy array)")
            dkind, ok = "device", depth.dtype == torch.uint16
        else:
            raise SspError("depth must be a (B, H, W) uint16 numpy array or CUDA tensor, got %s" % type(depth).__name__)
        if not ok:
            raise SspError("depth must be uint16, got %s" % depth.dtype)
        if tuple(depth.shape) != (self.batch, Hf, Wf):
            raise SspError("depth must be (B, H, W) = (%d, %d, %d), registered to the frames at their own size; got %s"
                           % (self.batch, Hf, Wf, tuple(depth.shape)))
        return dkind, depth

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
        if c.dsrc == "host":
            c.depth.copy_(c.dpin, non_blocking=True)
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

    def _chain(self, Wf, Hf, src, dsrc=None):
        key = (Wf, Hf, src, dsrc)
        c = self._chains.get(key)
        if c is None:
            c = _Chain(self, Wf, Hf, src, dsrc)
            self._chains[key] = c
            while len(self._chains) > self.max_graphs:
                self._chains.popitem(last=False)
        self._chains.move_to_end(key)
        return c

    def __call__(self, frames, to_host=False, events=None, depth=None):
        kind, arr = self._check(frames)
        dkind, darr = self._check_depth(depth, kind, arr)
        with torch.cuda.device(self.device):
            if kind == "jpeg":
                if self._jpeg is None:
                    from .jpeg import GpuJpegDecoder
                    self._jpeg = GpuJpegDecoder(self.device)
                arr, kind = torch.stack(self._jpeg(arr)), "device"
            Hf, Wf = int(arr.shape[1]), int(arr.shape[2])
            self._ensure_current()
            c = self._chain(Wf, Hf, kind, dkind)
            staged = kind == "host" or dkind == "host"
            if staged:
                c.copied.synchronize()            # the previous replay's copies out of the staging buffers have run
            if kind == "host":
                np.copyto(c.pin.numpy(), arr, casting="no")
            else:
                c.u8.copy_(arr)
            if dkind == "host":
                np.copyto(c.dpin.numpy(), darr.view(np.int16), casting="no")
            elif dkind == "device":
                c.depth.copy_(darr.view(torch.int16))
            if self.use_graph and not events:
                if c.graph is None:
                    self._capture(c)
                c.graph.replay()
            else:
                self._body(c, events)
            if staged:
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
    distCoeffs) of the raw keypoints and corners_px is cv2.projectPoints with them, on the raw frame; None or all zeros: no distortion.
    mesh=(vertices (Nv, 3), faces (Nf, 3)): refine each pose against a depth frame registered to the colour frame, which every call
    then takes as depth=(B, H, W) uint16 at the frames' size (host numpy or CUDA tensor): projective point-to-plane ICP of the mesh's
    vertices (utils.refine_depth_batched; depth_scale mesh units per depth unit, refine_iters iterations, refine_gate the pair gate
    range as fractions of the mesh's diameter).  The outputs add R_ref (B, 3, 3), t_ref (B, 3), corners_ref_px (B, 9, 2),
    refine_points (B,), refine_rmse (B,) and refine_status (B,) (utils.REFINE_STATUS bits; with a bit set R_ref, t_ref are R, t);
    R, t and the other outputs are the same bits as without a mesh.
    rig=utils.camera_rig(...) of C calibrated cameras (K=None; no dist_coeffs, each camera brings its own): batch is a multiple of
    C and frame g C + c is camera c of capture g.  R, t, corners_px are each frame's pose with its own camera; a frame's view takes
    part in the fusion when conf > conf_thresh (default the cfg's [net] conf_thresh).  The outputs add, per capture, R_world (G, 3, 3),
    t_world (G, 3) world-from-object, world_cov (G, 6, 6), views (G, C) bool, view_err (G, C), fuse_hyp (G,), fuse_status (G,)
    (utils.fuse_views_batched, fuse = (gate, reproj_thresh, keypoint_sigma)), and per frame corners_world_px (B, 9, 2), the fused
    pose in the frame's camera.  Not with pnp="consensus".  With a rig and mesh= every call takes depth=(B, H, W), row b registered
    to frame b's camera, and each capture's fused pose is refined against the depth of all its cameras at once
    (utils.refine_depth_rig_batched): the outputs add, per capture, R_world_ref (G, 3, 3), t_world_ref (G, 3), refine_points,
    refine_rmse, refine_status (G,), refine_view_points, refine_view_rmse (G, C), and per frame corners_world_ref_px (B, 9, 2);
    there is no per-frame R_ref."""

    def __init__(self, model, corners3D, K, frame_size=(640, 480), shape=None, batch=1, graph=True, max_graphs=4, pnp="plain",
                 reproj_thresh=8.0, dist_coeffs=None, mesh=None, depth_scale=0.001, refine_iters=10, refine_gate=(0.5, 0.02), rig=None,
                 conf_thresh=None, fuse=(40.0, 8.0, 2.0)):
        if rig is not None:
            from .predict_multi import cfg_conf_thresh
            self.conf_thresh = cfg_conf_thresh(model, conf_thresh)
        super().__init__(model, {0: corners3D}, K, frame_size, shape if shape is not None else (model.test_width, model.test_height),
                         batch, graph, max_graphs, pnp, reproj_thresh, dist_coeffs=dist_coeffs,
                         meshes=None if mesh is None else {0: mesh}, depth_scale=depth_scale, refine_iters=refine_iters,
                         refine_gate=refine_gate, rig=rig, fuse=fuse)

    def _head_buffers(self, c):
        dev, B, K = self.device, self.batch, self.num_keypoints
        c.boxes = torch.empty(B, 2 * K + 3, dtype=torch.float32, device=dev)
        c.conf = torch.empty(B, dtype=torch.float32, device=dev)

    def _head(self, c, s):
        B, K = self.batch, self.num_keypoints
        h, w = c.logits.shape[2:]
        call("ssp_region_decode_argmax", ptr(c.logits), B, K, self.num_classes, h, w, 1, ptr(c.boxes), ptr(c.conf), None, s)
        torch.mul(c.boxes[:, :2 * K].view(B, 1, K, 2), c.scale, out=c.kp)
        if self.rig is not None:
            torch.gt(c.conf.view(B, 1), self.conf_thresh, out=c.row_valid)
        self._tail(c, s, c.row_valid if self.rig is not None else None)

    def _outputs(self, c):
        one = {k: v[:, 0] for k, v in dict(self._consensus_outputs(c), **self._refine_outputs(c), **self._fuse_outputs(c)).items()}   # the one slot of each frame
        return dict(R=c.R[:, 0], t=c.t[:, 0], conf=c.conf, keypoints_px=c.kp[:, 0], corners_px=c.corners[:, 0], **one)


def check_rig_predictor(name, rig, K, dist_coeffs, pnp, meshes, batch, detects=False, num_classes=None):
    """SspError for what a predictor with a rig refuses: a rig that is not a utils.CameraRig, K or dist_coeffs given as well
    (each camera brings its own), pnp="consensus", or a batch that is not whole captures; on a detecting head (detects), whose
    detections are associated across the views (ssp_fuse_instances) and whose world instances are drawn to refine them against
    depth, meshes that utils.check_instance_meshes refuses (a class id outside [0, num_classes), a face index outside its
    vertices, a diameter that is not > 0 or no face of non-zero area)"""
    if not isinstance(rig, CameraRig):
        raise SspError("rig must be a CameraRig (utils.camera_rig)")
    if K is not None or dist_coeffs is not None:
        raise SspError("%s with a rig takes K=None and no dist_coeffs: each camera of the rig brings its own" % name)
    if pnp != "plain":
        raise SspError("%s with a rig fuses the plain per-view solves: pnp=%r is not supported with a rig" % (name, pnp))
    if meshes is not None and detects:
        check_instance_meshes(meshes, num_classes)
    if batch % len(rig.K):
        raise SspError("batch %d is not a multiple of the rig's %d cameras" % (batch, len(rig.K)))


# ---------------------------------------------------------------------------------------------- command line
FUSE_KEYS = ("R_world", "t_world", "world_cov", "views", "view_err", "fuse_hyp", "fuse_status", "corners_world_px")     # the --rig columns
CONSENSUS_KEYS = {"plain": (), "consensus": ("inliers", "hyp")}          # the .npz columns each --pnp adds
REFINE_KEYS = ("R_ref", "t_ref", "corners_ref_px", "refine_points", "refine_rmse", "refine_status")     # the --depth-dir columns
RIG_REFINE_KEYS = ("R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points", "refine_view_rmse",
                   "corners_world_ref_px")                                # the --rig --depth-dir columns
SIZE_KEYS = (("width", "height"),)                                      # the frame size entries of a single-object .data file


def add_pnp_args(ap):
    ap.add_argument("--pnp", choices=("plain", "consensus"), default="plain",
                    help="consensus: a pose that survives wrong keypoints (PnP over keypoint subsets); adds inliers and hyp columns")
    ap.add_argument("--reproj-thresh", type=float, default=8.0, help="inlier threshold of --pnp consensus, frame pixels")


def add_dist_arg(ap):
    ap.add_argument("--dist", type=float, nargs="+", metavar="K",
                    help="the camera's OpenCV distortion coefficients k1 k2 p1 p2 [k3 [k4 k5 k6]] (cv2.calibrateCamera's distCoeffs); "
                         "overrides the .data file's dist entry.  End the list with -- when the images follow it")


def add_depth_args(ap):
    ap.add_argument("--depth-dir", metavar="DIR",
                    help="refine each pose against DIR/<image stem>.png, a 16-bit depth PNG registered to the image (same size); adds "
                         "the columns " + " ".join(REFINE_KEYS))
    ap.add_argument("--depth-scale", type=float, default=0.001,
                    help="--depth-dir: mesh units per depth unit (0.001 for millimetre depth and metre meshes)")
    ap.add_argument("--refine-iters", type=int, default=10, help="--depth-dir: iterations of the refinement")


def add_rig_arg(ap):
    ap.add_argument("--rig", metavar="RIG.npz",
                    help="fuse the views of several calibrated cameras (utils_host.read_rig: K, R, t[, dist] per camera): the images come "
                         "in groups of C, image i is camera i %% C; adds the columns " + " ".join(FUSE_KEYS))


def check_rig_args(args):
    """-> the --rig file's CameraRig, or None; SspError for --rig with --dist or --pnp consensus, an image count that is not a
    multiple of the rig's cameras, and with --depth-dir an image whose depth file DIR/<stem>.png does not exist (checked before
    the .data file or the model is read)"""
    if args.rig is None:
        return None
    if args.dist is not None:
        raise SspError("--dist and --rig: each camera of the rig brings its own distortion coefficients (the rig's dist)")
    if args.depth_dir is not None:
        for p in args.images:
            path = os.path.join(args.depth_dir, os.path.splitext(os.path.basename(p))[0] + ".png")
            if not os.path.isfile(path):
                raise SspError("depth file %s does not exist" % path)
    if args.pnp != "plain":
        raise SspError("--pnp %s is not supported with --rig" % args.pnp)
    from .utils_host import read_rig
    rig = read_rig(args.rig)
    if len(args.images) % len(rig.K):
        raise SspError("%d images are not whole captures of the rig's %d cameras: give the images in groups of %d"
                       % (len(args.images), len(rig.K), len(rig.K)))
    return rig


def refine_keys(refine, rig):
    """the .npz columns --depth-dir adds: REFINE_KEYS, or RIG_REFINE_KEYS with --rig"""
    if not refine:
        return ()
    return RIG_REFINE_KEYS if rig is not None else REFINE_KEYS


def check_depth_args(args):
    """SspError for a bad --depth-scale or --refine-iters given with --depth-dir"""
    if args.depth_dir is not None:
        check_refine_args(args.depth_scale, args.refine_iters, (0.5, 0.02))


def refine_kwargs(args):
    """the predictor keywords of --depth-scale and --refine-iters"""
    return dict(depth_scale=args.depth_scale, refine_iters=args.refine_iters)


def read_depth_png(path, size):
    """(H, W) uint16 depth of a 16-bit grayscale PNG; SspError naming the file when it is missing, not 16-bit or not of
    size (width, height)"""
    from PIL import Image
    if not os.path.isfile(path):
        raise SspError("depth file %s does not exist" % path)
    with Image.open(path) as im:
        if im.mode not in ("I;16", "I;16B", "I;16L", "I"):
            raise SspError("depth file %s is not a 16-bit grayscale PNG (mode %s)" % (path, im.mode))
        d = np.asarray(im)
    if d.dtype != np.uint16:
        if d.size and (d.min() < 0 or d.max() > 65535):
            raise SspError("depth file %s holds values outside 0..65535" % path)
        d = d.astype(np.uint16)
    if (d.shape[1], d.shape[0]) != tuple(size):
        raise SspError("depth file %s is %dx%d, its image %dx%d: the depth must be registered to the image at its size"
                       % (path, d.shape[1], d.shape[0], size[0], size[1]))
    return d


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


def read_mesh(path):
    """(vertices, faces) of a PLY mesh (utils_host.read_ply_mesh)"""
    from .utils_host import read_ply_mesh
    return read_ply_mesh(path)


def mesh_corners(path):
    """(4, 8) box corners (utils.get_3D_corners) of the vertices of a PLY mesh"""
    from .utils import get_3D_corners
    from .utils_host import read_ply_vertices
    V = read_ply_vertices(path)
    return get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)


def predict_files(pred, paths, depth_dir=None, group=1):
    """yields pred's host result for each group of `group` image files, one call per group: JPEG files go to the GPU decoder, others
    (or a group that mixes them) through Pillow.  depth_dir: each call also takes depth_dir/<image stem>.png (read_depth_png)"""
    for i in range(0, len(paths), group):
        chunk = paths[i:i + group]
        datas = []
        for path in chunk:
            with open(path, "rb") as f:
                datas.append(f.read())
        if all(d[:2] == b"\xff\xd8" for d in datas):
            from .jpeg import read_jpeg_size
            frames, size = datas, read_jpeg_size(datas[0])
        else:
            from PIL import Image
            arrays = [np.asarray(Image.open(path).convert("RGB")) for path in chunk]
            if len({a.shape for a in arrays}) != 1:
                raise SspError("the images of one capture must have one size: %s" % ", ".join(chunk))
            frames = np.stack(arrays)
            size = (frames.shape[2], frames.shape[1])
        kw = {}
        if depth_dir is not None:
            stems = [os.path.splitext(os.path.basename(p))[0] for p in chunk]
            kw["depth"] = np.stack([read_depth_png(os.path.join(depth_dir, st + ".png"), size) for st in stems])
        yield pred(frames, to_host=True, **kw)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.predict",
                                 description="6-D pose of the object of a trained single-object model in each image")
    ap.add_argument("--datacfg", required=True, help=".data file: mesh, fx fy u0 v0, width height")
    ap.add_argument("--modelcfg", required=True)
    ap.add_argument("--weightfile", required=True)
    ap.add_argument("--out", default="poses.npz")
    add_pnp_args(ap)
    add_dist_arg(ap)
    add_depth_args(ap)
    add_rig_arg(ap)
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    check_pnp_args(a.pnp, a.reproj_thresh)
    check_depth_args(a)
    rig = check_rig_args(a)
    dist = camera_dist(a) if rig is None else None
    from .darknet import Darknet
    mesh, K, size = read_camera(a.datacfg, SIZE_KEYS)
    if mesh is None:
        raise SspError("%s has no mesh entry" % a.datacfg)
    corners3D = mesh_corners(mesh)
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    refine = dict(mesh=read_mesh(mesh), **refine_kwargs(a)) if a.depth_dir is not None else {}
    cams = dict(K=K) if rig is None else dict(K=None, rig=rig, batch=len(rig.K))
    pred = PosePredictor(model, corners3D, frame_size=size, pnp=a.pnp, reproj_thresh=a.reproj_thresh, dist_coeffs=dist, **cams, **refine)
    res = {k: [] for k in ("R", "t", "conf", "keypoints_px", "corners_px") + CONSENSUS_KEYS[a.pnp] + refine_keys(refine, rig)
           + (FUSE_KEYS if rig is not None else ())}
    for r in predict_files(pred, a.images, a.depth_dir, pred.batch):
        for k in res:
            res[k].extend(r[k])
    np.savez(a.out, paths=np.array(a.images), **{k: np.stack(v) for k, v in res.items()})
    print("%d poses -> %s" % (len(a.images), a.out))


if __name__ == "__main__":
    main()
