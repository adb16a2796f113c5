"""Camera frames -> the 6-D pose of every requested object of a multi-object model (yolo-pose-multi.cfg) in one CUDA graph replay.

    pred = MultiPosePredictor(model, {0: corners_ape, 4: corners_can}, K, frame_size=(640, 480), batch=1)
    r = pred(frames)            # (B, H, W, 3) uint8 numpy array / CUDA tensor, or a list of B JPEG files' bytes
    r["R"][b, q], r["t"][b, q], r["detected"][b, q], ...             # slot q is class r["classes"][q] (the sorted class ids)

Frames go through the chain PosePredictor runs (predict.py: resize + ToTensor, the split-K eval forward, the graph LRU, the weight
re-pack); only the head differs.  Slot (frame b, class c) is the box reference valid_multi.py chooses for a ground truth of class
c that is the image's first (valid_multi.py:105-123, get_multi_region_boxes(..., correspondingclass=c, only_objectness=0)):
  * the first box with the largest det_conf among the listed boxes (det_conf * cls_max_conf > conf_thresh) whose arg-max class
    is c -- detected = True;
  * otherwise the reference's fallback box for correspondingclass = c (the running maxima of det_conf and softmax[c] in visiting
    order) -- detected = False.  Every slot therefore has a pose, as valid_multi always has one for the object it evaluates.
Each frame is its own batch-1 call (utils_multi.evaluate_multi_poses_batched documents the same departure).  Then per slot, as
valid_multi.py:127-138 computes them: the keypoints times the frame size in fp32, PnP of the 9 points [0; corners3D_c[:3]] of
class c's own box with the fp32 K, and the projection of the centroid and the 8 corners under that pose.

The head is one ssp_predict_multi_select launch (one CTA per frame, all classes), one ssp_pnp_batched over the B x Q problems
and one ssp_project_points of every class's 9 points under every slot's pose, of which each slot keeps its own class's columns.

Returned device tensors are the predictor's static outputs: the next call overwrites them.

Command line: python -m singleshotpose_b200.predict_multi --datacfg cfg/occlusion.data --modelcfg cfg/yolo-pose-multi.cfg
              --weightfile w.weights --object 0=../LINEMOD/ape/ape.ply --object 4=../LINEMOD/can/can.ply --out poses.npz img...
              [--depth-dir DIR [--depth-scale 0.001 --refine-iters 10]]: refine against 16-bit depth PNGs, as predict's command line
              [--rig rig.npz]: fuse the views of several calibrated cameras, as predict's command line
"""
from __future__ import annotations

import argparse
import ctypes as C

import numpy as np
import torch

from ._lib import SspError, call, ptr
from .predict import (CONSENSUS_KEYS, FUSE_KEYS, _FramePredictor, add_depth_args, add_dist_arg, add_pnp_args, add_rig_arg, camera_dist,
                      check_depth_args, check_rig_args, mesh_corners, predict_files, read_camera, read_mesh, refine_keys, refine_kwargs)
from .utils import check_pnp_args

MAX_ENTRIES = 4096          # H*W*num_anchors the select kernel keeps in shared memory (eval_multi_core.h kMaxEntries)
OUTPUT_KEYS = ("R", "t", "conf", "cls_conf", "detected", "keypoints_px", "corners_px")


class MultiPosePredictor(_FramePredictor):
    """model: a singleshotpose_b200.darknet_multi.Darknet (multi-anchor head, 9 keypoints).  objects: {class id: (3|4, 8) box corners
    of that class's mesh (utils.get_3D_corners)}; the slots follow the sorted class ids.  K: (3, 3) camera matrix; frame_size:
    (width, height) of the camera frames (other sizes are accepted and captured separately); shape: network input (width,
    height), default the cfg's training size (valid_multi.py:71); batch: frames per call; conf_thresh: default the cfg net
    block's conf_thresh (valid_multi.py:40).  graph=False runs the same launches eagerly (no capture).

    Returns dict(classes (Q,), R (B, Q, 3, 3) fp64, t (B, Q, 3) fp64, conf (B, Q) det_conf of the box, cls_conf (B, Q),
    detected (B, Q) bool, keypoints_px (B, Q, 9, 2), corners_px (B, Q, 9, 2)): device tensors, or numpy with to_host=True.
    pnp="consensus" solves each slot with the consensus PnP (utils.pnp_consensus_batched, inliers within reproj_thresh frame
    pixels) and adds inliers (B, Q, 9) bool and hyp (B, Q) int32; pnp="plain" (default) is the all-point solve.
    dist_coeffs: the camera's OpenCV distortion coefficients, as predict.PosePredictor takes them.
    meshes={class id: (vertices, faces)}, one for every requested class: refine every slot's pose against the call's depth=(B, H, W)
    uint16 frames, as predict.PosePredictor's mesh= does, adding R_ref (B, Q, 3, 3), t_ref (B, Q, 3), corners_ref_px (B, Q, 9, 2),
    refine_points, refine_rmse and refine_status (B, Q).
    rig=utils.camera_rig(...) of C calibrated cameras (K=None, no dist_coeffs): frame g C + c is camera c of capture g, and each
    class's detected views are fused into one world pose, as predict.PosePredictor's rig= does; the outputs add R_world (G, Q, 3, 3),
    t_world (G, Q, 3), world_cov (G, Q, 6, 6), views (G, Q, C), view_err (G, Q, C), fuse_hyp, fuse_status (G, Q) and
    corners_world_px (B, Q, 9, 2).  With a rig and meshes= each class's fused pose is refined against the depth of all the
    capture's cameras, as predict.PosePredictor's rig= with mesh= does, adding R_world_ref (G, Q, 3, 3), t_world_ref (G, Q, 3),
    refine_points, refine_rmse, refine_status (G, Q), refine_view_points, refine_view_rmse (G, Q, C) and corners_world_ref_px
    (B, Q, 9, 2)."""

    def __init__(self, model, objects, K, frame_size=(640, 480), shape=None, batch=1, conf_thresh=None, graph=True, max_graphs=4,
                 pnp="plain", reproj_thresh=8.0, dist_coeffs=None, meshes=None, depth_scale=0.001, refine_iters=10, refine_gate=(0.5, 0.02),
                 rig=None, fuse=(40.0, 8.0, 2.0)):
        self.num_anchors = int(getattr(model, "num_anchors", 0))
        if self.num_anchors < 2:
            raise SspError("MultiPosePredictor needs a multi-anchor region head (yolo-pose-multi.cfg), got %d anchor(s)" % self.num_anchors)
        self.conf_thresh = cfg_conf_thresh(model, conf_thresh)
        super().__init__(model, objects, K, frame_size, shape if shape is not None else (model.width, model.height), batch, graph,
                         max_graphs, pnp, reproj_thresh, dist_coeffs=dist_coeffs, meshes=meshes, depth_scale=depth_scale,
                         refine_iters=refine_iters, refine_gate=refine_gate, rig=rig, fuse=fuse)
        check_grid(self, "select")
        self._classes = torch.from_numpy(self.classes).to(self.device)

    def _head_buffers(self, c):
        dev, B, Q = self.device, self.batch, len(self.classes)
        c.boxes = torch.empty(B, Q, 2 * self.num_keypoints + 3, dtype=torch.float32, device=dev)
        c.flags = torch.empty(B, Q, dtype=torch.int32, device=dev)
        c.detected = torch.empty(B, Q, dtype=torch.bool, device=dev)

    def _head(self, c, s):
        Wf, Hf = c.frame
        h, w = c.logits.shape[2:]
        call("ssp_predict_multi_select", ptr(c.logits), self.batch, self.num_keypoints, self.num_classes, self.num_anchors, h, w,
             C.c_void_p(self._cls_host.ctypes.data), len(self.classes), self.conf_thresh, float(Wf), float(Hf), ptr(c.boxes),
             ptr(c.flags), ptr(c.kp), s)
        torch.eq(c.flags, 0, out=c.detected)
        self._tail(c, s, c.detected)

    def _outputs(self, c):
        K = self.num_keypoints
        return dict(classes=self._classes, R=c.R, t=c.t, conf=c.boxes[..., 2 * K], cls_conf=c.boxes[..., 2 * K + 1], detected=c.detected,
                    keypoints_px=c.kp, corners_px=c.corners, **self._consensus_outputs(c), **self._refine_outputs(c), **self._fuse_outputs(c))


def cfg_conf_thresh(model, conf_thresh):
    """conf_thresh as a float, by default the model cfg's [net] conf_thresh (valid_multi.py:40)"""
    if conf_thresh is None:
        if "conf_thresh" not in model.blocks[0]:
            raise SspError("the model's cfg has no conf_thresh in its [net] block: pass conf_thresh")
        conf_thresh = model.blocks[0]["conf_thresh"]
    return float(conf_thresh)


def check_grid(pred, kernel):
    """SspError unless the predictor's grid of anchors fits the MAX_ENTRIES the select and detect kernels hold in shared memory"""
    h, w = pred.out_hw
    if h * w * pred.num_anchors > MAX_ENTRIES:
        raise SspError("network shape %dx%d gives a %dx%d grid of %d anchors: more than the %d entries the %s kernel holds"
                       % (pred.shape[0], pred.shape[1], h, w, pred.num_anchors, MAX_ENTRIES, kernel))


# ---------------------------------------------------------------------------------------------- command line
SIZE_KEYS = (("im_width", "im_height"),)            # the frame size entries of a multi-object .data file (valid_multi.py:30-35)


def parse_objects(specs):
    """['0=ape.ply', '4=can.ply'] -> {0: 'ape.ply', 4: 'can.ply'}; raises SspError for a malformed entry or a class given twice"""
    out = {}
    for s in specs or ():
        cls, sep, path = s.partition("=")
        try:
            c = int(cls)
        except ValueError:
            c = None
        if not sep or c is None or c < 0 or not path:
            raise SspError("--object takes CLASS=MESH.ply with a class id >= 0, got %r" % s)
        if c in out:
            raise SspError("class %d is given twice (%s and %s)" % (c, out[c], path))
        out[c] = path
    if not out:
        raise SspError("give at least one --object CLASS=MESH.ply")
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.predict_multi",
                                 description="6-D poses of the requested objects of a trained multi-object model in each image")
    ap.add_argument("--datacfg", required=True, help=".data file: fx fy u0 v0, im_width im_height")
    ap.add_argument("--modelcfg", required=True)
    ap.add_argument("--weightfile", required=True)
    ap.add_argument("--object", action="append", required=True, metavar="CLASS=MESH.ply",
                    help="a class id of the model and the mesh of its object; repeat for every object to predict")
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
    from .darknet_multi import Darknet
    _mesh, K, size = read_camera(a.datacfg, SIZE_KEYS)
    paths = parse_objects(a.object)
    objects = {c: mesh_corners(mesh) for c, mesh in paths.items()}
    refine = dict(meshes={c: read_mesh(p) for c, p in paths.items()}, **refine_kwargs(a)) if a.depth_dir is not None else {}
    model = Darknet(a.modelcfg)
    model.load_weights(a.weightfile)
    model.cuda().eval()
    cams = dict(K=K) if rig is None else dict(K=None, rig=rig, batch=len(rig.K))
    pred = MultiPosePredictor(model, objects, frame_size=size, pnp=a.pnp, reproj_thresh=a.reproj_thresh, dist_coeffs=dist, **cams, **refine)
    res = {k: [] for k in OUTPUT_KEYS + CONSENSUS_KEYS[a.pnp] + refine_keys(refine, rig) + (FUSE_KEYS if rig is not None else ())}
    for r in predict_files(pred, a.images, a.depth_dir, pred.batch):
        for k in res:
            res[k].extend(r[k])
    np.savez(a.out, paths=np.array(a.images), classes=pred.classes, **{k: np.stack(v) for k, v in res.items()})
    print("%d images x %d objects -> %s" % (len(a.images), len(pred.classes), a.out))


if __name__ == "__main__":
    main()
