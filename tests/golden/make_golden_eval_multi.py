"""Generate tests/golden/eval_multi.npz from the REFERENCE ITSELF: multi_obj_pose_estimation/valid_multi.py's valid(), run
unmodified on a synthetic LINEMOD tree (singleshotpose_b200.synth.write_linemod_multi_like) with planted network outputs.

Run where the reference checkout is available (path in REF below):
    python tests/golden/make_golden_eval_multi.py
Stubs, none of which touches the evaluation arithmetic: `matplotlib` (imported, unused) is an empty module, `.cuda()` is the
identity, and valid_multi.Darknet is a model whose forward returns the planted (1,160,13,13) outputs in loader order.  The
script writes the .data file, an ASCII .ply mesh (a box's 8 corners plus points inside it) and the test list; the chosen
labels_occlusion/ files hold exact projections of known poses of the mesh's box, stored in OCCLUSION corner order (the inverse
of fix_corner_order).  The reference's loader keeps 2K+1 of every 2K+3 values of a label file row while valid_multi reads the
label as rows of 2K+3, so the files are laid out (loader_rows) such that the loaded label holds whole rows.  A wrapper around valid_multi.pnp records every call's 2-D points, R and t; a wrapper around
get_multi_region_boxes records the box lists; the printed accuracy lines are captured.

Cases, one image each, in loader order (PLANTS): a plain match; several ground truths of different classes; the first ground
truth's class missing above the threshold (the fallback box); a later ground truth whose class has no box (the carry-over);
two boxes of one class with exactly equal logits (the first in list order wins); an empty label file; prediction noise of
1e-3 and 3e-2 in normalised image units.  Stored: outputs, targets, vertices, corners, intrinsics, per-pnp-call points and
poses, the chosen list position per ground truth, the per-object pixel errors recomputed from the recorded poses with the
reference's compute_projection, and the 10 accuracies.  The script asserts that no pixel error lies within 1e-2 px of an
accuracy threshold (so the table is an exact check) and that oracle/eval_multi_ref.py reproduces the selections and the
points bit for bit.

A separate script, not a flag of make_golden.py: that generator and the fixtures it writes are left exactly as they are.
"""
import contextlib
import io
import os
import re
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REPO)

from singleshotpose_b200 import synth          # noqa: E402
from oracle import eval_multi_ref as EM        # noqa: E402

K, NC, NA, H, W, NL = 9, 13, 5, 13, 13, 21
IM_W, IM_H = 640, 480
CONF_THRESH = 0.05                             # yolo-pose-multi.cfg:20
FIX = (0, 1, 3, 5, 7, 2, 4, 6, 8)
THRESHOLDS = (5, 10, 15, 20, 25, 30, 35, 40, 45, 50)

# (image path under the tree, ground-truth classes, planted boxes (class, anchor, noise, which ground truth's pose, cell shift),
#  fallback plant: ground truth whose pose the sub-threshold box of the first class carries, or None)
PLANTS = [
    ("LINEMOD/ape/JPEGImages/000000.png", [0], [(0, 2, 1e-3, 0, 0)], None),                                        # plain match
    ("LINEMOD/can/JPEGImages/000000.png", [4, 8, 1], [(4, 0, 1e-3, 0, 0), (8, 3, 1e-3, 1, 0), (1, 4, 1e-3, 2, 0)], None),
    ("LINEMOD/cat/JPEGImages/000000.png", [6, 2], [(2, 1, 1e-3, 1, 0)], 0),                                        # fallback
    ("LINEMOD/duck/JPEGImages/000000.png", [3, 11], [(3, 2, 1e-3, 0, 0)], None),                                   # carry-over
    ("LINEMOD/glue/JPEGImages/000000.png", [5], [(5, 1, 1e-3, 0, 0), (5, 1, 1e-3, 0, 2)], None),                    # equal logits
    ("LINEMOD/holepuncher/JPEGImages/000000.png", [], [], None),                                                  # empty label
    ("LINEMOD/iron/JPEGImages/000000.png", [7, 9], [(7, 0, 3e-2, 0, 0), (9, 4, 3e-2, 1, 0)], None),                 # noise 3e-2
]


def mesh_vertices(rng, n=300, half=(0.038, 0.039, 0.046)):
    """(n, 3): the box's 8 corners (so get_3D_corners gives the box) and n - 8 points inside it"""
    c = synth.box_points(half, with_center=False).astype(np.float64)
    inner = rng.uniform(-1, 1, size=(n - 8, 3)) * np.array(half)
    return np.round(np.concatenate([c, inner]), 6)


def project(P, R, t, Kc):
    Pc = P @ R.T + t
    return np.stack([Kc[0, 0] * Pc[:, 0] / Pc[:, 2] + Kc[0, 2], Kc[1, 1] * Pc[:, 1] / Pc[:, 2] + Kc[1, 2]], 1)


def poses(rng, n, zmin=.6, zmax=1.1):
    ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    rv = ax * rng.uniform(0.2, 2.5, size=(n, 1))
    t = np.stack([rng.uniform(-.1, .1, n), rng.uniform(-.07, .07, n), rng.uniform(zmin, zmax, n)], 1)
    return synth._rodrigues(rv), t


def plant_box(out, kp_norm, anchor, cell_shift, cls, det_logit, cls_logit):
    """write one (cell, anchor) of out (160, 13, 13) whose decoded keypoints are kp_norm (9, 2) (normalised), shifted by
    `cell_shift` cells to the right with identical raw values"""
    gx, gy = kp_norm[0, 0] * W, kp_norm[0, 1] * H
    cx, cy = int(gx), int(gy)
    base = anchor * (2 * K + 1 + NC)
    for k in range(K):
        vx, vy = kp_norm[k, 0] * W - cx, kp_norm[k, 1] * H - cy
        if k == 0:
            vx, vy = np.log(vx / (1 - vx)), np.log(vy / (1 - vy))
        assert 0 <= cx + cell_shift < W
        out[base + 2 * k, cy, cx + cell_shift] = vx
        out[base + 2 * k + 1, cy, cx + cell_shift] = vy
    out[base + 2 * K, cy, cx + cell_shift] = det_logit
    out[base + 2 * K + 1:base + 2 * K + 1 + NC, cy, cx + cell_shift] = 0.0
    out[base + 2 * K + 1 + cls, cy, cx + cell_shift] = cls_logit


def build_case(rng, classes, boxes, fallback_gt, corners, Kc):
    """-> (label rows (n, 21) in OCCLUSION order, planted output (1, 160, 13, 13) float32)"""
    out = np.zeros((NA * (2 * K + 1 + NC), H, W), np.float32)
    for a in range(NA):
        base = a * (2 * K + 1 + NC)
        out[base:base + 2 * K] = rng.normal(0, 0.5, size=(2 * K, H, W))
        out[base + 2 * K] = -8.0 + rng.normal(0, 0.01, size=(H, W))
        out[base + 2 * K + 1:base + 2 * K + 1 + NC] = rng.normal(0, 0.3, size=(NC, H, W))
    noisy = any(b[2] > 1e-2 for b in boxes)                              # closer objects, so 3e-2 noise leaves a usable pose
    R, t = poses(rng, max(len(classes), 1), *((.3, .4) if noisy else (.6, 1.1)))
    P9 = np.concatenate([np.zeros((1, 3)), corners.T[:, :3]])            # [0; corners3D] as valid_multi.py:135 builds it
    std = [project(P9, R[i], t[i], Kc) / np.array([IM_W, IM_H]) for i in range(len(classes))]    # (9, 2) normalised, box order
    rows = np.zeros((len(classes), NL))
    for i, c in enumerate(classes):
        occ = np.zeros((9, 2))
        for dst, src in enumerate(FIX):                                  # inverse of fix_corner_order
            occ[src] = std[i][dst]
        rows[i, 0] = c
        rows[i, 1:1 + 2 * K] = occ.reshape(-1)
        rows[i, -2:] = std[i].max(0) - std[i].min(0)
    for cls, anchor, noise, gi, shift in boxes:
        kp = std[gi] + rng.normal(0, noise, size=(9, 2))
        plant_box(out, kp, anchor, shift, cls, 4.0, 6.0)
    if fallback_gt is not None:                                          # below the threshold, but the running maximum
        kp = std[fallback_gt] + rng.normal(0, 1e-3, size=(9, 2))
        plant_box(out, kp, 3, 0, classes[0], -2.0, 1.5)
    if len(boxes) == 2 and boxes[0][:4] == boxes[1][:4]:                 # the equal-logit pair: identical raw values
        kp0 = std[boxes[0][3]]
        cx, cy = int(kp0[0, 0] * W), int(kp0[0, 1] * H)
        a = boxes[0][1] * (2 * K + 1 + NC)
        out[a:a + 2 * K + 1 + NC, cy, cx + boxes[1][4]] = out[a:a + 2 * K + 1 + NC, cy, cx]
    return rows, out[None]


def loader_rows(rows):
    """file rows whose loaded label holds `rows` at 2K+3 values per row: the reference's read_truths_args keeps the first 2K+1 of
    every 2K+3 values of a file row (utils_multi.py:394-401), while valid_multi.py:104 views the label with 2K+3 per row"""
    flat = rows.reshape(-1)
    n = -(-flat.size // (2 * K + 1))
    out = np.zeros((n, NL))
    out[:, :2 * K + 1] = np.pad(flat, (0, n * (2 * K + 1) - flat.size)).reshape(n, 2 * K + 1)
    return out


def write_ply(path, V):
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "element face 0\nproperty list uchar int vertex_indices\nend_header\n" % len(V))
        for v in V:
            f.write("%.6f %.6f %.6f\n" % tuple(v))


def main():
    import torch
    rng = np.random.default_rng(20261015)
    sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
    sys.modules.setdefault("matplotlib.pyplot", types.ModuleType("matplotlib.pyplot"))
    torch.Tensor.cuda = lambda self, *a, **k: self
    for d in (os.path.join(REF, "multi_obj_pose_estimation"), REF):
        sys.path.insert(0, d)
    with contextlib.redirect_stdout(io.StringIO()):
        import valid_multi as VM
    Kc = synth.intrinsics()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "tree")
        synth.write_linemod_multi_like(root, n=1)
        V = mesh_vertices(rng)
        write_ply(os.path.join(root, "mesh.ply"), V)
        vertices = np.c_[V, np.ones((len(V), 1))].transpose()
        corners = VM.get_3D_corners(vertices)
        outputs, targets = [], []
        for path, classes, boxes, fb in PLANTS:
            rows, o = build_case(rng, classes, boxes, fb, corners, Kc)
            lab = os.path.join(root, path.replace("JPEGImages", "labels_occlusion").replace(".png", ".txt"))
            with open(lab, "w") as f:
                if len(rows):
                    np.savetxt(f, loader_rows(rows))
            outputs.append(o)
        with open(os.path.join(root, "test.txt"), "w") as f:
            f.write("".join(os.path.join(root, p) + "\n" for p, *_ in PLANTS))
        k = synth.LINEMOD_INTRINSICS
        datacfg = os.path.join(root, "eval.data")
        with open(datacfg, "w") as f:
            f.write("valid = %s\nmesh = %s\nname = ape\ndiam = 0.103\nim_width = %d\nim_height = %d\nfx = %r\nfy = %r\nu0 = %r\nv0 = %r\n" % (
                os.path.join(root, "test.txt"), os.path.join(root, "mesh.ply"), IM_W, IM_H, k["fx"], k["fy"], k["u0"], k["v0"]))
        planted = [torch.from_numpy(o) for o in outputs]

        class PlantedModel:
            width, height = 416, 416

            def __init__(self, cfgfile):
                self.calls = 0

            def load_weights(self, f):
                pass

            def cuda(self):
                return self

            def eval(self):
                return self

            def __call__(self, x):
                o = planted[self.calls]
                self.calls += 1
                return o
        calls, lists, targets_seen = [], [], []
        orig_pnp, orig_gmrb = VM.pnp, VM.get_multi_region_boxes

        def rec_pnp(p3, p2, Km):
            R, t = orig_pnp(p3, p2, Km)
            calls.append((np.array(p3), np.array(p2), np.array(Km), np.array(R), np.array(t)))
            return R, t

        def rec_gmrb(output, *a, **kw):
            b = orig_gmrb(output, *a, **kw)
            lists.append(b[0])
            return b
        VM.Darknet, VM.pnp, VM.get_multi_region_boxes = PlantedModel, rec_pnp, rec_gmrb
        log = io.StringIO()
        cfgfile = os.path.join(REF, "multi_obj_pose_estimation", "cfg", "yolo-pose-multi.cfg")
        with contextlib.redirect_stdout(log):
            VM.valid(datacfg, cfgfile, "unused.weights")
        import dataset_multi as RD                                        # the reference's loader, for the stored targets
        ds = RD.listDataset(os.path.join(root, "test.txt"), shape=(416, 416), shuffle=False, objclass="ape")
        targets = [ds[i][1].numpy() for i in range(len(PLANTS))]

    printed = [float(m) for m in re.findall(r"Acc using \d+ px 2D Projection = ([0-9.]+)%", log.getvalue())]
    assert len(printed) == 10, log.getvalue()
    # per ground truth: the list position the pnp points came from, and the pixel error of the recorded poses
    pos, img_of, errs, flags, ci = [], [], [], [], 0
    for b, (boxes, tgt) in enumerate(zip(lists, targets)):
        truths = tgt.reshape(-1, NL)
        n = EM.truths_length(truths)
        n_listed = EM._count_listed(torch.from_numpy(outputs[b]), CONF_THRESH, NC, K, NA)
        for g in range(n):
            gt_call, pr_call = calls[ci], calls[ci + 1]
            ci += 2
            cand = [j for j, bx in enumerate(boxes)
                    if np.array_equal(np.array([[float(bx[2 * i]) * IM_W, float(bx[2 * i + 1]) * IM_H] for i in range(K)], np.float32),
                                      pr_call[1])]
            assert len(cand) == 1, (b, g, cand)
            pos.append(cand[0]); img_of.append(b)
            carried = int(truths[g][0]) not in [int(bx[2 * K + 2]) for bx in boxes]
            flags.append((1 if cand[0] >= n_listed else 0) | (2 if carried else 0))
            errs.append(EM.pixel_error(vertices, gt_call[3], gt_call[4], pr_call[3], pr_call[4], Kc))
    assert ci == len(calls)
    acc = EM.projection_accuracy_ref(errs)
    assert np.allclose(acc, printed, atol=5e-3), (acc, printed)
    for e in errs:
        assert min(abs(e - th) for th in THRESHOLDS) > 1e-2, e
    # the oracle reproduces every selection and every pnp point bit for bit
    ci = 0
    for b, (o, tgt) in enumerate(zip(outputs, targets)):
        res, _ = EM.evaluate_image_multi_ref(torch.from_numpy(o), tgt, CONF_THRESH, NC, K, synth.MULTI_ANCHORS, NA, vertices, corners, Kc,
                                             IM_W, IM_H, with_pose=False)
        for r in res:
            assert r["pos"] == pos[ci // 2] and r["fallback"] + 2 * r["carried"] == flags[ci // 2], (b, r, pos[ci // 2])
            assert np.array_equal(r["uv_gt"], calls[ci][1]) and np.array_equal(r["uv_pr"], calls[ci + 1][1]), b
            ci += 2
    out.update(outputs=np.concatenate(outputs), targets=np.stack(targets), vertices=vertices, corners3D=corners, K=Kc,
               conf_thresh=np.array(CONF_THRESH), anchors=np.array(synth.MULTI_ANCHORS), counts=np.array([len(p[1]) for p in PLANTS]),
               list_lengths=np.array([len(b) for b in lists]), pos=np.array(pos), flags=np.array(flags), image=np.array(img_of),
               pnp_points3d=np.stack([c[0] for c in calls]), pnp_points2d=np.stack([c[1] for c in calls]), pnp_K=calls[0][2],
               pnp_R=np.stack([c[3] for c in calls]), pnp_t=np.stack([c[4] for c in calls]),
               pixel_err=np.array(errs), accuracy=np.array(acc), printed_accuracy=np.array(printed))
    np.savez_compressed(os.path.join(HERE, "eval_multi.npz"), **out)
    print("eval_multi golden: %d images, %d ground truths, list positions %s, flags %s, pixel errors %s, accuracy %s" % (
        len(PLANTS), len(errs), pos, flags, np.round(errs, 3).tolist(), [round(a, 2) for a in acc]))


if __name__ == "__main__":
    main()
