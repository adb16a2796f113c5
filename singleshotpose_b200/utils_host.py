"""Host-side helpers of the reference's utils.py that train.py / valid.py / dataset.py pull in through `from utils import *`
(file and config readers, logging, 2-D box helpers, the CPU corner-confidence functions, mesh diameter / ADI metrics).  None of
them is on the GPU hot path; they exist so that the drop-in `utils` module resolves every name the reference's unchanged
scripts use.  Behaviour follows the reference function cited in each docstring (same arguments, same return conventions)."""
from __future__ import annotations

import math
import os
import struct
import time

import numpy as np
import torch


def makedirs(path):
    """utils.py:17-19"""
    if not os.path.exists(path):
        os.makedirs(path)


def get_all_files(directory):
    """utils.py:21-29: every file below `directory`, sub-directories expanded in place, os.listdir order"""
    found = []
    for name in os.listdir(directory):
        full = os.path.join(directory, name)
        if os.path.isfile(full):
            found.append(full)
        else:
            found += get_all_files(full)
    return found


def calc_pts_diameter(pts):
    """utils.py:50-58: largest pairwise distance of an (n,3) point set (blocked so that n = 10^4 vertices stays within memory)"""
    pts = np.asarray(pts)
    best = -1.0
    n = pts.shape[0]
    for i0 in range(0, n, 256):
        blk = pts[i0:i0 + 256]
        for j in range(blk.shape[0]):                       # pairs (i, k >= i), as the reference walks them
            d = blk[j][None, :] - pts[i0 + j:, :]
            m = float((d * d).sum(axis=1).max())
            if m > best:
                best = m
    return math.sqrt(best) if best >= 0 else -1


def adi(pts_est, pts_gt):
    """utils.py:60-64: mean nearest-neighbour distance from the ground-truth points to the estimated point set"""
    from scipy import spatial
    dists, _ = spatial.cKDTree(pts_est).query(pts_gt, k=1)
    return dists.mean()


def _extent(v):
    return np.min(v), np.max(v)


def get_2d_bb(box, size):
    """utils.py:102-112: [x0*size, y0*size, w*size, h*size] of a flat keypoint list (x, y interleaved)"""
    xy = np.reshape(box, [-1, 2])
    (x_lo, x_hi), (y_lo, y_hi) = _extent(xy[:, 0]), _extent(xy[:, 1])
    return [box[0] * size, box[1] * size, (x_hi - x_lo) * size, (y_hi - y_lo) * size]


def compute_2d_bb(pts):
    """utils.py:114-124: [cx, cy, w, h] of a (2,n) pixel array"""
    (x_lo, x_hi), (y_lo, y_hi) = _extent(pts[0, :]), _extent(pts[1, :])
    return [(x_hi + x_lo) / 2.0, (y_hi + y_lo) / 2.0, x_hi - x_lo, y_hi - y_lo]


def compute_2d_bb_from_orig_pix(pts, size):
    """utils.py:126-136: as compute_2d_bb on 640x480 pixel coordinates, normalised and scaled by `size`"""
    x_lo, x_hi = np.min(pts[0, :]) / 640.0, np.max(pts[0, :]) / 640.0
    y_lo, y_hi = np.min(pts[1, :]) / 480.0, np.max(pts[1, :]) / 480.0
    return [(x_hi + x_lo) / 2.0 * size, (y_hi + y_lo) / 2.0 * size, (x_hi - x_lo) * size, (y_hi - y_lo) * size]


def corner_confidences(gt_corners, pr_corners, th=80, sharpness=2, im_width=640, im_height=480):
    """utils.py:138-165 (CPU tensors): (2K,n) ground-truth and predicted corners -> (n,) mean confidence; the reference's
    batched variant divides without the 1e-5 guard of the scalar one."""
    n = gt_corners.size(1)
    K = gt_corners.numel() // (n * 2)
    scale = torch.tensor([im_width, im_height], dtype=torch.float32).repeat(K).view(2 * K, 1)
    d = ((gt_corners - pr_corners) * scale).view(K, 2, n)
    dist = torch.sqrt((d * d).sum(dim=1))                                     # (K, n) pixel distances
    inside = (dist < th).type_as(dist)
    conf = (torch.exp(sharpness * (1 - dist / th)) - 1) / (torch.exp(torch.tensor(float(sharpness))) - 1)
    return (inside * conf).mean(dim=0)


def corner_confidence(gt_corners, pr_corners, th=80, sharpness=2, im_width=640, im_height=480):
    """utils.py:167-187 (CPU tensors / lists): 2K-vectors -> scalar tensor.  The reference divides a (K,) tensor by a (K,1) tensor
    there, which broadcasts to (K,K) before the mean; reproduced because RegionLoss targets depend on it (region_loss.py:70)."""
    diff = torch.as_tensor(gt_corners, dtype=torch.float32) - pr_corners
    K = diff.numel() // 2
    scale = torch.tensor([im_width, im_height], dtype=torch.float32).repeat(K)
    d = (diff * scale).view(K, 2)
    dist = torch.sqrt((d * d).sum(dim=1))                                     # (K,)
    inside = (dist < th).type_as(dist)
    conf = torch.exp(sharpness * (1.0 - dist / th)) - 1
    conf0 = torch.exp(torch.tensor([float(sharpness)])) - 1 + 1e-5
    conf = inside * (conf / conf0.repeat(K, 1))                               # (K,) / (K,1) -> (K,K), times (K,)
    return torch.mean(conf)


def sigmoid(x):
    """utils.py:189-190"""
    return 1.0 / (math.exp(-x) + 1.)


def softmax(x):
    """utils.py:192-195 (over the whole tensor)"""
    e = torch.exp(x - torch.max(x))
    return e / e.sum()


def fix_corner_order(corners2D_gt):
    """utils.py:197-208"""
    out = np.zeros((9, 2), dtype='float32')
    for dst, src in enumerate((0, 1, 3, 5, 7, 2, 4, 6, 8)):
        out[dst, :] = corners2D_gt[src, :]
    return out


def read_truths(lab_path, num_keypoints=9):
    """utils.py:299-306"""
    num_labels = 2 * num_keypoints + 3
    if os.path.getsize(lab_path):
        truths = np.loadtxt(lab_path)
        return truths.reshape(truths.size // num_labels, num_labels)
    return np.array([])


def read_truths_args(lab_path, num_keypoints=9):
    """utils.py:308-315: class + 2K keypoint coordinates of every row, flattened (the two range columns are dropped).  Like the
    reference, the row width always comes from read_truths' default of 9 keypoints."""
    num_labels = 2 * num_keypoints + 1
    truths = read_truths(lab_path)
    if truths.size == 0:
        return np.array([])
    return np.ascontiguousarray(truths[:, :num_labels]).reshape(-1)


def label_rows_from_projection(px, width, height, class_id=0):
    """Label rows of label_file_creation.md from the projected keypoints px (n, 2, 9) -- column 0 the model origin [0, 0, 0],
    columns 1-8 the get_3D_corners corners, in pixels as compute_projection returns them -> (n, 21) float64:
    [class, x0/w, y0/h, ..., x8/w, y8/h, x range, y range], the ranges being the width and height of the tight box around the 8
    projected corners only (step 4), over the image size.  The pixel values are taken as float64, then divided."""
    P = np.asarray(px, dtype=np.float64)
    if P.ndim != 3 or P.shape[1:] != (2, 9):
        raise ValueError("projected keypoints must be (n, 2, 9), got %s" % (P.shape,))
    n = P.shape[0]
    rows = np.empty((n, 21))
    rows[:, 0] = class_id
    rows[:, 1:19:2] = P[:, 0] / float(width)
    rows[:, 2:19:2] = P[:, 1] / float(height)
    rows[:, 19] = (P[:, 0, 1:].max(1) - P[:, 0, 1:].min(1)) / float(width)
    rows[:, 20] = (P[:, 1, 1:].max(1) - P[:, 1, 1:].min(1)) / float(height)
    return rows


def read_pose(lab_path):
    """utils.py:419-424"""
    if os.path.getsize(lab_path):
        return np.loadtxt(lab_path)
    return np.array([])


def load_class_names(namesfile):
    """utils.py:325-332"""
    with open(namesfile, 'r') as fp:
        return [line.rstrip() for line in fp.readlines()]


def image2torch(img):
    """utils.py:334-341: PIL RGB image -> (1,3,H,W) float tensor in [0,1]"""
    a = torch.from_numpy(np.asarray(img, dtype=np.uint8).copy())
    return a.permute(2, 0, 1).contiguous().view(1, 3, img.height, img.width).float().div(255.0)


def read_ply_vertices(path):
    """(Nv, 3) float64 x, y, z of the `vertex` element of an ASCII PLY file (the format of the LINEMOD meshes the .data file's
    `mesh` entry names).  Binary PLY is refused."""
    return _read_ply(path, faces=False)[0]


def read_ply_mesh(path):
    """(vertices (Nv, 3) float64, faces (Nf, 3) int32) of an ASCII PLY file: the `vertex` element's x, y, z and the `face`
    element's vertex index lists.  Every face must be a triangle ("triangulate the mesh first") whose indices lie in [0, Nv).
    Binary PLY is refused."""
    return _read_ply(path, faces=True)


def _read_ply(path, faces):
    """Written from the PLY format: a header of `element <name> <count>` lines, each followed by its `property <type> <name>` /
    `property list <count type> <item type> <name>` lines, closed by `end_header`; then one text line per element item, the
    elements in header order.  faces=False stops after the vertex element and returns (V, None)."""
    V = F = None
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("%s: not a PLY file" % path)
        elements, fmt = [], None           # [name, count, [property names]]
        while True:
            line = f.readline()
            if not line:
                raise ValueError("%s: PLY header without end_header" % path)
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1] if len(tok) > 1 else None
            elif tok[0] == "element":
                elements.append([tok[1], int(tok[2]), []])
            elif tok[0] == "property" and elements:
                elements[-1][2].append(tok[-1])
        if fmt != "ascii":
            raise ValueError("%s: PLY format %r is not supported (ASCII PLY only)" % (path, fmt))
        for name, count, props in elements:
            if name == "vertex" and V is None:
                try:
                    cols = [props.index(a) for a in ("x", "y", "z")]
                except ValueError:
                    raise ValueError("%s: the vertex element has no x, y, z properties" % path)
                rows = [f.readline().split() for _ in range(count)]
                if any(len(r) < len(props) for r in rows):
                    raise ValueError("%s: truncated vertex data" % path)
                V = np.array([[float(r[c]) for c in cols] for r in rows], dtype=np.float64).reshape(count, 3)
                if not faces:
                    return V, None
            elif name == "face" and faces and F is None:
                if not props or props[0] not in ("vertex_indices", "vertex_index"):
                    raise ValueError("%s: the face element does not start with a vertex_indices list" % path)
                rows = [f.readline().split() for _ in range(count)]
                if any(not r for r in rows):
                    raise ValueError("%s: truncated face data" % path)
                for i, r in enumerate(rows):
                    if int(r[0]) != 3:
                        raise ValueError("%s: face %d has %s vertices: triangulate the mesh first" % (path, i, r[0]))
                    if len(r) < 4:
                        raise ValueError("%s: truncated face data" % path)
                F = np.array([[int(v) for v in r[1:4]] for r in rows], dtype=np.int64).reshape(count, 3)
            else:
                for _ in range(count):     # one text line per item, whatever its properties
                    f.readline()
    if V is None:
        raise ValueError("%s: no vertex element" % path)
    if F is None:
        raise ValueError("%s: no face element" % path)
    bad = (F < 0) | (F >= len(V))
    if bad.any():
        i = int(np.flatnonzero(bad.any(axis=1))[0])
        raise ValueError("%s: face %d has a vertex index outside [0, %d)" % (path, i, len(V)))
    return V, F.astype(np.int32)


def read_data_cfg(datacfg):
    """utils.py:343-358: `key = value` lines of a .data file; 'gpus' and 'num_workers' default to '0' and '10'"""
    options = {'gpus': '0', 'num_workers': '10'}
    with open(datacfg, 'r') as fp:
        for line in fp.readlines():
            line = line.strip()
            if line == '':
                continue
            key, value = line.split('=')
            options[key.strip()] = value.strip()
    return options


def scale_bboxes(bboxes, width, height):
    """utils.py:360-368: deep copy with x, w scaled by width and y, h by height"""
    import copy
    dets = copy.deepcopy(bboxes)
    for d in dets:
        d[0], d[1], d[2], d[3] = d[0] * width, d[1] * height, d[2] * width, d[3] * height
    return dets


def file_lines(thefilepath):
    """utils.py:370-379: number of newline bytes in the file"""
    count = 0
    with open(thefilepath, 'rb') as f:
        while True:
            buf = f.read(8192 * 1024)
            if not buf:
                break
            count += buf.count(b'\n')
    return count


def get_image_size(fname):
    """utils.py:381-414: (width, height) from the header of a PNG / GIF / JPEG file, None for anything else or a damaged header
    (file type from the magic bytes; the reference asks the `imghdr` module, removed in Python 3.13)"""
    with open(fname, 'rb') as fh:
        head = fh.read(24)
        if len(head) != 24:
            return None
        if head[:8] == b'\x89PNG\r\n\x1a\n':
            return struct.unpack('>ii', head[16:24])
        if head[:6] in (b'GIF87a', b'GIF89a'):
            return struct.unpack('<HH', head[6:10])
        if head[:2] == b'\xff\xd8':
            try:
                fh.seek(0)
                size, ftype = 2, 0
                while not 0xc0 <= ftype <= 0xcf:               # walk the segments up to a start-of-frame marker
                    fh.seek(size, 1)
                    byte = fh.read(1)
                    while ord(byte) == 0xff:
                        byte = fh.read(1)
                    ftype = ord(byte)
                    size = struct.unpack('>H', fh.read(2))[0] - 2
                fh.seek(1, 1)                                   # precision byte
                height, width = struct.unpack('>HH', fh.read(4))
                return width, height
            except Exception:
                return None
        return None


def logging(message):
    """utils.py:416-417"""
    print('%s %s' % (time.strftime("%Y-%m-%d %H:%M:%S", time.localtime()), message))


def read_rig(path):
    """utils.camera_rig of a .npz with the keys K (C, 3, 3), R (C, 3, 3), t (C, 3) and optionally dist (C, n), n in 4, 5, 8
    (camera-from-world extrinsics, x_c = R_c x_w + t_c); SspError naming the file for a missing file or key"""
    from ._lib import SspError
    from .utils import camera_rig
    if not os.path.isfile(path):
        raise SspError("rig file %s does not exist" % path)
    with np.load(path) as z:
        missing = [k for k in ("K", "R", "t") if k not in z.files]
        if missing:
            raise SspError("rig file %s has no %s" % (path, ", ".join(missing)))
        return camera_rig(z["K"], z["R"], z["t"], z["dist"] if "dist" in z.files else None)


def write_rig(path, rig):
    """write a utils.CameraRig to the .npz that read_rig reads back bit for bit: K, R, t and, for a rig with distortion, dist (C, 8)"""
    from ._lib import SspError
    from .utils import CameraRig
    if not isinstance(rig, CameraRig):
        raise SspError("write_rig takes a CameraRig (utils.camera_rig), got %s" % type(rig).__name__)
    arrays = dict(K=np.asarray(rig.K, np.float64), R=np.asarray(rig.R, np.float64), t=np.asarray(rig.t, np.float64))
    if rig.dist is not None:
        arrays["dist"] = np.asarray(rig.dist, np.float64)
    np.savez(path, **arrays)
