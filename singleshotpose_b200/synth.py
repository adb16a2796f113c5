"""Seeded synthetic inputs for tests, smoke and bench (SURVEY.md 8d): uniform RGB batches,
one-ground-truth label rows in the reference's 50x21 layout (dataset.py:107 / region_loss.py:29-36),
box-corner 3-D models and exact/noisy 2-D projections for PnP."""
from __future__ import annotations

import os

import numpy as np
import torch

from .cfgs import LINEMOD_INTRINSICS


def images(batch, height=416, width=416, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(batch, 3, height, width, generator=g)


def targets(batch, seed=1, num_keypoints=9, max_objs=50):
    """(batch, 50*21) float32: one object per image, class 0, centroid U(.1,.9), 8 corners =
    centroid + U(-.15,.15), then x/y range; remaining slots zero."""
    rng = np.random.default_rng(seed)
    nl = 2 * num_keypoints + 3
    t = np.zeros((batch, max_objs * nl), np.float32)
    for b in range(batch):
        c = rng.uniform(0.1, 0.9, size=2)
        pts = np.concatenate([c[None], c[None] + rng.uniform(-0.15, 0.15, size=(num_keypoints - 1, 2))])
        t[b, 0] = 0
        t[b, 1:1 + 2 * num_keypoints] = pts.reshape(-1)
        t[b, 1 + 2 * num_keypoints] = pts[:, 0].max() - pts[:, 0].min()
        t[b, 2 + 2 * num_keypoints] = pts[:, 1].max() - pts[:, 1].min()
    return torch.from_numpy(t)


def targets_multi(batch, seed=1, num_keypoints=9, max_objs=50, num_classes=13, min_objs=1, max_gts=3):
    """(batch, 50*21) float32 with 1..max_gts objects per image (SURVEY 8d config 4): class U{0..12}, centroid U(.1,.9),
    corners = centroid + U(-.15,.15), x/y range U(0.05, 0.4) (drives the anchor choice)."""
    rng = np.random.default_rng(seed)
    nl = 2 * num_keypoints + 3
    t = np.zeros((batch, max_objs * nl), np.float32)
    for b in range(batch):
        for k in range(int(rng.integers(min_objs, max_gts + 1))):
            c = rng.uniform(0.1, 0.9, size=2)
            pts = np.concatenate([c[None], c[None] + rng.uniform(-0.15, 0.15, size=(num_keypoints - 1, 2))])
            o = k * nl
            t[b, o] = rng.integers(0, num_classes)
            t[b, o + 1:o + 1 + 2 * num_keypoints] = pts.reshape(-1)
            t[b, o + 1 + 2 * num_keypoints] = rng.uniform(0.05, 0.4)
            t[b, o + 2 + 2 * num_keypoints] = rng.uniform(0.05, 0.4)
    return torch.from_numpy(t)


MULTI_ANCHORS = [1.4820, 2.2412, 2.0501, 3.1265, 2.3946, 4.6891, 3.1018, 3.9910, 3.4879, 5.8851]   # yolo-pose-multi.cfg:240


def intrinsics(dtype=np.float64):
    k = LINEMOD_INTRINSICS
    return np.array([[k["fx"], 0.0, k["u0"]], [0.0, k["fy"], k["v0"]], [0.0, 0.0, 1.0]], dtype)


def box_points(half_extents=(0.038, 0.039, 0.046), with_center=True):
    """(9,3) or (8,3) float32: origin + the 8 corners in get_3D_corners order (utils.py:66-84:
    x outermost, z fastest, min before max)."""
    hx, hy, hz = half_extents
    c = np.array([[sx * hx, sy * hy, sz * hz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
    if with_center:
        c = np.concatenate([np.zeros((1, 3)), c])
    return c.astype(np.float32)


def _rodrigues(r):
    th = np.linalg.norm(r, axis=-1, keepdims=True)
    u = r / np.maximum(th, 1e-300)
    c, s = np.cos(th)[..., None], np.sin(th)[..., None]
    ux = np.zeros(r.shape[:-1] + (3, 3))
    ux[..., 0, 1], ux[..., 0, 2] = -u[..., 2], u[..., 1]
    ux[..., 1, 0], ux[..., 1, 2] = u[..., 2], -u[..., 0]
    ux[..., 2, 0], ux[..., 2, 1] = -u[..., 1], u[..., 0]
    return c * np.eye(3) + (1 - c) * u[..., :, None] * u[..., None, :] + s * ux


def pnp_problems(n, sigma=0.5, seed=5, with_center=True):
    """n synthetic PnP problems sharing one 3-D model and K.  Returns dict with P3 (N,3) f32,
    uv (n,N,2) f32, K (3,3) f32, and the generating R (n,3,3), t (n,3) in f64."""
    rng = np.random.default_rng(seed)
    P3 = box_points(with_center=with_center)
    K = intrinsics()
    ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    rv = ax * rng.uniform(0, np.pi, size=(n, 1))
    t = np.stack([rng.uniform(-.2, .2, n), rng.uniform(-.15, .15, n), rng.uniform(.6, 1.2, n)], 1)
    R = _rodrigues(rv)
    Pc = np.einsum("nij,kj->nki", R, P3.astype(np.float64)) + t[:, None, :]
    uv = np.stack([K[0, 0] * Pc[..., 0] / Pc[..., 2] + K[0, 2], K[1, 1] * Pc[..., 1] / Pc[..., 2] + K[1, 2]], -1)
    uv = uv + rng.normal(size=uv.shape) * sigma
    return dict(P3=P3, uv=uv.astype(np.float32), K=K.astype(np.float32), R=R, t=t)


def photo_sample(seed, ow=640, oh=480, bw=500, bh=375):
    """One synthetic training sample for the image pipeline (image.py:129-142): (image, object mask, background), uint8 HxWx3 RGB.
    Integer arithmetic only, so every platform generates the same bytes.  The mask is an ellipse (255 inside, 0 outside) with
    an anti-aliased rim of intermediate values, like the LINEMOD masks after PNG decoding."""
    rng = np.random.default_rng(1000 + seed)
    yy, xx = np.mgrid[0:oh, 0:ow]
    base = np.stack([xx * 255 // max(ow - 1, 1), yy * 255 // max(oh - 1, 1), (xx + yy) * 255 // max(ow + oh - 2, 1)], -1)
    img = np.clip(base + rng.integers(-48, 49, (oh, ow, 3)), 0, 255).astype(np.uint8)
    cx, cy = int(rng.integers(ow // 4, 3 * ow // 4)), int(rng.integers(oh // 4, 3 * oh // 4))
    ax, ay = int(rng.integers(ow // 8, ow // 3)), int(rng.integers(oh // 8, oh // 3))
    d = ((xx - cx) * ay) ** 2 + ((yy - cy) * ax) ** 2                       # < (ax*ay)^2 inside the ellipse
    r2 = (ax * ay) ** 2
    m = np.where(d < r2 * 9 // 10, 255, np.where(d < r2, rng.integers(0, 256, (oh, ow)), 0)).astype(np.uint8)
    mask = np.repeat(m[:, :, None], 3, 2)
    by, bx = np.mgrid[0:bh, 0:bw]
    bbase = np.stack([255 - bx * 255 // max(bw - 1, 1), (bx * by) % 256, by * 255 // max(bh - 1, 1)], -1)
    bg = np.clip(bbase + rng.integers(-64, 65, (bh, bw, 3)), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(img), np.ascontiguousarray(mask), np.ascontiguousarray(bg)


def label_rows(seed, n=1, num_keypoints=9):
    """n label rows [cls, x0, y0, ..., x8, y8, xrange, yrange] like the reference's labels/*.txt"""
    rng = np.random.default_rng(2000 + seed)
    rows = np.zeros((n, 2 * num_keypoints + 3))
    for r in rows:
        c = rng.uniform(0.2, 0.8, 2)
        pts = c + rng.uniform(-0.15, 0.15, (num_keypoints, 2))
        pts[0] = c
        r[0] = 0
        r[1:1 + 2 * num_keypoints] = pts.reshape(-1)
        r[-2:] = pts.max(0) - pts.min(0)
    return rows


def write_linemod_like(root, n=4, ow=160, oh=120, num_bg=3, fmt="png"):
    """A tiny dataset tree with the reference's path conventions (image.py:130-131, train.py:309): JPEGImages/00000i.png, mask/000i.png,
    labels/00000i.txt, a background folder and the list file.  PNG throughout (lossless, so every decoder yields the same bytes).
    fmt="jpg": images and backgrounds are JPEG instead (JPEGImages/00000i.jpg, Pillow quality 95, its default 4:2:0), masks
    stay PNG -- the layout of the real LINEMOD and VOC trees.  Returns (list file path, background file names)."""
    if fmt not in ("png", "jpg"):
        raise ValueError("fmt must be 'png' or 'jpg'")
    kw = dict(quality=95) if fmt == "jpg" else {}
    from PIL import Image
    base = os.path.join(root, "LINEMOD", "ape")
    for d in ("JPEGImages", "mask", "labels"):
        os.makedirs(os.path.join(base, d), exist_ok=True)
    bgdir = os.path.join(root, "VOCdevkit", "VOC2012", "JPEGImages")
    os.makedirs(bgdir, exist_ok=True)
    lines = []
    for i in range(n):
        img, mask, _bg = photo_sample(50 + i, ow, oh, 8, 8)
        name = "%06d" % i
        Image.fromarray(img).save(os.path.join(base, "JPEGImages", name + "." + fmt), **kw)
        Image.fromarray(mask).save(os.path.join(base, "mask", "%04d.png" % i))
        rows = label_rows(50 + i, n=1 + i % 2)
        with open(os.path.join(base, "labels", name + ".txt"), "w") as f:
            if i != 3:                                   # sample 3 has an empty label file (os.path.getsize == 0 branch)
                np.savetxt(f, rows)
        lines.append(os.path.join(base, "JPEGImages", name + "." + fmt))
    bgs = []
    for j in range(num_bg):
        _i, _m, bg = photo_sample(70 + j, 8, 8, 100 + 13 * j, 75 + 7 * j)
        pth = os.path.join(bgdir, "bg%d.%s" % (j, fmt))
        Image.fromarray(bg).save(pth, **kw)
        bgs.append(pth)
    listfile = os.path.join(root, "train.txt")
    with open(listfile, "w") as f:
        f.write("\n".join(lines) + "\n")
    return listfile, bgs


def closed_mesh(rings=60, segments=100, half_extents=(0.038, 0.039, 0.046), bumps=0.15, seed=0):
    """A closed, LINEMOD-sized triangle mesh: a latitude-longitude ellipsoid (two poles, `rings` rings of `segments` vertices)
    whose radius is modulated by a few seeded bumps (bumps=0: the plain ellipsoid, which is convex).  The defaults give 6002
    vertices and 12000 faces, about the size of a LINEMOD mesh.  Returns (vertices (Nv, 3) float64, rounded to 6 decimals as an
    ASCII PLY stores them, faces (Nf, 3) int32), every face wound the same way."""
    rng = np.random.default_rng(seed)
    th = np.pi * (np.arange(rings) + 1) / (rings + 1)                       # polar angle of each ring
    ph = 2 * np.pi * np.arange(segments) / segments
    T, P = np.meshgrid(th, ph, indexing="ij")
    d = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    d = np.concatenate([[[0.0, 0.0, 1.0]], d, [[0.0, 0.0, -1.0]]])
    k = rng.normal(size=(4, 3))
    k /= np.linalg.norm(k, axis=1, keepdims=True)
    r = 1.0 + bumps * np.tanh(np.cos(3 * d @ k.T + rng.uniform(0, 2 * np.pi, 4)).sum(1))
    V = np.round(d * r[:, None] * np.asarray(half_extents), 6)
    ring = lambda i, j: 1 + i * segments + j % segments
    F = [[0, ring(0, j + 1), ring(0, j)] for j in range(segments)]
    for i in range(rings - 1):
        for j in range(segments):
            a, b, c, e = ring(i, j), ring(i, j + 1), ring(i + 1, j), ring(i + 1, j + 1)
            F += [[a, b, e], [a, e, c]]
    last = len(d) - 1
    F += [[last, ring(rings - 1, j), ring(rings - 1, j + 1)] for j in range(segments)]
    return V, np.array(F, dtype=np.int32)


def write_ply(path, vertices, faces):
    """ASCII PLY with a vertex element (x, y, z) and a face element (vertex_indices), the layout of the LINEMOD meshes"""
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(vertices), len(faces)))
        f.writelines("%.6f %.6f %.6f\n" % tuple(v) for v in vertices)
        f.writelines("3 %d %d %d\n" % tuple(t) for t in faces)


def object_poses(n, seed=0, depth=(0.6, 1.1)):
    """n poses (R (n, 3, 3), t (n, 3)) of an object-sized mesh in front of the LINEMOD camera, fully inside a 640 x 480 view"""
    rng = np.random.default_rng(seed)
    ax = rng.normal(size=(n, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    R = _rodrigues(ax * rng.uniform(0, np.pi, size=(n, 1)))
    t = np.stack([rng.uniform(-.08, .08, n), rng.uniform(-.06, .06, n), rng.uniform(*depth, n)], 1)
    return R, t


LINEMOD_OBJECTS = ("ape", "benchvise", "cam", "can", "cat", "driller", "duck", "eggbox", "glue", "holepuncher", "iron", "lamp", "phone")


def object_sample(seed, ow, oh, empty=False, spread=False):
    """One LINEMOD-like object view: (image, mask), uint8 HxWx3.  The mask is a SMALL ellipse (about 3 % of the frame, like the
    LINEMOD objects) near the centre, so that pasted objects overlap often enough to be rejected now and then but a scene of 8
    objects still fits; `empty=True` gives an all-zero mask.  `spread=True` places the object anywhere in the central 3/4 of the
    frame instead of the central 2/5 (fewer rejections; used for throughput runs on many samples).  Integer arithmetic only."""
    rng = np.random.default_rng(3000 + seed)
    yy, xx = np.mgrid[0:oh, 0:ow]
    base = np.stack([(xx * 7 + seed * 31) % 256, (yy * 5 + seed * 17) % 256, ((xx + yy) * 3) % 256], -1)
    img = np.clip(base + rng.integers(-40, 41, (oh, ow, 3)), 0, 255).astype(np.uint8)
    if spread:
        cx, cy = int(rng.integers(ow // 8, 7 * ow // 8)), int(rng.integers(oh // 8, 7 * oh // 8))
    else:
        cx, cy = int(rng.integers(3 * ow // 10, 7 * ow // 10)), int(rng.integers(3 * oh // 10, 7 * oh // 10))
    ax, ay = int(rng.integers(ow // 14, ow // 8)), int(rng.integers(oh // 14, oh // 8))
    d = ((xx - cx) * ay) ** 2 + ((yy - cy) * ax) ** 2
    r2 = (ax * ay) ** 2
    m = np.where(d < r2 * 8 // 10, 255, np.where(d < r2, rng.integers(0, 256, (oh, ow)), 0)).astype(np.uint8)
    if empty:
        m[:] = 0
    return np.ascontiguousarray(img), np.ascontiguousarray(np.repeat(m[:, :, None], 3, 2))


def write_linemod_multi_like(root, n=3, ow=160, oh=120, num_bg=2, spread=False):
    """All 13 LINEMOD object folders with the paths the multi-object pipeline reads (image_multi.py: LINEMOD/<obj>/train.txt
    listing LINEMOD/<obj>/JPEGImages/00000i.png relative to `root`, mask/000i.png, labels/00000i.txt), the test-mode labels of
    dataset_multi.py (labels_occlusion/00000i.txt, several objects per file, every 5th file empty), plus backgrounds under bg/.
    PNG throughout.  The mask of cat's image 1 is empty (the "no object pixels" rejection); every 4th label file is empty.
    Returns the background paths."""
    from PIL import Image
    for k, obj in enumerate(LINEMOD_OBJECTS):
        base = os.path.join(root, "LINEMOD", obj)
        for d in ("JPEGImages", "mask", "labels", "labels_occlusion"):
            os.makedirs(os.path.join(base, d), exist_ok=True)
        lines = []
        for i in range(n):
            seed = 100 * k + i
            img, mask = object_sample(seed, ow, oh, empty=(obj == "cat" and i == 1), spread=spread)
            name = "%06d" % i
            Image.fromarray(img).save(os.path.join(base, "JPEGImages", name + ".png"))
            Image.fromarray(mask).save(os.path.join(base, "mask", "%04d.png" % i))
            rows = label_rows(seed, n=1 + i % 2)
            rows[:, 0] = k
            with open(os.path.join(base, "labels", name + ".txt"), "w") as f:
                if (k * n + i) % 4 != 3:
                    np.savetxt(f, rows)
            with open(os.path.join(base, "labels_occlusion", name + ".txt"), "w") as f:      # the test-mode labels of dataset_multi
                if (k * n + i) % 5 != 4:
                    occ = label_rows(500 + seed, n=1 + (k + i) % 3)
                    occ[:, 0] = [(k + j) % 13 for j in range(len(occ))]
                    np.savetxt(f, occ)
            lines.append("LINEMOD/%s/JPEGImages/%s.png" % (obj, name))
        with open(os.path.join(base, "train.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
    bgdir = os.path.join(root, "bg")
    os.makedirs(bgdir, exist_ok=True)
    bgs = []
    for j in range(num_bg):
        _i, _m, bg = photo_sample(90 + j, 8, 8, ow * 5 // 4 + 13 * j, oh * 5 // 4 + 7 * j)
        pth = os.path.join(bgdir, "bg%d.png" % j)
        Image.fromarray(bg).save(pth)
        bgs.append(pth)
    return bgs
