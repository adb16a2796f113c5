"""Make a custom object's training set from camera poses: label files, silhouette masks and the .data file.

    python -m singleshotpose_b200.make_dataset --mesh obj.ply --poses poses.npz --fx 572.4 --fy 573.6 --u0 325.3 --v0 242.0 \\
        --name obj [--class-id 0] [--test-list test_images.txt] --data-out cfg/obj.data

poses.npz holds `paths` (n image paths, each containing a JPEGImages directory), `R` (n, 3, 3) and `t` (n, 3) in the mesh's
units: the keys `python -m singleshotpose_b200.predict --out` writes, so predicted poses can be fed back as pseudo-labels.
For every image it writes, at the paths the training loaders read (dataset.label_path, dataset.mask_path -- the reference's
image.py:130-131 rules, `/00` -> `/` included):
  * labels/<name>.txt: one row of label_file_creation.md (utils.pose_label_rows), written by np.savetxt's default %.18e, which
    reads back bit for bit;
  * mask/<name>.png: the 8-bit silhouette of the mesh under the pose (utils.render_masks: 255 object, 0 background).
Then train.txt (every image not in --test-list) and, with --test-list, test.txt, both in the parent of the first image's
JPEGImages directory, and the .data file with the keys train.py and valid.py read.

Everything is checked before anything is written.  It refuses, naming the file: a missing image, images of different sizes,
two images whose mask or label paths collide, a pose whose mask would be empty because a vertex is behind the camera or
projects outside +-2^20 px, and a test-list image that has no pose."""
from __future__ import annotations

import argparse
import os

import numpy as np

BATCH = 256          # poses per render_masks call: bounds the device memory of the masks


class DatasetError(ValueError):
    pass


def load_poses(path):
    z = np.load(path)
    for k in ("paths", "R", "t"):
        if k not in z.files:
            raise DatasetError("%s has no %r array (expected paths, R, t)" % (path, k))
    paths, R, t = [str(p) for p in z["paths"]], np.asarray(z["R"], np.float64), np.asarray(z["t"], np.float64)
    n = len(paths)
    if R.shape != (n, 3, 3) or t.reshape(n, -1).shape != (n, 3):
        raise DatasetError("%s: R must be (n, 3, 3) and t (n, 3) for n = %d paths, got %s and %s" % (path, n, R.shape, t.shape))
    return paths, np.concatenate([R, t.reshape(n, 3, 1)], 2)


def check_images(paths):
    """-> (width, height) shared by every image; refuses missing images, mixed sizes and colliding mask / label paths"""
    from PIL import Image
    from .dataset import label_path, mask_path
    if not paths:
        raise DatasetError("no images")
    size, owner = None, {}
    for p in paths:
        if "JPEGImages" not in p:
            raise DatasetError("%s: the image path must contain a JPEGImages directory (the labels and masks go beside it)" % p)
        if not os.path.isfile(p):
            raise DatasetError("%s: no such image" % p)
        with Image.open(p) as im:
            s = im.size
        if size is None:
            size = s
        elif s != size:
            raise DatasetError("%s is %d x %d, but %s is %d x %d: all images must have one size" % (p, s[0], s[1], paths[0], *size))
        for kind, q in (("mask", mask_path(p)), ("label", label_path(p))):
            q = os.path.normpath(q)
            if q in owner:
                raise DatasetError("%s and %s both map to the %s file %s" % (owner[q], p, kind, q))
            if q == os.path.normpath(p):
                raise DatasetError("%s: its %s path is the image itself" % (p, kind))
            owner[q] = p
    return size


def make_dataset(mesh, poses, K, name, data_out, class_id=0, test_list=None, log=print):
    from PIL import Image
    from . import utils
    from .dataset import label_path, mask_path
    from .utils_host import read_ply_mesh
    paths, Rt = load_poses(poses)
    W, H = check_images(paths)
    test = set()
    if test_list:
        with open(test_list) as f:
            test = {os.path.normpath(s.strip()) for s in f if s.strip()}
        unknown = sorted(test - {os.path.normpath(p) for p in paths})
        if unknown:
            raise DatasetError("%s lists %s, which has no pose in %s" % (test_list, unknown[0], poses))
    V, F = read_ply_mesh(mesh)
    n = len(paths)
    for p0 in range(0, n, BATCH):                   # every pose must render before a file is written
        status = utils.render_masks(V, F, Rt[p0:p0 + BATCH], K, W, H)[1].cpu().numpy()
        bad = np.flatnonzero(status)
        if len(bad):
            i = p0 + int(bad[0])
            why = "a vertex at camera depth <= 0" if status[bad[0]] & 1 else "a vertex projects outside +-2^20 px"
            raise DatasetError("%s: the pose puts %s (status %d)" % (paths[i], why, status[bad[0]]))
    corners = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    rows = utils.pose_label_rows(corners, Rt, K, W, H, class_id)
    for p0 in range(0, n, BATCH):
        masks = utils.render_masks(V, F, Rt[p0:p0 + BATCH], K, W, H)[0].cpu().numpy()
        for j, m in enumerate(masks):
            p = paths[p0 + j]
            for q in (label_path(p), mask_path(p)):
                os.makedirs(os.path.dirname(q) or ".", exist_ok=True)
            np.savetxt(label_path(p), rows[p0 + j][None])
            Image.fromarray(m).save(mask_path(p))
    root = os.path.dirname(os.path.dirname(paths[0]))
    train_txt = os.path.join(root, "train.txt")
    with open(train_txt, "w") as f:
        f.writelines(p + "\n" for p in paths if os.path.normpath(p) not in test)
    valid_txt = train_txt
    if test_list:
        valid_txt = os.path.join(root, "test.txt")
        with open(valid_txt, "w") as f:
            f.writelines(p + "\n" for p in paths if os.path.normpath(p) in test)
    diam = utils.mesh_diameter(V)
    opts = dict(train=train_txt, valid=valid_txt, backup=os.path.join("backup", name), mesh=mesh, name=name, diam=repr(diam),
                width=W, height=H, fx=repr(float(K[0, 0])), fy=repr(float(K[1, 1])), u0=repr(float(K[0, 2])), v0=repr(float(K[1, 2])))
    os.makedirs(os.path.dirname(data_out) or ".", exist_ok=True)
    with open(data_out, "w") as f:
        f.writelines("%s = %s\n" % kv for kv in opts.items())
    log("%d images (%d x %d): labels, masks, %s%s, %s" % (n, W, H, train_txt, ", " + valid_txt if test_list else "", data_out))
    return opts


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m singleshotpose_b200.make_dataset",
                                 description="label files, silhouette masks and the .data file of a custom object's training set")
    ap.add_argument("--mesh", required=True, help="ASCII PLY triangle mesh of the object")
    ap.add_argument("--poses", required=True, help=".npz with paths, R (n, 3, 3), t (n, 3) in the mesh's units")
    for k in ("fx", "fy", "u0", "v0"):
        ap.add_argument("--" + k, type=float, required=True)
    ap.add_argument("--name", required=True)
    ap.add_argument("--class-id", type=int, default=0)
    ap.add_argument("--test-list", default=None, help="file of image paths (one per line) that go to test.txt")
    ap.add_argument("--data-out", required=True, help="the .data file to write")
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    from .utils import get_camera_intrinsic
    K = get_camera_intrinsic(a.u0, a.v0, a.fx, a.fy)
    try:
        make_dataset(a.mesh, a.poses, K, a.name, a.data_out, a.class_id, a.test_list)
    except DatasetError as e:
        raise SystemExit("make_dataset: %s" % e)


if __name__ == "__main__":
    main()
