"""TEST INFRASTRUCTURE ONLY (next to oracle/augment_ref.py; imported by the tests, smoke() and the golden generator) -- CPU restatement (numpy, byte arithmetic) of the reference's multi-object training-image pipeline,
multi_obj_pose_estimation/image_multi.py:
  mask_background                      :38-50    a * round(m / 255) per channel
  fill_truth_detection                 :123-165  ranges recomputed from the moved keypoints, stops at max_num_gt, flip ignored
  shifted_data_augmentation_with_mask  :184-228  crop -> resize -> ImageChops.offset (wrap-around roll) -> FLIP_LEFT_RIGHT
  data_augmentation_with_mask          :230-263  crop -> resize -> FLIP_LEFT_RIGHT
  superimpose_masked_imgs / _masks     :265-297  per-channel select by the pasted mask / clip(m + t * round(1 - m / 255))
  augment_objects, load_data_detection :299-382  rejection sampling of the pasted objects, main object on top, background
The resize, crop and point() tables are those of oracle/augment_ref.py (pinned against Pillow there).  File access goes through
callbacks so that the tests can feed in the synthetic tree of singleshotpose_b200.synth.write_linemod_multi_like.  The
resizes of already network-sized images (:317-318 and inside superimpose_*) return copies in Pillow and are left out.
"""
from __future__ import annotations

import os
import random as _random

import numpy as np

from oracle import augment_ref as A

PIXEL_THRESHOLD = 200
JITTER, NUM_KEYPOINTS, MAX_NUM_GT = 0.1, 9, 50      # dataset_multi.py:62, listDataset defaults

# the cases of tests/golden/augment_multi.npz (tests/golden/make_golden_augment_multi.py): name, source size of the synthetic
# tree (singleshotpose_b200.synth.write_linemod_multi_like), network shape, random.seed, main images (relative to the tree's
# root; several = one random stream across consecutive calls), background index
GOLDEN_CASES = [
    ("s96", (160, 120), (96, 96), 0, ["LINEMOD/ape/JPEGImages/000000.png"], 0),
    ("s128", (160, 120), (128, 128), 1, ["LINEMOD/eggbox/JPEGImages/000002.png"], 1),
    ("s416", (640, 480), (416, 416), 2, ["LINEMOD/cat/JPEGImages/000001.png"], 0),
    ("seq", (160, 120), (96, 96), 5, ["LINEMOD/duck/JPEGImages/000001.png", "LINEMOD/benchvise/JPEGImages/000000.png",
                                      "LINEMOD/holepuncher/JPEGImages/000002.png"], 1),
]
# dataset_multi.listDataset cases of the same golden (160x120 tree; list files of these paths, batch_size 2, cell_size 8):
# train mode at one `seen` per band of the resolution schedule (bands of 20 * nbatches * batch_size = 120), test mode with
# objclass 'ape' (the benchvise paths read ape's labels_occlusion/)
DATASET_TRAIN_LIST = ["LINEMOD/%s/JPEGImages/%06d.png" % (o, i) for o, i in
                      (("ape", 0), ("duck", 1), ("can", 2), ("eggbox", 0), ("glue", 1), ("phone", 2))]
DATASET_SEEN = (0, 130, 250, 370, 500)
DATASET_TEST_LIST = ["LINEMOD/benchvise/JPEGImages/%06d.png" % i for i in range(3)] + ["LINEMOD/duck/JPEGImages/000000.png"]

ADD_OBJS = {
    "ape": ["can", "cat", "duck", "glue", "holepuncher", "iron", "phone"],
    "benchvise": ["ape", "can", "cat", "driller", "duck", "glue", "holepuncher"],
    "cam": ["ape", "benchvise", "can", "cat", "driller", "duck", "holepuncher"],
    "can": ["ape", "benchvise", "cat", "driller", "duck", "eggbox", "holepuncher"],
    "cat": ["ape", "can", "duck", "glue", "holepuncher", "eggbox", "phone"],
    "driller": ["ape", "benchvise", "can", "cat", "duck", "glue", "holepuncher"],
    "duck": ["ape", "can", "cat", "eggbox", "glue", "holepuncher", "phone"],
    "eggbox": ["ape", "benchvise", "cam", "can", "cat", "duck", "glue", "holepuncher"],
    "glue": ["ape", "benchvise", "cam", "driller", "duck", "eggbox", "holepuncher"],
    "holepuncher": ["benchvise", "cam", "can", "cat", "driller", "duck", "eggbox"],
    "iron": ["ape", "benchvise", "can", "cat", "driller", "duck", "glue"],
    "lamp": ["ape", "benchvise", "can", "driller", "eggbox", "holepuncher", "iron"],
    "phone": ["ape", "benchvise", "cam", "can", "driller", "duck", "holepuncher"],
}


def mask_background(img, mask):
    pos, _neg = A.mask_luts()
    return (img.astype(np.int64) * pos[mask]).clip(0, 255).astype(np.uint8)


def offset(a, dx, dy):
    """ImageChops.offset(im, dx, dy)"""
    return np.roll(a, (dy, dx), (0, 1))


def superimpose_masks(mask, total_mask):
    _pos, neg = A.mask_luts()
    return np.clip(mask.astype(np.int64) + total_mask.astype(np.int64) * neg[mask], 0, 255).astype(np.uint8)


def superimpose_masked_imgs(masked_img, mask, total_img):
    pos, neg = A.mask_luts()
    return np.clip(masked_img.astype(np.int64) * pos[mask] + total_img.astype(np.int64) * neg[mask], 0, 255).astype(np.uint8)


def _jitter(ow, oh, jitter, rng):
    dw, dh = int(ow * jitter), int(oh * jitter)
    pleft, pright = rng.randint(-dw, dw), rng.randint(-dw, dw)
    ptop, pbot = rng.randint(-dh, dh), rng.randint(-dh, dh)
    swidth, sheight = ow - pleft - pright, oh - ptop - pbot
    sx, sy = float(swidth) / ow, float(sheight) / oh
    flip = rng.randint(1, 10000) % 2
    return pleft, ptop, swidth, sheight, sx, sy, flip


def _crop_resize(a, pleft, ptop, swidth, sheight, shape, resample):
    return A.resize_u8(A.crop_u8(a, (pleft, ptop, pleft + swidth - 1, ptop + sheight - 1)), shape, resample)


def shifted_data_augmentation_with_mask(img, mask, shape, jitter, rng=_random, resample=A.BICUBIC):
    oh, ow = img.shape[:2]
    pleft, ptop, swidth, sheight, sx, sy, flip = _jitter(ow, oh, jitter, rng)
    shift_x, shift_y = rng.randint(-80, 80), rng.randint(-80, 80)
    dx = (float(pleft) / ow) / sx - (float(shift_x) / shape[0])
    dy = (float(ptop) / oh) / sy - (float(shift_y) / shape[1])
    sized = offset(_crop_resize(img, pleft, ptop, swidth, sheight, shape, resample), shift_x, shift_y)
    msized = offset(_crop_resize(mask, pleft, ptop, swidth, sheight, shape, resample), shift_x, shift_y)
    if flip:
        sized, msized = sized[:, ::-1], msized[:, ::-1]
    return np.ascontiguousarray(sized), np.ascontiguousarray(msized), flip, dx, dy, sx, sy


def data_augmentation_with_mask(img, mask, shape, jitter, rng=_random, resample=A.BICUBIC):
    oh, ow = img.shape[:2]
    pleft, ptop, swidth, sheight, sx, sy, flip = _jitter(ow, oh, jitter, rng)
    dx, dy = (float(pleft) / ow) / sx, (float(ptop) / oh) / sy
    sized = _crop_resize(img, pleft, ptop, swidth, sheight, shape, resample)
    msized = _crop_resize(mask, pleft, ptop, swidth, sheight, shape, resample)
    if flip:
        sized, msized = sized[:, ::-1], msized[:, ::-1]
    return np.ascontiguousarray(sized), np.ascontiguousarray(msized), flip, dx, dy, sx, sy


def fill_truth_detection(bs, dx, dy, sx, sy, num_keypoints, max_num_gt):
    """image_multi.py:123-165 with the label rows already parsed (None / empty: the empty-file branch)"""
    num_labels = 2 * num_keypoints + 3
    label = np.zeros((max_num_gt, num_labels))
    if bs is None or np.size(bs) == 0:
        return label.reshape(-1)
    bs = np.array(bs, np.float64).reshape(-1, num_labels)
    cc = 0
    for i in range(bs.shape[0]):
        xs = [bs[i][2 * j + 1] for j in range(num_keypoints)]
        ys = [bs[i][2 * j + 2] for j in range(num_keypoints)]
        xs[0] = min(0.999, max(0, xs[0] * sx - dx))
        ys[0] = min(0.999, max(0, ys[0] * sy - dy))
        for j in range(1, num_keypoints):
            xs[j] = xs[j] * sx - dx
            ys[j] = ys[j] * sy - dy
        for j in range(num_keypoints):
            bs[i][2 * j + 1] = xs[j]
            bs[i][2 * j + 2] = ys[j]
        bs[i][2 * num_keypoints + 1] = max(xs) - min(xs)
        bs[i][2 * num_keypoints + 2] = max(ys) - min(ys)
        label[cc] = bs[i]
        cc += 1
        if cc >= max_num_gt:
            break
    return label.reshape(-1)


def mask_path(imgpath):
    return imgpath.replace("JPEGImages", "mask").replace("/00", "/").replace(".jpg", ".png")


def label_path(imgpath):
    return imgpath.replace("images", "labels").replace("JPEGImages", "labels").replace(".jpg", ".txt").replace(".png", ".txt")


def read_rgb(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"))


def read_label(path):
    return np.loadtxt(path) if os.path.getsize(path) else None


def read_lines(path):
    with open(path) as f:
        return f.readlines()


def load_data_detection(imgpath, shape, jitter, bgpath, num_keypoints, max_num_gt, rng=_random, root="..", resample=A.BICUBIC,
                        read_image=read_rgb, read_labels=read_label, read_list=read_lines):
    """image_multi.py:367-382 (+ augment_objects :299-365).  Returns (uint8 HxWx3 image, label, attempts per pasted object)."""
    shape = (int(shape[0]), int(shape[1]))
    num_labels = 2 * num_keypoints + 3
    bg = read_image(bgpath)
    objname = os.path.basename(os.path.dirname(os.path.dirname(imgpath)))
    add_objs = list(ADD_OBJS[objname])
    rng.shuffle(add_objs)
    img, mask = read_image(imgpath), read_image(mask_path(imgpath))
    img, mask, _flip, dx, dy, sx, sy = shifted_data_augmentation_with_mask(img, mask, shape, jitter, rng, resample)
    total_label = fill_truth_detection(read_labels(label_path(imgpath)), dx, dy, 1. / sx, 1. / sy, num_keypoints, max_num_gt)
    total_label = total_label.reshape(-1, num_labels)
    masked_img = mask_background(img, mask)
    total_mask, total_img = mask, masked_img
    attempts, count = [], 1
    for obj in add_objs:
        n = 0
        while True:
            n += 1
            lines = read_list(os.path.join(root, "LINEMOD", obj, "train.txt"))
            path = os.path.join(root, lines[rng.randint(0, len(lines) - 1)].rstrip())
            cimg = mask_background(read_image(path), read_image(mask_path(path)))
            cmask = read_image(mask_path(path))
            cimg, cmask, _f, cdx, cdy, csx, csy = data_augmentation_with_mask(cimg, cmask, shape, jitter, rng, resample)
            xx = cmask > PIXEL_THRESHOLD
            s = int(xx.sum())
            if s == 0:
                continue
            inter = int((xx & (total_mask > PIXEL_THRESHOLD)).sum())
            if float(inter) / float(s) < 0.2:
                total_mask = superimpose_masks(cmask, total_mask)
                total_img = superimpose_masked_imgs(cimg, cmask, total_img)
                clab = fill_truth_detection(read_labels(label_path(path)), cdx, cdy, 1. / csx, 1. / csy, num_keypoints, max_num_gt)
                total_label[count, :] = clab.reshape(-1, num_labels)[0, :]
                count += 1
                break
        attempts.append(n)
    total_img = superimpose_masked_imgs(masked_img, mask, total_img)
    out = A.change_background(total_img, total_mask, bg, resample)
    return out, total_label.reshape(-1), attempts
