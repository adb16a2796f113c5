"""CPU tests of the multi-object training-image pipeline (image_multi.py of the reference's multi_obj_pose_estimation):
  * the numpy restatement (oracle/augment_multi_ref.py) against the reference's own load_data_detection through the
    committed golden (tests/golden/augment_multi.npz, written by tests/golden/make_golden_augment_multi.py): image, label,
    attempts per pasted object and the random-stream fingerprint;
  * the multi-object ops of the kernel core (singleshotpose_b200/csrc/augment_core.h) compiled for the host by
    tests/helpers/augment_multi_host.cpp and run through the op table: against Pillow directly (ImageChops.offset,
    transpose, ImageMath) and, driven by the product's host draws and labels (singleshotpose_b200/image_multi.py), against
    every golden case."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from oracle import augment_multi_ref as M
from singleshotpose_b200 import image_multi as IM
from singleshotpose_b200 import synth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = M.GOLDEN_CASES
JITTER, K, MAX_GT = M.JITTER, M.NUM_KEYPOINTS, M.MAX_NUM_GT


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_multi.npz"))


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    """the synthetic LINEMOD trees the golden was made on, keyed by source size"""
    out = {}
    for size in sorted({c[1] for c in CASES}):
        root = str(tmp_path_factory.mktemp("linemod%dx%d" % size))
        out[size] = (root, synth.write_linemod_multi_like(root, ow=size[0], oh=size[1]))
    return out


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("augmhost") / "libaugmhost.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", "augment_multi_host.cpp")])
    lib = C.CDLL(so)
    for f in ("h_multi_op_bytes", "h_multi_item_bytes", "h_multi_work_bytes"):
        getattr(lib, f).restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data


def _case_paths(trees, size, rels, bgi):
    root, bgs = trees[size]
    return root, [os.path.join(root, r) for r in rels], bgs[bgi]


# ------------------------------------------------------------------------------------------------ oracle vs reference golden
def test_oracle_matches_reference_golden(golden, trees):
    for name, size, shape, seed, rels, bgi in CASES:
        root, paths, bgpath = _case_paths(trees, size, rels, bgi)
        rng = random.Random(seed)
        for k, path in enumerate(paths):
            img, label, att = M.load_data_detection(path, shape, JITTER, bgpath, K, MAX_GT, rng=rng, root=root)
            tag = "%s_%d" % (name, k)
            assert np.array_equal(img, golden["img_" + tag]), tag
            assert np.array_equal(label, golden["label_" + tag]), tag
            assert att == list(golden["attempts_" + tag]), tag
        assert rng.getrandbits(64) == int(golden["rng_" + name]), name


def test_golden_exercises_rejection_and_empty_masks(golden, trees):
    """the cases include rejected candidates, and the tree has an empty mask (the S == 0 branch)"""
    assert max(int(golden[k].max()) for k in golden.files if k.startswith("attempts_")) > 10
    root, _bgs = trees[(160, 120)]
    assert not M.read_rgb(os.path.join(root, "LINEMOD/cat/mask/0001.png")).any()


# ------------------------------------------------------------------------------------------------ host build of the kernel ops
class HostPipeline:
    """GpuMultiAugmenter's sequence (begin, attempt rounds, finish) for ONE sample, on the host build of the op table, driven by
    the product's host code (draws, label transform, accept check)"""

    def __init__(self, host, W, H):
        self.h, self.W, self.H = host, W, H
        pos, neg = IM.mask_luts()
        self.luts = np.ascontiguousarray(np.concatenate([pos, neg]))
        self.state = np.zeros((4, H, W, 3), np.uint8)
        self.counts = np.zeros(4, np.uint32)
        assert host.h_multi_item_bytes() == C.sizeof(IM._MultiItem)

    def run(self, phase, img, mask, sw, sh, p, mask_bg=0, out_u8=None):
        W, H = self.W, self.H
        iw, ih = (sw, sh) if phase == 2 else (p["cw"], p["ch"])
        wb = self.h.h_multi_work_bytes(iw, ih, W, H, 3)
        work = np.zeros(wb, np.uint8)
        st = [self.state[k].ctypes.data for k in range(4)]
        it = IM._MultiItem(_p(img), _p(mask) if mask is not None else None, sw, sh, p.get("pleft", 0), p.get("ptop", 0), p.get("cw", 0),
                           p.get("ch", 0), p.get("flip", 0), p.get("shift_x", 0), p.get("shift_y", 0), mask_bg, *st, _p(self.counts),
                           _p(self.luts), _p(work), wb, _p(out_u8) if out_u8 is not None else None, None)
        table = np.zeros(self.h.h_multi_max_stages() * self.h.h_multi_op_bytes(), np.uint8)
        dims = (C.c_int * 32)()
        assert self.h.h_multi_run(phase, C.byref(it), 1, W, H, 3, _p(table), dims) == 0


def host_load_data_detection(host, imgpath, shape, bgpath, rng, root):
    W, H = shape
    nl = 2 * K + 3
    s = IM._Sample(imgpath, rng)
    bg, img, mask = M.read_rgb(bgpath), M.read_rgb(imgpath), M.read_rgb(IM.mask_path(imgpath))
    s.rng.shuffle(s.add_objs)
    p = IM.draw_main(img.shape[1], img.shape[0], shape, JITTER, s.rng)
    label = IM.fill_truth_detection(IM.read_label_rows(IM.label_path(imgpath)), 0, 0, p["flip"], p["dx"], p["dy"], 1. / p["sx"],
                                    1. / p["sy"], K, MAX_GT).reshape(-1, nl)
    hp = HostPipeline(host, W, H)
    hp.run(0, img, mask, img.shape[1], img.shape[0], p)
    attempts = []
    for obj in s.add_objs:
        n = 0
        while True:
            n += 1
            with open(os.path.join(root, "LINEMOD", obj, "train.txt")) as f:
                lines = f.readlines()
            path = os.path.join(root, lines[s.rng.randint(0, len(lines) - 1)].rstrip())
            view, vmask = M.read_rgb(path).copy(), M.read_rgb(IM.mask_path(path))
            c = IM.draw_crop(view.shape[1], view.shape[0], JITTER, s.rng)
            hp.run(1, view, vmask, view.shape[1], view.shape[0], c, mask_bg=1)
            S, I, acc = (int(v) for v in hp.counts[:3])
            assert bool(acc) == (S != 0 and float(I) / float(S) < 0.2)
            if acc:
                lab = IM.fill_truth_detection(IM.read_label_rows(IM.label_path(path)), 0, 0, c["flip"], c["dx"], c["dy"], 1. / c["sx"],
                                              1. / c["sy"], K, MAX_GT)
                label[len(attempts) + 1] = lab.reshape(-1, nl)[0]
                break
        attempts.append(n)
    out = np.zeros((H, W, 3), np.uint8)
    hp.run(2, bg, None, bg.shape[1], bg.shape[0], {}, out_u8=out)
    return out, label.reshape(-1), attempts


def test_kernel_ops_and_product_host_logic_match_reference_golden(host, golden, trees):
    """the whole sequence on the host build of the kernel core, with the product's draws and labels: every golden case is
    reproduced byte for byte (image), exactly (label), with the same attempts and the same random-stream fingerprint"""
    for name, size, shape, seed, rels, bgi in CASES:
        root, paths, bgpath = _case_paths(trees, size, rels, bgi)
        rng = random.Random(seed)
        for k, path in enumerate(paths):
            tag = "%s_%d" % (name, k)
            img, label, att = host_load_data_detection(host, path, shape, bgpath, rng, root)
            assert att == list(golden["attempts_" + tag]), tag
            assert np.array_equal(label, golden["label_" + tag]), tag
            assert np.array_equal(img, golden["img_" + tag]), tag
        assert rng.getrandbits(64) == int(golden["rng_" + name]), name


def test_place_main_equals_pillow_offset_and_transpose(host):
    """begin with a same-size crop (the resize is then a copy): offset + flip + mask_background equal ImageChops.offset and
    transpose(FLIP_LEFT_RIGHT) of Pillow itself, for shifts beyond the image size in both directions"""
    from PIL import Image, ImageChops
    rng = np.random.default_rng(5)
    W, H = 23, 17
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    mask = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    pos, _neg = IM.mask_luts()
    for dx, dy in [(0, 0), (5, -3), (-80, 80), (23, 17), (-23, -40), (47, -1), (80, 79)]:
        for flip in (0, 1):
            hp = HostPipeline(host, W, H)
            hp.run(0, img, mask, W, H, dict(pleft=0, ptop=0, cw=W, ch=H, flip=flip, shift_x=dx, shift_y=dy))
            a, m = ImageChops.offset(Image.fromarray(img), dx, dy), ImageChops.offset(Image.fromarray(mask), dx, dy)
            if flip:
                a, m = a.transpose(Image.FLIP_LEFT_RIGHT), m.transpose(Image.FLIP_LEFT_RIGHT)
            a, m = np.asarray(a), np.asarray(m)
            assert np.array_equal(hp.state[1], m) and np.array_equal(hp.state[3], m), (dx, dy, flip)
            assert np.array_equal(hp.state[0], (a * pos[m]).astype(np.uint8)) and np.array_equal(hp.state[2], hp.state[0]), (dx, dy, flip)


def test_superimpose_equals_pillow_imagemath(host):
    """one accepted attempt with a same-size, unflipped view: the new totals equal the reference's ImageMath expressions
    (image_multi.py:265-297) evaluated by Pillow; a heavily overlapping view is rejected and leaves the totals alone"""
    from PIL import Image, ImageMath
    ev = getattr(ImageMath, "unsafe_eval", None) or ImageMath.eval
    rng = np.random.default_rng(6)
    W, H = 31, 19
    hp = HostPipeline(host, W, H)
    tm = np.zeros((H, W, 3), np.uint8)
    tm[:, :8] = rng.integers(0, 256, (H, 8, 3))
    hp.state[3] = tm
    hp.state[2] = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    t_img, t_mask = hp.state[2].copy(), hp.state[3].copy()
    view = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    vmask = np.zeros((H, W, 3), np.uint8)
    vmask[:, 6:20] = rng.integers(0, 256, (H, 14, 3))
    masked = M.mask_background(view, vmask)
    hp.run(1, view.copy(), vmask, W, H, dict(pleft=0, ptop=0, cw=W, ch=H, flip=0), mask_bg=1)
    S, I = int((vmask > 200).sum()), int(((vmask > 200) & (t_mask > 200)).sum())
    assert (int(hp.counts[0]), int(hp.counts[1])) == (S, I) and hp.counts[2] == (float(I) / S < 0.2) == 1

    def band(a, c):
        return Image.fromarray(np.ascontiguousarray(a[..., c]))
    for c in range(3):
        m = band(vmask, c)
        neg, posm = m.point(lambda i: 1 - i / 255), m.point(lambda i: i / 255)
        want_m = np.asarray(ev("c + b * d", b=band(t_mask, c), c=m.point(lambda i: i), d=neg).convert("L"))
        want_i = np.asarray(ev("a * c + b * d", a=band(masked, c), b=band(t_img, c), c=posm, d=neg).convert("L"))
        assert np.array_equal(hp.state[3][..., c], want_m) and np.array_equal(hp.state[2][..., c], want_i), c
    before = hp.state.copy()
    hp.run(1, view.copy(), hp.state[3].copy(), W, H, dict(pleft=0, ptop=0, cw=W, ch=H, flip=0), mask_bg=1)
    assert hp.counts[2] == 0 and np.array_equal(hp.state, before)


def test_empty_candidate_is_rejected(host):
    W, H = 16, 12
    hp = HostPipeline(host, W, H)
    z = np.zeros((H, W, 3), np.uint8)
    hp.run(1, z.copy() + 7, z, W, H, dict(pleft=0, ptop=0, cw=W, ch=H, flip=1), mask_bg=1)
    assert list(hp.counts[:3]) == [0, 0, 0]


def test_product_host_helpers():
    assert IM.get_add_objs("eggbox") == M.ADD_OBJS["eggbox"] and len(IM.get_add_objs("ape")) == 7
    assert all(IM.get_add_objs(o) == M.ADD_OBJS[o] for o in synth.LINEMOD_OBJECTS)
    assert IM.mask_path("../LINEMOD/ape/JPEGImages/000012.png") == "../LINEMOD/ape/mask/0012.png"
    assert IM.label_path("../LINEMOD/ape/JPEGImages/000012.png") == "../LINEMOD/ape/labels/000012.txt"
    rows = synth.label_rows(3, n=3)
    for args in [(0.1, -0.05, 1.2, 0.9), (-0.2, 0.3, 0.8, 1.1)]:
        assert np.array_equal(IM.fill_truth_detection(rows.copy(), 0, 0, 1, *args, K, 2), M.fill_truth_detection(rows.copy(), *args, K, 2))
    assert not IM.fill_truth_detection(None, 0, 0, 0, 0, 0, 1, 1, K, MAX_GT).any()


def test_multi_pipeline_has_no_cpu_path():
    from singleshotpose_b200._lib import SspError
    with pytest.raises(SspError):
        IM.GpuMultiAugmenter("cpu")
