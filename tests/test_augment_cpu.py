"""CPU tests of the training-image pipeline (SURVEY 8f.3):
  * the oracle (oracle/augment_ref.py) against Pillow itself -- the library whose arithmetic the reference's image.py calls --
    and against the reference's own functions through the committed golden (tests/golden/augment.npz);
  * the KERNEL arithmetic and pass sequencing (singleshotpose_b200/csrc/augment_core.h, shared by the CUDA kernels) compiled
    for the host by tests/helpers/augment_host.cpp and checked bit-exactly the same way;
  * the product's host logic (random draws, point() tables, label transform)."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import augment_ref as A
from singleshotpose_b200 import image as I
from singleshotpose_b200 import synth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUG_CASES = [(0, (160, 120), (100, 75), (96, 96)), (1, (160, 120), (211, 97), (128, 128)),
             (2, (320, 240), (250, 187), (224, 224)), (3, (96, 128), (64, 64), (160, 160))]
RESIZE_CASES = [(48, 64, 32, 32), (120, 160, 104, 104), (37, 53, 111, 97), (100, 100, 100, 50), (60, 80, 60, 80), (13, 200, 208, 7),
                (5, 5, 64, 64), (300, 2, 3, 300), (300, 2, 30, 2), (50, 50, 20, 50)]          # (in_h, in_w, out_h, out_w)
FILTERS = (A.BICUBIC, A.BILINEAR, A.NEAREST)


def _all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.ascontiguousarray(np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8))


@pytest.fixture(scope="module")
def pil():
    return pytest.importorskip("PIL.Image")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    """the kernel core compiled for the host"""
    so = str(tmp_path_factory.mktemp("aughost") / "libaughost.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", "augment_host.cpp")])
    lib = C.CDLL(so)
    lib.h_resize_work_bytes.restype = C.c_longlong
    lib.h_augment_work_bytes.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _host_resize(lib, img, size, rs, box=None):
    ih, iw = img.shape[:2]
    ow, oh = size
    l, t, r, b = box if box else (0, 0, iw, ih)
    wb = lib.h_resize_work_bytes(r - l, b - t, ow, oh, rs)
    work, dst = np.empty(wb, np.uint8), np.empty((oh, ow, 3), np.uint8)
    assert lib.h_resize(_p(img), iw, ih, l, t, r - l, b - t, _p(dst), ow, oh, rs, _p(work), C.c_longlong(wb)) == 0
    return dst


# ------------------------------------------------------------------------------------------------ oracle vs Pillow / reference
def test_oracle_hsv_vs_pillow(pil):
    """numpy oracle vs Pillow's convert(): every 7th of the 2^24 byte triples (2.4 M colours, all residues of r, g, b) by default,
    all of them with SSP_FULL_HSV=1 (~1 min; zero mismatches when the oracle was written).  The kernel arithmetic itself
    (augment_core.h) is checked over ALL triples below -- it is C and takes seconds."""
    rgb = _all_colours()
    if os.environ.get("SSP_FULL_HSV", "0") != "1":
        rgb = np.ascontiguousarray(rgb[::7])
    n = rgb.shape[0]
    rgb = rgb[: n - n % 1024].reshape(-1, 1024, 3)
    assert np.array_equal(A.rgb2hsv_u8(rgb), np.asarray(pil.fromarray(rgb, "RGB").convert("HSV")))
    assert np.array_equal(A.hsv2rgb_u8(rgb), np.asarray(pil.fromarray(rgb, "HSV").convert("RGB")))


def test_oracle_resize_crop_point_vs_pillow(pil):
    rng = np.random.default_rng(0)
    for (ih, iw, oh, ow) in RESIZE_CASES:
        img = rng.integers(0, 256, (ih, iw, 3), dtype=np.uint8)
        for rs in FILTERS:
            assert np.array_equal(A.resize_u8(img, (ow, oh), rs), np.asarray(pil.fromarray(img).resize((ow, oh), rs))), (ih, iw, oh, ow, rs)
    img = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    for box in [(-5, -3, 70, 50), (5, 3, 40, 30), (-10, -10, 20, 20), (30, 20, 80, 60), (0, 0, 64, 48), (-50, -50, -10, -10)]:
        assert np.array_equal(A.crop_u8(img, box), np.asarray(pil.fromarray(img).crop(box)))
    ramp = pil.fromarray(np.arange(256, dtype=np.uint8).reshape(16, 16))
    for f in (lambda i: i * 1.5, lambda i: i * 0.66, lambda i: i / 255, lambda i: 1 - i / 255, lambda i: i - 300.5):
        assert np.array_equal(np.asarray(ramp.point(f)).reshape(-1), A.point_lut(f))


def test_oracle_matches_reference_golden(golden):
    """the golden holds the outputs of the reference's own image.py functions (make_golden.py main_augment)"""
    for seed, (ow, oh), (bw, bh), shape in AUG_CASES:
        img, mask, bg = synth.photo_sample(seed, ow, oh, bw, bh)
        comp = A.change_background(img, mask, bg)
        assert np.array_equal(comp, golden["comp_%d" % seed])
        res, flip, dx, dy, sx, sy = A.data_augmentation(comp, shape, 0.2, 0.1, 1.5, 1.5, rng=random.Random(seed))
        assert np.array_equal(res, golden["img_%d" % seed])
        assert np.array_equal(np.array([flip, dx, dy, sx, sy]), golden["xform_%d" % seed])
        rows = synth.label_rows(seed, n=1 + seed % 2)
        assert np.array_equal(A.fill_truth_detection(rows, flip, dx, dy, 1. / sx, 1. / sy, 9, 50), golden["label_%d" % seed])


# ------------------------------------------------------------------------------------------------ kernel core on the host
def test_kernel_core_hsv_all_colours(host, pil):
    rgb = _all_colours()
    out = np.empty_like(rgb)
    host.h_rgb2hsv(_p(rgb), _p(out), C.c_longlong(1 << 24))
    assert np.array_equal(out.reshape(4096, 4096, 3), np.asarray(pil.fromarray(rgb.reshape(4096, 4096, 3), "RGB").convert("HSV")))
    host.h_hsv2rgb(_p(rgb), _p(out), C.c_longlong(1 << 24))
    assert np.array_equal(out.reshape(4096, 4096, 3), np.asarray(pil.fromarray(rgb.reshape(4096, 4096, 3), "HSV").convert("RGB")))


def test_kernel_core_resize_vs_oracle(host):
    rng = np.random.default_rng(1)
    for (ih, iw, oh, ow) in RESIZE_CASES:
        img = rng.integers(0, 256, (ih, iw, 3), dtype=np.uint8)
        for rs in FILTERS:
            assert np.array_equal(_host_resize(host, img, (ow, oh), rs), A.resize_u8(img, (ow, oh), rs)), (ih, iw, oh, ow, rs)
    img = rng.integers(0, 256, (120, 160, 3), dtype=np.uint8)
    for box in [(-20, -10, 150, 100), (10, 5, 120, 90), (-30, 20, 200, 60), (100, 100, 101, 101), (-50, -50, -10, -10)]:
        for rs in FILTERS:                                            # the jitter crop is fused into the first pass's reads
            assert np.array_equal(_host_resize(host, img, (96, 64), rs, box), A.resize_u8(A.crop_u8(img, box), (96, 64), rs)), (box, rs)
    work = np.empty(16, np.uint8)
    assert host.h_resize(_p(img), 160, 120, 0, 0, 160, 120, _p(img), 80, 60, 3, _p(work), C.c_longlong(16)) == -2     # work too small
    assert host.h_resize(_p(img), 160, 120, 0, 0, 0, 120, _p(img), 80, 60, 3, _p(work), C.c_longlong(16)) == -1       # empty window


def test_kernel_core_full_sample_vs_reference_golden(host, golden):
    for seed, (ow, oh), (bw, bh), shape in AUG_CASES:
        img, mask, bg = synth.photo_sample(seed, ow, oh, bw, bh)
        p = I.draw_augmentation(ow, oh, 0.2, 0.1, 1.5, 1.5, random.Random(seed))
        luts = np.ascontiguousarray(np.concatenate(I.mask_luts() + I.distort_luts(p["dhue"], p["dsat"], p["dexp"])))
        wb = host.h_augment_work_bytes(ow, oh, bw, bh, p["cw"], p["ch"], shape[0], shape[1], 3)
        work = np.empty(wb, np.uint8)
        o8, of = np.empty((shape[1], shape[0], 3), np.uint8), np.empty((3, shape[1], shape[0]), np.float32)
        rc = host.h_augment_sample(_p(img), _p(mask), ow, oh, _p(bg), bw, bh, _p(luts), p["pleft"], p["ptop"], p["cw"], p["ch"],
                                   shape[0], shape[1], 3, _p(work), C.c_longlong(wb), _p(o8), _p(of))
        assert rc == 0
        assert np.array_equal(o8, golden["img_%d" % seed])
        assert np.array_equal(of, np.transpose(o8, (2, 0, 1)).astype(np.float32) / np.float32(255))       # ToTensor


# ------------------------------------------------------------------------------------------------ product host logic
def test_product_draws_tables_and_labels_follow_the_reference(golden):
    for seed in range(40):
        a = I.draw_augmentation(640, 480, 0.2, 0.1, 1.5, 1.5, random.Random(seed))
        b = A.draw_augmentation(640, 480, 0.2, 0.1, 1.5, 1.5, random.Random(seed))
        assert all(a[k] == b[k] for k in ("pleft", "ptop", "flip", "dhue", "dsat", "dexp"))
        assert (a["cw"], a["ch"]) == (640 - b["pleft"] - b["pright"] - 1, 480 - b["ptop"] - b["pbot"] - 1)
    r = random.Random(7)
    cases = [(0.07, 1.3, 0.8), (0.1, 1.5, 1.5), (-0.1, 1 / 1.5, 1 / 1.5), (0, 1, 1), (0.5 / 255, 0.5, 2.5 / 255)]
    cases += [(r.uniform(-0.1, 0.1), I.rand_scale(1.5, r), I.rand_scale(1.5, r)) for _ in range(300)]
    for hsv in cases:          # the product builds the point() tables vectorised; the oracle calls the reference's lambdas
        for f, g in zip(I.mask_luts() + I.distort_luts(*hsv), A.mask_luts() + A.distort_luts(*hsv)):
            assert np.array_equal(f, g), hsv
    for seed, (ow, oh), _bg, shape in AUG_CASES:
        p = I.draw_augmentation(ow, oh, 0.2, 0.1, 1.5, 1.5, random.Random(seed))
        assert np.array_equal(np.array([p["flip"], p["dx"], p["dy"], p["sx"], p["sy"]]), golden["xform_%d" % seed])
        lab = I.fill_truth_detection(synth.label_rows(seed, n=1 + seed % 2), shape[0], shape[1], p["flip"], p["dx"], p["dy"],
                                     1. / p["sx"], 1. / p["sy"], 9, 50)
        assert np.array_equal(lab, golden["label_%d" % seed])


def test_image_pipeline_has_no_cpu_path():
    import torch
    from singleshotpose_b200._lib import SspError
    with pytest.raises(SspError):
        I.resize_u8(torch.zeros(4, 4, 3, dtype=torch.uint8), (2, 2))
    with pytest.raises(SspError):
        I.GpuAugmenter("cpu")


def test_staging_layout_feeds_the_kernel_core(host):
    """GpuAugmenter's host half (batch plan, pinned-buffer fill with the thread pool, argument order of augment_sample_driver) driven
    into the host build of the kernel core: a mixed-size batch equals the oracle sample by sample."""
    sizes = [((160, 120), (100, 75)), ((96, 128), (64, 64)), ((200, 150), (333, 41)), ((160, 120), (160, 120)), ((64, 48), (20, 30))]
    samples = [synth.photo_sample(10 + i, ow, oh, bw, bh) for i, ((ow, oh), (bw, bh)) in enumerate(sizes)]
    imgs, masks, bgs = zip(*samples)
    W = H = 104
    rng = random.Random(100)
    params = [I.draw_augmentation(im.shape[1], im.shape[0], 0.2, 0.1, 1.5, 1.5, rng) for im in imgs]
    offs, total, work_bytes = I._stage_plan(imgs, masks, bgs, params, W, H, I.BICUBIC)
    assert all(o[k] % 16 == 0 for o in offs for k in o) and total % 16 == 0
    st = np.full(total, 0xAB, np.uint8)
    I._stage_fill(st, imgs, masks, bgs, params, offs)
    work = np.empty(work_bytes, np.uint8)
    rng = random.Random(100)
    base = st.ctypes.data
    for i, (im, bg, p, o) in enumerate(zip(imgs, bgs, params, offs)):
        assert host.h_augment_work_bytes(im.shape[1], im.shape[0], bg.shape[1], bg.shape[0], p["cw"], p["ch"], W, H, 3) <= work_bytes
        o8 = np.empty((H, W, 3), np.uint8)
        rc = host.h_augment_sample(C.c_void_p(base + o["img"]), C.c_void_p(base + o["mask"]), im.shape[1], im.shape[0],
                                   C.c_void_p(base + o["bg"]), bg.shape[1], bg.shape[0], C.c_void_p(base + o["luts"]), p["pleft"], p["ptop"],
                                   p["cw"], p["ch"], W, H, 3, _p(work), C.c_longlong(work_bytes), _p(o8), None)
        assert rc == 0
        want = A.data_augmentation(A.change_background(*samples[i]), (W, H), 0.2, 0.1, 1.5, 1.5, rng=rng)[0]
        assert np.array_equal(o8, want), i
    with pytest.raises(ValueError):
        I._stage_plan(imgs, [m[:10] for m in masks], bgs, params, W, H, I.BICUBIC)


def test_batched_op_table_matches_per_sample_driver(host):
    """the batched path (one launch per stage per batch): the recording back end + op_element() of augment_core.h, executed by the
    host harness stage by stage over a mixed-size batch, produce the bytes of the oracle for every sample (uint8 and float32 CHW)"""
    from singleshotpose_b200.image import _AugItem
    host.h_aug_op_bytes.restype = C.c_longlong; host.h_aug_item_bytes.restype = C.c_longlong
    assert host.h_aug_item_bytes() == C.sizeof(_AugItem)
    sizes = [((160, 120), (100, 75)), ((96, 128), (64, 64)), ((200, 150), (333, 41)), ((160, 120), (160, 120)), ((64, 48), (20, 30)), ((104, 104), (104, 104))]
    samples = [synth.photo_sample(30 + i, ow, oh, bw, bh) for i, ((ow, oh), (bw, bh)) in enumerate(sizes)]
    imgs, masks, bgs = zip(*samples)
    W = H = 104
    rng = random.Random(200)
    params = [I.draw_augmentation(im.shape[1], im.shape[0], 0.2, 0.1, 1.5, 1.5, rng) for im in imgs]
    params[-1].update(pleft=0, ptop=0, cw=104, ch=104)            # same-size crop: Image.resize returns a copy (nearest op, fewer stages)
    offs, total, work_bytes = I._stage_plan(imgs, masks, bgs, params, W, H, I.BICUBIC)
    st = np.zeros(total, np.uint8)
    I._stage_fill(st, imgs, masks, bgs, params, offs)
    B = len(imgs)
    each = (work_bytes + 15) & ~15
    work = np.zeros(each * B + 16, np.uint8)
    wbase = (work.ctypes.data + 15) & ~15
    o8 = np.zeros((B, H, W, 3), np.uint8); of = np.zeros((B, 3, H, W), np.float32)
    items = (_AugItem * B)()
    base = st.ctypes.data
    for i, (im, bg, p, o) in enumerate(zip(imgs, bgs, params, offs)):
        items[i] = _AugItem(base + o["img"], base + o["mask"], im.shape[1], im.shape[0], base + o["bg"], bg.shape[1], bg.shape[0], base + o["luts"],
                            p["pleft"], p["ptop"], p["cw"], p["ch"], wbase + i * each, each, o8[i].ctypes.data, of[i].ctypes.data)
    table = np.zeros(10 * B * host.h_aug_op_bytes(), np.uint8)
    dims = (C.c_int * 20)()
    assert host.h_augment_batch(items, B, W, H, 3, _p(table), dims) == 0
    assert sum(1 for k in range(10) if dims[2 * k] > 0) == 10 and max(dims) <= 3 * 200
    rng = random.Random(200)
    for i in range(B):
        if i == B - 1:
            want = A.distort_image(A.change_background(*samples[i]), params[i]["dhue"], params[i]["dsat"], params[i]["dexp"]) if hasattr(A, "distort_image") else None
        else:
            want = A.data_augmentation(A.change_background(*samples[i]), (W, H), 0.2, 0.1, 1.5, 1.5, rng=rng)[0]
        if want is not None:
            assert np.array_equal(o8[i], want), i
        assert np.array_equal(of[i], (o8[i].transpose(2, 0, 1).astype(np.float32) / np.float32(255.0))), i


def test_validation_batch_glue_with_oracle_resize():
    """load_validation_batch = per-image resize_u8 + to_tensor_u8; with both kernels swapped for the oracle (the GPU kernel itself is
    tested in test_gpu_augment.py) the stacking / dtype / layout glue is checked on the CPU"""
    import torch
    from singleshotpose_b200._lib import SspError
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((48, 64), (30, 30), (64, 48))]
    oracle_resize = lambda t, size, resample: torch.from_numpy(A.resize_u8(t.numpy(), size, resample))
    oracle_to_tensor = lambda r, out: out.copy_(r.permute(2, 0, 1).float().div(255))
    x = I._validation_batch(imgs, (32, 24), torch.device("cpu"), I.BICUBIC, oracle_resize, oracle_to_tensor)
    assert x.shape == (3, 3, 24, 32) and x.dtype == torch.float32
    for i, im in enumerate(imgs):
        assert torch.equal(x[i], torch.from_numpy(A.resize_u8(im, (32, 24))).permute(2, 0, 1).float().div(255))
    with pytest.raises(SspError):
        I.load_validation_batch(imgs, (32, 24), "cpu")
