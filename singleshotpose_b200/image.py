"""GPU training-image pipeline: the reference's image.py (change_background, data_augmentation, distort_image,
fill_truth_detection, load_data_detection) with the pixel work on the GPU and byte-identical results.

Split of work, per sample:
  host   - the random draws, in the reference's order (image.py:46-75, 34-44), so that a seeded `random` gives the same
           crop / flip / hue / saturation / exposure as the reference; the five 256-entry point() tables (image.py:17-27,
           121-122), built the way Pillow's Image.point() builds them (round, then clip to 8 bits); the label transform
           (fill_truth_detection, image.py:77-108).  JPEG/PNG decoding stays with PIL in the loader workers.
  device - background resize, mask compositing, jitter crop (zero fill), resize to the network shape, RGB->HSV->RGB
           distortion, ToTensor: libssp_b200.so `ssp_aug_batch_plan` + `ssp_aug_batch_run` for the whole batch
           (csrc/augment.cu), byte-exact with Pillow's
           ImagingResample / rgb2hsv / hsv2rgb, which the reference calls through PIL.

There is no CPU fallback: the tensors come back on the CUDA device, and a missing library raises.
`resample` is Pillow's Image.resize() filter.  The reference calls resize() without one (image.py:69,114); that means
BICUBIC on every Pillow since 7.0 (the default here) and NEAREST on the Pillow 5 of the reference's era -- pass
`resample=NEAREST` to reproduce the latter.
"""
from __future__ import annotations

import random as _random

import numpy as np
import torch

from ._lib import C, STRUCTS, SspError, call, load, ptr, stream_ptr

NEAREST, BILINEAR, BICUBIC = 0, 2, 3          # PIL.Image.Resampling values


# ---------------------------------------------------------------------------------------------- host side
def point_lut(fn):
    """Image.point(callable) on an 8-bit band: [round(fn(i)) for i in range(256)] stored as bytes with saturation."""
    return np.clip(np.array([round(fn(i)) for i in range(256)], np.int64), 0, 255).astype(np.uint8)


_RAMP = np.arange(256, dtype=np.float64)


def _store_u8(values):
    """round() (half to even, like Python's) then saturate to a byte: what Image.point() does with a float table"""
    return np.clip(np.rint(values), 0, 255).astype(np.uint8)


_MASK_LUTS = None


def mask_luts():
    """posmask, negmask of change_background (image.py:121-122): point(i / 255), point(1 - i / 255)"""
    global _MASK_LUTS
    if _MASK_LUTS is None:
        _MASK_LUTS = (_store_u8(_RAMP / 255), _store_u8(1 - _RAMP / 255))
    return _MASK_LUTS


def distort_luts(hue, sat, val):
    """hue / saturation / value tables of distort_image (image.py:17-27), including the reference's +-255 hue wrap.
    Vectorised over the 256 entries; the same float64 operations, in the same order, as the reference's lambdas."""
    x = _RAMP + hue * 255
    x = np.where(x > 255, x - 255, x)
    x = np.where(x < 0, x + 255, x)
    return _store_u8(x), _store_u8(_RAMP * sat), _store_u8(_RAMP * val)


def rand_scale(s, rng=_random):
    """image.py:34-38"""
    scale = rng.uniform(1, s)
    if rng.randint(1, 10000) % 2:
        return scale
    return 1. / scale


def draw_augmentation(ow, oh, jitter, hue, saturation, exposure, rng=_random):
    """All random draws of data_augmentation + random_distort_image, in the reference's order (image.py:46-75, 40-44).
    Returns the crop window, the label transform (flip, dx, dy, sx, sy) and the three distortion factors."""
    dw, dh = int(ow * jitter), int(oh * jitter)
    pleft, pright = rng.randint(-dw, dw), rng.randint(-dw, dw)
    ptop, pbot = rng.randint(-dh, dh), rng.randint(-dh, dh)
    swidth, sheight = ow - pleft - pright, oh - ptop - pbot
    sx, sy = float(swidth) / ow, float(sheight) / oh
    flip = rng.randint(1, 10000) % 2
    dx, dy = (float(pleft) / ow) / sx, (float(ptop) / oh) / sy
    dhue = rng.uniform(-hue, hue)
    dsat = rand_scale(saturation, rng)
    dexp = rand_scale(exposure, rng)
    return dict(pleft=pleft, ptop=ptop, cw=swidth - 1, ch=sheight - 1, flip=flip, dx=dx, dy=dy, sx=sx, sy=sy,
                dhue=dhue, dsat=dsat, dexp=dexp)


def fill_truth_detection(bs, w, h, flip, dx, dy, sx, sy, num_keypoints, max_num_gt):
    """image.py:77-108 on parsed label rows `bs` ((n, 2K+3) floats; the reference np.loadtxt()s them from labpath).
    As in the reference, `flip`, `w` and `h` are accepted and unused, and at most 50 rows are kept."""
    num_labels = 2 * num_keypoints + 3
    label = np.zeros((max_num_gt, num_labels))
    bs = np.array(bs, np.float64).reshape(-1, num_labels)
    cc = 0
    for i in range(bs.shape[0]):
        row = bs[i].copy()
        row[1] = min(0.999, max(0, row[1] * sx - dx))            # the centroid stays inside the image
        row[2] = min(0.999, max(0, row[2] * sy - dy))
        for j in range(1, num_keypoints):
            row[2 * j + 1] = row[2 * j + 1] * sx - dx
            row[2 * j + 2] = row[2 * j + 2] * sy - dy
        label[cc] = row
        cc += 1
        if cc >= 50:
            break
    return np.reshape(label, (-1))


# ---------------------------------------------------------------------------------------------- device side
def _u8_hwc(a, what):
    """PIL.Image / numpy / torch -> contiguous uint8 HWC numpy array (host) or torch tensor (any device)"""
    if torch.is_tensor(a):
        if a.dtype != torch.uint8 or a.dim() != 3 or a.shape[2] != 3:
            raise ValueError("%s: expected a uint8 HxWx3 tensor, got %s %s" % (what, a.dtype, tuple(a.shape)))
        return a.contiguous()
    a = np.asarray(a)                                            # PIL images convert through the array interface
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("%s: expected a uint8 HxWx3 RGB image, got %s %s" % (what, a.dtype, a.shape))
    return np.ascontiguousarray(a)


def _work(nbytes, device):
    return torch.empty(int(nbytes) + 16, dtype=torch.uint8, device=device)       # torch allocations are >= 256-B aligned


def _require_cuda(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise SspError("%s runs on CUDA tensors only (no CPU fallback)" % what)


def resize_u8(img, size, resample=BICUBIC, box=None):
    """Image.crop(box).resize(size, resample) of a uint8 HxWx3 CUDA tensor; size = (width, height), box = (l, t, r, b) may
    stick out of the image (zero fill) -- image.py:64,69 and dataset.py:103."""
    _require_cuda(img, "resize_u8")
    img = _u8_hwc(img, "img")
    sh, sw = img.shape[:2]
    l, t, r, b = box if box is not None else (0, 0, sw, sh)
    ow, oh = int(size[0]), int(size[1])
    nb = load().ssp_aug_resize_work_bytes(r - l, b - t, ow, oh, resample)
    if nb < 0:
        raise SspError("resize_u8: empty crop window or output size")
    work = _work(nb, img.device)
    out = torch.empty(oh, ow, 3, dtype=torch.uint8, device=img.device)
    call("ssp_aug_resize_u8", ptr(img), sw, sh, l, t, r - l, b - t, ptr(out), ow, oh, resample, ptr(work), work.numel(), stream_ptr())
    return out


def rgb2hsv_u8(rgb):
    """Image.convert('HSV') of uint8 (...,3) CUDA pixels (image.py:15)"""
    _require_cuda(rgb, "rgb2hsv_u8")
    rgb = rgb.contiguous()
    out = torch.empty_like(rgb)
    call("ssp_aug_rgb2hsv_u8", ptr(rgb), ptr(out), rgb.numel() // 3, stream_ptr())
    return out


def hsv2rgb_u8(hsv):
    """Image.convert('RGB') of uint8 HSV (...,3) CUDA pixels (image.py:30)"""
    _require_cuda(hsv, "hsv2rgb_u8")
    hsv = hsv.contiguous()
    out = torch.empty_like(hsv)
    call("ssp_aug_hsv2rgb_u8", ptr(hsv), ptr(out), hsv.numel() // 3, stream_ptr())
    return out


def to_tensor_u8(img, out=None):
    """torchvision ToTensor of a uint8 HxWx3 CUDA image -> float32 (3,H,W) in [0,1] (byte / 255 as an IEEE division, in-kernel)."""
    _require_cuda(img, "to_tensor_u8")
    img = _u8_hwc(img, "img")
    h, w = img.shape[:2]
    if out is None:
        out = torch.empty(3, h, w, dtype=torch.float32, device=img.device)
    call("ssp_aug_to_tensor_u8", ptr(img), h * w, ptr(out), stream_ptr())
    return out


def _validation_batch(imgs, shape, dev, resample, resize_fn, to_tensor_fn):
    W, H = int(shape[0]), int(shape[1])
    out = torch.empty(len(imgs), 3, H, W, dtype=torch.float32, device=dev)
    for i, a in enumerate(imgs):
        a = _u8_hwc(a, "img")
        d = a.to(dev, non_blocking=True) if torch.is_tensor(a) else torch.from_numpy(a).to(dev, non_blocking=True)
        r = resize_fn(d, (W, H), resample)                    # (H, W, 3) uint8, byte-identical to PIL
        to_tensor_fn(r, out[i])                               # torchvision ToTensor
    return out


def load_validation_batch(imgs, shape, device, resample=BICUBIC):
    """The test-mode branch of listDataset.__getitem__ (dataset.py:100-103) + ToTensor for a batch: every image is resized to
    `shape` = (width, height) with Image.resize's arithmetic on the GPU (ssp_aug_resize_u8) and returned as one float32
    (B,3,H,W) CUDA tensor in [0,1].  imgs: uint8 HxWx3 RGB arrays / PIL images of any sizes."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise SspError("load_validation_batch needs a CUDA device (no CPU fallback); got %s" % dev)
    return _validation_batch(imgs, shape, dev, resample, resize_u8, to_tensor_u8)


def _a16(n):
    return (n + 15) & ~15


def _stage_plan(imgs, masks, bgs, params, W, H, resample):
    """staging layout of one batch: per sample img | mask | bg | 5 tables, each 16-B aligned -> (offsets, total bytes, scratch bytes)"""
    lib = load()
    offs, total, work_bytes = [], 0, 0
    for im, mk, bg, p in zip(imgs, masks, bgs, params):
        if tuple(mk.shape) != tuple(im.shape):
            raise ValueError("mask %s and image %s differ in size" % (tuple(mk.shape), tuple(im.shape)))
        if p["cw"] <= 0 or p["ch"] <= 0:
            raise ValueError("empty crop window %dx%d" % (p["cw"], p["ch"]))
        o = {}
        for k, a in (("img", im), ("mask", mk), ("bg", bg)):
            if torch.is_tensor(a) and a.is_cuda:            # already on the device: the kernels read it in place
                o[k] = None
                continue
            o[k] = total
            total += _a16(int(np.prod(a.shape)))
        o["luts"] = total
        total += _a16(5 * 256)
        offs.append(o)
        nb = lib.ssp_aug_sample_work_bytes(im.shape[1], im.shape[0], bg.shape[1], bg.shape[0], p["cw"], p["ch"], W, H, resample)
        if nb < 0:
            raise SspError("ssp_aug_sample_work_bytes: bad sizes")
        work_bytes = max(work_bytes, nb)
    return offs, total, work_bytes


_POOL = None


def _stage_fill(st, imgs, masks, bgs, params, offs):
    """copy the batch's bytes and point() tables into the (pinned) staging array `st`; the big copies release the GIL, so a small
    thread pool moves them in parallel"""
    global _POOL
    pos, neg = mask_luts()

    def one(args):
        im, mk, bg, p, o = args
        for k, a in (("img", im), ("mask", mk), ("bg", bg)):
            if o[k] is None:
                continue
            a = a.numpy() if torch.is_tensor(a) else a
            st[o[k]:o[k] + a.size] = a.reshape(-1)
        lh, ls, lv = distort_luts(p["dhue"], p["dsat"], p["dexp"])
        st[o["luts"]:o["luts"] + 1280] = np.concatenate([pos, neg, lh, ls, lv])
    jobs = list(zip(imgs, masks, bgs, params, offs))
    if len(jobs) < 4:
        for j in jobs:
            one(j)
        return
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _POOL = ThreadPoolExecutor(max_workers=4, thread_name_prefix="ssp-stage")
    list(_POOL.map(one, jobs))


_AugItem = STRUCTS["ssp_aug_item"]


class GpuAugmenter:
    """change_background + data_augmentation + ToTensor for a whole batch: one pinned staging buffer, ONE host->device copy,
    then one launch per pipeline stage for the whole batch on the current stream, writing straight into the (B,3,H,W) float32 network input.

        aug = GpuAugmenter(device)
        x, params = aug(imgs, masks, bgs, shape=(416, 416), jitter=0.2, hue=0.1, saturation=1.5, exposure=1.5)
        labels = [fill_truth_detection(rows, ow, oh, p["flip"], p["dx"], p["dy"], 1./p["sx"], 1./p["sy"], 9, 50) ...]

    imgs / masks / bgs: sequences of uint8 HxWx3 RGB arrays (or PIL images), what `Image.open(path).convert('RGB')` gives in
    load_data_detection (image.py:134-136).  `params` (optional argument) replays earlier draws instead of drawing."""

    def __init__(self, device, resample=BICUBIC, keep_u8=False):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise SspError("GpuAugmenter needs a CUDA device (no CPU fallback); got %s" % self.device)
        self.resample = resample
        self.keep_u8 = keep_u8              # also return the uint8 HWC result (parity tests)
        self._stage = None                  # pinned host staging, grown on demand
        self._dev = None
        self._work = None
        self._copied = None
        self.launches = 0
        self.h2d_bytes = 0

    def __call__(self, imgs, masks, bgs, shape, jitter=0.2, hue=0.1, saturation=1.5, exposure=1.5, rng=_random, params=None):
        B = len(imgs)
        if not (len(masks) == len(bgs) == B) or B == 0:
            raise ValueError("imgs, masks and bgs must be non-empty sequences of the same length")
        W, H = int(shape[0]), int(shape[1])
        imgs = [_u8_hwc(a, "img") for a in imgs]
        masks = [_u8_hwc(a, "mask") for a in masks]
        bgs = [_u8_hwc(a, "bg") for a in bgs]
        here = self.device.index if self.device.index is not None else torch.cuda.current_device()
        for a in imgs + masks + bgs:
            if torch.is_tensor(a) and a.is_cuda and a.device.index != here:
                raise ValueError("input tensor on %s, the augmenter runs on cuda:%d" % (a.device, here))
        if params is None:
            params = [draw_augmentation(im.shape[1], im.shape[0], jitter, hue, saturation, exposure, rng) for im in imgs]
        offs, total, work_bytes = _stage_plan(imgs, masks, bgs, params, W, H, self.resample)
        lib = load()
        table_off = _a16(total)
        table_bytes = int(lib.ssp_aug_batch_table_bytes(B))
        work_each = _a16(work_bytes)
        work_total = work_each * B          # concurrent samples need their own scratch
        total = table_off + table_bytes
        if self._stage is None or self._stage.numel() < total:
            self._stage = torch.empty(total, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty(total, dtype=torch.uint8, device=self.device)
        if self._work is None or self._work.numel() < work_total + 16:
            self._work = _work(work_total, self.device)
        if self._copied is not None:
            self._copied.synchronize()      # the previous batch's host->device copy has drained the pinned staging buffer
        _stage_fill(self._stage.numpy(), imgs, masks, bgs, params, offs)
        out = torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)
        u8 = torch.empty(B, H, W, 3, dtype=torch.uint8, device=self.device) if self.keep_u8 else None
        base = self._dev.data_ptr()

        def at(a, o, k):                    # device address of an input: in place if it is a CUDA tensor, else its staged copy
            return a.data_ptr() if o[k] is None else base + o[k]
        # the op table (device pointers, per-sample geometry) is planned on the host straight into the tail of the pinned
        # staging buffer and travels in the batch's single host->device copy
        items = (_AugItem * B)()
        wbase = self._work.data_ptr()
        for i, (im, bg, p, o) in enumerate(zip(imgs, bgs, params, offs)):
            items[i] = _AugItem(at(im, o, "img"), at(masks[i], o, "mask"), im.shape[1], im.shape[0], at(bg, o, "bg"), bg.shape[1], bg.shape[0],
                                base + o["luts"], p["pleft"], p["ptop"], p["cw"], p["ch"], wbase + i * work_each, work_each,
                                u8[i].data_ptr() if u8 is not None else None, out[i].data_ptr())
        dims = (C.c_int * 20)()
        call("ssp_aug_batch_plan", items, B, W, H, self.resample, C.c_void_p(self._stage.data_ptr() + table_off), table_bytes, dims)
        self._dev[:total].copy_(self._stage[:total], non_blocking=True)
        self._copied = torch.cuda.Event()
        self._copied.record()
        self.h2d_bytes = total
        call("ssp_aug_batch_run", C.c_void_p(base + table_off), B, dims, stream_ptr())
        self.launches += sum(1 for k in range(10) if dims[2 * k] > 0)
        return (out, params, u8) if self.keep_u8 else (out, params)


def load_data_detection_arrays(img, mask, bg, label_rows, shape, jitter, hue, saturation, exposure, num_keypoints, max_num_gt,
                               device, rng=_random, resample=BICUBIC):
    """load_data_detection (image.py:129-142) after the three Image.open() calls: returns (float32 (3,H,W) CUDA tensor, label)."""
    aug = GpuAugmenter(device, resample)
    x, params = aug([img], [mask], [bg], shape, jitter, hue, saturation, exposure, rng)
    p = params[0]
    label = fill_truth_detection(label_rows, shape[0], shape[1], p["flip"], p["dx"], p["dy"], 1. / p["sx"], 1. / p["sy"], num_keypoints, max_num_gt)
    return x[0], label


from .jpeg import decode_jpeg  # noqa: E402,F401  (JPEG decode on the GPU, byte-identical to Pillow: jpeg.py)
