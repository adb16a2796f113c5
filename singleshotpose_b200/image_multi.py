"""GPU multi-object training-image pipeline: the reference's multi_obj_pose_estimation/image_multi.py (load_data_detection,
augment_objects and the functions they call) with the pixel work on the GPU and byte-identical results.

Each sample pastes the 7 other LINEMOD objects of get_add_objs() (8 for eggbox) into its scene.  Every pasted object is drawn
by rejection sampling: a random view of the object is cropped, resized and flipped, and kept only if less than 20 % of its
mask overlaps the masks placed so far.  Split of work:
  host   - the random draws in the reference's order (shuffle, the main object's crop / flip / shift, then per attempt the view
           index and its crop / flip), PNG/JPEG decoding (a thread pool), the label transform (fill_truth_detection).
  device - everything on pixels, through libssp_b200.so `ssp_augm_plan_*` / `ssp_augm_run` (csrc/augment.cu, arithmetic in
           csrc/augment_core.h): crop + resize (Pillow's ImagingResample), ImageChops.offset, FLIP_LEFT_RIGHT,
           mask_background, the overlap counts, the accept decision, superimpose_masks / superimpose_masked_imgs,
           change_background and ToTensor.

All samples of a batch advance in LOCKSTEP ROUNDS: each round draws one attempt for every sample still placing objects, copies
the candidates that are not on the device yet in one host->device copy, launches one stage sequence for the whole batch and
reads back 16 bytes per sample (the counts and the device's accept flag).  Rounds per batch = the largest number of attempts
of any sample, not their sum.  Candidate views come from the finite lists LINEMOD/<obj>/train.txt, so decoded views stay on
the device (already masked, at source resolution) in an LRU "object bank" of `bank_bytes`; once it is warm an attempt costs
no decode and no copy.

There is no CPU fallback: a missing library or a non-CUDA device raises SspError.
"""
from __future__ import annotations

import collections
import os
import random as _random

import numpy as np
import torch

from ._lib import C, STRUCTS, SspError, call, load, stream_ptr
from .image import BICUBIC, mask_luts

PIXEL_THRESHOLD = 200                 # image_multi.py:301

_ADD_OBJS = {
    "ape": ("can", "cat", "duck", "glue", "holepuncher", "iron", "phone"),
    "benchvise": ("ape", "can", "cat", "driller", "duck", "glue", "holepuncher"),
    "cam": ("ape", "benchvise", "can", "cat", "driller", "duck", "holepuncher"),
    "can": ("ape", "benchvise", "cat", "driller", "duck", "eggbox", "holepuncher"),
    "cat": ("ape", "can", "duck", "glue", "holepuncher", "eggbox", "phone"),
    "driller": ("ape", "benchvise", "can", "cat", "duck", "glue", "holepuncher"),
    "duck": ("ape", "can", "cat", "eggbox", "glue", "holepuncher", "phone"),
    "eggbox": ("ape", "benchvise", "cam", "can", "cat", "duck", "glue", "holepuncher"),
    "glue": ("ape", "benchvise", "cam", "driller", "duck", "eggbox", "holepuncher"),
    "holepuncher": ("benchvise", "cam", "can", "cat", "driller", "duck", "eggbox"),
    "iron": ("ape", "benchvise", "can", "cat", "driller", "duck", "glue"),
    "lamp": ("ape", "benchvise", "can", "driller", "eggbox", "holepuncher", "iron"),
    "phone": ("ape", "benchvise", "cam", "can", "driller", "duck", "holepuncher"),
}


def get_add_objs(objname):
    """the objects pasted into a scene of `objname` (image_multi.py:8-36), as a new list (the caller shuffles it)"""
    return list(_ADD_OBJS[objname])


def mask_path(imgpath):
    """image_multi.py:305,333"""
    return imgpath.replace("JPEGImages", "mask").replace("/00", "/").replace(".jpg", ".png")


def label_path(imgpath):
    """image_multi.py:304,334"""
    return imgpath.replace("images", "labels").replace("JPEGImages", "labels").replace(".jpg", ".txt").replace(".png", ".txt")


def read_label_rows(path):
    """the rows fill_truth_detection np.loadtxt()s, or None for an empty file (image_multi.py:127-129)"""
    return np.loadtxt(path) if os.path.getsize(path) else None


def fill_truth_detection(bs, w, h, flip, dx, dy, sx, sy, num_keypoints, max_num_gt):
    """image_multi.py:123-165 on parsed label rows (None: empty file).  Unlike image.py's version it recomputes the two range
    columns from the moved keypoints and keeps at most max_num_gt rows; `flip`, `w` and `h` are accepted and unused, as there."""
    num_labels = 2 * num_keypoints + 3
    label = np.zeros((max_num_gt, num_labels))
    if bs is None:
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


def draw_crop(ow, oh, jitter, rng):
    """the jitter crop and flip draws of (shifted_)data_augmentation_with_mask (image_multi.py:187-201, 233-247)"""
    dw, dh = int(ow * jitter), int(oh * jitter)
    pleft, pright = rng.randint(-dw, dw), rng.randint(-dw, dw)
    ptop, pbot = rng.randint(-dh, dh), rng.randint(-dh, dh)
    swidth, sheight = ow - pleft - pright, oh - ptop - pbot
    sx, sy = float(swidth) / ow, float(sheight) / oh
    flip = rng.randint(1, 10000) % 2
    return dict(pleft=pleft, ptop=ptop, cw=swidth - 1, ch=sheight - 1, flip=flip, sx=sx, sy=sy,
                dx=(float(pleft) / ow) / sx, dy=(float(ptop) / oh) / sy, shift_x=0, shift_y=0)


def draw_main(ow, oh, shape, jitter, rng):
    """shifted_data_augmentation_with_mask's draws (image_multi.py:184-210): crop, flip, then the wrap-around shift"""
    p = draw_crop(ow, oh, jitter, rng)
    p["shift_x"], p["shift_y"] = rng.randint(-80, 80), rng.randint(-80, 80)
    p["dx"] -= float(p["shift_x"]) / shape[0]
    p["dy"] -= float(p["shift_y"]) / shape[1]
    return p


def _decode_rgb(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.ascontiguousarray(np.asarray(im.convert("RGB")))


def _image_size(path):
    from PIL import Image
    with Image.open(path) as im:          # reads the header only
        return im.size


def _a16(n):
    return (int(n) + 15) & ~15


_MultiItem = STRUCTS["ssp_augm_item"]

_POOL = None


def _pool_map(fn, jobs):
    global _POOL
    if len(jobs) < 2:
        return [fn(j) for j in jobs]
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _POOL = ThreadPoolExecutor(max_workers=8, thread_name_prefix="ssp-multi")
    return list(_POOL.map(fn, jobs))


class _Sample:
    """host state of one sample while its objects are being placed"""
    def __init__(self, imgpath, rng):
        self.imgpath, self.rng = imgpath, rng
        self.add_objs = get_add_objs(os.path.basename(os.path.dirname(os.path.dirname(imgpath))))
        self.k = 0                         # index of the object being placed
        self.count = 1                     # next label row
        self.attempts = [0] * len(self.add_objs)
        self.label = None
        self.cand = None                   # (bank key, draws) of the current attempt

    @property
    def done(self):
        return self.k >= len(self.add_objs)


class GpuMultiAugmenter:
    """load_data_detection of image_multi.py for a whole batch on the GPU:

        aug = GpuMultiAugmenter("cuda", root="..")
        x, labels = aug([(imgpath, bgpath), ...], shape=(416, 416), rngs=[random.Random(s) for s in seeds])

    x: float32 (B,3,H,W) CUDA tensor (ToTensor of the reference's image), labels: (B, max_num_gt*(2K+3)) float64 numpy.
    Sample i consumes rngs[i] exactly as the reference consumes `random` in one load_data_detection call.  `root` replaces the
    reference's hard-coded '../' in front of LINEMOD/<obj>/train.txt and its lines.  max_attempts (None: unbounded, as in the
    reference) bounds the attempts for one object; exceeding it raises SspError.  After a call: `rounds`, `attempts`
    (per sample and object), `decodes` and `h2d_bytes` describe that call; `u8` holds the (B,H,W,3) bytes if keep_u8;
    with timing=True, `timing` holds one (start, end) CUDA event pair per phase / round around its copy and launches."""

    def __init__(self, device, root="..", resample=BICUBIC, bank_bytes=1 << 30, keep_u8=False, max_attempts=None, timing=False):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise SspError("GpuMultiAugmenter needs a CUDA device (no CPU fallback); got %s" % self.device)
        self.root, self.resample, self.bank_bytes = root, resample, int(bank_bytes)
        self.keep_u8, self.max_attempts, self._timing = keep_u8, max_attempts, timing
        self.timing = []
        self._bank = collections.OrderedDict()        # view path -> (device bytes: masked image | mask, w, h)
        self._bank_used = 0
        self._sizes = {}                              # view path -> (w, h), from the file header
        self._lists = {}                              # train.txt path -> lines
        self._labels = {}                             # label path -> rows
        self._stage = None
        self._copied = None
        self._work = None
        pos, neg = mask_luts()
        self._luts = torch.from_numpy(np.concatenate([pos, neg])).to(self.device)
        self.rounds = self.decodes = self.h2d_bytes = 0
        self.attempts = []
        self.u8 = None

    # ------------------------------------------------------------------------------------------------ host helpers
    def _lines(self, obj):
        p = os.path.join(self.root, "LINEMOD", obj, "train.txt")
        if p not in self._lists:
            with open(p) as f:
                self._lists[p] = f.readlines()
        return self._lists[p]

    def _label_rows(self, path):
        lp = label_path(path)
        if lp not in self._labels:
            self._labels[lp] = read_label_rows(lp)
        return self._labels[lp]

    def _size(self, path):
        if path in self._bank:
            return self._bank[path][1:]
        if path not in self._sizes:
            self._sizes[path] = _image_size(path)
        return self._sizes[path]

    def _staging(self, nbytes):
        if self._stage is None or self._stage.numel() < nbytes:
            self._stage = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8).pin_memory()
            self._dev = torch.empty(self._stage.numel(), dtype=torch.uint8, device=self.device)
        return self._stage.numpy()

    def _work_for(self, B, each):
        each = _a16(each)
        if self._work is None or self._work.numel() < B * each + 16:
            self._work = torch.empty(B * each + 16, dtype=torch.uint8, device=self.device)
        return self._work.data_ptr(), each

    def _plan_and_copy(self, plan, items, n, W, H, table_off):
        """plan into the staging tail, then ONE host->device copy of staging[:table_off + table]; returns the launch extents"""
        table_bytes = int(load().ssp_augm_table_bytes(n))
        dims = (C.c_int * 32)()
        call(plan, items, n, W, H, self.resample, C.c_void_p(self._stage.data_ptr() + table_off), table_bytes, dims)
        total = table_off + table_bytes
        if self._timing:
            self.timing.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            self.timing[-1][0].record()
        self._dev[:total].copy_(self._stage[:total], non_blocking=True)
        self.h2d_bytes += total
        return dims

    def _launch(self, n, dims, table_off):
        call("ssp_augm_run", C.c_void_p(self._dev.data_ptr() + table_off), n, dims, stream_ptr())
        if self._timing:
            self.timing[-1][1].record()

    def _evict_for(self, nbytes, keep):
        while self._bank and self._bank_used + nbytes > self.bank_bytes:
            key = next((k for k in self._bank if k not in keep), None)
            if key is None:
                break
            t, _w, _h = self._bank.pop(key)
            self._bank_used -= t.numel()

    # ------------------------------------------------------------------------------------------------ the batch
    def _refill_staging(self, nbytes):
        """the pinned staging buffer once the previous host->device copy out of it has completed"""
        if self._copied is not None:
            self._copied.synchronize()
        return self._staging(nbytes)

    def _copy_launched(self):
        self._copied = torch.cuda.Event()
        self._copied.record()

    def __call__(self, samples, shape, rngs, jitter=0.1, num_keypoints=9, max_num_gt=50):
        """samples: sequence of (image path, background path), or of dicts with keys imgpath, bgpath and optionally the already
        decoded img, mask, bg (uint8 HxWx3) and the label rows (`rows`, None for an empty label file), as dataset_multi.listDataset
        returns them; rngs: one random.Random (or the `random` module) per sample.
        Returns (float32 (B,3,H,W) CUDA tensor, float64 (B, max_num_gt*(2K+3)) labels)."""
        B = len(samples)
        if B == 0 or len(rngs) != B:
            raise ValueError("samples and rngs must be non-empty sequences of the same length")
        W, H = int(shape[0]), int(shape[1])
        lib = load()
        num_labels = 2 * num_keypoints + 3
        self.rounds = self.decodes = self.h2d_bytes = 0
        self.timing = []
        samples = [s if isinstance(s, dict) else dict(imgpath=s[0], bgpath=s[1]) for s in samples]
        st = [_Sample(s["imgpath"], r) for s, r in zip(samples, rngs)]
        # -- main objects and backgrounds: decode, then the draws of each sample in the reference's order
        def main_inputs(s):
            got = (s.get("bg"), s.get("img"), s.get("mask"))
            paths = (s["bgpath"], s["imgpath"], mask_path(s["imgpath"]))
            return tuple(np.ascontiguousarray(a) if a is not None else _decode_rgb(p) for a, p in zip(got, paths))
        dec = _pool_map(main_inputs, samples)
        self.decodes += sum(1 for s in samples for k in ("bg", "img", "mask") if s.get(k) is None)
        mains = []
        for s, sd, (_bg, img, mask) in zip(st, samples, dec):
            if mask.shape != img.shape:
                raise ValueError("%s: mask %s and image %s differ in size" % (s.imgpath, mask.shape, img.shape))
            s.rng.shuffle(s.add_objs)
            p = draw_main(img.shape[1], img.shape[0], (W, H), jitter, s.rng)
            if p["cw"] <= 0 or p["ch"] <= 0:
                raise ValueError("%s: empty crop window" % s.imgpath)
            rows = sd["rows"] if "rows" in sd else self._label_rows(s.imgpath)
            s.label = fill_truth_detection(rows, 0, 0, p["flip"], p["dx"], p["dy"], 1. / p["sx"], 1. / p["sy"],
                                           num_keypoints, max_num_gt).reshape(-1, num_labels)
            mains.append(p)
        state = torch.empty(B, 4, H, W, 3, dtype=torch.uint8, device=self.device)    # main img, main mask, total img, total mask
        counts = torch.zeros(B, 4, dtype=torch.int32, device=self.device)
        sp = lambda i, k: state[i, k].data_ptr()
        luts = self._luts.data_ptr()
        # -- begin.  staging: all backgrounds, then img | mask per sample, then the op table
        bg_offs, off = [], 0
        for bg, _i, _m in dec:
            bg_offs.append(off)
            off += _a16(bg.size)
        bg_end, img_offs = off, []
        for _b, img, _m in dec:
            img_offs.append(off)
            off += 2 * _a16(img.size)
        table_off = _a16(off)
        stg = self._refill_staging(table_off + int(lib.ssp_augm_table_bytes(B)))

        def fill(args):
            (bg, img, mask), bo, io = args
            stg[bo:bo + bg.size] = bg.reshape(-1)
            stg[io:io + img.size] = img.reshape(-1)
            stg[io + _a16(img.size):io + _a16(img.size) + mask.size] = mask.reshape(-1)
        _pool_map(fill, list(zip(dec, bg_offs, img_offs)))
        base = self._dev.data_ptr()
        wbase, each = self._work_for(B, max(lib.ssp_augm_work_bytes(p["cw"], p["ch"], W, H, self.resample) for p in mains))
        items = (_MultiItem * B)()
        for i, ((_bg, img, _m), p, o) in enumerate(zip(dec, mains, img_offs)):
            items[i] = _MultiItem(base + o, base + o + _a16(img.size), img.shape[1], img.shape[0], p["pleft"], p["ptop"], p["cw"], p["ch"],
                                  p["flip"], p["shift_x"], p["shift_y"], 0, sp(i, 0), sp(i, 1), sp(i, 2), sp(i, 3),
                                  counts[i].data_ptr(), luts, wbase + i * each, each, None, None)
        dims = self._plan_and_copy("ssp_augm_plan_begin", items, B, W, H, table_off)
        bgs = self._dev[:bg_end].clone()               # the backgrounds wait on the device for finish; the rounds reuse staging
        self._launch(B, dims, table_off)
        self._copy_launched()
        # -- attempt rounds: one candidate for every sample that is still placing objects
        while True:
            active = [i for i, s in enumerate(st) if not s.done]
            if not active:
                break
            order = []
            for i in active:
                s = st[i]
                lines = self._lines(s.add_objs[s.k])
                path = os.path.join(self.root, lines[s.rng.randint(0, len(lines) - 1)].rstrip())
                w, h = self._size(path)                        # the crop draws need the view's size before its pixels
                s.cand = (path, draw_crop(w, h, jitter, s.rng))
                s.attempts[s.k] += 1
                if self.max_attempts is not None and s.attempts[s.k] > self.max_attempts:
                    raise SspError("%s: object %s not placed after %d attempts" % (s.imgpath, s.add_objs[s.k], self.max_attempts))
                if s.cand[1]["cw"] <= 0 or s.cand[1]["ch"] <= 0:
                    raise ValueError("%s: empty crop window" % path)
                if path not in self._bank and path not in order:
                    order.append(path)
            # views not on the device yet: decode, add to the bank, stage them ahead of the op table
            decoded = _pool_map(lambda p: (_decode_rgb(p), _decode_rgb(mask_path(p))), order)
            self.decodes += 2 * len(order)
            in_use = {st[i].cand[0] for i in active}
            new, off = {}, 0
            for path, (img, mask) in zip(order, decoded):
                if mask.shape != img.shape:
                    raise ValueError("%s: mask %s and image %s differ in size" % (path, mask.shape, img.shape))
                nb = 2 * _a16(img.size)
                self._evict_for(nb, in_use)
                t = torch.empty(nb, dtype=torch.uint8, device=self.device)
                self._bank[path] = (t, img.shape[1], img.shape[0])
                self._bank_used += nb
                self._sizes[path] = (img.shape[1], img.shape[0])
                new[path] = (off, img, mask, t)
                off += nb
            n = len(active)
            table_off = _a16(off)
            stg = self._refill_staging(table_off + int(lib.ssp_augm_table_bytes(n)))
            for o, img, mask, _t in new.values():
                stg[o:o + img.size] = img.reshape(-1)
                stg[o + _a16(img.size):o + _a16(img.size) + mask.size] = mask.reshape(-1)
            wbase, each = self._work_for(n, max(lib.ssp_augm_work_bytes(st[i].cand[1]["cw"], st[i].cand[1]["ch"], W, H, self.resample)
                                                for i in active))
            items = (_MultiItem * n)()
            masked = set()
            for j, i in enumerate(active):
                path, p = st[i].cand
                t, w, h = self._bank[path]
                self._bank.move_to_end(path)
                mask_bg = int(path in new and path not in masked)      # mask_background once, in the bank, at source resolution
                masked.add(path)
                items[j] = _MultiItem(t.data_ptr(), t.data_ptr() + _a16(3 * w * h), w, h, p["pleft"], p["ptop"], p["cw"], p["ch"],
                                      p["flip"], 0, 0, mask_bg, sp(i, 0), sp(i, 1), sp(i, 2), sp(i, 3),
                                      counts[i].data_ptr(), luts, wbase + j * each, each, None, None)
            dims = self._plan_and_copy("ssp_augm_plan_attempt", items, n, W, H, table_off)
            for o, _img, _m, t in new.values():
                t.copy_(self._dev[o:o + t.numel()], non_blocking=True)
            self._launch(n, dims, table_off)
            self._copy_launched()
            got = counts.cpu().numpy()                     # the round's only device->host copy
            self.rounds += 1
            for i in active:
                s = st[i]
                S, I, acc = int(got[i, 0]), int(got[i, 1]), int(got[i, 2])
                want = S != 0 and float(I) / float(S) < 0.2
                if bool(acc) != want:
                    raise SspError("device accept flag %d disagrees with its counts S=%d I=%d" % (acc, S, I))
                if want:
                    path, p = s.cand
                    lab = fill_truth_detection(self._label_rows(path), 0, 0, p["flip"], p["dx"], p["dy"], 1. / p["sx"], 1. / p["sy"],
                                               num_keypoints, max_num_gt)
                    s.label[s.count, :] = lab.reshape(-1, num_labels)[0, :]
                    s.count += 1
                    s.k += 1
        # -- finish: background, main object on top, change_background, ToTensor
        out = torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)
        self.u8 = torch.empty(B, H, W, 3, dtype=torch.uint8, device=self.device) if self.keep_u8 else None
        wbase, each = self._work_for(B, max(lib.ssp_augm_work_bytes(bg.shape[1], bg.shape[0], W, H, self.resample) for bg, _i, _m in dec))
        items = (_MultiItem * B)()
        for i, ((bg, _i, _m), o) in enumerate(zip(dec, bg_offs)):
            items[i] = _MultiItem(bgs.data_ptr() + o, None, bg.shape[1], bg.shape[0], 0, 0, 0, 0, 0, 0, 0, 0, sp(i, 0), sp(i, 1), sp(i, 2),
                                  sp(i, 3), None, luts, wbase + i * each, each, self.u8[i].data_ptr() if self.u8 is not None else None,
                                  out[i].data_ptr())
        self._refill_staging(int(lib.ssp_augm_table_bytes(B)))
        dims = self._plan_and_copy("ssp_augm_plan_finish", items, B, W, H, 0)
        self._launch(B, dims, 0)
        self._copy_launched()
        self.attempts = [s.attempts for s in st]
        return out, np.stack([s.label.reshape(-1) for s in st])


def load_data_detection(imgpath, shape, jitter, hue, saturation, exposure, bgpath, num_keypoints, max_num_gt, device, rng=_random,
                        root="..", resample=BICUBIC, augmenter=None):
    """image_multi.py:367-382 on the GPU: (float32 (3,H,W) CUDA tensor, label).  hue / saturation / exposure are accepted and
    unused, as in the reference.  Calling it repeatedly with one shared `rng` reproduces the reference's sequential stream."""
    aug = augmenter if augmenter is not None else GpuMultiAugmenter(device, root=root, resample=resample)
    x, labels = aug([(imgpath, bgpath)], shape, [rng], jitter, num_keypoints, max_num_gt)
    return x[0], labels[0]
