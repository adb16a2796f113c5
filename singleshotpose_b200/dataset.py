"""``listDataset`` for the GPU image pipeline -- the reference's dataset.py:14-143 with the pixel work moved out of the loader
workers: `__getitem__` does what must stay on the host (file paths, `Image.open(...).convert('RGB')`, label file, the random
draws in the reference's order) and returns the RAW bytes plus the drawn parameters; `GpuCollate` turns a list of such samples
into the (B,3,H,W) float32 CUDA batch and the (B, 50*21) target tensor with `image.GpuAugmenter` / `image.load_validation_batch`.

    train_loader = DataLoader(listDataset(trainlist, shape=(w, h), shuffle=True, train=True, seen=model.seen, batch_size=bs,
                                          num_workers=nw, bg_file_names=bg_file_names),
                              batch_size=bs, shuffle=False, num_workers=nw, collate_fn=lambda samples: samples)
    collate = GpuCollate("cuda")
    for samples in train_loader:            # the workers only decode; CUDA work happens here, in the training process
        data, target = collate(samples)

Same constructor, same attributes (`seen`, `shape`, `nbatches`, ...), same multi-resolution schedule (dataset.py:66-90), same
path conventions (image.py:130-131) and -- with the same `random` state -- the same draws as the reference, so the batch equals
what `listDataset` + `transforms.ToTensor()` + default collate produce there (tests/test_dataset_cpu.py checks this against the
reference's own output through the committed golden).

`listDataset(..., gpu_decode=True)`: for files that start with a JPEG's SOI marker (by content, not by extension) the workers
return the file's bytes instead of decoding them, and take the image size from the frame header (`jpeg.read_jpeg_size`), so the
draws do not change; `GpuCollate` then decodes all of a batch's JPEGs in one `jpeg.GpuJpegDecoder` call, byte-identical to Pillow.
PNG masks and other formats decode in the workers as before.  The default, False, keeps the workers decoding everything.
"""
from __future__ import annotations

import os
import random

import numpy as np
import torch
from torch.utils.data import Dataset

from . import image as _image
from .jpeg import read_jpeg_size
from .utils_host import read_truths, read_truths_args          # noqa: F401  (dataset.py:12 imports them from utils)


def label_path(imgpath):
    """image.py:130"""
    return imgpath.replace('images', 'labels').replace('JPEGImages', 'labels').replace('.jpg', '.txt').replace('.png', '.txt')


def mask_path(imgpath):
    """image.py:131"""
    return imgpath.replace('JPEGImages', 'mask').replace('/00', '/').replace('.jpg', '.png')


def _open_rgb(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert('RGB'))


def _load(path, gpu_decode):
    """decoded RGB array, or -- with gpu_decode, for a JPEG -- the file's bytes (decoded later by GpuCollate on the device)"""
    if gpu_decode:
        with open(path, "rb") as f:
            data = f.read()
        if data[:2] == b"\xff\xd8" and read_jpeg_size(data) is not None:
            return data
    return _open_rgb(path)


def _size(img):
    """(width, height) of a decoded array or of JPEG bytes"""
    return read_jpeg_size(img) if isinstance(img, bytes) else (img.shape[1], img.shape[0])


class listDataset(Dataset):
    def __init__(self, root, shape=None, shuffle=True, transform=None, target_transform=None, train=False, seen=0, batch_size=64,
                 num_workers=4, cell_size=32, bg_file_names=None, num_keypoints=9, max_num_gt=50, gpu_decode=False):
        with open(root, 'r') as file:
            self.lines = file.readlines()
        if shuffle:
            random.shuffle(self.lines)
        self.nSamples = len(self.lines)
        self.transform = transform                       # kept for signature compatibility; ToTensor happens on the GPU
        self.target_transform = target_transform
        self.train = train
        self.shape = shape
        self.seen = seen
        self.batch_size = batch_size
        self.num_workers = num_workers
        self.bg_file_names = bg_file_names
        self.cell_size = cell_size
        self.nbatches = self.nSamples // self.batch_size
        self.num_keypoints = num_keypoints
        self.max_num_gt = max_num_gt
        self.gpu_decode = gpu_decode

    def __len__(self):
        return self.nSamples

    def _schedule_shape(self, index):
        """multi-resolution training (dataset.py:66-90): a new square size every batch, the range widening every 10 epochs"""
        if not (self.train and index % self.batch_size == 0):
            return
        unit = 10 * self.nbatches * self.batch_size
        if self.seen < unit:
            width = 13 * self.cell_size
        else:
            k = 7                                        # after 70 "epochs": randint(0, 19) + 7
            for kk in range(1, 7):
                if self.seen < (kk + 1) * unit:
                    k = kk
                    break
            width = (random.randint(0, 2 * k + 5) + 14 - k) * self.cell_size      # k = 1: randint(0,7)+13 ... k = 7: randint(0,19)+7
        self.shape = (width, width)

    def __getitem__(self, index):
        assert index <= len(self), 'index range error'
        imgpath = self.lines[index].rstrip()
        self._schedule_shape(index)
        if self.train:
            jitter, hue, saturation, exposure = 0.2, 0.1, 1.5, 1.5                         # dataset.py:93-97
            bgpath = self.bg_file_names[random.randint(0, len(self.bg_file_names) - 1)]
            g = self.gpu_decode
            img, mask, bg = _load(imgpath, g), _load(mask_path(imgpath), g), _load(bgpath, g)
            # change_background keeps the image size, so the draws of data_augmentation see (ow, oh) of the image
            ow, oh = _size(img)
            params = _image.draw_augmentation(ow, oh, jitter, hue, saturation, exposure, random)
            labpath = label_path(imgpath)
            rows = np.loadtxt(labpath) if os.path.getsize(labpath) else np.zeros((0, 2 * self.num_keypoints + 3))
            sample = dict(train=True, img=img, mask=mask, bg=bg, params=params, rows=rows, shape=tuple(self.shape),
                          num_keypoints=self.num_keypoints, max_num_gt=self.max_num_gt)
        else:
            img = _load(imgpath, self.gpu_decode)
            labpath = label_path(imgpath)
            num_labels = 2 * self.num_keypoints + 3
            label = torch.zeros(self.max_num_gt * num_labels)
            if os.path.getsize(labpath):
                tmp = torch.from_numpy(read_truths_args(labpath, self.num_keypoints)).view(-1)
                tsz = tmp.numel()
                if tsz > self.max_num_gt * num_labels:
                    label = tmp[0:self.max_num_gt * num_labels]
                elif tsz > 0:
                    label[0:tsz] = tmp
            sample = dict(train=False, img=img, label=label, shape=tuple(self.shape) if self.shape else None)
        self.seen = self.seen + self.num_workers
        return sample


def host_labels(samples):
    """the label half of load_data_detection for a list of training samples: (B, max_num_gt*(2K+3)) float64 tensor"""
    out = []
    for s in samples:
        p, (w, h) = s["params"], s["shape"]
        out.append(torch.from_numpy(_image.fill_truth_detection(s["rows"], w, h, p["flip"], p["dx"], p["dy"], 1. / p["sx"], 1. / p["sy"],
                                                                s["num_keypoints"], s["max_num_gt"])))
    return torch.stack(out)


class GpuCollate:
    """list of `listDataset` samples -> (data, target): data is the (B,3,H,W) float32 CUDA tensor train.py:82-92 feeds the model,
    target stays on the host like the reference's (region_loss.py consumes it from the CPU)."""

    def __init__(self, device, resample=_image.BICUBIC):
        self.device = torch.device(device)
        self.resample = resample
        self._aug = None
        self._jpeg = None

    def _decoded(self, samples, keys):
        """the samples' images with every JPEG given as bytes (listDataset(gpu_decode=True)) decoded on the device, in one call"""
        cols = {k: [s[k] for s in samples] for k in keys}
        todo = [(k, i) for k in keys for i, a in enumerate(cols[k]) if isinstance(a, bytes)]
        if todo:
            if self._jpeg is None:
                from .jpeg import GpuJpegDecoder
                self._jpeg = GpuJpegDecoder(self.device)
            for (k, i), t in zip(todo, self._jpeg([cols[k][i] for k, i in todo])):
                cols[k][i] = t
        return cols

    def __call__(self, samples):
        if not samples:
            raise ValueError("empty batch")
        train = samples[0]["train"]
        shapes = {s["shape"] for s in samples}
        if any(s["train"] != train for s in samples) or len(shapes) != 1:
            raise ValueError("a batch must come from one loader worker: mixed train/test samples or network shapes %s" % sorted(map(str, shapes)))
        shape = samples[0]["shape"]
        if train:
            if self._aug is None:
                self._aug = _image.GpuAugmenter(self.device, self.resample)
            cols = self._decoded(samples, ("img", "mask", "bg"))
            data, _ = self._aug(cols["img"], cols["mask"], cols["bg"], shape, params=[s["params"] for s in samples])
            return data, host_labels(samples)
        if shape is None:
            raise ValueError("test-mode batches need a network shape (listDataset(shape=...)) to be stackable")
        data = _image.load_validation_batch(self._decoded(samples, ("img",))["img"], shape, self.device, self.resample)
        return data, torch.stack([s["label"] for s in samples])
