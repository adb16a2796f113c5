"""``listDataset`` of the multi-object driver for the GPU image pipeline: the reference's multi_obj_pose_estimation/dataset_multi.py
with the pixel work moved out of the loader workers.  `__getitem__` does what stays on the host: the file paths, the decoding of
the main image, its mask and the background, the label rows, and the random draws in the reference's order.  `GpuMultiCollate`
turns a list of such samples into the (B,3,H,W) float32 CUDA batch and the (B, max_num_gt*(2K+3)) target with
`image_multi.GpuMultiAugmenter` (train) or `image.load_validation_batch` (test).

    train_loader = DataLoader(listDataset(trainlist, shape=(w, h), shuffle=True, objclass=objclass, train=True, seen=model.seen,
                                          batch_size=bs, num_workers=nw, bg_file_names=bg_file_names),
                              batch_size=bs, shuffle=False, num_workers=nw, collate_fn=lambda samples: samples)
    collate = GpuMultiCollate("cuda")
    for samples in train_loader:            # the workers only decode and draw; CUDA work happens here, in the training process
        data, target = collate(samples)

Same constructor, attributes and resolution schedule (dataset_multi.py:43-58, its own: not dataset.py's) as the reference.
Train mode draws the schedule (at a batch start) and the background index from the worker's `random` exactly as the
reference, then ONE 63-bit seed per sample in place of the augmentation draws.  Deliberate departure: the pixels and label of
a sample equal the reference's `load_data_detection` after `random.seed(seed)`, but the augmentation draws no longer share one
stream across samples.  A shared stream would force the rejection loop to be resolved one attempt at a time (hundreds of
synchronising rounds per batch instead of the largest attempt count of one sample); and with DataLoader workers the
reference's stream already depends on each worker's random seed, so nothing could rely on it.  Test mode is the reference's
plain resize + labels_occlusion/ labels (dataset_multi.py:73-89).
"""
from __future__ import annotations

import os
import random

import numpy as np
import torch
from torch.utils.data import Dataset

from . import image as _image
from . import image_multi as _im
from .utils_host import read_truths_args


def _open_rgb(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.ascontiguousarray(np.asarray(im.convert("RGB")))


def occlusion_label_path(imgpath, objclass):
    """dataset_multi.py:78"""
    return imgpath.replace('benchvise', objclass).replace('images', 'labels_occlusion').replace('JPEGImages', 'labels_occlusion') \
        .replace('.jpg', '.txt').replace('.png', '.txt')


class listDataset(Dataset):
    def __init__(self, root, shape=None, shuffle=True, transform=None, objclass=None, target_transform=None, train=False, seen=0,
                 batch_size=64, num_workers=4, cell_size=32, bg_file_names=None, num_keypoints=9, max_num_gt=50):
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
        self.objclass = objclass
        self.cell_size = cell_size
        self.nbatches = self.nSamples // self.batch_size
        self.num_keypoints = num_keypoints
        self.max_num_gt = max_num_gt

    def __len__(self):
        return self.nSamples

    def _schedule_shape(self, index):
        """dataset_multi.py:43-58: 13 cells for 20 epochs, then randint(0,3)+13, randint(0,5)+12, randint(0,7)+11 for 20 epochs each,
        then randint(0,9)+10 cells"""
        if not (self.train and index % self.batch_size == 0):
            return
        unit = 20 * self.nbatches * self.batch_size
        if self.seen < unit:
            width = 13 * self.cell_size
        else:
            k = 4
            for kk in (1, 2, 3):
                if self.seen < (kk + 1) * unit:
                    k = kk
                    break
            width = (random.randint(0, 2 * k + 1) + 14 - k) * self.cell_size
        self.shape = (width, width)

    def __getitem__(self, index):
        assert index <= len(self), 'index range error'
        imgpath = self.lines[index].rstrip()
        self._schedule_shape(index)
        if self.train:
            bgpath = self.bg_file_names[random.randint(0, len(self.bg_file_names) - 1)]
            labpath = _im.label_path(imgpath)
            sample = dict(train=True, imgpath=imgpath, bgpath=bgpath, img=_open_rgb(imgpath), mask=_open_rgb(_im.mask_path(imgpath)),
                          bg=_open_rgb(bgpath), rows=_im.read_label_rows(labpath), seed=random.getrandbits(63), shape=tuple(self.shape),
                          num_keypoints=self.num_keypoints, max_num_gt=self.max_num_gt)
        else:
            img = _open_rgb(imgpath)
            labpath = occlusion_label_path(imgpath, self.objclass)
            num_labels = 2 * self.num_keypoints + 3
            label = torch.zeros(self.max_num_gt * num_labels)
            if os.path.getsize(labpath):
                tmp = torch.from_numpy(read_truths_args(labpath)).view(-1)
                tsz = tmp.numel()
                if tsz > self.max_num_gt * num_labels:
                    label = tmp[0:self.max_num_gt * num_labels]
                elif tsz > 0:
                    label[0:tsz] = tmp
            sample = dict(train=False, img=img, label=label, shape=tuple(self.shape) if self.shape else (img.shape[1], img.shape[0]))
        self.seen = self.seen + self.num_workers
        return sample


class GpuMultiCollate:
    """list of `listDataset` samples -> (data, target): data is the (B,3,H,W) float32 CUDA tensor train_multi.py feeds the model,
    target the (B, max_num_gt*(2K+3)) float64 host tensor (float32 in test mode, as the reference's).  `root` is the directory
    the reference reaches as '..' (LINEMOD/<obj>/train.txt of the pasted objects); the object bank lives as long as the collate."""

    def __init__(self, device, root="..", resample=_image.BICUBIC, bank_bytes=1 << 30, max_attempts=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _im.SspError("GpuMultiCollate needs a CUDA device (no CPU fallback); got %s" % self.device)
        self.root, self.resample, self.bank_bytes, self.max_attempts = root, resample, bank_bytes, max_attempts
        self.aug = None

    def __call__(self, samples):
        if not samples:
            raise ValueError("empty batch")
        train = samples[0]["train"]
        shapes = {s["shape"] for s in samples}
        if any(s["train"] != train for s in samples) or len(shapes) != 1:
            raise ValueError("a batch must come from one loader worker: mixed train/test samples or network shapes %s" % sorted(map(str, shapes)))
        shape = samples[0]["shape"]
        if not train:
            data = _image.load_validation_batch([s["img"] for s in samples], shape, self.device, self.resample)
            return data, torch.stack([s["label"] for s in samples])
        if self.aug is None:
            self.aug = _im.GpuMultiAugmenter(self.device, root=self.root, resample=self.resample, bank_bytes=self.bank_bytes,
                                             max_attempts=self.max_attempts)
        k, g = samples[0]["num_keypoints"], samples[0]["max_num_gt"]
        data, labels = self.aug(samples, shape, [random.Random(s["seed"]) for s in samples], 0.1, k, g)
        return data, torch.from_numpy(labels)
