"""GPU parity of the training-image pipeline (SURVEY 8f.3): csrc/augment.cu through the C ABI vs the oracle
(oracle/augment_ref.py, pinned to Pillow) and vs the reference's own image.py outputs (tests/golden/augment.npz).
Byte work: every comparison is exact."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import augment_ref as A
from singleshotpose_b200 import image as I
from singleshotpose_b200 import synth
from singleshotpose_b200._lib import SspError

pytestmark = pytest.mark.gpu

AUG_CASES = [(0, (160, 120), (100, 75), (96, 96)), (1, (160, 120), (211, 97), (128, 128)),
             (2, (320, 240), (250, 187), (224, 224)), (3, (96, 128), (64, 64), (160, 160))]
RESIZE_CASES = [(48, 64, 32, 32), (120, 160, 104, 104), (37, 53, 111, 97), (100, 100, 100, 50), (60, 80, 60, 80), (13, 200, 208, 7),
                (5, 5, 64, 64), (300, 2, 3, 300), (300, 2, 30, 2), (50, 50, 20, 50), (480, 640, 416, 416)]
FILTERS = (A.BICUBIC, A.BILINEAR, A.NEAREST)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


def test_hsv_all_colours():
    """RGB->HSV and HSV->RGB over all 2^24 byte triples: equal to Pillow's convert() (the oracle is pinned to it on the CPU)"""
    c = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.ascontiguousarray(np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8))
    d = torch.from_numpy(rgb).cuda()
    try:
        from PIL import Image
        want_hsv = np.asarray(Image.fromarray(rgb.reshape(4096, 4096, 3), "RGB").convert("HSV")).reshape(-1, 3)
        want_rgb = np.asarray(Image.fromarray(rgb.reshape(4096, 4096, 3), "HSV").convert("RGB")).reshape(-1, 3)
    except ImportError:
        want_hsv, want_rgb = A.rgb2hsv_u8(rgb), A.hsv2rgb_u8(rgb)
    assert np.array_equal(I.rgb2hsv_u8(d).cpu().numpy(), want_hsv)
    assert np.array_equal(I.hsv2rgb_u8(d).cpu().numpy(), want_rgb)


def test_resize_and_crop_vs_oracle():
    rng = np.random.default_rng(1)
    for (ih, iw, oh, ow) in RESIZE_CASES:
        img = rng.integers(0, 256, (ih, iw, 3), dtype=np.uint8)
        d = torch.from_numpy(img).cuda()
        for rs in FILTERS:
            assert np.array_equal(I.resize_u8(d, (ow, oh), rs).cpu().numpy(), A.resize_u8(img, (ow, oh), rs)), (ih, iw, oh, ow, rs)
    img = rng.integers(0, 256, (120, 160, 3), dtype=np.uint8)
    d = torch.from_numpy(img).cuda()
    for box in [(-20, -10, 150, 100), (10, 5, 120, 90), (-30, 20, 200, 60), (100, 100, 101, 101), (-50, -50, -10, -10)]:
        for rs in FILTERS:
            assert np.array_equal(I.resize_u8(d, (96, 64), rs, box).cpu().numpy(), A.resize_u8(A.crop_u8(img, box), (96, 64), rs)), (box, rs)
    with pytest.raises(SspError):
        I.resize_u8(d, (96, 64), A.BICUBIC, (10, 10, 10, 40))            # empty crop window
    with pytest.raises(SspError):
        I.resize_u8(d, (96, 64), 5)                                       # unsupported filter


def test_augmenter_matches_reference_golden(golden):
    """whole pipeline, one sample per call: bytes equal to the reference's change_background + data_augmentation output"""
    aug = I.GpuAugmenter("cuda", keep_u8=True)
    for seed, (ow, oh), (bw, bh), shape in AUG_CASES:
        img, mask, bg = synth.photo_sample(seed, ow, oh, bw, bh)
        x, params, u8 = aug([img], [mask], [bg], shape, 0.2, 0.1, 1.5, 1.5, rng=random.Random(seed))
        p = params[0]
        assert np.array_equal(u8[0].cpu().numpy(), golden["img_%d" % seed]), seed
        assert np.array_equal(np.array([p["flip"], p["dx"], p["dy"], p["sx"], p["sy"]]), golden["xform_%d" % seed])
        want = torch.from_numpy(golden["img_%d" % seed]).permute(2, 0, 1).float().div(255)        # torchvision ToTensor
        assert x.shape == (1, 3, shape[1], shape[0]) and torch.equal(x[0].cpu(), want)
    x1, lab = I.load_data_detection_arrays(img, mask, bg, synth.label_rows(3, n=2), shape, 0.2, 0.1, 1.5, 1.5, 9, 50, "cuda",
                                           rng=random.Random(3))
    assert torch.equal(x1.cpu(), want) and np.array_equal(lab, golden["label_3"])


def test_batched_augmenter_mixed_sources_vs_oracle():
    """a batch whose samples differ in image and background size (one staging copy, shared scratch), all three filters, and
    a second call that reuses the pinned staging buffer"""
    sizes = [((160, 120), (100, 75)), ((96, 128), (64, 64)), ((200, 150), (333, 41)), ((160, 120), (160, 120))]
    samples = [synth.photo_sample(10 + i, ow, oh, bw, bh) for i, ((ow, oh), (bw, bh)) in enumerate(sizes)]
    imgs, masks, bgs = zip(*samples)
    for rs in FILTERS:
        aug = I.GpuAugmenter("cuda", resample=rs, keep_u8=True)
        for rep in range(2):
            rng = random.Random(100 + rep)
            x, params, u8 = aug(imgs, masks, bgs, (104, 104), 0.2, 0.1, 1.5, 1.5, rng=rng)
            rng = random.Random(100 + rep)
            for i, (img, mask, bg) in enumerate(samples):
                want = A.data_augmentation(A.change_background(img, mask, bg, rs), (104, 104), 0.2, 0.1, 1.5, 1.5, rng=rng, resample=rs)[0]
                assert np.array_equal(u8[i].cpu().numpy(), want), (rs, rep, i)
            assert torch.equal(x.cpu(), u8.cpu().permute(0, 3, 1, 2).float().div(255))
    # replaying recorded draws gives the same batch
    x2, _p, _u = aug(imgs, masks, bgs, (104, 104), params=params)
    assert torch.equal(x2, x)
    # one launch per pipeline stage for the whole batch
    l0 = aug.launches; aug(imgs, masks, bgs, (104, 104), params=params)
    assert aug.launches - l0 <= 10
    with pytest.raises(ValueError):
        aug(imgs, masks[:2], bgs, (104, 104))


def test_validation_batch_matches_oracle():
    """dataset.py:100-103 (test mode): img.resize(shape) + ToTensor for a batch of differently sized images"""
    rng = np.random.default_rng(4)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((120, 160), (97, 131), (160, 120))]
    x = I.load_validation_batch(imgs, (104, 104), "cuda")
    assert x.shape == (3, 3, 104, 104) and x.is_cuda
    for i, im in enumerate(imgs):
        assert torch.equal(x[i].cpu(), torch.from_numpy(A.resize_u8(im, (104, 104))).permute(2, 0, 1).float().div(255))


def test_dataset_collate_matches_reference_golden(golden_dir, tmp_path):
    """listDataset (host half) + GpuCollate (device half) vs the reference's listDataset + ToTensor outputs (golden/dataset.npz)"""
    from singleshotpose_b200 import dataset as D
    g = np.load(os.path.join(golden_dir, "dataset.npz"))
    listfile, bgs = synth.write_linemod_like(str(tmp_path))
    collate = D.GpuCollate("cuda")
    random.seed(6)
    ds = D.listDataset(listfile, shape=(96, 96), shuffle=True, train=True, seen=10 ** 6, batch_size=2, num_workers=2, cell_size=8,
                       bg_file_names=bgs)
    samples = [ds[i] for i in range(4)]
    for b in (0, 2):
        data, target = collate(samples[b:b + 2])
        assert data.is_cuda and not target.is_cuda and target.dtype == torch.float64
        for j in range(2):
            want = torch.from_numpy(g["train_late_img_%d" % (b + j)]).permute(2, 0, 1).float().div(255)
            assert torch.equal(data[j].cpu(), want), (b, j)
            assert np.array_equal(target[j].numpy(), g["train_late_label_%d" % (b + j)])
    random.seed(9)
    dt = D.listDataset(listfile, shape=(64, 48), shuffle=False, train=False, num_workers=3)
    data, target = collate([dt[i] for i in range(4)])
    for i in range(4):
        assert torch.equal(data[i].cpu(), torch.from_numpy(g["test_img_%d" % i]).permute(2, 0, 1).float().div(255))
        assert np.array_equal(target[i].numpy(), g["test_label_%d" % i])

