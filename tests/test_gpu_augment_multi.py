"""GPU tests of the multi-object training-image pipeline (singleshotpose_b200/image_multi.py, csrc/augment.cu): every comparison
is exact, against the reference's own image_multi.load_data_detection through tests/golden/augment_multi.npz."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import augment_multi_ref as M
from singleshotpose_b200 import image_multi as IM
from singleshotpose_b200 import synth
from singleshotpose_b200._lib import SspError

pytestmark = pytest.mark.gpu

CASES = M.GOLDEN_CASES
JITTER, K, MAX_GT = M.JITTER, M.NUM_KEYPOINTS, M.MAX_NUM_GT
MARGIN = 20          # attempts beyond the golden count before a divergence fails instead of looping


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_multi.npz"))


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    out = {}
    for size in sorted({c[1] for c in CASES}):
        root = str(tmp_path_factory.mktemp("linemod%dx%d" % size))
        out[size] = (root, synth.write_linemod_multi_like(root, ow=size[0], oh=size[1]))
    return out


def _max_attempts(golden):
    return max(int(golden[k].max()) for k in golden.files if k.startswith("attempts_")) + MARGIN


def test_golden_cases_through_load_data_detection(golden, trees):
    """each case with one shared `random.Random` per case, as the reference's sequential stream: image bytes, label, attempts and the
    stream fingerprint; the 3-sample case continues one stream across calls"""
    for name, size, shape, seed, rels, bgi in CASES:
        root, bgs = trees[size]
        aug = IM.GpuMultiAugmenter("cuda", root=root, keep_u8=True, max_attempts=_max_attempts(golden))
        rng = random.Random(seed)
        for k, rel in enumerate(rels):
            tag = "%s_%d" % (name, k)
            x, label = IM.load_data_detection(os.path.join(root, rel), shape, JITTER, 0.05, 1.5, 1.5, bgs[bgi], K, MAX_GT, "cuda", rng=rng,
                                              root=root, augmenter=aug)
            assert np.array_equal(aug.u8[0].cpu().numpy(), golden["img_" + tag]), tag
            assert np.array_equal(label, golden["label_" + tag]), tag
            assert aug.attempts[0] == list(golden["attempts_" + tag]), tag
            assert x.shape == (3, shape[1], shape[0]) and x.dtype == torch.float32 and x.is_cuda
        assert rng.getrandbits(64) == int(golden["rng_" + name]), name


def _batch_96(trees, golden, one):
    """the four 96x96 samples of the 160x120 tree with the rng state each has in its golden run (the 3-sample case's stream is
    advanced by running its samples one at a time through `one`)"""
    root, bgs = trees[(160, 120)]
    samples, states, tags = [], [], []
    for name, size, shape, seed, rels, bgi in CASES:
        if size != (160, 120) or shape != (96, 96):
            continue
        r = random.Random(seed)
        for k, rel in enumerate(rels):
            samples.append((os.path.join(root, rel), bgs[bgi]))
            states.append(r.getstate())
            tags.append("%s_%d" % (name, k))
            one([samples[-1]], (96, 96), [r], JITTER, K, MAX_GT)
            assert np.array_equal(one.u8[0].cpu().numpy(), golden["img_" + tags[-1]]), tags[-1]
    return samples, states, tags


def _rngs(states):
    out = []
    for st in states:
        out.append(random.Random())
        out[-1].setstate(st)
    return out


def test_lockstep_batch_equals_samples_one_at_a_time(golden, trees):
    """a batch with one rng per sample gives every sample's golden bytes, label and attempts; it takes as many rounds as the
    sample with the most attempts; float output = uint8 / 255; a second run from the warm object bank is identical and copies
    fewer bytes"""
    root, _bgs = trees[(160, 120)]
    one = IM.GpuMultiAugmenter("cuda", root=root, keep_u8=True, max_attempts=_max_attempts(golden))
    samples, states, tags = _batch_96(trees, golden, one)
    aug = IM.GpuMultiAugmenter("cuda", root=root, keep_u8=True, max_attempts=_max_attempts(golden))
    x, labels = aug(samples, (96, 96), _rngs(states), JITTER, K, MAX_GT)
    for i, tag in enumerate(tags):
        assert np.array_equal(aug.u8[i].cpu().numpy(), golden["img_" + tag]), tag
        assert np.array_equal(labels[i], golden["label_" + tag]), tag
        assert aug.attempts[i] == list(golden["attempts_" + tag]), tag
    assert aug.rounds == max(int(np.sum(golden["attempts_" + t])) for t in tags)
    u8 = aug.u8.clone()
    want = u8.permute(0, 3, 1, 2).cpu().numpy().astype(np.float32) / np.float32(255)      # ToTensor: IEEE byte / 255
    assert np.array_equal(x.cpu().numpy(), want)
    cold_h2d, cold_dec = aug.h2d_bytes, aug.decodes
    x2, labels2 = aug(samples, (96, 96), _rngs(states), JITTER, K, MAX_GT)
    assert torch.equal(aug.u8, u8) and torch.equal(x2, x) and np.array_equal(labels2, labels)
    assert aug.decodes == 3 * len(samples) < cold_dec and aug.h2d_bytes < cold_h2d


def test_cpu_device_raises():
    with pytest.raises(SspError):
        IM.GpuMultiAugmenter("cpu")
    with pytest.raises(SspError):
        IM.load_data_detection("x", (96, 96), JITTER, 0, 1, 1, "y", K, MAX_GT, "cpu")


def test_dataset_collate_train_and_test_batches(golden, trees):
    """dataset_multi.listDataset + GpuMultiCollate: a train batch equals the oracle run with each sample's seed (bytes through the
    float output, labels); a test batch equals the reference listDataset's test-mode output"""
    from singleshotpose_b200 import dataset_multi as D
    root, bgs = trees[(160, 120)]
    lst = os.path.join(root, "ds_train.txt")
    with open(lst, "w") as f:
        f.write("".join(os.path.join(root, p) + "\n" for p in M.DATASET_TRAIN_LIST))
    random.seed(3)
    ds = D.listDataset(lst, shape=(104, 104), shuffle=True, objclass="ape", train=True, seen=0, batch_size=4, num_workers=1, cell_size=8,
                       bg_file_names=bgs)
    samples = [ds[i] for i in range(4)]
    collate = D.GpuMultiCollate("cuda", root=root, max_attempts=_max_attempts(golden))
    data, target = collate(samples)
    assert data.shape == (4, 3, 104, 104) and data.is_cuda and target.shape == (4, MAX_GT * (2 * K + 3)) and target.dtype == torch.float64
    for i, s in enumerate(samples):
        want, want_label, _att = M.load_data_detection(s["imgpath"], (104, 104), JITTER, s["bgpath"], K, MAX_GT, rng=random.Random(s["seed"]),
                                                       root=root)
        assert np.array_equal(data[i].cpu().numpy(), want.transpose(2, 0, 1).astype(np.float32) / np.float32(255)), i
        assert np.array_equal(target[i].numpy(), want_label), i
    tst = os.path.join(root, "ds_test.txt")
    with open(tst, "w") as f:
        f.write("".join(os.path.join(root, p) + "\n" for p in M.DATASET_TEST_LIST))
    ds = D.listDataset(tst, shape=(64, 48), shuffle=False, objclass="ape", train=False, num_workers=3)
    data, target = collate([ds[i] for i in range(len(M.DATASET_TEST_LIST))])
    for i in range(len(M.DATASET_TEST_LIST)):
        want = golden["ds_test_img_%d" % i]
        assert np.array_equal(data[i].cpu().numpy(), want.transpose(2, 0, 1).astype(np.float32) / np.float32(255)), i
        assert np.array_equal(target[i].numpy(), golden["ds_test_label_%d" % i]), i
