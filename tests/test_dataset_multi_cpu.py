"""CPU tests of singleshotpose_b200.dataset_multi (host half of the multi-object loader) against the reference's own
dataset_multi.listDataset, run unmodified on the synthetic LINEMOD tree (tests/golden/augment_multi.npz, keys ds_*):
train mode -- the resolution schedule, background draw, `seen` bookkeeping and the per-sample seed drawn from the same
stream state; test mode -- labels_occlusion/ labels with the objclass path replace, and the resized image (the resize done by
the oracle here; the GPU kernel in tests/test_gpu_augment_multi.py)."""
import os
import random

import numpy as np
import pytest

from oracle import augment_ref as A
from oracle import augment_multi_ref as M
from singleshotpose_b200 import dataset_multi as D
from singleshotpose_b200 import synth


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_multi.npz"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("linemod_ds"))
    bgs = synth.write_linemod_multi_like(root, ow=160, oh=120)
    for name, paths in (("train_list.txt", M.DATASET_TRAIN_LIST), ("test_list.txt", M.DATASET_TEST_LIST)):
        with open(os.path.join(root, name), "w") as f:
            f.write("".join(os.path.join(root, p) + "\n" for p in paths))
    return root, bgs


def test_train_mode_schedule_background_and_seed_follow_the_reference(golden, tree):
    root, bgs = tree
    for j, seen in enumerate(M.DATASET_SEEN):
        random.seed(20 + j)
        ds = D.listDataset(os.path.join(root, "train_list.txt"), shape=(104, 104), shuffle=True, objclass="ape", train=True, seen=seen,
                           batch_size=2, num_workers=2, cell_size=8, bg_file_names=bgs)
        s = ds[0]
        assert s["shape"] == tuple(golden["ds_train_%d_shape" % j]), seen
        assert os.path.basename(s["bgpath"]) == str(golden["ds_train_%d_bg" % j]), seen
        assert os.path.relpath(s["imgpath"], root) == str(golden["ds_train_%d_img" % j]), seen
        assert s["seed"] == int(golden["ds_train_%d_seed63" % j]), seen
        assert ds.seen == int(golden["ds_train_%d_seen" % j])
        assert np.array_equal(s["img"], M.read_rgb(s["imgpath"])) and np.array_equal(s["bg"], M.read_rgb(s["bgpath"]))
        assert np.array_equal(s["mask"], M.read_rgb(M.mask_path(s["imgpath"])))
    # every band of the schedule is visited, and only its sizes come out
    bands = [(13, 13), (13, 16), (12, 17), (11, 18), (10, 19)]
    for seen, (lo, hi) in zip(M.DATASET_SEEN, bands):
        ds = D.listDataset(os.path.join(root, "train_list.txt"), shuffle=False, train=True, seen=seen, batch_size=2, cell_size=8,
                           bg_file_names=bgs)
        widths = set()
        for _ in range(60):
            ds.seen = seen
            widths.add(ds[0]["shape"][0] // 8)
        assert widths <= set(range(lo, hi + 1)) and (lo == hi or len(widths) > 1), (seen, widths)


def test_test_mode_equals_the_reference(golden, tree):
    root, _bgs = tree
    random.seed(9)
    ds = D.listDataset(os.path.join(root, "test_list.txt"), shape=(64, 48), shuffle=False, objclass="ape", train=False, num_workers=3)
    for i in range(len(M.DATASET_TEST_LIST)):
        s = ds[i]
        assert np.array_equal(s["label"].numpy(), golden["ds_test_label_%d" % i]), i
        assert s["shape"] == (64, 48)
        assert np.array_equal(A.resize_u8(s["img"], s["shape"]), golden["ds_test_img_%d" % i]), i
    assert ds.seen == int(golden["ds_test_seen"])


def test_collate_has_no_cpu_path():
    from singleshotpose_b200._lib import SspError
    with pytest.raises(SspError):
        D.GpuMultiCollate("cpu")
