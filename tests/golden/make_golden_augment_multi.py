"""Generate tests/golden/augment_multi.npz from the REFERENCE ITSELF: multi_obj_pose_estimation/image_multi.py's
load_data_detection, run unmodified with a seeded `random` on the synthetic LINEMOD tree of
singleshotpose_b200.synth.write_linemod_multi_like.

Run where the reference checkout is available (path in REF below):
    python tests/golden/make_golden_augment_multi.py
The reference opens '../LINEMOD/<obj>/train.txt' and '../' + <line>, so it runs with the working directory one level below the
tree's root.  One shim: Pillow 12 renamed ImageMath.eval (image_multi.py:48) to unsafe_eval.  Every case is also run through
the numpy restatement (oracle/augment_multi_ref.py) and must be byte-identical.  Stored per case: the uint8 image,
the label, the attempts per pasted object (counted by a wrapper around the module's data_augmentation_with_mask) and
random.getrandbits(64) after the call, which pins the exact amount of randomness consumed.

It also runs dataset_multi.listDataset unmodified on the 160x120 tree: test mode (resize + labels_occlusion/ labels) for four
images, and ds[0] in train mode at one `seen` value in every band of its resolution schedule.  Stored for train mode: the
network shape and background the reference passed to load_data_detection, ds.seen afterwards, and the 63-bit number a
random.Random in the state of that moment draws first (what dataset_multi of this package draws as the per-sample seed).

A separate script, not a flag of make_golden.py: that generator and the fixtures it writes are left exactly as they are.
"""
import contextlib
import io
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REPO)

from singleshotpose_b200 import synth          # noqa: E402
from oracle import augment_multi_ref as M     # noqa: E402

CASES = M.GOLDEN_CASES
JITTER, NUM_KEYPOINTS, MAX_NUM_GT = M.JITTER, M.NUM_KEYPOINTS, M.MAX_NUM_GT


def dataset_cases(ref_dataset, out):
    """dataset_multi.listDataset, cwd = <tree>/work; the list files hold '../LINEMOD/...' paths as the reference's do"""
    import torch
    to_tensor = lambda img: torch.from_numpy(np.asarray(img).copy()).permute(2, 0, 1).float().div(255)       # transforms.ToTensor
    seen_calls = []
    orig = ref_dataset.load_data_detection

    def recording(imgpath, shape, jitter, hue, saturation, exposure, bgpath, *a):
        r = random.Random()
        r.setstate(random.getstate())
        seen_calls.append((imgpath, tuple(shape), bgpath, r.getrandbits(63)))
        return orig(imgpath, shape, jitter, hue, saturation, exposure, bgpath, *a)
    ref_dataset.load_data_detection = recording
    with open("train_list.txt", "w") as f:
        f.write("".join("../%s\n" % p for p in M.DATASET_TRAIN_LIST))
    with open("test_list.txt", "w") as f:
        f.write("".join("../%s\n" % p for p in M.DATASET_TEST_LIST))
    bgs = ["../bg/bg0.png", "../bg/bg1.png"]
    for j, seen in enumerate(M.DATASET_SEEN):
        random.seed(20 + j)
        ds = ref_dataset.listDataset("train_list.txt", shape=(104, 104), shuffle=True, objclass="ape", train=True, seen=seen,
                                     batch_size=2, num_workers=2, cell_size=8, bg_file_names=bgs)
        img, label = ds[0]
        imgpath, shape, bgpath, seed63 = seen_calls[-1]
        out["ds_train_%d_shape" % j] = np.array(shape)
        out["ds_train_%d_img" % j] = os.path.relpath(imgpath, "..")
        out["ds_train_%d_bg" % j] = os.path.basename(bgpath)
        out["ds_train_%d_seed63" % j] = np.array(seed63, np.uint64)
        out["ds_train_%d_seen" % j] = np.array(ds.seen)
        print("dataset_multi golden train seen=%d: shape %s, bg %s" % (seen, shape, bgpath))
    random.seed(9)
    ds = ref_dataset.listDataset("test_list.txt", shape=(64, 48), shuffle=False, transform=to_tensor, objclass="ape", train=False,
                                 num_workers=3)
    for i in range(len(M.DATASET_TEST_LIST)):
        img, label = ds[i]
        out["ds_test_img_%d" % i] = (img * 255).round().to(torch.uint8).permute(1, 2, 0).numpy()
        out["ds_test_label_%d" % i] = label.numpy()
    out["ds_test_seen"] = np.array(ds.seen)
    ref_dataset.load_data_detection = orig


def main():
    from PIL import ImageMath
    if not hasattr(ImageMath, "eval"):
        ImageMath.eval = ImageMath.unsafe_eval
    mdir = os.path.join(REF, "multi_obj_pose_estimation")
    sys.path.insert(0, mdir)
    with contextlib.redirect_stdout(io.StringIO()):
        import image_multi as ref
    counts = []
    orig_aug, orig_sup = ref.data_augmentation_with_mask, ref.superimpose_masks

    def counting_aug(*a, **k):
        counts[-1] += 1
        return orig_aug(*a, **k)

    def counting_sup(*a, **k):
        counts.append(0)
        return orig_sup(*a, **k)
    ref.data_augmentation_with_mask, ref.superimpose_masks = counting_aug, counting_sup
    with contextlib.redirect_stdout(io.StringIO()):
        import dataset_multi as ref_dataset
    out = {}
    cwd = os.getcwd()
    trees = {}
    with tempfile.TemporaryDirectory() as tmp:
        try:
            for name, (ow, oh), shape, seed, mains, bgi in CASES:
                if (ow, oh) not in trees:
                    root = os.path.join(tmp, "t%dx%d" % (ow, oh))
                    os.makedirs(os.path.join(root, "work"))
                    trees[(ow, oh)] = (root, synth.write_linemod_multi_like(root, ow=ow, oh=oh))
                root, bgs = trees[(ow, oh)]
                os.chdir(os.path.join(root, "work"))
                bgpath = "../bg/" + os.path.basename(bgs[bgi])
                random.seed(seed)
                orng = random.Random(seed)
                for k, rel in enumerate(mains):
                    counts[:] = [0]
                    img, label = ref.load_data_detection("../" + rel, shape, JITTER, 0.05, 1.5, 1.5, bgpath, NUM_KEYPOINTS, MAX_NUM_GT)
                    img = np.asarray(img)
                    attempts = counts[:-1]
                    o_img, o_label, o_att = M.load_data_detection("../" + rel, shape, JITTER, bgpath, NUM_KEYPOINTS, MAX_NUM_GT, rng=orng)
                    assert np.array_equal(o_img, img), (name, k, "image")
                    assert np.array_equal(o_label, label), (name, k, "label")
                    assert o_att == attempts, (name, k, o_att, attempts)
                    tag = "%s_%d" % (name, k)
                    out["img_" + tag], out["label_" + tag], out["attempts_" + tag] = img, np.asarray(label), np.array(attempts)
                    print("augment_multi golden %s: %s -> %s, attempts %s, oracle byte-identical" % (tag, (ow, oh), shape, attempts))
                fp = random.getrandbits(64)
                assert orng.getrandbits(64) == fp, name
                out["rng_" + name] = np.array(fp, np.uint64)
            os.chdir(os.path.join(trees[(160, 120)][0], "work"))
            dataset_cases(ref_dataset, out)
        finally:
            os.chdir(cwd)
    import PIL
    out["pillow_version"] = np.array(PIL.__version__)
    np.savez_compressed(os.path.join(HERE, "augment_multi.npz"), **out)


if __name__ == "__main__":
    main()
