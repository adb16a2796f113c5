"""CPU tests of the multi-object evaluation tail (valid_multi.py:97-158 of the reference's multi_obj_pose_estimation):
  * the restatement (oracle/eval_multi_ref.py) against the reference's own valid() through the committed golden
    (tests/golden/eval_multi.npz, written by tests/golden/make_golden_eval_multi.py): chosen box list positions, the points of
    every pnp call bit for bit, pixel errors and the accuracy table;
  * the selection rules of the kernel core (singleshotpose_b200/csrc/eval_multi_core.h) compiled for the host by
    tests/helpers/eval_multi_host.cpp, driven by the product's host code (utils_multi.truths_lengths for the offsets);
  * the host helpers (truths_lengths, projection_accuracy) and the argument checks of ssp_eval_multi_select."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import eval_multi_ref as EM
from singleshotpose_b200 import _lib
from singleshotpose_b200 import utils_multi as UM

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, NC, NA, NL = 9, 13, 5, 21


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "eval_multi.npz"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("evmhost") / "libevmhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", "eval_multi_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host_select(host, outputs, targets, conf_thresh, im_width=640, im_height=480):
    """run the host build over a batch; offsets from the product's host code"""
    out = np.ascontiguousarray(outputs, np.float32)
    tgt = np.ascontiguousarray(targets, np.float32)
    B, _, H, W = out.shape
    counts = UM.truths_lengths(torch.from_numpy(tgt), K)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    G = int(off[-1])
    boxes = np.zeros((G, NL), np.float32)
    flags = np.zeros(G, np.int32)
    uv = np.zeros((2 * G, K, 2), np.float32)
    pos = np.zeros(G, np.int32)
    rc = host.h_eval_multi_select(_p(out), B, K, NC, NA, H, W, _p(tgt), tgt.shape[1], _p(off), C.c_float(conf_thresh), C.c_float(im_width),
                                  C.c_float(im_height), _p(boxes), _p(flags), _p(uv), _p(pos))
    assert rc == 0
    return dict(boxes=boxes, flags=flags, uv=uv, pos=pos, counts=counts)


# ------------------------------------------------------------------------------------------------ oracle vs reference golden
def test_oracle_matches_reference_golden(golden):
    Kc, V, corners = golden["K"], golden["vertices"], golden["corners3D"]
    errs, gi = [], 0
    for b in range(golden["outputs"].shape[0]):
        res, boxes = EM.evaluate_image_multi_ref(torch.from_numpy(golden["outputs"][b:b + 1]), golden["targets"][b], float(golden["conf_thresh"]),
                                                 NC, K, list(golden["anchors"]), NA, V, corners, Kc)
        assert len(boxes) == golden["list_lengths"][b]
        for r in res:
            assert r["pos"] == golden["pos"][gi] and r["fallback"] + 2 * r["carried"] == golden["flags"][gi], (b, gi)
            assert np.array_equal(r["uv_gt"], golden["pnp_points2d"][2 * gi]), (b, gi)
            assert np.array_equal(r["uv_pr"], golden["pnp_points2d"][2 * gi + 1]), (b, gi)
            assert r["pixel_err"] == pytest.approx(float(golden["pixel_err"][gi]), rel=1e-4), (b, gi)
            errs.append(r["pixel_err"])
            gi += 1
    assert gi == len(golden["pos"])
    assert EM.projection_accuracy_ref(errs) == list(golden["accuracy"])
    np.testing.assert_allclose(golden["accuracy"], golden["printed_accuracy"], atol=5e-3)


def test_golden_covers_the_selection_cases(golden):
    """fallback, carry-over, an empty label file, several ground truths of one image, and the equal-logit tie (two boxes in
    one image's list whose det_conf is equal, the first chosen)"""
    f = golden["flags"]
    assert (f & 1).any() and (f & 2).any()
    counts = golden["counts"]
    assert 0 in counts and counts.max() >= 3
    assert len(golden["pos"]) == counts.sum()


# ------------------------------------------------------------------------------------------------ host build of the kernel core
def test_host_build_matches_golden(golden, host):
    r = host_select(host, golden["outputs"], golden["targets"], float(golden["conf_thresh"]))
    assert list(r["counts"]) == list(golden["counts"])
    np.testing.assert_array_equal(r["pos"], golden["pos"])
    np.testing.assert_array_equal(r["flags"], golden["flags"])
    G = len(golden["pos"])
    pts = golden["pnp_points2d"]
    np.testing.assert_allclose(r["uv"][:G], pts[0::2], rtol=1e-5)
    np.testing.assert_allclose(r["uv"][G:], pts[1::2], rtol=1e-5)
    np.testing.assert_array_equal(r["uv"][:G], pts[0::2])          # the ground truth takes no transcendental: bit-equal


def test_host_build_matches_oracle_random(host):
    """seeded random outputs with many boxes above the threshold and 1-3 ground truths per image, several sharing a class"""
    from singleshotpose_b200 import synth
    gen = torch.Generator().manual_seed(7)
    B = 4
    out = torch.randn(B, 160, 13, 13, generator=gen)
    out[:, [18 + 32 * a for a in range(5)]] += 1.0
    tgt = synth.targets_multi(B, seed=11, num_classes=4)
    r = host_select(host, out.numpy(), tgt.numpy(), 0.05)
    gi = 0
    for b in range(B):
        res, boxes = EM.evaluate_image_multi_ref(out[b:b + 1], tgt[b].numpy(), 0.05, NC, K, synth.MULTI_ANCHORS, NA, None, None, np.eye(3),
                                                 with_pose=False)
        assert len(boxes) > 20
        for x in res:
            assert r["pos"][gi] == x["pos"] and r["flags"][gi] == x["fallback"] + 2 * x["carried"], (b, gi)
            np.testing.assert_allclose(r["boxes"][gi], x["box"], rtol=1e-5, atol=1e-7)
            gi += 1
    assert gi == len(r["pos"])


def test_host_build_fallback_when_nothing_is_listed(host):
    gen = torch.Generator().manual_seed(21)
    out = torch.randn(2, 160, 13, 13, generator=gen) * 0.5
    out[:, [18 + 32 * a for a in range(5)]] -= 6.0
    tgt = torch.zeros(2, 50 * NL)
    tgt[:, 0], tgt[:, 1:19] = 7, 0.5
    tgt[1, NL] = 2
    tgt[1, NL + 1:NL + 19] = 0.25
    r = host_select(host, out.numpy(), tgt.numpy(), 0.05)
    assert list(r["flags"]) == [1, 1, 3]                              # image 1's second ground truth carries the fallback over
    for b in range(2):
        res, _ = EM.evaluate_image_multi_ref(out[b:b + 1], tgt[b].numpy(), 0.05, NC, K, [], NA, None, None, np.eye(3), with_pose=False)
        assert res[0]["fallback"] and r["pos"][b] == res[0]["pos"] == 0


# ------------------------------------------------------------------------------------------------ host helpers and the C ABI
def test_truths_lengths_and_offsets():
    t = np.zeros((4, 50 * NL), np.float32)
    t[1, 1] = 0.3                                                     # one ground truth
    for k in range(3):
        t[2, k * NL + 1] = 0.1 * (k + 1)
    t[2, 4 * NL + 1] = 0.5                                            # a row after the first x0 == 0 does not count
    t[3, 1::NL] = 0.7                                                 # all 50 rows filled
    n = UM.truths_lengths(torch.from_numpy(t))
    assert list(n) == [0, 1, 3, 50]
    assert [EM.truths_length(t[b].reshape(-1, NL)) for b in range(3)] == [0, 1, 3]
    assert EM.truths_length(t[3].reshape(-1, NL)) is None             # the reference's range(None)
    assert list(UM.truths_lengths(t)) == list(n)


def test_projection_accuracy_matches_reference_formula():
    rng = np.random.default_rng(3)
    errs = np.concatenate([rng.uniform(0, 60, 97), [5.0, 10.0, 50.0]]).astype(np.float32)
    want = [len(np.where(np.array(errs) <= px)[0]) * 100. / (len(errs) + 1e-5) for px in (5, 10, 15, 20, 25, 30, 35, 40, 45, 50)]
    assert UM.projection_accuracy(errs) == want
    assert UM.projection_accuracy(torch.from_numpy(errs)) == want
    assert UM.projection_accuracy([]) == [0.0] * 10
    assert UM.projection_accuracy(errs, thresholds=(1, 2)) == EM.projection_accuracy_ref(errs, (1, 2))


def test_eval_multi_select_rejects_bad_arguments():
    dummy = C.c_void_p(1)
    args = lambda K, H, W: (dummy, 1, K, 13, 5, H, W, dummy, 50 * (2 * K + 3), dummy, C.c_float(0.05), C.c_float(640), C.c_float(480),
                            dummy, dummy, dummy, None)
    with pytest.raises(_lib.SspError, match="num_keypoints must be 9"):
        _lib.call("ssp_eval_multi_select", *args(8, 13, 13))
    with pytest.raises(_lib.SspError, match="grid too large"):
        _lib.call("ssp_eval_multi_select", *args(9, 29, 29))
