"""CPU checks of the multi-object pose predictor's pieces (singleshotpose_b200/predict_multi.py): the ssp_predict_multi_select ABI
(symbol, argument checks), the prediction rules of singleshotpose_b200/csrc/eval_multi_core.h compiled for the host by
tests/helpers/predict_multi_host.cpp against the oracle of valid_multi.py's loop and against the reference's own run
(tests/golden/eval_multi.npz), and the command line's parsing.  No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import eval_multi_ref as EM
from singleshotpose_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, NC, NA, NL = 9, 13, 5, 21
SSP_ERR_ARG = -1


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "eval_multi.npz"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pmhost") / "libpmhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", "predict_multi_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host_predict(host, outputs, classes, conf_thresh, frame=(640, 480)):
    out = np.ascontiguousarray(outputs, np.float32)
    cls = np.ascontiguousarray(classes, np.int32)
    B, _, H, W = out.shape
    Q = len(cls)
    boxes = np.zeros((B, Q, NL), np.float32)
    flags = np.zeros((B, Q), np.int32)
    uv = np.zeros((B, Q, K, 2), np.float32)
    pos = np.zeros((B, Q), np.int32)
    rc = host.h_predict_multi_select(_p(out), B, K, NC, NA, H, W, _p(cls), Q, C.c_float(conf_thresh), C.c_float(frame[0]), C.c_float(frame[1]),
                                     _p(boxes), _p(flags), _p(uv), _p(pos))
    assert rc == 0
    return dict(boxes=boxes, flags=flags, uv=uv, pos=pos)


def one_row_target(c):
    """a label holding one ground truth of class c (the oracle's selection reads only the class of each row)"""
    t = np.zeros(50 * NL, np.float32)
    t[0], t[1:NL] = c, 0.5
    return t


# ------------------------------------------------------------------------------------------------ ABI
def test_symbol_is_declared_and_exported():
    assert "ssp_predict_multi_select" in _lib.SIGNATURES
    assert hasattr(_lib.load(), "ssp_predict_multi_select")
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        assert "int ssp_predict_multi_select(" in f.read()


def _select(out=1, K_=9, nC=13, nA=5, H=13, W=13, classes=(0, 4), n_req=None, boxes=1, flags=1, uv=1):
    cls = None if classes is None else (C.c_int * max(1, len(classes)))(*classes)
    fake = lambda a: C.c_void_p(0x10000 * a) if a else None
    return _lib.load().ssp_predict_multi_select(fake(out), 1, K_, nC, nA, H, W, cls, len(classes or ()) if n_req is None else n_req,
                                                C.c_float(0.05), C.c_float(640), C.c_float(480), fake(boxes), fake(flags), fake(uv), None)


def test_predict_multi_select_rejects_bad_arguments():
    bad = [dict(out=0), dict(boxes=0), dict(flags=0), dict(uv=0), dict(classes=None, n_req=1),      # null pointers
           dict(K_=8),                                                                                # not the 9 keypoints of a box
           dict(H=29, W=29), dict(nC=257),                                                            # 29x29x5 > 4096 entries; > 256 classes
           dict(n_req=0), dict(n_req=-1),
           dict(classes=(0, 13)), dict(classes=(-1,)), dict(classes=(3, 5, 3))]                       # out of range, duplicate
    for kw in bad:
        assert _select(**kw) == SSP_ERR_ARG, kw
    lib = _lib.load()
    _select(K_=8)
    assert b"num_keypoints must be 9" in lib.ssp_last_error()
    _select(classes=(3, 5, 3))
    assert b"twice" in lib.ssp_last_error()
    _select(H=29, W=29)
    assert b"grid too large" in lib.ssp_last_error()


# ------------------------------------------------------------------------------------------------ host build against the oracle
@pytest.mark.parametrize("thr_scale", [0.2, 1.0, 4.0])
def test_host_build_matches_oracle_for_every_class(golden, host, thr_scale):
    """slot (image, class c) = evaluate_image_multi_ref on the image with a one-row target of class c: the chosen list position and
    the fallback flag exactly, the box and the PnP points, for all 13 classes at the golden threshold and a lower and a higher one"""
    thr = float(golden["conf_thresh"]) * thr_scale
    outs = golden["outputs"]
    r = host_predict(host, outs, np.arange(NC), thr)
    kinds = set()
    for b in range(outs.shape[0]):
        for c in range(NC):
            (x,), _boxes = EM.evaluate_image_multi_ref(torch.from_numpy(outs[b:b + 1]), one_row_target(c), thr, NC, K, list(golden["anchors"]),
                                                       NA, None, None, np.eye(3), with_pose=False)
            assert not x["carried"]
            assert r["pos"][b, c] == x["pos"] and r["flags"][b, c] == int(x["fallback"]), (b, c)
            # the oracle's torch sigmoid / softmax and libm's expf may differ in the last bit: the choice is exact, the values
            # within fp32 rounding (the GPU test pins the kernel to ssp_eval_multi_select bit for bit)
            np.testing.assert_allclose(r["boxes"][b, c], x["box"], rtol=1e-5, atol=1e-7, err_msg="image %d class %d" % (b, c))
            np.testing.assert_allclose(r["uv"][b, c], x["uv_pr"], rtol=1e-5, err_msg="image %d class %d" % (b, c))
            assert r["boxes"][b, c, 2 * K + 2] == c
            kinds.add(bool(x["fallback"]))
    assert kinds == {True, False}                             # both listed and fallback slots occur


def test_host_build_slots_follow_the_requested_order(golden, host):
    outs = golden["outputs"]
    order = [7, 0, 12, 4]
    a = host_predict(host, outs, np.arange(NC), 0.05)
    b = host_predict(host, outs, order, 0.05, frame=(320, 240))
    for k in ("boxes", "flags", "pos"):
        np.testing.assert_array_equal(b[k], a[k][:, order])
    np.testing.assert_array_equal(b["uv"], b["boxes"][..., :2 * K].reshape(-1, len(order), K, 2) * np.float32([320, 240]))


def test_host_build_pins_to_the_reference_run(golden, host):
    """the slot of each image's first ground-truth class is the box the reference's own valid() chose for that ground truth"""
    outs, tgts, counts = golden["outputs"], golden["targets"], golden["counts"]
    r = host_predict(host, outs, np.arange(NC), float(golden["conf_thresh"]))
    offs = np.concatenate([[0], np.cumsum(counts)])
    checked = 0
    for b in range(outs.shape[0]):
        if counts[b] == 0:
            continue
        c, g = int(tgts[b][0]), int(offs[b])
        assert r["pos"][b, c] == golden["pos"][g] and r["flags"][b, c] == golden["flags"][g], (b, c)
        np.testing.assert_allclose(r["uv"][b, c], golden["pnp_points2d"][2 * g + 1], rtol=1e-5)
        checked += 1
    assert checked == int((counts > 0).sum()) >= 5


# ------------------------------------------------------------------------------------------------ command line
def test_cli_parsing(tmp_path):
    from singleshotpose_b200.predict import read_camera
    from singleshotpose_b200.predict_multi import SIZE_KEYS, parse_objects, main
    p = tmp_path / "occlusion.data"
    p.write_text("train  = cfg/train_occlusion.txt\nmesh1 = ../LINEMOD/ape/ape.ply\ngpus = 0\nim_width = 640\nim_height = 480\n"
                 "fx = 572.4114 \nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    _mesh, Km, size = read_camera(str(p), SIZE_KEYS)
    assert size == (640, 480)
    assert np.array_equal(Km, np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]]))
    for missing in ("im_width", "im_height", "fx", "v0"):
        q = tmp_path / ("no_%s.data" % missing)
        q.write_text("".join(l + "\n" for l in p.read_text().splitlines() if not l.startswith(missing)))
        with pytest.raises(_lib.SspError, match=missing):
            read_camera(str(q), SIZE_KEYS)
    q = tmp_path / "single.data"
    q.write_text("mesh = m.ply\nwidth = 640\nheight = 480\nfx = 1\nfy = 1\nu0 = 1\nv0 = 1\n")   # the single-object keys are not read
    with pytest.raises(_lib.SspError, match="im_width"):
        read_camera(str(q), SIZE_KEYS)
    assert parse_objects(["4=can.ply", "0=a=b.ply"]) == {4: "can.ply", 0: "a=b.ply"}
    for bad in (["ape.ply"], ["x=ape.ply"], ["1="], ["-1=ape.ply"], ["=ape.ply"], ["0=a.ply", "0=b.ply"], []):
        with pytest.raises(_lib.SspError):
            parse_objects(bad)
    with pytest.raises(SystemExit):
        main(["--datacfg", str(p), "--modelcfg", "m.cfg", "--weightfile", "w", "img.png"])      # --object is required
