"""CPU checks of every-instance detection (singleshotpose_b200/predict_instances.py): the ABI of ssp_detect_instances and
ssp_pnp_batched_counted (symbols, argument checks), the ordering / IoU / suppression stage of singleshotpose_b200/csrc/detect_core.h
compiled for the host by tests/helpers/detect_host.cpp against the numpy oracle (oracle/detect_ref.py), the oracle's candidate
listing against the reference's own (tests/golden/decode_multi.npz), and the command line's checks.  No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import detect_ref as DR
from singleshotpose_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSP_ERR_ARG = -1
F32 = np.float32


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dethost") / "libdethost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "detect_host.cpp")])
    lib = C.CDLL(so)
    lib.h_iou.restype = C.c_float
    return lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host_stage(host, det, cmax, cls_id, uv, classes, conf_thresh, nms_thresh, max_inst, num_classes=13):
    det, cmax = np.ascontiguousarray(det, F32), np.ascontiguousarray(cmax, F32)
    cls_id = np.ascontiguousarray(cls_id, np.int32)
    uv = np.ascontiguousarray(uv, F32)
    req = np.zeros(256, np.uint8)
    req[list(classes)] = 1
    entries = np.zeros(max_inst, np.int32)
    count, kept = C.c_int(), C.c_int()
    rc = host.h_detect_stage(_p(det), _p(cmax), _p(cls_id), _p(uv), len(det), _p(req), C.c_float(conf_thresh), C.c_float(nms_thresh),
                             max_inst, _p(entries), C.byref(count), C.byref(kept))
    assert rc == 0
    assert (entries[count.value:] == -1).all()
    return list(entries[:count.value]), kept.value


def _check(host, det, cmax, cls_id, uv, classes, thr, nms, M):
    got = host_stage(host, det, cmax, cls_id, uv, classes, thr, nms, M)
    want = DR.detect_ref(det, cmax, cls_id, uv, thr, nms, classes, M)
    assert got[0] == want[0] and got[1] == want[1], (got, want)
    return got


def _random_frame(rng, n, nC=13, spread=60.0, size=40.0, ties=False):
    det = rng.random(n).astype(F32)
    if ties:
        det = (np.round(det * 8) / 8).astype(F32)                    # many exact ties of det
    cmax = (0.3 + 0.7 * rng.random(n)).astype(F32)
    cls_id = rng.integers(0, nC, n)
    centre = rng.random((n, 1, 2)) * spread
    uv = (centre + (rng.random((n, 9, 2)) - 0.5) * size).astype(F32)
    return det, cmax, cls_id, uv


# ------------------------------------------------------------------------------------------------ ABI
def test_symbols_are_declared_and_exported():
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        text = f.read()
    for name in ("ssp_detect_instances", "ssp_pnp_batched_counted"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
        assert "int %s(" % name in text


def _detect(out=1, K_=9, nC=13, nA=5, H=13, W=13, classes=(0, 4), n_req=None, nms=0.4, M=32, boxes=1, cls=1, uv=1, count=1, kept=1):
    c = None if classes is None else (C.c_int * max(1, len(classes)))(*classes)
    fake = lambda a: C.c_void_p(0x10000 * a) if a else None
    return _lib.load().ssp_detect_instances(fake(out), 1, K_, nC, nA, H, W, c, len(classes or ()) if n_req is None else n_req, C.c_float(0.05),
                                            C.c_float(nms), M, C.c_float(640), C.c_float(480), fake(boxes), fake(cls), fake(uv), fake(count),
                                            fake(kept), None)


def test_detect_instances_rejects_bad_arguments():
    bad = [dict(out=0), dict(boxes=0), dict(cls=0), dict(uv=0), dict(count=0), dict(kept=0), dict(classes=None, n_req=1),
           dict(K_=8), dict(H=29, W=29), dict(nC=257), dict(n_req=0),
           dict(classes=(0, 13)), dict(classes=(-1,)), dict(classes=(3, 5, 3)),
           dict(nms=-0.01), dict(nms=1.01), dict(nms=float("nan")), dict(M=0), dict(M=257)]
    for kw in bad:
        assert _detect(**kw) == SSP_ERR_ARG, kw
    lib = _lib.load()
    for kw, msg in ((dict(K_=8), b"num_keypoints must be 9"), (dict(classes=(3, 5, 3)), b"twice"), (dict(H=29, W=29), b"grid too large"),
                    (dict(nms=2.0), b"nms_thresh"), (dict(M=300), b"max_instances")):
        _detect(**kw)
        assert msg in lib.ssp_last_error(), kw


def test_pnp_counted_rejects_bad_arguments():
    fake = lambda a: C.c_void_p(0x10000 * a) if a else None
    lib = _lib.load()

    def run(P3=1, uv=1, K=1, np_=9, groups=2, per=4, count=1, R=1, t=1):
        return lib.ssp_pnp_batched_counted(fake(P3), fake(uv), fake(K), np_, groups, per, fake(count), 20, fake(R), fake(t), None)
    for kw in (dict(P3=0), dict(uv=0), dict(K=0), dict(count=0), dict(R=0), dict(t=0), dict(np_=5), dict(np_=17), dict(groups=-1),
               dict(per=0)):
        assert run(**kw) == SSP_ERR_ARG, kw
    assert run(groups=0) == 0                                          # nothing to solve: no launch


# ------------------------------------------------------------------------------------------------ host build against the oracle
def test_iou_arithmetic_matches_oracle(host):
    rng = np.random.default_rng(0)
    x, y = np.sort(rng.random((500, 2)) * 50, 1), np.sort(rng.random((500, 2)) * 50, 1)
    a = np.ascontiguousarray(np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1), F32)     # rows [x0, y0, x1, y1]
    b = np.ascontiguousarray(np.roll(a, 1, 0))
    for i in range(len(a)):
        assert np.float32(host.h_iou(_p(a[i]), _p(b[i]))).tobytes() == DR.iou_ref(a[i], b[i:i + 1])[0].tobytes(), i
    sq = np.float32([0, 0, 2, 2]); sh = np.float32([1, 0, 3, 2]); pt = np.float32([1, 1, 1, 1]); ln = np.float32([0, 1, 2, 1])
    assert host.h_iou(_p(sq), _p(sh)) == DR.iou_ref(sq, sh)[0] == np.float32(2) / np.float32(6)
    assert host.h_iou(_p(sq), _p(sq)) == DR.iou_ref(sq, sq)[0] == 1.0
    assert host.h_iou(_p(pt), _p(pt)) == DR.iou_ref(pt, pt)[0] == 0.0        # zero-area rectangles: union 0 -> IoU 0
    assert host.h_iou(_p(ln), _p(sq)) == DR.iou_ref(ln, sq)[0] == 0.0


@pytest.mark.parametrize("nms", [0.0, 0.2, 0.4, 0.7, 1.0])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_stage_equals_oracle_on_random_boxes(host, seed, nms):
    rng = np.random.default_rng(seed)
    n = [845, 3380, 4096][seed]
    det, cmax, cls_id, uv = _random_frame(rng, n, ties=seed == 1)
    for classes, thr, M in ((range(13), 0.3, 256), ([2, 7, 11], 0.1, 32), ([5], 0.05, 4)):
        entries, kept = _check(host, det, cmax, cls_id, uv, list(classes), thr, nms, M)
        assert len(entries) == min(kept, M)
        if nms == 1.0:                                                # IoU > 1 never holds: every candidate is kept
            assert kept == int(((det * cmax > F32(thr)) & np.isin(cls_id, list(classes))).sum())


def test_stage_ties_threshold_edges_zero_area_and_truncation(host):
    n = 12
    det = np.full(n, 0.5, F32)                                        # exact ties everywhere: entry order decides
    cmax = np.ones(n, F32)
    cls_id = np.zeros(n, np.int64)
    cls_id[6:] = 1
    uv = np.zeros((n, 9, 2), F32)

    def rect(i, x0, y0, x1, y1):
        uv[i, 1:, 0] = [x0, x1] * 4
        uv[i, 1:, 1] = [y0, y0, y1, y1] * 2
    for i in range(n):
        rect(i, 100 * i, 0, 100 * i + 2, 2)                           # disjoint
    rect(1, 1, 0, 3, 2)                                               # IoU(0, 1) = 2 / 6 exactly
    rect(2, 5, 5, 5, 5)                                               # a point: zero area
    rect(3, 5, 5, 5, 5)                                               # the same point
    rect(7, 600, 0, 602, 2)                                           # class 1 duplicate of entry 6
    at = F32(2) / F32(6)
    e, k = _check(host, det, cmax, cls_id, uv, [0, 1], 0.1, float(at), 32)
    assert 1 in e and 7 not in e and k == n - 1                     # IoU == threshold keeps; a duplicate (IoU 1) goes
    e, k = _check(host, det, cmax, cls_id, uv, [0, 1], 0.1, float(np.nextafter(at, F32(0))), 32)
    assert 1 not in e and 2 in e and 3 in e and k == n - 2          # just below: suppressed; zero-area boxes never suppress
    e, k = _check(host, det, cmax, cls_id, uv, [0, 1], 0.1, 0.0, 32)
    assert 1 not in e and k == n - 2
    e, k = _check(host, det, cmax, cls_id, uv, [0, 1], 0.1, 0.0, 3)
    assert e == [0, 2, 3] and k == n - 2                               # truncation keeps the key order
    e, k = _check(host, det, cmax, cls_id, uv, [1], 0.1, 0.5, 32)
    assert e == [6, 8, 9, 10, 11] and k == 5                           # class subset
    det[9] = F32(0.75)
    e, k = _check(host, det, cmax, cls_id, uv, [1], 0.1, 0.5, 2)
    assert e == [9, 6] and k == 5
    rect(6, 600, 0, 602, 2); rect(7, 600, 0, 602, 2)
    cls_id[7] = 0                                                     # same rectangle, other class: not suppressed
    e, k = _check(host, det, cmax, cls_id, uv, [0, 1], 0.1, 0.0, 32)
    assert 6 in e and 7 in e
    assert _check(host, det, cmax, cls_id, uv, [0, 1], 0.8, 0.4, 32) == ([], 0)      # no candidate at all


# ------------------------------------------------------------------------------------------------ oracle against the reference
def test_oracle_listing_is_the_reference_listing(golden_dir):
    """listing_ref = the reference's box list (decode_multi.npz: get_multi_region_boxes(..., correspondingclass=4,
    only_objectness=0) as the reference computed it) without its fallback box, which it appends when no listed box has class 4"""
    g = np.load(os.path.join(golden_dir, "decode_multi.npz"))
    assert int(g["correspondingclass"]) == 4
    lists = DR.listing_ref(torch.from_numpy(g["output"]), float(g["conf_thresh"]), 13, 9, list(g["anchors"]), 5)
    off = 0
    seen_fallback = seen_listed = False
    for b, n in enumerate(g["counts"]):
        ref = g["boxes"][off:off + n]
        off += n
        mine = np.array([[float(v) for v in bx] for bx in lists[b]]).reshape(-1, 21)
        has4 = bool((mine[:, 20] == 4).any())
        assert len(ref) == len(mine) + (0 if has4 else 1), b
        np.testing.assert_array_equal(ref[:len(mine)], mine)
        seen_fallback |= not has4
        seen_listed |= len(mine) > 0
    assert seen_listed


# ------------------------------------------------------------------------------------------------ command line
def test_cli_checks(tmp_path):
    from singleshotpose_b200.predict import read_camera
    from singleshotpose_b200.predict_instances import SIZE_KEYS, parse_args
    base = ["--datacfg", "d.data", "--modelcfg", "m.cfg", "--weightfile", "w"]
    a = parse_args(base + ["a.png", "b.png"])
    assert a.objects is None and a.nms_thresh == 0.4 and a.max_instances == 32 and a.images == ["a.png", "b.png"]
    a = parse_args(base + ["--object", "4=can.ply", "--object", "0=ape.ply", "--nms-thresh", "0", "--max-instances", "256", "x.jpg"])
    assert a.objects == {4: "can.ply", 0: "ape.ply"} and a.nms_thresh == 0.0 and a.max_instances == 256
    for bad in (["--nms-thresh", "1.5"], ["--nms-thresh", "-0.1"], ["--max-instances", "0"], ["--max-instances", "257"],
                ["--object", "x=a.ply"], ["--object", "0=a.ply", "--object", "0=b.ply"]):
        with pytest.raises(_lib.SspError):
            parse_args(base + bad + ["a.png"])
    with pytest.raises(SystemExit):
        parse_args(base)                                              # no image
    with pytest.raises(SystemExit):
        parse_args(["--modelcfg", "m.cfg", "--weightfile", "w", "a.png"])   # --datacfg is required
    single = tmp_path / "ape.data"
    single.write_text("mesh = ape.ply\nwidth = 640\nheight = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    mesh, Km, size = read_camera(str(single), SIZE_KEYS)
    assert mesh == "ape.ply" and size == (640, 480) and Km[0, 0] == 572.4114 and Km[1, 2] == 242.0489
    multi = tmp_path / "occlusion.data"
    multi.write_text("mesh1 = a.ply\nim_width = 320\nim_height = 240\nfx = 1\nfy = 2\nu0 = 3\nv0 = 4\n")
    mesh, Km, size = read_camera(str(multi), SIZE_KEYS)
    assert mesh is None and size == (320, 240) and Km[1, 1] == 2
    for missing in ("fx", "height"):
        q = tmp_path / ("no_%s.data" % missing)
        q.write_text("".join(l + "\n" for l in single.read_text().splitlines() if not l.startswith(missing)))
        with pytest.raises(_lib.SspError, match=missing):
            read_camera(str(q), SIZE_KEYS)
