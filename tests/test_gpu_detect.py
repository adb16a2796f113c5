"""GPU checks of every-instance detection: the ssp_detect_instances kernel against the numpy oracle (oracle/detect_ref.py) on the
per-entry values of ssp_region_decode_multi, ssp_pnp_batched_counted, utils_multi.detect_instances and
predict_instances.InstancePosePredictor (agreement with the one-pose predictors, planted detections, graph plumbing, the CLI)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import detect_ref as DR
from oracle.pnp_ref import pnp_ref
from singleshotpose_b200 import FlatSGD, synth, utils
from singleshotpose_b200 import Darknet as SingleDarknet
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from singleshotpose_b200.darknet_multi import Darknet
from singleshotpose_b200.predict import PosePredictor
from singleshotpose_b200.predict_instances import OUTPUT_KEYS, ROW_KEYS, InstancePosePredictor, main
from singleshotpose_b200.predict_multi import MultiPosePredictor
from singleshotpose_b200.region_loss_multi import RegionLoss
from singleshotpose_b200.utils_multi import detect_instances, get_3D_corners, multi_region_dense

pytestmark = pytest.mark.gpu
DEV = "cuda"
K9, NC, NA, NL = 9, 13, 5, 21
KM = synth.intrinsics()
A = synth.MULTI_ANCHORS
F32 = np.float32


def _corners(c):
    """a distinct (3, 8) box per class, in get_3D_corners order"""
    s = 1.0 + 0.1 * c
    return synth.box_points((0.038 * s, 0.039 * s, 0.046 * (2.0 - 0.05 * c)), with_center=False).T.astype(np.float64)


OBJECTS = {c: _corners(c) for c in range(NC)}


def _frames(n, seed, w=640, h=480):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _clone(r):
    return {k: v.clone() for k, v in r.items()}


def _equal(a, b):
    return all(torch.equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------- kernel against the oracle
def _detect(out, nC, nA, classes, thr, nms, M, frame=(640.0, 480.0)):
    B, _, H, W = out.shape
    cls = np.ascontiguousarray(classes, np.int32)
    boxes = torch.full((B, M, NL), float("nan"), device=DEV)
    kcls = torch.full((B, M), 7, dtype=torch.int32, device=DEV)
    uv = torch.full((B, M, K9, 2), float("nan"), device=DEV)
    count = torch.full((B,), -5, dtype=torch.int32, device=DEV)
    kept = torch.full((B,), -5, dtype=torch.int32, device=DEV)
    call("ssp_detect_instances", ptr(out), B, K9, nC, nA, H, W, C.c_void_p(cls.ctypes.data), len(cls), thr, nms, M, frame[0], frame[1],
         ptr(boxes), ptr(kcls), ptr(uv), ptr(count), ptr(kept), stream_ptr())
    return dict(boxes=boxes, cls=kcls, uv=uv, count=count, kept=kept)


def _oracle(out, nC, nA, classes, thr, nms, M, frame=(640.0, 480.0)):
    """the oracle's NMS on the per-entry values of ssp_region_decode_multi (decode_entry on the device) -> the kernel's outputs"""
    B = out.shape[0]
    dense = multi_region_dense(out, nC, K9, nA, -1, only_objectness=0)["boxes"].cpu().numpy()      # (B, n, 21)
    boxes = np.zeros((B, M, NL), F32)
    cls = np.full((B, M), -1, np.int32)
    uv = np.zeros((B, M, K9, 2), F32)
    count = np.zeros(B, np.int32)
    kept = np.zeros(B, np.int32)
    for b in range(B):
        d = dense[b]
        px = d[:, :2 * K9].reshape(-1, K9, 2) * np.array(frame, F32)
        entries, kept[b] = DR.detect_ref(d[:, 2 * K9], d[:, 2 * K9 + 1], d[:, 2 * K9 + 2].astype(np.int64), px, thr, nms, classes, M)
        count[b] = len(entries)
        for m, e in enumerate(entries):
            boxes[b, m], cls[b, m], uv[b, m] = d[e], int(d[e, 2 * K9 + 2]), px[e]
    return dict(boxes=boxes, cls=cls, uv=uv, count=count, kept=kept)


def _logits(B, H, nC, nA, shifts, seed):
    gen = torch.Generator().manual_seed(seed)
    out = torch.randn(B, (2 * K9 + 1 + nC) * nA, H, H, generator=gen)
    for b, s in enumerate(shifts):
        out[b, [2 * K9 + (2 * K9 + 1 + nC) * a for a in range(nA)]] += s
    return out.to(DEV)


HEADS = {"multi": (NC, NA, 0.05, (-2.5, 2.0, -12.0)), "single": (1, 1, 0.1, (-3.5, 1.0, -12.0))}   # few, thousands (or all), none


@pytest.mark.parametrize("head", sorted(HEADS))
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [13, 21, 26])
def test_kernel_equals_oracle_bit_for_bit(H, B, head):
    nC, nA, thr, shifts = HEADS[head]
    shifts = shifts[1:2] if B == 1 else shifts
    out = _logits(B, H, nC, nA, shifts, seed=10 * H + B)
    classes = list(range(nC))
    for cls_req, nms, M in ((classes, 0.4, 64), (classes[::3], 0.0, 256), (classes, 1.0, 8)):
        got = _detect(out, nC, nA, cls_req, thr, nms, M)
        want = _oracle(out, nC, nA, cls_req, thr, nms, M)
        for k in want:
            assert np.array_equal(got[k].cpu().numpy(), want[k]), (k, cls_req, nms, M)
        again = _detect(out, nC, nA, cls_req, thr, nms, M)
        assert _equal(got, again)
        for b in range(B):                                            # a frame alone gives what it gives inside the batch
            alone = _detect(out[b:b + 1].contiguous(), nC, nA, cls_req, thr, nms, M)
            assert all(torch.equal(alone[k][0], got[k][b]) for k in got)
    cnt = _detect(out, nC, nA, classes, thr, 0.4, 256)
    if B == 3:
        assert cnt["count"][2] == 0 and 0 < cnt["kept"][0] < cnt["kept"][1]
        assert (cnt["cls"][2] == -1).all() and not cnt["boxes"][2].any()


def test_pnp_counted_solves_only_the_counted_slots():
    pr = synth.pnp_problems(12, sigma=0.5, seed=3)
    P3 = torch.as_tensor(np.repeat(np.asarray(pr["P3"], F32)[None], 12, 0)).to(DEV).contiguous()
    uv = torch.as_tensor(np.asarray(pr["uv"], F32)).to(DEV).contiguous()
    Kc = torch.as_tensor(np.asarray(pr["K"], F32)).to(DEV)
    count = torch.tensor([4, 0, 2], dtype=torch.int32, device=DEV)
    R = torch.full((12, 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    t = torch.full((12, 3), float("nan"), dtype=torch.float64, device=DEV)
    call("ssp_pnp_batched_counted", ptr(P3), ptr(uv), ptr(Kc), 9, 3, 4, ptr(count), 20, ptr(R), ptr(t), stream_ptr())
    Rw, tw = utils.pnp_batched(P3[0], uv, Kc)                          # the same solve, every problem
    run = [g * 4 + m for g, c in enumerate((4, 0, 2)) for m in range(c)]
    skip = [i for i in range(12) if i not in run]
    assert torch.equal(R[run], Rw[run]) and torch.equal(t[run], tw[run])
    assert not R[skip].any() and not t[skip].any()


# ---------------------------------------------------------------------------------------------------- planted detections
def _pose(ang, t):
    ang = np.asarray(ang, float)
    th = np.linalg.norm(ang); kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]]) / th
    return np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx, np.asarray(t, float)


def _project(c, R, t):
    P = np.concatenate([np.zeros((3, 1)), OBJECTS[c]], 1)
    cam = KM @ (R @ P + t[:, None])
    return (cam[:2] / cam[2]).T                                           # (9, 2) pixels


def _plant(o, b, a, c, uv, H, objectness=4.0):
    """write entry (cell of uv's centroid, anchor a) of image b as a detection of class c with pixel keypoints uv"""
    gx, gy = uv[:, 0] / 640 * H, uv[:, 1] / 480 * H
    cx, cy = int(gx[0]), int(gy[0])
    base = a * (2 * K9 + 1 + NC)
    fx, fy = gx[0] - cx, gy[0] - cy
    o[b, base, cy, cx], o[b, base + 1, cy, cx] = np.log(fx / (1 - fx)), np.log(fy / (1 - fy))
    o[b, base + 2:base + 18:2, cy, cx] = torch.from_numpy(gx[1:] - cx).float()
    o[b, base + 3:base + 18:2, cy, cx] = torch.from_numpy(gy[1:] - cy).float()
    o[b, base + 18, cy, cx] = objectness
    o[b, base + 19 + c, cy, cx] = 8.0
    return cy * H + cx


def test_two_planted_instances_are_recovered_and_a_duplicate_is_suppressed():
    H, c = 13, 6
    o = torch.zeros(1, NA * (2 * K9 + 1 + NC), H, H)
    o[:, [18 + 32 * a for a in range(NA)]] = -10.0
    poses = [_pose([0.3, -0.2, 0.1], [-0.12, -0.05, 0.7]), _pose([-0.2, 0.4, 0.3], [0.1, 0.06, 0.8])]
    truth = [_project(c, R, t) for R, t in poses]
    _plant(o, 0, 0, c, truth[0], H, objectness=5.0)
    _plant(o, 0, 1, c, truth[1], H, objectness=4.0)
    _plant(o, 0, 2, c, truth[1] + 2.0, H, objectness=3.0)                # near-duplicate of the second, lower score
    out = o.to(DEV)
    r = detect_instances(out, 0.05, 0.4, NC, K9, NA, (640, 480), classes=[c, 3])
    assert int(r["count"][0]) == 2 and int(r["kept"][0]) == 2
    assert r["cls"][0, :2].tolist() == [c, c] and (r["cls"][0, 2:] == -1).all()
    kp = r["keypoints_px"][0, :2].cpu().numpy()
    P3 = np.concatenate([np.zeros((1, 3)), OBJECTS[c].T]).astype(F32)
    for m in range(2):
        assert np.abs(kp[m] - truth[m]).max() < 1e-3, m
        Ro, to = pnp_ref(P3, kp[m], KM.astype(F32))
        ang = np.degrees(np.arccos(np.clip((np.trace(poses[m][0] @ Ro.T) - 1) / 2, -1, 1)))
        assert ang < 1e-2 and np.abs(to.reshape(3) - poses[m][1]).max() * 1e3 < 1e-1, m
    P3d = torch.from_numpy(np.repeat(P3[None], 32, 0)).to(DEV)
    R = torch.empty(32, 3, 3, dtype=torch.float64, device=DEV)
    t = torch.empty(32, 3, dtype=torch.float64, device=DEV)
    call("ssp_pnp_batched_counted", ptr(P3d), ptr(r["keypoints_px"]), ptr(torch.from_numpy(KM.astype(F32)).to(DEV)), 9, 1, 32, ptr(r["count"]),
         20, ptr(R), ptr(t), stream_ptr())
    for m in range(2):
        ang = np.degrees(np.arccos(np.clip((np.trace(R[m].cpu().numpy() @ poses[m][0].T) - 1) / 2, -1, 1)))
        assert ang < 1e-2 and np.abs(t[m].cpu().numpy() - poses[m][1]).max() * 1e3 < 1e-1, m
    r3 = detect_instances(out, 0.05, 1.0, NC, K9, NA, (640, 480), classes=[c])
    assert int(r3["count"][0]) == 3                                       # no suppression: the duplicate is the third
    r1 = detect_instances(out, 0.05, 0.4, NC, K9, NA, (640, 480), classes=[c], max_instances=1)
    assert int(r1["count"][0]) == 1 and int(r1["kept"][0]) == 2 and torch.equal(r1["keypoints_px"][0, 0], r["keypoints_px"][0, 0])


PLANTED = (2, 5, 11)                                                # anchors 0, 1, 2 detect these classes at every cell


def _planted_model(cfg_multi_path):
    """a network whose last layer outputs constant logits (test_gpu_predict_multi.py's construction): anchor a (0..2) is a confident
    detection of class PLANTED[a] whose keypoints at cell (0, 0) are that class's box projected under a known pose; every other
    cell lists the same box shifted by one cell.  -> model, {class: (9, 2) planted pixels}, {class: (R, t)}"""
    torch.manual_seed(5)
    planted, poses = {}, {}
    m = Darknet(cfg_multi_path)
    last = m.models[30][0]
    b = np.zeros(160)
    b[[18 + 32 * a for a in range(NA)]] = -8.0
    for a, c in enumerate(PLANTED):
        R, t = _pose([0.3, -0.2 + 0.1 * a, 0.1], np.array([-0.315, -0.235, 0.6]) * (1 + 0.1 * a))
        uv = _project(c, R, t).T
        planted[c], poses[c] = uv.T, (R, t)
        gx, gy = uv[0] / 640 * 13, uv[1] / 480 * 13
        assert 0 < gx[0] < 1 and 0 < gy[0] < 1
        o = 32 * a
        b[o], b[o + 1] = np.log(gx[0] / (1 - gx[0])), np.log(gy[0] / (1 - gy[0]))
        b[o + 2:o + 18:2], b[o + 3:o + 18:2] = gx[1:], gy[1:]
        b[o + 18] = 4.0
        b[o + 19 + c] = 8.0
    with torch.no_grad():
        last.weight.zero_()
        last.bias.copy_(torch.from_numpy(b).float())
    return m.cuda().eval(), planted, poses


def test_planted_lattice(cfg_multi_path):
    m, planted, poses = _planted_model(cfg_multi_path)
    pred = InstancePosePredictor(m, OBJECTS, KM, batch=2, max_instances=256)
    assert pred.shape == (416, 416) and pred.conf_thresh == 0.05 and pred.nms_thresh == 0.4
    r = _clone(pred(_frames(2, seed=5)))
    want = _oracle(pred.logits, NC, NA, list(range(NC)), 0.05, 0.4, 256)
    assert np.array_equal(r["count"].cpu().numpy(), want["count"]) and np.array_equal(r["kept"].cpu().numpy(), want["kept"])
    assert np.array_equal(r["cls"].cpu().numpy(), want["cls"]) and np.array_equal(r["keypoints_px"].cpu().numpy(), want["uv"])
    assert set(np.unique(want["cls"][want["cls"] >= 0])) == set(PLANTED) and want["kept"][0] > len(PLANTED)
    K32 = KM.astype(F32)
    for b in range(2):
        for a, c in enumerate(PLANTED):
            m0 = int(np.nonzero(want["cls"][b] == c)[0][0])             # instance 0 of class c: the entry (cell 0, anchor a)
            assert m0 == a
            kp = r["keypoints_px"][b, m0].cpu().numpy()
            assert np.abs(kp - planted[c]).max() < 1e-3
            P3 = np.concatenate([np.zeros((1, 3)), OBJECTS[c].T]).astype(F32)
            Ro, to = pnp_ref(P3, kp, K32)
            ang = np.degrees(np.arccos(np.clip((np.trace(r["R"][b, m0].cpu().numpy() @ Ro.T) - 1) / 2, -1, 1)))
            assert ang < 1e-2 and np.abs(r["t"][b, m0].cpu().numpy() - to.reshape(3)).max() * 1e3 < 1e-2, (b, c)
            X = np.concatenate([np.concatenate([np.zeros((3, 1)), OBJECTS[c]], 1), np.ones((1, 9))]).astype(F32)
            Rt = torch.cat([r["R"][b, m0], r["t"][b, m0].unsqueeze(1)], 1)[None]
            assert torch.equal(r["corners_px"][b, m0], utils.project_points_batched(X, Rt, KM)[0].transpose(0, 1))


# ---------------------------------------------------------------------------------------------------- agreement with the predictors
@pytest.fixture(scope="module")
def multi_model(cfg_multi_path):
    torch.manual_seed(0)
    return Darknet(cfg_multi_path).cuda().eval()


def test_instance_zero_is_the_multi_predictor_slot(multi_model):
    fr = _frames(2, seed=21)
    mp = MultiPosePredictor(multi_model, OBJECTS, KM, batch=2, conf_thresh=0.02)
    ip = InstancePosePredictor(multi_model, OBJECTS, KM, batch=2, conf_thresh=0.02, max_instances=256)
    rm, ri = _clone(mp(fr)), _clone(ip(fr))
    assert torch.equal(mp.logits, ip.logits)
    det = rm["detected"].cpu().numpy()
    cls = ri["cls"].cpu().numpy()
    checked = 0
    for b in range(2):
        for c in range(NC):
            if not det[b, c]:
                assert not (cls[b] == c).any()
                continue
            hit = np.nonzero(cls[b] == c)[0]
            if len(hit) == 0:                                         # the class's best box ranks past the 256 slots
                assert int(ri["kept"][b]) > int(ri["count"][b]) == 256
                continue
            m0 = int(hit[0])
            assert torch.equal(ip._last.boxes[b, m0], mp._last.boxes[b, c]), (b, c)
            for k in ("keypoints_px", "R", "t", "corners_px", "conf", "cls_conf"):
                assert torch.equal(ri[k][b, m0], rm[k][b, c]), (b, c, k)
            checked += 1
    assert checked >= 4


def test_single_object_instance_zero_is_the_pose_predictor(cfg_path):
    torch.manual_seed(1)
    m = SingleDarknet(cfg_path).cuda().eval()
    corners = OBJECTS[0]
    fr = _frames(2, seed=22)
    pp = PosePredictor(m, corners, KM, batch=2)
    ip = InstancePosePredictor(m, corners, KM, batch=2)
    assert ip.shape == pp.shape == (m.test_width, m.test_height) and ip.conf_thresh == 0.1
    rp, ri = _clone(pp(fr)), _clone(ip(fr))
    assert torch.equal(pp.logits, ip.logits)
    checked = 0
    for b in range(2):
        if not float(rp["conf"][b]) > 0.1:
            continue
        assert int(ri["count"][b]) >= 1 and int(ri["cls"][b, 0]) == 0
        for k in ("keypoints_px", "R", "t", "corners_px", "conf"):
            assert torch.equal(ri[k][b, 0], rp[k][b]), (b, k)
        checked += 1
    assert checked >= 1


# ---------------------------------------------------------------------------------------------------- the predictor's plumbing
def test_graph_replay_equals_eager_repeats_and_empty_slots_are_zero(multi_model):
    fr = _frames(2, seed=6)
    objs = {c: OBJECTS[c] for c in (12, 0, 6)}
    g = InstancePosePredictor(multi_model, objs, KM, batch=2, conf_thresh=0.02, max_instances=16)
    e = InstancePosePredictor(multi_model, objs, KM, batch=2, conf_thresh=0.02, max_instances=16, graph=False)
    r_e = _clone(e(fr))
    r1 = _clone(g(fr))
    r2 = _clone(g(fr))
    assert g._last.graph is not None
    assert _equal(r1, r_e) and _equal(r1, r2)
    assert torch.equal(g(torch.from_numpy(fr).cuda())["R"], r_e["R"])
    assert set(r1["cls"][r1["cls"] >= 0].cpu().tolist()) <= {0, 6, 12}
    for b in range(2):
        n = int(r1["count"][b])
        assert n == min(int(r1["kept"][b]), 16)
        assert (r1["cls"][b, n:] == -1).all() and (r1["cls"][b, :n] >= 0).all()
        for k in ("R", "t", "conf", "cls_conf", "keypoints_px", "corners_px"):
            assert not r1[k][b, n:].any(), k
            assert torch.isfinite(r1[k][b]).all(), k
    sparse = InstancePosePredictor(multi_model, objs, KM, batch=2, conf_thresh=0.9)
    rs = sparse(fr)
    assert (rs["count"] == 0).all() and (rs["cls"] == -1).all() and not rs["corners_px"].any() and not rs["R"].any()


def test_replay_follows_load_weights_and_sgd_step(cfg_multi_path, tmp_path):
    torch.manual_seed(1)
    m = Darknet(cfg_multi_path).cuda().eval()
    fr = _frames(1, seed=7)
    pred = InstancePosePredictor(m, OBJECTS, KM, conf_thresh=0.02)
    pred(fr)
    l0 = pred.logits.clone()
    torch.manual_seed(2)
    wf = str(tmp_path / "other.weights")
    Darknet(cfg_multi_path).save_weights(wf)
    m.load_weights(wf)
    r1 = _clone(pred(fr))
    l1 = pred.logits.clone()
    assert not torch.equal(l0, l1)
    fresh = InstancePosePredictor(m, OBJECTS, KM, conf_thresh=0.02)
    assert _equal(r1, fresh(fr)) and torch.equal(l1, fresh.logits)
    m.train()
    opt = FlatSGD(m, lr=1e-3, momentum=0.9, weight_decay=5e-4)
    crit = RegionLoss(anchors=A); crit.verbose = False
    loss = crit(m(synth.images(2, seed=1).cuda()), synth.targets_multi(2, seed=1), 20)
    opt.zero_grad(); loss.backward(); opt.step()
    m.eval()
    r2 = _clone(pred(fr))
    l2 = pred.logits.clone()
    assert not torch.equal(l1, l2)
    fresh = InstancePosePredictor(m, OBJECTS, KM, conf_thresh=0.02)
    assert _equal(r2, fresh(fr)) and torch.equal(l2, fresh.logits)


def test_model_call_and_training_step_between_replays_change_nothing(cfg_multi_path):
    torch.manual_seed(3)
    m = Darknet(cfg_multi_path).cuda().eval()
    fr = _frames(1, seed=8)
    pred = InstancePosePredictor(m, OBJECTS, KM, conf_thresh=0.02)
    r1 = _clone(pred(fr))
    l1 = pred.logits.clone()
    state = copy.deepcopy(m.state_dict())
    with torch.no_grad():
        m(synth.images(1, seed=9).cuda())
    for bn in (x for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d)):
        bn.momentum = 0.0
    m.train()
    opt = FlatSGD(m, lr=0.0, momentum=0.0, weight_decay=0.0)
    crit = RegionLoss(anchors=A); crit.verbose = False
    loss = crit(m(synth.images(1, seed=10).cuda()), synth.targets_multi(1, seed=2), 20)
    opt.zero_grad(); loss.backward(); opt.step()
    m.eval()
    assert all(torch.equal(a, b) for a, b in zip(state.values(), m.state_dict().values()))
    r2 = pred(fr)
    assert _equal(r1, r2) and torch.equal(l1, pred.logits)


def test_bad_inputs_and_arguments_raise_before_any_launch(multi_model):
    m = multi_model
    eng = m._engine
    pred = InstancePosePredictor(m, OBJECTS, KM, batch=2)
    n0 = eng.launches
    good = _frames(2, seed=11)
    for b in [good.astype(np.float32), good[0], good[..., :2], good[:1], torch.from_numpy(good), [b"\xff\xd8junk", b"abc"], "frames"]:
        with pytest.raises(SspError):
            pred(b)
    assert pred._last is None
    for args, kw in (((m, {}, KM), {}), ((m, {13: OBJECTS[0]}, KM), {}), ((m, {-1: OBJECTS[0]}, KM), {}),
                     ((m, {0: OBJECTS[0][:, :7]}, KM), {}), ((m, OBJECTS, KM[:2]), {}),
                     ((m, OBJECTS, KM), dict(nms_thresh=-0.1)), ((m, OBJECTS, KM), dict(nms_thresh=1.5)),
                     ((m, OBJECTS, KM), dict(nms_thresh=float("nan"))),
                     ((m, OBJECTS, KM), dict(max_instances=0)), ((m, OBJECTS, KM), dict(max_instances=257)),
                     ((m, OBJECTS, KM), dict(max_instances=2.5)), ((m, OBJECTS, KM), dict(max_instances=True)),
                     ((m, OBJECTS, KM), dict(shape=(928, 928)))):          # a 29 x 29 x 5 grid: more than 4096 entries
        with pytest.raises(SspError):
            InstancePosePredictor(*args, **kw)
    assert eng.launches == n0
    with pytest.raises(SspError):
        detect_instances(torch.zeros(1, 160, 13, 13), 0.05, 0.4, NC, K9, NA, (640, 480))                    # CPU tensor
    with pytest.raises(SspError):
        detect_instances(torch.zeros(1, 150, 13, 13, device=DEV), 0.05, 0.4, NC, K9, NA, (640, 480))        # channels
    with pytest.raises(SspError):
        detect_instances(torch.zeros(1, 160, 13, 13, device=DEV), 0.05, 0.4, NC, K9, NA, (640, 480), classes=[13])


def test_cli_writes_what_the_api_returns(cfg_multi_path, tmp_path):
    import glob
    import os
    root = str(tmp_path)
    synth.write_linemod_multi_like(root, n=2)
    paths = sorted(glob.glob(os.path.join(root, "LINEMOD", "*", "JPEGImages", "*.png")))[:3]
    assert len(paths) == 3
    meshes = {}
    for c in (0, 4):
        V = np.random.default_rng(c).normal(size=(40, 3)) * 0.03
        ply = str(tmp_path / ("obj%d.ply" % c))
        with open(ply, "w") as f:
            f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n" % len(V))
            for v in V:
                f.write("%.17g %.17g %.17g\n" % tuple(v))
        meshes[c] = (ply, get_3D_corners(np.c_[V, np.ones((len(V), 1))].T))
    data = tmp_path / "occlusion.data"
    data.write_text("mesh1 = ignored.ply\nim_width = 640\nim_height = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    torch.manual_seed(4)
    wf = str(tmp_path / "m.weights")
    Darknet(cfg_multi_path).save_weights(wf)
    out = str(tmp_path / "det.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_multi_path, "--weightfile", wf, "--out", out, "--nms-thresh", "0.3",
          "--max-instances", "8", "--object", "4=%s" % meshes[4][0], "--object", "0=%s" % meshes[0][0]] + paths)
    got = np.load(out)
    m = Darknet(cfg_multi_path)
    m.load_weights(wf)
    m.cuda().eval()
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    pred = InstancePosePredictor(m, {c: meshes[c][1] for c in meshes}, Km, nms_thresh=0.3, max_instances=8)
    assert list(got["paths"]) == paths
    from PIL import Image
    rows = {k: [] for k in ROW_KEYS}
    image = []
    for i, p in enumerate(paths):
        r = pred(np.asarray(Image.open(p).convert("RGB"))[None], to_host=True)
        assert set(r) == set(OUTPUT_KEYS)
        n = int(r["count"][0])
        image += [i] * n
        for k in rows:
            rows[k].append(r[k][0, :n])
    assert np.array_equal(got["image"], np.array(image, np.int64))
    for k in ROW_KEYS:
        assert np.array_equal(got[k], np.concatenate(rows[k])), k
