"""GPU checks of the multi-object pose predictor (singleshotpose_b200/predict_multi.py) and its select kernel
(ssp_predict_multi_select)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import eval_multi_ref as EM
from oracle.darknet_ref import RefDarknet
from oracle.pnp_ref import pnp_ref
from singleshotpose_b200 import FlatSGD, synth, utils
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from singleshotpose_b200.darknet_multi import Darknet
from singleshotpose_b200.image import load_validation_batch
from singleshotpose_b200.predict_multi import OUTPUT_KEYS, MultiPosePredictor, main
from singleshotpose_b200.region_loss_multi import RegionLoss
from singleshotpose_b200.utils_multi import evaluate_multi_poses_batched, get_3D_corners

pytestmark = pytest.mark.gpu
DEV = "cuda"
K9, NC, NA, NL = 9, 13, 5, 21
KM = synth.intrinsics()
A = synth.MULTI_ANCHORS


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


def _one_row_targets(classes):
    t = torch.zeros(len(classes), 50 * NL)
    t[:, 0] = torch.tensor([float(c) for c in classes])
    t[:, 1:NL] = 0.5
    return t


def _populate_eval(model):
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.reset_running_stats(); bn.momentum = None
    model.train()
    with torch.no_grad():
        for s in (0, 10, 11):
            model(synth.images(2, seed=s))
    for bn in bns:
        bn.momentum = 0.1


@pytest.fixture(scope="module")
def pair(cfg_multi_path):
    torch.manual_seed(0)
    ref = RefDarknet(cfg_multi_path)
    _populate_eval(ref)
    ref.eval()
    dut = Darknet(cfg_multi_path)
    dut.load_state_dict(ref.state_dict())
    return ref, dut.cuda().eval()


# ---------------------------------------------------------------------------------------------------- select kernel
def _select(out, classes, thr=0.05, frame=(640.0, 480.0)):
    B, _, H, W = out.shape
    cls = np.ascontiguousarray(classes, np.int32)
    Q = len(cls)
    boxes = torch.empty(B, Q, NL, device=DEV)
    flags = torch.empty(B, Q, dtype=torch.int32, device=DEV)
    uv = torch.empty(B, Q, K9, 2, device=DEV)
    call("ssp_predict_multi_select", ptr(out), B, K9, NC, NA, H, W, C.c_void_p(cls.ctypes.data), Q, thr, frame[0], frame[1], ptr(boxes),
         ptr(flags), ptr(uv), stream_ptr())
    return boxes, flags, uv


def _eval_select(out, classes, thr=0.05, frame=(640.0, 480.0)):
    """ssp_eval_multi_select on every frame replicated once per class, with a one-row target of that class"""
    B, _, H, W = out.shape
    Q = len(classes)
    rep = out.repeat_interleave(Q, 0).contiguous()
    tgt = _one_row_targets(list(classes) * B).to(DEV).contiguous()
    off = torch.arange(B * Q + 1, dtype=torch.int32, device=DEV)
    G = B * Q
    boxes = torch.empty(G, NL, device=DEV)
    flags = torch.empty(G, dtype=torch.int32, device=DEV)
    uv = torch.empty(2 * G, K9, 2, device=DEV)
    call("ssp_eval_multi_select", ptr(rep), G, K9, NC, NA, H, W, ptr(tgt), tgt.shape[1], ptr(off), thr, frame[0], frame[1], ptr(boxes),
         ptr(flags), ptr(uv), stream_ptr())
    return boxes.view(B, Q, NL), flags.view(B, Q), uv[G:].view(B, Q, K9, 2)


@pytest.mark.parametrize("classes", [list(range(NC)), [9, 2, 5]])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [13, 21, 26])
def test_select_kernel_equals_eval_kernel(H, B, classes):
    gen = torch.Generator().manual_seed(100 * H + B)
    out = torch.randn(B, (2 * K9 + 1 + NC) * NA, H, H, generator=gen)
    shift = [-1.5, 1.0, -9.0][:B]                                   # fewer listed boxes, many, none
    for b, s in enumerate(shift):
        out[b, [18 + 32 * a for a in range(NA)]] += s
    out = out.to(DEV)
    got = _select(out, classes)
    again = _select(out, classes)
    want = _eval_select(out, classes)
    for g, a, w, name in zip(got, again, want, ("boxes", "flags", "uv")):
        assert torch.equal(g, w), name
        assert torch.equal(g, a), name
    if B == 3:
        f = got[1].cpu().numpy()
        assert (f == 0).any() and (f[2] == 1).all()                 # listed slots, and the fallback of every class


# ---------------------------------------------------------------------------------------------------- planted model
PLANTED = (2, 5, 11)                                                # anchors 0, 1, 2 detect these classes at every cell


def _pose(ang, t):
    ang = np.asarray(ang, float)
    th = np.linalg.norm(ang); kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]]) / th
    return np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx, np.asarray(t, float)


def _planted_model(cfg_multi_path):
    """a network whose last layer outputs constant logits: anchor a (0..2) is a confident detection of class PLANTED[a] whose
    keypoints at cell (0, 0) are that class's box projected under a known pose (as test_gpu_predict.py's _posed_model does);
    anchors 3 and 4 are not confident.  -> model, {class: (9, 2) planted pixels}"""
    torch.manual_seed(5)
    planted = {}
    m = Darknet(cfg_multi_path)
    last = m.models[30][0]
    b = np.zeros(160)
    b[[18 + 32 * a for a in range(NA)]] = -8.0                     # not confident
    for a, c in enumerate(PLANTED):
        R, t = _pose([0.3, -0.2 + 0.1 * a, 0.1], np.array([-0.315, -0.235, 0.6]) * (1 + 0.1 * a))   # the centroid stays in cell (0, 0)
        P = np.concatenate([np.zeros((3, 1)), OBJECTS[c]], 1)
        cam = KM @ (R @ P + t[:, None])
        uv = cam[:2] / cam[2]
        planted[c] = uv.T
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
    return m.cuda().eval(), planted


def test_planted_model(cfg_multi_path):
    m, planted = _planted_model(cfg_multi_path)
    pred = MultiPosePredictor(m, OBJECTS, KM, batch=2)
    assert pred.shape == (416, 416) and pred.conf_thresh == 0.05
    r = _clone(pred(_frames(2, seed=5)))
    assert r["classes"].cpu().tolist() == list(range(NC))
    det = r["detected"].cpu().numpy()
    assert (det[:, list(PLANTED)]).all() and det.sum() == 2 * len(PLANTED)
    boxes = pred._last.boxes
    kp = boxes[..., :18].reshape(2, NC, 9, 2) * torch.tensor([640.0, 480.0], device=DEV)
    assert torch.equal(r["keypoints_px"], kp)
    lg = pred.logits.cpu()
    K32 = KM.astype(np.float32)
    for c in range(NC):
        P3 = np.concatenate([np.zeros((1, 3)), OBJECTS[c].T]).astype(np.float32)
        X = np.concatenate([np.concatenate([np.zeros((3, 1)), OBJECTS[c]], 1), np.ones((1, 9))]).astype(np.float32)
        Rt = torch.cat([r["R"][:, c], r["t"][:, c].unsqueeze(2)], 2)
        assert torch.equal(r["corners_px"][:, c], utils.project_points_batched(X, Rt, KM).transpose(1, 2)), c
        for b in range(2):
            (x,), _ = EM.evaluate_image_multi_ref(lg[b:b + 1], _one_row_targets([c])[0].numpy(), 0.05, NC, K9, A, NA, None, None, np.eye(3),
                                                  with_pose=False)
            assert x["fallback"] == (c not in PLANTED), (b, c)
            np.testing.assert_allclose(boxes[b, c].cpu().numpy(), x["box"], rtol=1e-5, atol=1e-7)
            if c in PLANTED:
                assert x["pos"] == PLANTED.index(c) and float(boxes[b, c, 2 * K9 + 2]) == c       # entry (cell 0, anchor a)
                assert np.abs(kp[b, c].cpu().numpy() - planted[c]).max() < 1e-3
                Ro, to = pnp_ref(P3, kp[b, c].cpu().numpy(), K32)
                Rg = r["R"][b, c].cpu().numpy()
                ang = np.degrees(np.arccos(np.clip((np.trace(Rg @ Ro.T) - 1) / 2, -1, 1)))
                assert ang < 1e-2 and np.abs(r["t"][b, c].cpu().numpy() - to.reshape(3)).max() * 1e3 < 1e-2, (b, c)
    host = pred(_frames(2, seed=5), to_host=True)
    assert set(host) == set(OUTPUT_KEYS) | {"classes"}
    assert isinstance(host["R"], np.ndarray) and np.array_equal(host["R"], r["R"].cpu().numpy())


# ---------------------------------------------------------------------------------------------------- network and inputs
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("size", [416, 672])
def test_logits_match_oracle_and_model_and_head_uses_own_logits(pair, size, batch):
    ref, m = pair
    pred = MultiPosePredictor(m, OBJECTS, KM, shape=(size, size), batch=batch)
    r = _clone(pred(_frames(batch, seed=size + batch)))
    x = pred.input.clone()
    logits = pred.logits.clone()
    with torch.no_grad():
        o_ref = ref(x.cpu())
        o_model = m(x)
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
    assert rel(logits.cpu(), o_ref) < 1e-3
    assert rel(logits, o_model) < 5e-4
    # the selection is discrete and split-K changes the last bits of the logits: compare the head on the predictor's own logits
    V = np.c_[np.random.default_rng(0).normal(size=(30, 3)) * 0.03, np.ones(30)].T
    boxes = pred._last.boxes
    for c in range(NC):
        e = evaluate_multi_poses_batched(logits, _one_row_targets([c] * batch), pred.conf_thresh, NC, K9, NA, V, OBJECTS[c], KM)
        assert torch.equal(e["box"], boxes[:, c]), c
        assert torch.equal(e["fallback"], ~r["detected"][:, c]), c
        assert torch.equal(e["R_pr"], r["R"][:, c]) and torch.equal(e["t_pr"], r["t"][:, c]), c


def test_input_is_load_validation_batch(pair, tmp_path):
    _ref, m = pair
    from PIL import Image
    from singleshotpose_b200.jpeg import GpuJpegDecoder
    fr = _frames(2, seed=4, w=320, h=240)
    pred = MultiPosePredictor(m, {3: OBJECTS[3]}, KM, frame_size=(320, 240), batch=2)
    assert pred.shape == (m.width, m.height)
    want = load_validation_batch(list(fr), pred.shape, DEV)
    pred(fr)
    assert torch.equal(pred.input, want)
    pred(torch.from_numpy(fr).cuda())
    assert torch.equal(pred.input, want)
    blobs = []
    for i, a in enumerate(fr):
        p = str(tmp_path / ("%d.jpg" % i))
        Image.fromarray(a).save(p, quality=95)
        blobs.append(open(p, "rb").read())
    dec = GpuJpegDecoder(DEV)(blobs)
    pred(blobs)
    assert torch.equal(pred.input, load_validation_batch(dec, pred.shape, DEV))


# ---------------------------------------------------------------------------------------------------- graph behaviour
def test_graph_replay_equals_eager_and_repeats(pair):
    _ref, m = pair
    fr = _frames(2, seed=6)
    objs = {c: OBJECTS[c] for c in (12, 0, 6)}
    g = MultiPosePredictor(m, objs, KM, batch=2)
    e = MultiPosePredictor(m, objs, KM, batch=2, graph=False)
    r_e = _clone(e(fr))
    r1 = _clone(g(fr))
    r2 = _clone(g(fr))
    assert g._last.graph is not None
    assert _equal(r1, r_e) and _equal(r1, r2)
    assert r1["classes"].cpu().tolist() == [0, 6, 12]
    assert torch.equal(g(torch.from_numpy(fr).cuda())["R"], r_e["R"])


def test_replay_follows_load_weights_and_sgd_step(cfg_multi_path, tmp_path):
    torch.manual_seed(1)
    m = Darknet(cfg_multi_path).cuda().eval()
    fr = _frames(1, seed=7)
    pred = MultiPosePredictor(m, OBJECTS, KM)
    pred(fr)
    l0 = pred.logits.clone()
    torch.manual_seed(2)
    wf = str(tmp_path / "other.weights")
    Darknet(cfg_multi_path).save_weights(wf)
    m.load_weights(wf)
    r1 = _clone(pred(fr))
    l1 = pred.logits.clone()
    assert not torch.equal(l0, l1)
    fresh = MultiPosePredictor(m, OBJECTS, KM)
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
    fresh = MultiPosePredictor(m, OBJECTS, KM)
    assert _equal(r2, fresh(fr)) and torch.equal(l2, fresh.logits)


def test_model_call_and_training_step_between_replays_change_nothing(cfg_multi_path):
    torch.manual_seed(3)
    m = Darknet(cfg_multi_path).cuda().eval()
    fr = _frames(1, seed=8)
    pred = MultiPosePredictor(m, OBJECTS, KM)
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


def test_bad_inputs_and_arguments_raise_before_any_launch(pair, cfg_path):
    _ref, m = pair
    eng = m._engine
    pred = MultiPosePredictor(m, OBJECTS, KM, batch=2)
    n0 = eng.launches
    good = _frames(2, seed=11)
    bad = [good.astype(np.float32), good[0], good[..., :2], good[:1], torch.from_numpy(good), [b"\xff\xd8junk", b"abc"],
           [b"abc"], "frames", good[:, :0]]
    for b in bad:
        with pytest.raises(SspError):
            pred(b)
    assert pred._last is None
    from singleshotpose_b200 import Darknet as SingleDarknet
    single = SingleDarknet(cfg_path).cuda().eval()
    for args, kw in (((single, {0: OBJECTS[0]}, KM), {}),               # one anchor: not a multi-object head
                     ((m, {}, KM), {}), ((m, {13: OBJECTS[0]}, KM), {}), ((m, {-1: OBJECTS[0]}, KM), {}),
                     ((m, {0: OBJECTS[0][:, :7]}, KM), {}), ((m, [OBJECTS[0]], KM), {}),
                     ((m, OBJECTS, KM[:2]), {}),
                     ((m, OBJECTS, KM), dict(shape=(928, 928)))):          # a 29 x 29 x 5 grid: more than 4096 entries
        with pytest.raises(SspError):
            MultiPosePredictor(*args, **kw)
    assert eng.launches == n0
    blocks = m.blocks[0]
    saved = blocks.pop("conf_thresh")
    try:
        with pytest.raises(SspError, match="conf_thresh"):
            MultiPosePredictor(m, OBJECTS, KM)
        assert MultiPosePredictor(m, OBJECTS, KM, conf_thresh=0.2).conf_thresh == 0.2
    finally:
        blocks["conf_thresh"] = saved


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
    out = str(tmp_path / "poses.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_multi_path, "--weightfile", wf, "--out", out,
          "--object", "4=%s" % meshes[4][0], "--object", "0=%s" % meshes[0][0]] + paths)
    got = np.load(out)
    m = Darknet(cfg_multi_path)
    m.load_weights(wf)
    m.cuda().eval()
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    pred = MultiPosePredictor(m, {c: meshes[c][1] for c in meshes}, Km)
    assert list(got["classes"]) == [0, 4] and list(got["paths"]) == paths
    from PIL import Image
    for i, p in enumerate(paths):
        r = pred(np.asarray(Image.open(p).convert("RGB"))[None], to_host=True)
        for k in OUTPUT_KEYS:
            assert np.array_equal(got[k][i], r[k][0]), (p, k)
