"""GPU checks of tracking across frames: ssp_track_associate / ssp_track_commit against the host harness
(tests/helpers/track_host.cpp) on ssp_detect_instances outputs, ssp_pnp_batched_guess against cv2 (tests/golden/pnp_guess.npz) and
ssp_pnp_batched_counted, utils_multi.InstanceTracker on planted moving objects, and predict_instances.TrackingPosePredictor
(agreement with InstancePosePredictor, graph and state plumbing, argument checks, the CLI)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle.track_ref import pnp_guess_ref
from singleshotpose_b200 import synth
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from singleshotpose_b200.darknet_multi import Darknet
from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor, main
from singleshotpose_b200.utils_multi import InstanceTracker, detect_instances, get_3D_corners

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K9, NC, NA = 9, 13, 5
KM = synth.intrinsics()
F32 = np.float32


def _corners(c):
    s = 1.0 + 0.1 * c
    return synth.box_points((0.038 * s, 0.039 * s, 0.046 * (2.0 - 0.05 * c)), with_center=False).T.astype(np.float64)


OBJECTS = {c: _corners(c) for c in range(NC)}


def _p(a):
    return C.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("trackhost") / "libtrackhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "track_host.cpp")])
    return C.CDLL(so)


def _ang(a, b):
    return np.degrees(np.arccos(np.clip((np.trace(a @ b.T) - 1) / 2, -1, 1)))


# ---------------------------------------------------------------------------------------------------- kernels against the harness
HEADS = {"multi": (NC, NA, 0.05), "single": (1, 1, 0.1)}


@pytest.mark.parametrize("head", sorted(HEADS))
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [13, 21, 26])
def test_kernels_equal_harness_bit_for_bit(host, H, B, head):
    nC, nA, thr = HEADS[head]
    T, M = (64, 256) if H != 21 else (8, 32)                          # 21: a small table that fills up
    gen = torch.Generator().manual_seed(100 * H + B)
    base = torch.randn(B, (2 * K9 + 1 + nC) * nA, H, H, generator=gen)
    obj = [2 * K9 + (2 * K9 + 1 + nC) * a for a in range(nA)]
    d_state = [torch.zeros(B, T, 5, dtype=torch.int32, device=DEV), torch.zeros(B, T, 4, device=DEV),
               torch.zeros(B, T, 6, dtype=torch.float64, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)]
    h_state = [np.zeros((B, T, 5), np.int32), np.zeros((B, T, 4), F32), np.zeros((B, T, 6)), np.zeros(B, np.int32)]
    slot = torch.empty(B, M, dtype=torch.int32, device=DEV); tid = torch.empty_like(slot); use = torch.empty_like(slot)
    guess = torch.empty(B, M, 6, dtype=torch.float64, device=DEV)
    rng = np.random.default_rng(H * B)
    seen = dict(warm=0, born=0, empty=0, many=0)
    for f in range(24):
        o = base + 0.05 * torch.randn(base.shape, generator=gen)      # a slowly changing scene: detections persist
        shift = (2.0, -1.5, -12.0)[(f // 4) % 3] if B == 1 else 0.0
        o[:, obj] += shift
        if B == 3:
            o[1, obj] += 2.0; o[2, obj] -= 12.0 if f % 5 == 4 else 1.5
        out = o.to(DEV)
        d = detect_instances(out, thr, 0.4, nC, K9, nA, (640, 480), max_instances=M)
        count, cls, uv = d["count"], d["cls"], d["keypoints_px"]
        call("ssp_track_associate", B, T, M, ptr(count), ptr(cls), ptr(uv), 0.3, 2, ptr(d_state[0]), ptr(d_state[1]), ptr(d_state[2]),
             ptr(d_state[3]), ptr(slot), ptr(tid), ptr(guess), ptr(use), stream_ptr())
        hc, hcls, huv = count.cpu().numpy(), cls.cpu().numpy(), np.ascontiguousarray(uv.cpu().numpy())
        h_slot = np.zeros((B, M), np.int32); h_tid = np.zeros((B, M), np.int32); h_use = np.zeros((B, M), np.int32)
        h_guess = np.zeros((B, M, 6))
        assert host.h_track_associate(B, T, M, _p(hc), _p(hcls), _p(huv), C.c_float(0.3), 2, _p(h_state[0]), _p(h_state[1]), _p(h_state[2]),
                                      _p(h_state[3]), _p(h_slot), _p(h_tid), _p(h_guess), _p(h_use)) == 0
        for got, want in ((slot, h_slot), (tid, h_tid), (use, h_use), (guess, h_guess)):
            assert np.array_equal(got.cpu().numpy(), want), f
        params = np.ascontiguousarray(np.where(h_use[..., None] != 0, h_guess + 1e-3, rng.normal(size=(B, M, 6))))
        dp = torch.from_numpy(params).to(DEV)
        call("ssp_track_commit", B, T, M, ptr(count), ptr(uv), ptr(slot), ptr(dp), ptr(d_state[0]), ptr(d_state[1]), ptr(d_state[2]),
             stream_ptr())
        assert host.h_track_commit(B, T, M, _p(hc), _p(huv), _p(h_slot), _p(params), _p(h_state[0]), _p(h_state[1]), _p(h_state[2])) == 0
        for got, want in zip(d_state, h_state):
            assert got.cpu().numpy().tobytes() == want.tobytes(), f
        seen["warm"] += int(h_use.sum()); seen["empty"] += int((hc == 0).sum()); seen["many"] += int((hc >= min(100, M)).sum())
    seen["born"] = int(h_state[3].sum())
    assert seen["warm"] > 0 and seen["born"] > 0 and seen["empty"] > 0, seen
    if head == "multi":
        assert seen["many"] > 0, seen


# ---------------------------------------------------------------------------------------------------- warm PnP kernel
def _pnp_guess(P3, uv, K, guess, use, groups, per, count):
    n = groups * per
    R = torch.full((n, 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    t = torch.full((n, 3), float("nan"), dtype=torch.float64, device=DEV)
    params = torch.full((n, 6), float("nan"), dtype=torch.float64, device=DEV)
    work = torch.full((n, 3), -99, dtype=torch.int32, device=DEV)
    call("ssp_pnp_batched_guess", ptr(P3), ptr(uv), ptr(K), uv.shape[1], groups, per, ptr(count), ptr(guess), ptr(use), 20, ptr(R), ptr(t),
         ptr(params), ptr(work), stream_ptr())
    return R, t, params, work


@pytest.mark.parametrize("npts", [9, 8])
def test_warm_pnp_kernel_meets_the_cv2_golden(golden_dir, npts):
    g = np.load(os.path.join(golden_dir, "pnp_guess.npz"))
    Kd = torch.from_numpy(g["K"]).to(DEV)
    for sigma in (0, 1, 5, 20, 80):
        tag = "p%d_s%d" % (npts, sigma)
        uv = torch.from_numpy(g["uv_" + tag]).to(DEV).contiguous()
        n = uv.shape[0]
        P3 = torch.from_numpy(np.repeat(g["P3_%d" % npts][None], n, 0)).to(DEV).contiguous()
        guess = torch.from_numpy(g["guess_" + tag]).to(DEV).contiguous()
        count = torch.tensor([n], dtype=torch.int32, device=DEV)
        R, t, params, work = _pnp_guess(P3, uv, Kd, guess, torch.ones(n, dtype=torch.int32, device=DEV), 1, n, count)
        R, t, params = R.cpu().numpy(), t.cpu().numpy(), params.cpu().numpy()
        ang = np.array([_ang(R[i], g["R_" + tag][i]) for i in range(n)])
        assert ang.max() < 1e-2 and np.abs(t - g["tvec_" + tag]).max() * 1e3 < 1e-2, (tag, ang.max())
        assert np.degrees(np.abs(params[:, :3] - g["rvec_" + tag])).max() < 1e-2 and np.array_equal(params[:, 3:], t)
        assert (work[:, 0] == 0).all()


def test_cold_slots_are_bit_identical_to_the_counted_solve(golden_dir):
    g = np.load(os.path.join(golden_dir, "pnp_guess.npz"))
    uv = torch.from_numpy(g["uv_p9_s5"][:48]).to(DEV).contiguous()
    P3 = torch.from_numpy(np.repeat(g["P3_9"][None], 48, 0)).to(DEV).contiguous()
    Kd = torch.from_numpy(g["K"]).to(DEV)
    guess = torch.from_numpy(g["guess_p9_s5"][:48]).to(DEV).contiguous()
    count = torch.tensor([16, 0, 9], dtype=torch.int32, device=DEV)
    R0 = torch.empty(48, 3, 3, dtype=torch.float64, device=DEV); t0 = torch.empty(48, 3, dtype=torch.float64, device=DEV)
    call("ssp_pnp_batched_counted", ptr(P3), ptr(uv), ptr(Kd), 9, 3, 16, ptr(count), 20, ptr(R0), ptr(t0), stream_ptr())
    R, t, params, work = _pnp_guess(P3, uv, Kd, guess, torch.zeros(48, dtype=torch.int32, device=DEV), 3, 16, count)
    assert torch.equal(R, R0) and torch.equal(t, t0) and torch.equal(params[:, 3:], t)
    run = [gi * 16 + m for gi, c in enumerate((16, 0, 9)) for m in range(c)]
    skip = [i for i in range(48) if i not in run]
    assert not params[skip].any() and not work[skip].any() and (work[run, 0] != 0).all()
    use = (torch.arange(48, device=DEV) % 2).int()
    Rm, tm, _pm, wm = _pnp_guess(P3, uv, Kd, guess, use, 3, 16, count)
    cold = [i for i in run if i % 2 == 0]
    assert torch.equal(Rm[cold], R0[cold]) and torch.equal(tm[cold], t0[cold])
    assert (wm[[i for i in run if i % 2], 0] == 0).all()


# ---------------------------------------------------------------------------------------------------- planted moving objects
def _pose(ang, t):
    ang = np.asarray(ang, float)
    th = np.linalg.norm(ang); kx = np.array([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]]) / th
    return np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx, np.asarray(t, float)


def _project(c, R, t):
    P = np.concatenate([np.zeros((3, 1)), OBJECTS[c]], 1)
    cam = KM @ (R @ P + t[:, None])
    return (cam[:2] / cam[2]).T


def _plant(o, b, a, c, uv, H, objectness=4.0):
    gx, gy = uv[:, 0] / 640 * H, uv[:, 1] / 480 * H
    cx, cy = int(gx[0]), int(gy[0])
    base = a * (2 * K9 + 1 + NC)
    fx, fy = gx[0] - cx, gy[0] - cy
    o[b, base, cy, cx], o[b, base + 1, cy, cx] = np.log(fx / (1 - fx)), np.log(fy / (1 - fy))
    o[b, base + 2:base + 18:2, cy, cx] = torch.from_numpy(gx[1:] - cx).float()
    o[b, base + 3:base + 18:2, cy, cx] = torch.from_numpy(gy[1:] - cy).float()
    o[b, base + 18, cy, cx] = objectness
    o[b, base + 19 + c, cy, cx] = 8.0


def _scene(objs, H=13):
    """logits of one frame: objs = [(anchor, class, R, t, objectness)]"""
    o = torch.zeros(1, NA * (2 * K9 + 1 + NC), H, H)
    o[:, [18 + 32 * a for a in range(NA)]] = -10.0
    for a, c, R, t, s in objs:
        _plant(o, 0, a, c, _project(c, R, t), H, s)
    return o.to(DEV)


def test_planted_moving_objects_keep_their_ids():
    tr = InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), max_tracks=8, max_misses=2)
    P3 = {c: np.concatenate([np.zeros((1, 3)), OBJECTS[c].T]).astype(F32) for c in OBJECTS}

    def frame(objs):
        r = tr.update(_scene(objs))
        n = int(r["count"][0])
        return {int(r["cls"][0, m]): (int(r["track_id"][0, m]), bool(r["warm"][0, m]), r) for m in range(n)}, r
    poses = lambda k: (_pose([0.3, -0.2 + 0.01 * k, 0.1], [-0.12 + 0.004 * k, -0.05, 0.7]), _pose([-0.2, 0.4, 0.3 + 0.01 * k], [0.1, 0.06 - 0.003 * k, 0.8]))
    ids_a, ids_b = [], []
    for k in range(6):                                                 # two objects of classes 6 and 2 move
        (Ra, ta), (Rb, tb) = poses(k)
        got, r = frame([(0, 6, Ra, ta, 5.0), (1, 2, Rb, tb, 4.0)])
        ids_a.append(got[6][:2]); ids_b.append(got[2][:2])
        if k:                                                          # a warm solve meets cv2 started from the stored pose
            m = int(np.nonzero(r["cls"][0].cpu().numpy() == 6)[0][0])
            Ro, to = pnp_guess_ref(P3[6], r["keypoints_px"][0, m].cpu().numpy(), KM.astype(F32), prev_a[:3], prev_a[3:])
            assert _ang(r["R"][0, m].cpu().numpy(), Ro) < 1e-2 and np.abs(r["t"][0, m].cpu().numpy() - to.reshape(3)).max() * 1e3 < 1e-2
            assert _ang(r["R"][0, m].cpu().numpy(), Ra) < 1e-2
        prev_a = r["params"][0, int(np.nonzero(r["cls"][0].cpu().numpy() == 6)[0][0])].cpu().numpy()
    assert ids_a == [(0, False)] + [(0, True)] * 5 and ids_b == [(1, False)] + [(1, True)] * 5
    (Ra, ta), (Rb, tb) = poses(6)
    got, _ = frame([(0, 6, Ra, ta, 5.0), (1, 2, Rb, tb, 4.0), (2, 9, Ra, ta + np.array([0.15, 0.1, 0.0]), 3.0)])
    assert got[9][:2] == (2, False)                                    # a new object gets the next id
    got, _ = frame([(0, 6, Ra, ta, 5.0), (1, 2, Rb, tb, 4.0), (2, 3, Ra, ta, 4.0)])   # another class at the same place: its own id
    assert got[6][:2] == (0, True) and got[3][:2] == (3, False) and got[2][:2] == (1, True)
    for _ in range(2):                                                 # 2 is absent max_misses frames: still tracked
        frame([(0, 6, Ra, ta, 5.0)])
    got, _ = frame([(0, 6, Ra, ta, 5.0), (1, 2, Rb, tb, 4.0)])
    assert got[2][:2] == (1, True)
    for _ in range(3):                                                 # absent max_misses + 1 frames: its id is gone
        frame([(0, 6, Ra, ta, 5.0)])
    got, _ = frame([(0, 6, Ra, ta, 5.0), (1, 2, Rb, tb, 4.0)])
    assert got[2][:2] == (4, False) and got[6][:2] == (0, True)
    t = tr.tracks(to_host=True)
    assert sorted(t["id"].tolist()) == [0, 4] and (t["stream"] == 0).all()
    tr.reset()
    got, _ = frame([(0, 6, Ra, ta, 5.0)])
    assert got[6][:2] == (0, False)


def test_streams_never_interact():
    B, H = 3, 13
    gen = torch.Generator().manual_seed(7)
    base = torch.randn(B, (2 * K9 + 1 + NC) * NA, H, H, generator=gen)
    base[:, [18 + 32 * a for a in range(NA)]] += torch.tensor([1.0, -1.0, 0.0])[:, None, None, None]
    kw = dict(conf_thresh=0.05, max_instances=64, max_tracks=16, max_misses=1)
    t3 = InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), batch=3, **kw)
    t1 = [InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), batch=1, **kw) for _ in range(B)]
    warm = 0
    for f in range(8):
        out = (base + 0.05 * torch.randn(base.shape, generator=gen)).to(DEV)
        r3 = _clone(t3.update(out))
        for b in range(B):
            r1 = t1[b].update(out[b:b + 1].contiguous())
            for k in r3:
                assert torch.equal(r3[k][b], r1[k][0]), (f, b, k)
        warm += int(r3["warm"].sum())
    assert warm > 0
    for a, b1 in zip(t3._state(), zip(*[t._state() for t in t1])):
        assert torch.equal(a, torch.cat(b1))


# ---------------------------------------------------------------------------------------------------- the predictor
@pytest.fixture(scope="module")
def multi_model(cfg_multi_path):
    torch.manual_seed(0)
    return Darknet(cfg_multi_path).cuda().eval()


def _frames(n, seed, w=640, h=480):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _sequence(n, B, seed, w=640, h=480):
    """frames of a slowly changing scene: each is the first plus a little noise"""
    rng = np.random.default_rng(seed)
    f0 = rng.integers(0, 256, size=(B, h, w, 3)).astype(np.int16)
    return [np.clip(f0 + rng.integers(-6, 7, size=f0.shape), 0, 255).astype(np.uint8) for _ in range(n)]


def _clone(r):
    return {k: v.clone() for k, v in r.items()}


def _equal(a, b):
    return all(torch.equal(a[k], b[k]) for k in a)


def test_agrees_with_the_instance_predictor(multi_model):
    objs = {c: OBJECTS[c] for c in (0, 4, 7, 11)}
    kw = dict(batch=2, conf_thresh=0.02, max_instances=64)
    tp = TrackingPosePredictor(multi_model, objs, KM, **kw)
    ip = InstancePosePredictor(multi_model, objs, KM, **kw)
    P3 = {c: np.concatenate([np.zeros((1, 3)), objs[c].T]).astype(F32) for c in objs}
    warm_seen = 0
    for f, fr in enumerate(_sequence(5, 2, seed=3)):
        before = tp.tracks(to_host=True)
        stored = {(int(b), int(s)): None for b, s in zip(before["stream"], before["slot"])}
        poses = tp._tracker.state_poses.cpu().numpy()
        rt, ri = _clone(tp(fr)), _clone(ip(fr))
        for k in ("count", "kept", "cls", "conf", "cls_conf", "keypoints_px"):
            assert torch.equal(rt[k], ri[k]), (f, k)
        warm = rt["warm"].cpu().numpy()
        if f == 0:
            assert not warm.any()
        cold = torch.from_numpy(~warm).to(DEV)
        for k in ("R", "t", "corners_px"):
            assert torch.equal(rt[k][cold], ri[k][cold]), (f, k)
        slot = tp._last.slot.cpu().numpy()
        for b, m in zip(*np.nonzero(warm)):
            assert (int(b), int(slot[b, m])) in stored
            g = poses[b, slot[b, m]]
            c = int(rt["cls"][b, m])
            Ro, to = pnp_guess_ref(P3[c], rt["keypoints_px"][b, m].cpu().numpy(), KM.astype(F32), g[:3], g[3:])
            if not np.abs(to).max() < 10.0:                             # LM ran away from the stored pose: no pose to compare
                continue
            assert _ang(rt["R"][b, m].cpu().numpy(), Ro) < 1e-2 and np.abs(rt["t"][b, m].cpu().numpy() - to.reshape(3)).max() * 1e3 < 1e-2
            warm_seen += 1
        tid = rt["track_id"].cpu().numpy()
        n = rt["count"].cpu().numpy()
        for b in range(2):
            assert (tid[b, n[b]:] == -1).all() and not warm[b, n[b]:].any()
            ids = tid[b, :n[b]][tid[b, :n[b]] >= 0]
            assert len(set(ids.tolist())) == len(ids)                   # an id appears once per frame
    assert warm_seen > 0


def test_graph_replay_equals_eager_and_state_plumbing(multi_model):
    objs = {c: OBJECTS[c] for c in (0, 6, 12)}
    kw = dict(batch=3, conf_thresh=0.02, max_instances=32, max_tracks=16)
    seq = _sequence(4, 3, seed=4)
    small = _sequence(4, 3, seed=5, w=320, h=240)
    g = TrackingPosePredictor(multi_model, objs, KM, **kw)
    e = TrackingPosePredictor(multi_model, objs, KM, graph=False, **kw)
    for f in range(4):                                                  # two frame sizes interleaved share one track table
        for fr in (seq[f], small[f]):
            rg, re_ = _clone(g(fr)), _clone(e(fr))
            assert g._last.graph is not None and _equal(rg, re_), f
    assert int(g._tracker.state_next_id.sum()) > 0
    assert all(torch.equal(a, b) for a, b in zip(g._tracker._state(), e._tracker._state()))
    assert len(g._chains) == 2
    # reset mid-sequence behaves like a fresh predictor
    g.reset()
    fresh = TrackingPosePredictor(multi_model, objs, KM, **kw)
    for f in range(3):
        assert _equal(_clone(g(seq[f])), _clone(fresh(seq[f]))), f
    g.reset(streams=[1])
    t = g.tracks()
    assert not (t["stream"] == 1).any() and (t["stream"] != 1).any()


def test_bad_arguments_raise_before_any_launch(multi_model):
    eng = multi_model._engine
    n0 = eng.launches
    for kw in (dict(max_tracks=0), dict(max_tracks=257), dict(max_tracks=2.5), dict(max_tracks=True), dict(match_iou=-0.1),
               dict(match_iou=1.5), dict(match_iou=float("nan")), dict(max_misses=-1), dict(max_misses=1.5)):
        with pytest.raises(SspError):
            TrackingPosePredictor(multi_model, OBJECTS, KM, **kw)
        with pytest.raises(SspError):
            InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), **kw)
    assert eng.launches == n0
    tr = InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), batch=2)
    with pytest.raises(SspError):
        tr.update(torch.zeros(1, 160, 13, 13, device=DEV))              # one stream short
    with pytest.raises(SspError):
        tr.update(torch.zeros(2, 150, 13, 13, device=DEV))              # channels


def test_cli_writes_what_the_api_returns(cfg_multi_path, tmp_path):
    import glob
    root = str(tmp_path)
    synth.write_linemod_multi_like(root, n=2)
    paths = sorted(glob.glob(os.path.join(root, "LINEMOD", "*", "JPEGImages", "*.png")))[:3]
    paths = paths + paths[::-1]
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
    out = str(tmp_path / "trk.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_multi_path, "--weightfile", wf, "--out", out, "--max-instances", "8", "--track",
          "--match-iou", "0.2", "--max-misses", "1", "--max-tracks", "4", "--object", "4=%s" % meshes[4][0], "--object", "0=%s" % meshes[0][0]]
         + paths)
    got = np.load(out)
    m = Darknet(cfg_multi_path)
    m.load_weights(wf)
    m.cuda().eval()
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    pred = TrackingPosePredictor(m, {c: meshes[c][1] for c in meshes}, Km, max_instances=8, match_iou=0.2, max_misses=1, max_tracks=4)
    from PIL import Image
    keys = ("cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px", "track_id")
    rows = {k: [] for k in keys}
    for p in paths:
        r = pred(np.asarray(Image.open(p).convert("RGB"))[None], to_host=True)
        n = int(r["count"][0])
        for k in rows:
            rows[k].append(r[k][0, :n])
    for k in keys:
        assert np.array_equal(got[k], np.concatenate(rows[k])), k
    assert "track_id" in got.files
