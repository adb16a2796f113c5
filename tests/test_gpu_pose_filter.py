"""GPU checks of the pose covariance and the pose filter of tracked instances: ssp_pose_covariance, ssp_track_predict and
ssp_track_filter_update against the host harness (tests/helpers/pose_filter_host.cpp) and cv2's empirical covariance
(tests/golden/pose_cov.npz); utils.pose_covariance_batched; InstanceTracker with motion on planted fast objects;
TrackingPosePredictor with motion (graph replay against eager, state plumbing, timestamps, argument checks) and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle.pose_filter_ref import pose_covariance, so3_exp
from singleshotpose_b200 import synth
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from singleshotpose_b200.darknet_multi import Darknet
from singleshotpose_b200.predict_instances import TrackingPosePredictor, main
from singleshotpose_b200.utils import pnp_batched, pose_covariance_batched
from singleshotpose_b200.utils_multi import InstanceTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K9, NC, NA, FD = 9, 13, 5, 163
KM = synth.intrinsics()
P3 = synth.box_points((0.038, 0.039, 0.046)).astype(np.float32)
F32 = np.float32


def _corners(c):
    s = 1.0 + 0.1 * c
    return synth.box_points((0.038 * s, 0.039 * s, 0.046 * (2.0 - 0.05 * c)), with_center=False).T.astype(np.float64)


OBJECTS = {c: _corners(c) for c in range(NC)}


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pfhost") / "libpfhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "pose_filter_host.cpp")])
    return C.CDLL(so)


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


# ---------------------------------------------------------------------------------------------------- covariance
@pytest.mark.parametrize("tag", ["plain", "barrel"])
def test_covariance_kernel_equals_harness_and_meets_cv2(host, golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "pose_cov.npz"))
    dist = None if tag == "plain" else g["dist_barrel"]
    rng = np.random.default_rng(1)
    n = 300
    R = np.stack([so3_exp(rng.normal(size=3)) for _ in range(n)])
    t = np.c_[rng.uniform(-0.2, 0.2, (n, 2)), rng.uniform(0.4, 1.2, n)]
    R[:4], t[:4] = g["R_" + tag], g["t_" + tag]
    t[5, 2] = -0.3                                                      # behind the camera: status DEPTH
    cov, st = pose_covariance_batched(g["P3"], g["K"], R, t, 1.0, dist)
    cov, st = cov.cpu().numpy(), st.cpu().numpy()
    hc, hs = np.zeros((n, 6, 6)), np.zeros(n, np.int32)
    Pc, Kc, Rc, tc = (np.ascontiguousarray(a, d) for a, d in ((g["P3"], F32), (g["K"], F32), (R, np.float64), (t, np.float64)))
    dc = None if dist is None else np.ascontiguousarray(dist)
    assert host.h_pose_covariance(_p(Pc), 1, _p(Kc), _p(dc), 9, C.c_longlong(n), _p(Rc), _p(tc), C.c_double(1.0), _p(hc), _p(hs)) == 0
    assert np.array_equal(st, hs) and st[5] == 2 and (np.delete(st, 5) == 0).all()
    assert max(_rel(cov[i], hc[i]) for i in range(n)) < 1e-12
    for i in range(4):
        assert np.abs(np.diag(cov[i]) / np.diag(g["cov_" + tag][i]) - 1).max() < 0.10
    # per problem: the same bits whatever the batch
    one, _ = pose_covariance_batched(g["P3"], g["K"], R[7:8], t[7:8], 1.0, dist)
    assert np.array_equal(one.cpu().numpy()[0], cov[7])


def test_covariance_of_the_batched_pnp():
    rng = np.random.default_rng(2)
    n = 64
    R = np.stack([so3_exp(rng.normal(size=3)) for _ in range(n)])
    t = np.c_[rng.uniform(-0.1, 0.1, (n, 2)), rng.uniform(0.5, 1.0, n)]
    uv = np.stack([((P3 @ R[i].T + t[i]) @ KM.T)[:, :2] / ((P3 @ R[i].T + t[i]) @ KM.T)[:, 2:] for i in range(n)]).astype(F32)
    Rp, tp = pnp_batched(P3, uv, KM)
    cov, st = pose_covariance_batched(P3, KM, Rp, tp, 2.0)
    assert (st == 0).all()
    want = np.stack([pose_covariance(P3, R[i], t[i], KM, 2.0)[0] for i in range(n)])
    assert max(_rel(cov[i].cpu().numpy(), want[i]) for i in range(n)) < 1e-6        # at the solved pose, not the true one
    with pytest.raises(SspError):
        pose_covariance_batched(P3, KM, Rp, tp, 0.0)


# ---------------------------------------------------------------------------------------------------- filter kernels
BARREL = np.array([-0.3, 0.12, 1e-3, -5e-4, -0.02, 0, 0, 0])          # pnp_dist.npz's "barrel"


def _predict(B, T, args, f, out, dist, acc):
    tracks, rects, poses, dt, table, Kd = args
    call("ssp_track_predict", B, T, ptr(tracks), ptr(rects), ptr(poses), ptr(f), ptr(dt), ptr(table), 2, ptr(Kd), None if dist is None else ptr(dist),
         acc[0], acc[1], ptr(out[0]), ptr(out[1]), stream_ptr())


def _update(B, T, M, args, f, out, v0, gate):
    call("ssp_track_filter_update", B, T, M, *map(ptr, args), ptr(f), v0[0], v0[1], gate, *map(ptr, out), stream_ptr())


def _update_outputs(B, M):
    return [torch.empty(B, M, k, dtype=torch.float64, device=DEV) for k in (9, 3, 36, 6)] + [torch.empty(B, M, dtype=torch.int32, device=DEV)]


@pytest.mark.parametrize("distorted", [False, True])
def test_filter_kernels_equal_harness(host, distorted):
    """ssp_track_predict and ssp_track_filter_update against the harness to 1e-12 (the predicted rectangles through the distorted
    projection with the barrel coefficients), and each stream's outputs bit-identical when it is launched alone (B = 1)"""
    rng = np.random.default_rng(4)
    B, T, M, acc, v0, gate = 3, 8, 6, (0.8, 0.3), (1.0, 0.5), 22.46
    table = np.ascontiguousarray(np.stack([P3, P3 * 1.3]), F32)
    Kd = np.ascontiguousarray(KM)
    h_dist = np.ascontiguousarray(BARREL) if distorted else None
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    d_dist = None if h_dist is None else d(h_dist)
    h_f = np.zeros((B, T, FD)); d_f = torch.zeros(B, T, FD, dtype=torch.float64, device=DEV)
    tracks = np.zeros((B, T, 5), np.int32)
    predicted = 0
    for f in range(12):
        tracks[..., 2] = rng.integers(0, 2, (B, T))
        rects, poses = rng.uniform(0, 400, (B, T, 4)).astype(F32), rng.normal(size=(B, T, 6))
        dt = rng.uniform(0.02, 0.05, B)
        hp, hr = np.zeros((B, T, 6)), np.zeros((B, T, 4), F32)
        assert host.h_track_predict(B, T, _p(tracks), _p(rects), _p(poses), _p(h_f), _p(dt), _p(table), 2, _p(Kd), _p(h_dist),
                                    C.c_double(acc[0]), C.c_double(acc[1]), _p(hp), _p(hr)) == 0
        args = [d(a) for a in (tracks, rects, poses, dt, table, Kd)]          # alive until the launches have run
        f0 = d_f.clone()
        out = [torch.empty(B, T, 6, dtype=torch.float64, device=DEV), torch.empty(B, T, 4, device=DEV)]
        _predict(B, T, args, d_f, out, d_dist, acc)
        torch.cuda.synchronize()
        assert _rel(out[0].cpu().numpy(), hp) < 1e-12 and _rel(d_f.cpu().numpy(), h_f) < 1e-12
        assert np.abs(out[1].cpu().numpy() - hr).max() <= 1e-3                   # fp32 pixels of fp64 poses equal to 1e-12
        predicted += int((hr != rects).any(-1).sum())
        for b in range(B):                                                       # one stream alone: the same bits
            fb = f0[b:b + 1].clone()
            ob = [torch.empty(1, T, 6, dtype=torch.float64, device=DEV), torch.empty(1, T, 4, device=DEV)]
            _predict(1, T, [x[b:b + 1].contiguous() for x in args[:4]] + args[4:], fb, ob, d_dist, acc)
            assert torch.equal(fb[0], d_f[b]) and torch.equal(ob[0][0], out[0][b]) and torch.equal(ob[1][0], out[1][b])
        count = rng.integers(0, M + 1, B).astype(np.int32)
        slot = np.full((B, M), -1, np.int32); use = np.zeros((B, M), np.int32)
        for b in range(B):
            for m, s in enumerate(rng.permutation(T)[:count[b]]):
                slot[b, m] = s
                use[b, m] = int(tracks[b, s, 0] and rng.random() < 0.8)
                tracks[b, s, 0] = 1
        Rm = np.stack([so3_exp(rng.normal(0, 0.3, 3)) for _ in range(B * M)]).reshape(B, M, 9)
        tm = np.c_[rng.normal(0, 0.05, (B * M, 2)), rng.uniform(0.5, 0.8, B * M)].reshape(B, M, 3)
        A = rng.normal(size=(B, M, 6, 6))
        Sm = (1e-5 * (A @ A.transpose(0, 1, 3, 2) + np.eye(6))).reshape(B, M, 36)
        st = (rng.random((B, M)) < 0.05).astype(np.int32)
        ho = [np.zeros((B, M, 9)), np.zeros((B, M, 3)), np.zeros((B, M, 36)), np.zeros((B, M, 6)), np.zeros((B, M), np.int32)]
        assert host.h_track_filter_update(B, T, M, _p(count), _p(slot), _p(use), _p(Rm), _p(tm), _p(Sm), _p(st), _p(h_f), C.c_double(v0[0]),
                                          C.c_double(v0[1]), C.c_double(gate), *map(_p, ho)) == 0
        args = [d(a) for a in (count, slot, use, Rm, tm, Sm, st)]
        f0 = d_f.clone()
        do = _update_outputs(B, M)
        _update(B, T, M, args, d_f, do, v0, gate)
        torch.cuda.synchronize()
        for a, b_ in zip(do, ho):
            assert _rel(a.cpu().numpy(), b_) < 1e-12 if b_.dtype != np.int32 else np.array_equal(a.cpu().numpy(), b_)
        assert _rel(d_f.cpu().numpy(), h_f) < 1e-12
        for b in range(B):
            fb, ob = f0[b:b + 1].clone(), _update_outputs(1, M)
            _update(1, T, M, [x[b:b + 1].contiguous() for x in args], fb, ob, v0, gate)
            assert torch.equal(fb[0], d_f[b]) and all(torch.equal(x[0], y[b]) for x, y in zip(ob, do))
        h_f = d_f.cpu().numpy().copy()                                          # libm may differ in the last bits: go on from one state
    assert predicted > 10                                                       # the predicted rectangles were exercised


# ---------------------------------------------------------------------------------------------------- planted fast objects
def _pose(ang, t):
    return so3_exp(np.asarray(ang, float)), np.asarray(t, float)


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
    o = torch.zeros(1, NA * (2 * K9 + 1 + NC), H, H)
    o[:, [18 + 32 * a for a in range(NA)]] = -10.0
    for a, c, R, t, s in objs:
        _plant(o, 0, a, c, _project(c, R, t), H, s)
    return o.to(DEV)


def _fast(k):
    """class 6, 1.2 m away (its corner rectangle about 0.16 m wide): speeding up to 0.1 m (48 px) per frame sideways, then steady
    (3 m/s at 30 fps), so consecutive rectangles overlap with IoU about 0.2"""
    x = -0.6 + sum(0.1 * min(j, 3) / 3 for j in range(k + 1))
    return _pose([0.3, -0.2, 0.1], [x, -0.02, 1.2])


def test_planted_fast_object_keeps_its_id_with_motion():
    kw = dict(max_tracks=16, max_misses=2)
    plain = InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), **kw)
    cv = InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), motion="constant_velocity", keypoint_sigma=1.0, init_velocity_sigma=(1.0, 3.0),
                         accel_sigma=(2.0, 30.0), **kw)                 # it speeds up by 1 m/s per frame: 30 m/s^2
    ids = {"plain": [], "cv": []}
    for k in range(11):
        R, t = _fast(k)
        logits = _scene([(0, 6, R, t, 5.0)])
        for name, tr in (("plain", plain), ("cv", cv)):
            r = tr.update(logits, timestamps=[k / 30.0]) if name == "cv" else tr.update(logits)
            assert int(r["count"][0]) == 1
            ids[name].append(int(r["track_id"][0, 0]))
            if name == "cv":
                assert r["pose_cov"][0, 0].diagonal().min() > 0 and (k > 0 or bool(r["reinit"][0, 0]))   # born at frame 0
                if k > 5:                                           # the filter has found the velocity, 3 m/s sideways
                    v = r["velocity"][0, 0, 3:].cpu().numpy()
                    assert abs(v[0] - 3.0) < 0.4 and np.abs(v[1:]).max() < 0.4, v
                    assert not bool(r["reinit"][0, 0])
    assert ids["cv"] == [0] * 11, ids
    assert len(set(ids["plain"])) > 4, ids                         # without motion the fast object gets new ids
    t = cv.tracks(to_host=True)
    assert list(t["id"]) == [0] and t["filter_valid"].all()
    # a coasting track reports its prediction and is found again after a 2-frame gap
    for k in (11, 12):
        r = cv.update(_scene([]), timestamps=[k / 30.0])
    t = cv.tracks(to_host=True)
    assert list(t["misses"]) == [2] and abs(t["t_filt"][0, 0] - _fast(12)[1][0]) < 0.02
    r = cv.update(_scene([(0, 6, *_fast(13), 5.0)]), timestamps=[13 / 30.0])
    assert int(r["track_id"][0, 0]) == 0
    with pytest.raises(SspError):
        cv.update(_scene([]), timestamps=[13 / 30.0])               # not after the last one
    saved = cv.snapshot()
    cv.reset()
    assert not cv.state_filter.any() and len(cv.tracks()["id"]) == 0
    cv.restore(saved)
    assert torch.equal(cv.state_filter, saved[4]) and list(cv.tracks(to_host=True)["id"]) == [0]


# ---------------------------------------------------------------------------------------------------- the predictor
@pytest.fixture(scope="module")
def multi_model(cfg_multi_path):
    torch.manual_seed(0)
    return Darknet(cfg_multi_path).cuda().eval()


def _sequence(n, B, seed, w=640, h=480):
    rng = np.random.default_rng(seed)
    f0 = rng.integers(0, 256, size=(B, h, w, 3)).astype(np.int16)
    return [np.clip(f0 + rng.integers(-6, 7, size=f0.shape), 0, 255).astype(np.uint8) for _ in range(n)]


def _clone(r):
    return {k: v.clone() for k, v in r.items()}


@pytest.mark.parametrize("distorted", [False, True])
def test_predictor_motion_graph_equals_eager_and_state(multi_model, distorted):
    """With the barrel coefficients the predict and the PnP run distorted.  The random network's PnP solutions collapse onto the
    camera centre (|t| about 1e-5 m, most of them behind it), so their covariance is unusable (SSP_POSE_COV_DEPTH) and a matched
    track's filter restarts from each of them; the Kalman update itself is exercised on planted objects
    (test_planted_fast_object_keeps_its_id_with_motion), through the same launches."""
    objs = {c: OBJECTS[c] for c in (0, 6, 12)}
    dist = BARREL[:5] if distorted else None
    kw = dict(batch=3, conf_thresh=0.02, max_instances=32, max_tracks=16, dist_coeffs=dist)
    seq = _sequence(5, 3, seed=4)
    g = TrackingPosePredictor(multi_model, objs, KM, motion="constant_velocity", **kw)
    e = TrackingPosePredictor(multi_model, objs, KM, graph=False, motion="constant_velocity", **kw)
    base = TrackingPosePredictor(multi_model, objs, KM, **kw)
    started = matched = 0
    for f in range(5):
        ts = [f * 0.05, f * 0.04 + 1.0, f / 30.0]
        rg, re_ = _clone(g(seq[f], timestamps=ts)), _clone(e(seq[f], timestamps=ts))
        assert g._last.graph is not None and rg.keys() == re_.keys()
        for k in rg:
            assert torch.equal(rg[k], re_[k]), (f, k)
        rb = _clone(base(seq[f]))
        for k in ("count", "cls", "keypoints_px"):                  # the same detections
            assert torch.equal(rb[k], rg[k])
        assert set(rg) - set(rb) == {"R_filt", "t_filt", "pose_cov", "velocity", "reinit"}
        n = rg["count"].cpu().numpy()
        tid = rg["track_id"].cpu().numpy()
        for b in range(3):
            has = tid[b, :n[b]] >= 0
            assert (rg["pose_cov"][b, :n[b]][torch.from_numpy(has).to(DEV)].diagonal(dim1=1, dim2=2) >= 0).all()
            assert not rg["R_filt"][b, n[b]:].any()
        born = (rg["track_id"] >= 0) & ~rg["warm"]
        assert bool(rg["reinit"][born].all())                      # a new track starts its filter from its PnP
        assert torch.equal(rg["R_filt"][born], rg["R"][born]) and torch.equal(rg["t_filt"][born], rg["t"][born])
        started += int(born.sum())
        unusable = g._last.cov_status != 0
        assert torch.equal(rg["reinit"] & rg["warm"], unusable & rg["warm"])   # a matched track restarts exactly when its PnP is unusable
        matched += int(rg["warm"].sum())
    assert started > 0 and matched > 0, (started, matched)
    assert all(torch.equal(a, b) for a, b in zip(g._tracker._state(), e._tracker._state()))
    g.reset(streams=[1])
    assert not g._tracker.state_filter[1].any() and np.isnan(g._tracker._last_time[1]) and not np.isnan(g._tracker._last_time[0])
    with pytest.raises(SspError):
        g(seq[0], timestamps=[0.0, 5.0, 0.0])                       # stream 0 goes back in time
    with pytest.raises(SspError):
        g(seq[0], timestamps=[1.0, 2.0])


def test_motion_none_is_the_tracker_before_the_filter(golden_dir):
    """motion=None: every output of every frame and the track state equal, bit for bit, what the tracker wrote before the pose filter
    existed (tests/golden/make_golden_track_motion_none.py)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_track_motion_none",
                                                  os.path.join(golden_dir, "make_golden_track_motion_none.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    want = np.load(os.path.join(golden_dir, "track_motion_none.npz"))
    got = gen.run()
    assert sorted(got) == sorted(want.files)
    for k in want.files:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
    assert sum(int(want[k].sum()) for k in want.files if k.startswith("warm_")) > 0


def test_bad_motion_arguments_raise_before_any_launch(multi_model):
    eng = multi_model._engine
    n0 = eng.launches
    for kw in (dict(motion="cv"), dict(keypoint_sigma=0.0), dict(accel_sigma=(1.0, float("nan"))), dict(init_velocity_sigma=(1.0,)),
               dict(gate=-1.0), dict(frame_dt=0.0)):
        kw = dict(dict(motion="constant_velocity"), **kw)
        with pytest.raises(SspError):
            TrackingPosePredictor(multi_model, OBJECTS, KM, **kw)
        with pytest.raises(SspError):
            InstanceTracker(OBJECTS, KM, NC, NA, (640, 480), **kw)
    assert eng.launches == n0


def test_cli_motion_writes_what_the_api_returns(cfg_multi_path, tmp_path):
    import glob
    root = str(tmp_path)
    synth.write_linemod_multi_like(root, n=2)
    paths = sorted(glob.glob(os.path.join(root, "LINEMOD", "*", "JPEGImages", "*.png")))[:3]
    paths = paths + paths[::-1]
    V = np.random.default_rng(0).normal(size=(40, 3)) * 0.03
    ply = str(tmp_path / "obj0.ply")
    with open(ply, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n" % len(V))
        for v in V:
            f.write("%.17g %.17g %.17g\n" % tuple(v))
    from singleshotpose_b200.utils_multi import get_3D_corners
    corners = get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    data = tmp_path / "occlusion.data"
    data.write_text("mesh1 = ignored.ply\nim_width = 640\nim_height = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    torch.manual_seed(4)
    wf = str(tmp_path / "m.weights")
    Darknet(cfg_multi_path).save_weights(wf)
    out = str(tmp_path / "trk.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_multi_path, "--weightfile", wf, "--out", out, "--max-instances", "8", "--track",
          "--match-iou", "0.2", "--max-tracks", "4", "--motion", "cv", "--keypoint-sigma", "1.5", "--fps", "10", "--object", "0=%s" % ply] + paths)
    got = np.load(out)
    m = Darknet(cfg_multi_path)
    m.load_weights(wf)
    m.cuda().eval()
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    pred = TrackingPosePredictor(m, {0: corners}, Km, max_instances=8, match_iou=0.2, max_tracks=4, motion="constant_velocity",
                                 keypoint_sigma=1.5, frame_dt=0.1)
    from PIL import Image
    keys = ("cls", "R", "t", "track_id", "R_filt", "t_filt", "velocity", "pose_cov")
    rows = {k: [] for k in keys}
    for p in paths:
        r = pred(np.asarray(Image.open(p).convert("RGB"))[None], to_host=True)
        n = int(r["count"][0])
        for k in rows:
            rows[k].append(r[k][0, :n])
    for k in keys:
        assert np.array_equal(got[k], np.concatenate(rows[k])), k
