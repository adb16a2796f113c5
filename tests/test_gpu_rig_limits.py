"""GPU checks of the rig kernels at the sizes they are declared for: ssp_fuse_views, ssp_fuse_instances, ssp_world_track_associate /
_commit and ssp_calibrate_rig against their host harnesses, each started from the device's own per-row poses, with 16 cameras,
more than 128 hypotheses per capture, 33 and 256 track and world slots with planted ties, more than 256 observations and more
than 256 co-observations per camera pair, and the calibration's opted-in shared memory from 11 cameras; the pose predictors with a
16-camera rig and with 256 instances and tracks; the refusals one past each limit.  Each case asserts the size it is there for.
The scenes come from tests/test_rig_limits_cpu.py, where the harnesses are held to the numpy oracles at the same sizes."""
import numpy as np
import pytest
import torch

from oracle.calibrate_rig_ref import MAX_PAIR_HYP
from singleshotpose_b200 import utils
from singleshotpose_b200._lib import SspError
from singleshotpose_b200.utils_multi import WorldInstanceTracker
from test_calibrate_rig_cpu import cal, host_calibrate, record, moving_object, relative, scene as cal_scene  # noqa: F401
from test_fuse_instances_cpu import TABLE, host_instances, ihost, scene as inst_scene, scene_rig  # noqa: F401
from test_gpu_calibrate_rig import KEYS as CAL_KEYS, _same, device as cal_device
from test_gpu_multiview import _frames, _rig2
from test_multiview_cpu import P9, host, host_fuse, observe, random_object, random_rig  # noqa: F401
from test_rig_limits_cpu import (WARP, co_observations, limit_frames, planted_hypothesis_won, planted_subsample_scene, sixteen_camera_instances,
                                 subsample_picks, tie_slots)
from test_world_track_cpu import host_step, whost  # noqa: F401

pytestmark = pytest.mark.gpu
ROW_KEYS = ("R", "t", "corners_px")
OBJECTS = {k: TABLE[k, 1:].T.astype(np.float64) for k in (0, 1)}


def _host(r):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in r.items()}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _rot_deg(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


# ---------------------------------------------------------------------------------------------------- ssp_fuse_views
@pytest.mark.parametrize("S", [1, 13])
def test_fuse_views_sixteen_cameras(host, S):
    """16 cameras, the even ones distorted (8 distorted-row launches), 12 captures of S slots, a view shifted 90 px and an
    invalid view: every slot bit for bit as the harness gives it from the device's rows"""
    rng = np.random.default_rng(1700 + S)
    Cn, G = 16, 12
    rig = random_rig(rng, Cn, True)
    assert rig.dist[::2].any(1).all() and not rig.dist[1::2].any()
    uv = np.stack([np.stack([observe(rig, *random_object(rng), rng) for _ in range(S)], 1) for _ in range(G)])   # (G, C, S, 9, 2)
    uv = uv.reshape(G * Cn, S, 9, 2)
    valid = np.ones((G * Cn, S), bool)
    uv[Cn + 5, S - 1] += 90.0                                           # a shifted view: capture 1, camera 5, the last slot
    valid[3 * Cn + 10, S // 2] = False                                  # an invalid view: capture 3, camera 10
    d = _host(utils.fuse_views_batched(P9, uv if S > 1 else uv[:, 0], rig, valid if S > 1 else valid[:, 0]))
    if S == 1:
        d = {k: v[:, None] for k, v in d.items()}
    h = host_fuse(host, rig, uv[:, 0], valid[:, 0])                     # step 1 on the host: within a tolerance
    assert np.abs(d["R"][:, 0] - h["R"]).max() < 1e-6 and np.abs(d["t"][:, 0] - h["t"]).max() < 1e-6
    fused = 0
    for s in range(S):
        h = host_fuse(host, rig, uv[:, s], valid[:, s], rows=(d["R"][:, s], d["t"][:, s]))
        for k in ("R_world", "t_world", "world_cov", "views", "view_err", "fuse_hyp", "fuse_status", "corners_world_px"):
            assert np.array_equal(d[k][:, s], h[k]), (s, k, np.argwhere(d[k][:, s] != h[k])[:5])
        fused += int((d["fuse_status"][:, s] == 0).sum())
        assert (d["views"][:, s].sum(1) >= 12).all(), s
    assert fused == G * S
    assert not d["views"][1, S - 1, 5] and not d["views"][3, S // 2, 10] and d["view_err"][3, S // 2, 10] == -1


def test_fuse_views_sixteen_cameras_noise_free():
    """keypoints without noise in 16 cameras, the even ones distorted: the fused pose is the truth to the rounding of the
    keypoints to fp32, ~3e-5 px at 300-600 px (measured on an H100: 7.7e-9 m and 5.2e-8 rad over six captures)"""
    rng = np.random.default_rng(1616)
    rig = random_rig(rng, 16, True)
    poses = [random_object(rng) for _ in range(6)]
    uv = np.concatenate([observe(rig, R, t, rng, noise=0.0) for R, t in poses])
    d = _host(utils.fuse_views_batched(P9, uv, rig))
    t_err = max(np.abs(d["t_world"][g] - t).max() for g, (R, t) in enumerate(poses))
    r_err = max(np.radians(_rot_deg(d["R_world"][g], R)) for g, (R, t) in enumerate(poses))
    print("\n16-camera noise-free fusion: translation %.3g m, rotation %.3g rad" % (t_err, r_err))
    assert (d["fuse_status"] == 0).all() and d["views"].all()
    assert t_err < 2e-8 and r_err < 1e-7, (t_err, r_err)


# ---------------------------------------------------------------------------------------------------- ssp_fuse_instances
def test_fuse_instances_sixteen_cameras(ihost):
    """16 cameras, 5-6 instances of each class, 16 slots: captures of more than 128 hypotheses on one 128-thread CTA"""
    rig, caps = sixteen_camera_instances(1717, 3)
    uv, cls, count = (np.concatenate([c[i] for c in caps]) for i in range(3))
    hyps = count.reshape(3, 16).sum(1)
    assert (hyps > 128).any(), hyps
    d = _host(utils.fuse_instances_batched(TABLE, uv, cls, count, rig))
    h = host_instances(ihost, rig, uv, cls, count)                       # step 1 (ssp_pnp's cold solve) on the host: within a tolerance
    err = np.maximum(np.abs(d["R"] - h["R"]).max((2, 3)), np.abs(d["t"] - h["t"]).max(2))
    assert (err < 1e-6).mean() > 0.99 and err.max() < 1e-3, np.sort(err.ravel())[-5:]      # measured: one of 768 solves at 5.7e-5
    h = host_instances(ihost, rig, uv, cls, count, rows=(d["R"], d["t"]))
    for k in h:
        if k not in ROW_KEYS:
            assert np.array_equal(d[k], h[k]), (k, np.argwhere(d[k] != h[k])[:5])
    assert (d["world_count"] >= 8).all()


def test_fuse_instances_sixteen_cameras_noise_free(ihost):
    """noise-free keypoints, no missed and no spurious detection: every true instance is one world instance holding all of its
    16 detections"""
    rng = np.random.default_rng(1818)
    rig = scene_rig(rng, 16, True)
    uv, cls, count, truth, poses = inst_scene(rng, rig, n_per_class=(3, 4), M=10, miss=0.0, spurious=0.0, noise=0.0)
    d = _host(utils.fuse_instances_batched(TABLE, uv, cls, count, rig))
    assert d["world_count"][0] == len(poses) and d["unfused"][0] == 0 and count.sum() == 16 * len(poses)
    got = {tuple(d["members"][0, w]) for w in range(len(poses))}
    want = {tuple(int(np.flatnonzero(truth[c] == j)[0]) for c in range(16)) for j in range(len(poses))}
    assert got == want
    h = host_instances(ihost, rig, uv, cls, count, rows=(d["R"], d["t"]))
    for k in h:
        if k not in ROW_KEYS:
            assert np.array_equal(d[k], h[k]), k


def test_fuse_instances_full_256_slots(ihost, cfg_multi_path):
    """InstancePosePredictor(rig=..., max_instances=256) on a random multi-object network at conf_thresh 0.02 fills all 256 slots
    of both views (512 hypotheses): the fusion equals the harness run on the predictor's keypoints, classes and counts, at the
    default gate and at a 1000 px gate.  Measured on an H100: no hypothesis of the random keypoints keeps a view at either gate, so
    this pins the scoring of 512 hypotheses (4 per thread) and the pick over them, not the rounds that follow an emission; those
    run in the 16-camera scenes"""
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    objects = {c: utils.get_3D_corners(np.c_[np.random.default_rng(c).normal(0, 0.04, (50, 3)), np.ones((50, 1))].T) for c in (0, 3, 7)}
    rig = _rig2(True)
    r = _host(InstancePosePredictor(m, objects, None, batch=2, conf_thresh=0.02, max_instances=256, rig=rig)(_frames(2, 8)))
    assert (r["count"] == 256).all() and r["keypoints_px"].shape[1] == 256
    table = np.zeros((m.num_classes, 9, 3), np.float32)
    for c, corners in objects.items():
        table[c, 1:] = corners[:3].T
    h = host_instances(ihost, rig, r["keypoints_px"], r["cls"], r["count"], table=table, rows=(r["R"], r["t"]))
    for k in h:
        if k not in ROW_KEYS:
            assert np.array_equal(r[k], h[k]), (k, np.argwhere(r[k] != h[k])[:5])
    wide = _host(utils.fuse_instances_batched(table, r["keypoints_px"], r["cls"], r["count"], rig, gate=1000.0, reproj_thresh=1000.0))
    h = host_instances(ihost, rig, r["keypoints_px"], r["cls"], r["count"], table=table, gate=1000.0, thr=1000.0, rows=(r["R"], r["t"]))
    for k in h:
        if k not in ROW_KEYS:
            assert np.array_equal(wide[k], h[k]), (k, np.argwhere(wide[k] != h[k])[:5])
    print("\n256 slots: world_count %s at the default gate, %s at 1000 px" % (r["world_count"], wide["world_count"]))


# ---------------------------------------------------------------------------------------------------- ssp_world_track_*
@pytest.mark.parametrize("motion", [None, "constant_velocity"])
@pytest.mark.parametrize("T,M", [(33, 33), (33, 256), (256, 33), (256, 256)])
def test_world_track_at_the_limits(whost, T, M, motion):
    """the CPU test's synthesised fused outputs of G = 3 streams: ints and stored poses bit for bit, the filter within 1e-12
    (the device's sin, cos and atan2); the planted ties go to the lower slot within a lane and across lanes"""
    G, Cn = 3, 3
    frames, ties = limit_frames(T, M, G, Cn)
    assert T > WARP and M > WARP and (M == 256 or (G * M) % 128)
    params = ((2.0, 3.0), (1.0, 2.0), 22.46)
    rig = utils.camera_rig(_rig2(False).K[[0, 1, 0]], _rig2(False).R[[0, 1, 0]], _rig2(False).t[[0, 1, 0]])
    tr = WorldInstanceTracker(OBJECTS, rig, 2, G, max_tracks=T, match_dist=0.5, max_misses=1, motion=motion, accel_sigma=params[0],
                              init_velocity_sigma=params[1], gate=params[2])
    dev = torch.device("cuda")
    high = 0
    for f, fr in enumerate(frames):
        st = {k: v.cpu().numpy().copy() for k, v in zip(("tracks", "poses", "next_id", "filter"), tr._state())}
        if motion:
            st["params"] = params
        dt = np.zeros(G) if f == 0 else np.full(G, 1 / 32)
        fused = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in fr.items()}
        h = host_step(whost, st, fr, match_dist=0.5, max_misses=1, dt=dt, size=tr.class_size)
        d = _host(tr.update(fused, timestamps=[f / 32] * G if motion else None))
        for k in ("world_track_id", "track_id"):
            assert np.array_equal(d[k], h[k]), (f, k, np.argwhere(d[k] != h[k])[:5])
        assert np.array_equal(d["matched"], h["matched"] != 0), f
        assert np.array_equal(tr._bufs.wslot.cpu().numpy()[:, :M], h["wslot"]), f
        state = [v.cpu().numpy() for v in tr._state()]
        assert np.array_equal(state[0], st["tracks"]) and np.array_equal(state[1], st["poses"]) and np.array_equal(state[2], st["next_id"]), f
        if motion:
            assert np.array_equal(d["reinit"], h["reinit"] != 0), f
            for k in ("R_filt", "t_filt", "pose_cov", "velocity"):
                assert _rel(d[k], h[k]) < 1e-12, (f, k)
            assert _rel(state[3], st["filter"]) < 1e-12
        for _f, g, w, lo, _hi in (x for x in ties if x[0] == f):
            assert h["wslot"][g, w] == lo and d["matched"][g, w], (f, g, lo)
        high += int((d["matched"] & (h["wslot"] >= WARP)).sum())
    lo_other, lo_same, hi = tie_slots(T, M)
    assert lo_other % WARP != hi % WARP and lo_same % WARP == hi % WARP and len(ties) == 2 and high > 0


# ---------------------------------------------------------------------------------------------------- ssp_calibrate_rig
def _calibrate(cal, rig, uv, valid, tol, tag, iters=0):
    """the device's calibration, then the harness from its rows: every output as _same checks it, the LM iteration counts within
    iters of each other -> (device dict, harness dict)"""
    d = cal_device(uv, rig, valid)
    h = host_calibrate(cal, rig.K, rig.dist, uv, valid, rows=(d["R_rows"], d["t_rows"]))
    diff = max(_rel(d[k], h[k]) for k in CAL_KEYS if np.asarray(h[k]).dtype == np.float64)
    print("\n%s: doubles within %.3g relative, rounds %d / %d, iterations %d / %d" % (tag, diff, d["rounds"], h["rounds"], d["iterations"],
                                                                                   h["iterations"]))
    assert abs(d["iterations"] - h["iterations"]) <= iters, (tag, d["iterations"], h["iterations"])
    _same(d, dict(h, iterations=d["iterations"]), tag, tol)
    return d, h


# measured on an H100: (11, 40) and (16, 40) bit for bit, and held to that.  (16, 300): every int, flag and round exact and the
# doubles within 2.3e-9 relative, but 28 LM iterations on the device against 36 in the harness.  Past convergence each step's
# cost and the current cost differ in their last bits, so whether a step is accepted (lambda / 10) or rejected (lambda x 10)
# until |delta| < 1e-12 follows the rounding of the device's sin and cos in so3_exp; the iteration count is the one output that
# counts those steps.  The bit-exact runs at 262 observations (test_calibrate_subsampled_pairs) hold the lane partials past 256
@pytest.mark.parametrize("n_cams,G,distorted,tol,iters", [(11, 40, False, 0.0, 0), (16, 40, True, 0.0, 0), (16, 300, False, 1e-8, 8)])
def test_calibrate_many_cameras(cal, n_cams, G, distorted, tol, iters):
    """n = 6 (C - 1) unknowns: cov_kernel's 16 n^2 B of dynamic shared memory passes the 48 KiB default from C = 11 (n = 60,
    57.6 KB) and factor_kernel's 8 n^2 B at C = 16 (n = 90: 64.8 and 129.6 KB), which only the opt-in allows"""
    assert 16 * (6 * (n_cams - 1)) ** 2 > 48 * 1024 and (n_cams < 16 or 8 * (6 * (n_cams - 1)) ** 2 > 48 * 1024)
    rig, uv, valid = cal_scene(7100 + n_cams + G, n_cams, G=G, distorted=distorted, miss=0.1, wrong=0.1)
    if G > 256:
        assert len(valid) // n_cams > 256
    d, _h = _calibrate(cal, rig, uv, valid, tol, (n_cams, G), iters)
    assert (d["cam_status"] == 0).all() and d["rig"] is not None


@pytest.mark.parametrize("planted", [False, True])
def test_calibrate_subsampled_pairs(cal, planted):
    """C = 3 with 262 co-observations in every pair, bit for bit: the pair hypotheses at floor(i n / 256), and sums over more than
    256 observations in the lane partials.  In the planted scene (the CPU test's) the winner of every pair is the one noise-free
    capture, at an index only floor(i n / 256) takes, so a kernel that strides otherwise starts its bundle adjustment elsewhere"""
    if planted:
        rig, uv, valid, j = planted_subsample_scene(4102, 3, False)
        assert j >= MAX_PAIR_HYP and j in subsample_picks(262) and j not in subsample_picks(262, MAX_PAIR_HYP + 1)
    else:
        rig, uv, valid = cal_scene(4030, 3, G=262, wrong=0.1)
    assert min(co_observations(valid, 3).values()) > MAX_PAIR_HYP
    d, _h = _calibrate(cal, rig, uv, valid, 0.0, ("C3 subsampled", planted))
    assert (d["cam_status"] == 0).all()
    if planted:
        tree = host_calibrate(cal, rig.K, rig.dist, uv, valid, rows=(d["R_rows"], d["t_rows"]), tree_only=True)
        assert planted_hypothesis_won(tree, 3, j)


def test_calibrate_slotted_equals_one_slot_per_row():
    """S = 13 slots per row give the outputs of the same 260 observations laid out one slot per row"""
    rng = np.random.default_rng(13)
    n, G, S = 4, 20, 13
    assert G * S > 256
    rig = random_rig(rng, n)
    uv, valid = record(rig, moving_object(rng, G * S), rng, 2.0, 0.1, 0.1)          # capture q = g S + s
    one = cal_device(uv, rig, valid)
    uvs = uv.reshape(G, S, n, 9, 2).transpose(0, 2, 1, 3, 4).reshape(G * n, S, 9, 2)
    vs = valid.reshape(G, S, n).transpose(0, 2, 1).reshape(G * n, S)
    many = cal_device(uvs, rig, vs)
    for k in ("R", "t", "cam_cov", "cam_obs", "cam_rmse", "tree_parent", "edge_agree", "cam_status"):
        assert np.array_equal(one[k], many[k]), k
    for k in ("R_world", "t_world", "views", "view_err", "linked"):
        assert np.array_equal(one[k].reshape(G * S, *one[k].shape[1:]), many[k].reshape(G * S, *many[k].shape[2:])), k
    assert (one["rounds"], one["iterations"]) == (many["rounds"], many["iterations"]) and (one["cam_status"] == 0).all()


def test_calibrate_sixteen_cameras_noise_free(cal):
    """16 cameras, 40 captures without keypoint noise: the true rig within 1e-7 rad and 1e-7 m, as the harness gives it"""
    rig, uv, valid = cal_scene(60, 16, G=40, noise=0.0)
    d, _h = _calibrate(cal, rig, uv, valid, 0.0, "C16 noise-free")
    Rt, tt = relative(rig)
    assert (d["cam_status"] == 0).all()
    assert np.abs(d["R"] - Rt).max() < 1e-7 and np.abs(d["t"] - tt).max() < 1e-7, (np.abs(d["R"] - Rt).max(), np.abs(d["t"] - tt).max())


# ---------------------------------------------------------------------------------------------------- the predictors
def test_pose_predictor_with_sixteen_cameras(cfg_path):
    """a 16-camera rig, batch 16: graph replay equals eager launches equals utils.fuse_views_batched on the predictor's rows"""
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = random_rig(np.random.default_rng(16), 16, True)
    fr = _frames(16, 3)
    kw = dict(shape=(416, 416), batch=16, rig=rig, conf_thresh=0.0)
    r = _host(PosePredictor(m, CORNERS, None, **kw)(fr))
    e = _host(PosePredictor(m, CORNERS, None, graph=False, **kw)(fr))
    assert set(r) == set(e) and all(np.array_equal(r[k], e[k]) for k in r)
    P9c = np.concatenate([np.zeros((1, 3)), CORNERS[:3].T]).astype(np.float32)
    want = _host(utils.fuse_views_batched(P9c, r["keypoints_px"], rig, r["conf"] > 0.0))
    for key in want:
        assert np.array_equal(r[key], want[key]), key
    assert r["views"].shape == (1, 16)


def test_world_tracking_predictor_256(cfg_multi_path):
    """WorldTrackingPosePredictor(max_tracks=256, max_instances=256) on a random multi-object network, three captures: graph
    replay equals eager launches in every output and in the tracker's state.  The random detections fuse into no world instance,
    so both trackers start from the same restored state of 240 alive tracks in slots 0-239 (misses 0, 1, 2 in turn, max_misses
    3): the associate kernel ages 240 tracks over 8 warps; those that start with 2 misses die in the second capture, with 1 in the
    third, and those with none stay alive"""
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import WorldTrackingPosePredictor
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    objects = {c: utils.get_3D_corners(np.c_[np.random.default_rng(c).normal(0, 0.04, (50, 3)), np.ones((50, 1))].T) for c in (0, 3, 7)}
    rig = _rig2(True)
    kw = dict(batch=2, conf_thresh=0.02, max_instances=256, max_tracks=256, fuse=(1000.0, 1000.0, 2.0))
    kw.update(max_misses=3)
    g = WorldTrackingPosePredictor(m, objects, rig, **kw)
    e = WorldTrackingPosePredictor(m, objects, rig, graph=False, **kw)
    n0, T = 240, 256
    tracks = np.zeros((1, T, 5), np.int32)
    s = np.arange(n0)
    tracks[0, :n0] = np.stack([np.ones(n0), s, np.array([0, 3, 7])[s % 3], s % 3, np.ones(n0)], 1)
    poses = np.zeros((1, T, 12))
    poses[0, :, [0, 4, 8]] = 1.0
    poses[0, :, 9:] = 0.25 * np.stack([np.arange(T) % 16, np.arange(T) // 16, np.zeros(T)], 1) + 10.0
    planted = (torch.from_numpy(tracks).cuda(), torch.from_numpy(poses).cuda(), torch.tensor([n0], dtype=torch.int32, device="cuda"))
    for p in (g, e):
        p._tracker.restore(planted)
    for f, fr in enumerate((_frames(2, 8), _frames(2, 9), _frames(2, 8))):
        rg = {k: v.clone() for k, v in g(fr).items()}
        re_ = {k: v.clone() for k, v in e(fr).items()}
        assert set(rg) == set(re_) and (rg["count"] == 256).all(), f
        for k in rg:
            assert torch.equal(rg[k], re_[k]), (f, k)
    assert g._last.graph is not None
    assert all(torch.equal(a, b) for a, b in zip(g._tracker._state(), e._tracker._state()))
    alive = g._tracker.state_tracks[0, :, 0].cpu().numpy() != 0
    print("\n256 tracks: %d alive after three captures, %d born" % (alive.sum(), int(g._tracker.state_next_id[0]) - n0))
    assert np.array_equal(np.flatnonzero(alive[:n0]), s[s % 3 == 0]) and alive[WARP:n0].any()


# ---------------------------------------------------------------------------------------------------- refusals one past the limits
def test_refusals_past_the_limits():
    """17 cameras, 257 detection slots, 257 world slots: SspError before any launch (17 cameras in camera_rig and
    calibrate_rig_batched, and 257 tracks, are refused by the CPU tests)"""
    rig = _rig2(False)
    big = utils.CameraRig(np.repeat(rig.K[:1], 17, 0), np.repeat(np.eye(3)[None], 17, 0), np.zeros((17, 3)), None)
    with pytest.raises(SspError, match="views"):
        utils.fuse_views_batched(P9, np.zeros((17, 9, 2), np.float32), big)
    with pytest.raises(SspError, match="views"):
        utils.fuse_instances_batched(TABLE, np.zeros((17, 1, 9, 2), np.float32), np.zeros((17, 1)), np.zeros(17), big)
    with pytest.raises(SspError, match="slots"):
        utils.fuse_instances_batched(TABLE, np.zeros((2, 257, 9, 2), np.float32), np.zeros((2, 257)), np.zeros(2), rig)
    tr = WorldInstanceTracker(OBJECTS, rig, 2, 1, max_tracks=256)
    fused = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in limit_frames(33, 257, 1, 2, 1)[0][0].items()}
    before = [v.clone() for v in tr._state()]
    with pytest.raises(SspError, match="slots"):
        tr.update(fused)
    assert all(torch.equal(a, b) for a, b in zip(before, tr._state()))
