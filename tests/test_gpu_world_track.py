"""GPU checks of tracking the world instances of a rig over time: ssp_world_track_associate / ssp_world_track_commit against the
host harness (tests/helpers/world_track_host.cpp) on the fused outputs of seeded moving scenes, WorldInstanceTracker.update keeping
the ids of planted moving objects, WorldTrackingPosePredictor against InstancePosePredictor(rig=...) (every shared output bit
for bit, graph replay against eager launches, the warm-up before capture, reset of one stream), the refusals, and the
predict_instances --rig --track --motion cv command line against the predictor."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import utils
from singleshotpose_b200._lib import SspError
from singleshotpose_b200.utils_multi import WorldInstanceTracker
from test_fuse_instances_cpu import TABLE, ihost, scene_rig  # noqa: F401
from test_gpu_multiview import _frames, _rig2, _same
from test_multiview_cpu import BARREL, KM
from test_world_track_cpu import FAST, detections, host_step, new_state, trajectories, whost  # noqa: F401

pytestmark = pytest.mark.gpu
OBJECTS = {k: TABLE[k, 1:].T.astype(np.float64) for k in (0, 1)}


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _scene_batch(rng, rig, trajs, f):
    """capture f of every stream's trajectories, fused on the GPU -> the dict of utils.fuse_instances_batched"""
    caps = [detections(rng, rig, [(k, R[f], t[f]) for k, R, t in tr], M=12) for tr in trajs]
    uv, cls, count = (np.concatenate([c[i] for c in caps]) for i in range(3))
    return utils.fuse_instances_batched(TABLE, uv, cls, count, rig)


@pytest.mark.parametrize("motion", [None, "constant_velocity"])
def test_kernels_equal_harness(whost, motion):
    """both launches against the harness, each capture started from the device's state: ints and stored poses bit for bit, the
    filter to 1e-12 (sin, cos, atan2 and acos of pose_filter_core.h may round differently on the device); the ids of the slow
    scenes are kept"""
    rng = np.random.default_rng(40 + (motion is not None))
    rig = scene_rig(rng, 3, True)
    G, n_caps = 3, 12
    trajs = [trajectories(rng, (1, 3), n_caps, (0.0, 0.2)) for _ in range(G)]
    params = ((2.0, 1.0), (1.0, 0.5), 22.46)
    tr = WorldInstanceTracker(OBJECTS, rig, 2, G, max_tracks=16, max_misses=2, motion=motion, accel_sigma=params[0],
                              init_velocity_sigma=params[1], gate=params[2])
    assert np.array_equal(tr.class_size, utils_sizes())
    matched = 0
    for f in range(n_caps):
        fused = _scene_batch(rng, rig, trajs, f)
        st = {k: v.cpu().numpy().copy() for k, v in zip(("tracks", "poses", "next_id", "filter"), tr._state())}
        if motion:
            st["params"] = params
        ts = [f / 30.0] * G
        dt = np.zeros(G) if f == 0 else np.full(G, ts[0] - (f - 1) / 30.0)
        hf = {k: v.cpu().numpy() for k, v in fused.items()}
        h = host_step(whost, st, hf, max_misses=2, dt=dt, size=tr.class_size)
        d = _host(tr.update(fused, timestamps=ts if motion else None))
        for k in ("world_track_id", "track_id"):
            assert np.array_equal(d[k], h[k]), (f, k)
        assert np.array_equal(d["matched"], h["matched"] != 0)
        state = [v.cpu().numpy() for v in tr._state()]
        assert np.array_equal(state[0], st["tracks"]) and np.array_equal(state[1], st["poses"]) and np.array_equal(state[2], st["next_id"])
        if motion:
            assert np.array_equal(d["reinit"], h["reinit"] != 0), f
            for k in ("R_filt", "t_filt", "pose_cov", "velocity"):
                assert _rel(d[k], h[k]) < 1e-12, (f, k)
            assert _rel(state[3], st["filter"]) < 1e-12
        matched += int(d["matched"].sum())
    assert matched >= 3 * n_caps
    # a stream alone: the same bits as in the batch
    one = WorldInstanceTracker(OBJECTS, rig, 2, 1, max_tracks=16, max_misses=2, motion=motion)
    assert one.update(_scene_batch(np.random.default_rng(1), rig, trajs[:1], 0))["world_track_id"].shape == (1, 12)


def utils_sizes():
    from oracle.world_track_ref import class_size
    return class_size(TABLE)


def test_planted_moving_objects_keep_their_ids():
    """three objects moving 0.1-0.2 box diagonals per capture, seen by three cameras without noise: every capture's world
    instances carry ids 0, 1, 2 without motion and with it; the filter finds their velocity"""
    rng = np.random.default_rng(3)
    rig = scene_rig(rng, 3)
    traj = trajectories(rng, (1, 2), 20, (0.1, 0.2))[:3]
    plain = WorldInstanceTracker(OBJECTS, rig, 2, 1)
    cv = WorldInstanceTracker(OBJECTS, rig, 2, 1, motion="constant_velocity", init_velocity_sigma=(1.0, 2.0))
    for f in range(20):
        caps = detections(rng, rig, [(k, R[f], t[f]) for k, R, t in traj], miss=0.0, spurious=0.0, noise=0.3)
        fused = utils.fuse_instances_batched(TABLE, *caps[:3], rig)
        n = int(fused["world_count"][0])
        assert n == len(traj)
        for tr in (plain, cv):
            r = _host(tr.update(fused, timestamps=[f / 30.0] if tr.motion else None))
            assert sorted(r["world_track_id"][0, :n]) == list(range(n)), (f, r["world_track_id"])
            assert (r["track_id"][r["track_id"] >= 0] < n).all()
        if f > 8:
            t_world = fused["t_world"][0, :n].cpu().numpy()
            for w in range(n):
                j = int(np.argmin([np.linalg.norm(t_world[w] - t[f]) for _k, _R, t in traj]))
                v_true = (traj[j][2][f] - traj[j][2][f - 1]) * 30.0
                assert np.linalg.norm(r["velocity"][0, w, 3:] - v_true) < 0.25 * np.linalg.norm(v_true) + 0.05
    t = cv.tracks(to_host=True)
    assert sorted(t["id"]) == list(range(len(traj))) and t["filter_valid"].all() and (t["hits"] == 20).all()
    saved = cv.snapshot()
    cv.reset()
    assert len(cv.tracks()["id"]) == 0
    cv.restore(saved)
    assert sorted(cv.tracks(to_host=True)["id"]) == list(range(len(traj)))


# ---------------------------------------------------------------------------------------------------- the predictor
def _clone(r):
    return {k: v.clone() for k, v in r.items()}


@pytest.mark.parametrize("motion", [None, "constant_velocity"])
def test_predictor_with_a_rig(cfg_path, motion):
    """a posed network whose views fuse into world instances: every output of InstancePosePredictor(rig=...) keeps its bits call
    after call, graph replay equals eager launches in outputs and state, the warm-up does not advance the tracks, and
    reset(streams=[g]) clears stream g only"""
    from singleshotpose_b200.predict_instances import InstancePosePredictor, WorldTrackingPosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    objects = {0: CORNERS}
    rig = _rig2(True)
    kw = dict(shape=(416, 416), batch=4, conf_thresh=0.5, max_instances=32, rig=rig)
    base = InstancePosePredictor(m, objects, None, **kw)
    g = WorldTrackingPosePredictor(m, objects, motion=motion, max_tracks=24, **kw)
    e = WorldTrackingPosePredictor(m, objects, motion=motion, max_tracks=24, graph=False, **kw)
    frames = [_frames(4, 30), _frames(4, 30), _frames(4, 31), _frames(4, 30)]
    extra = {"track_id", "world_track_id"} | ({"R_filt", "t_filt", "pose_cov", "velocity", "reinit"} if motion else set())
    matched = 0
    for f, fr in enumerate(frames):
        ts = [f * 0.05, f * 0.04 + 1.0] if motion else None
        rb = _clone(base(fr))
        rg = _clone(g(fr, timestamps=ts))
        if f == 0:                                                  # the warm-up runs before the capture did not advance the tracks
            assert int(g._tracker.state_next_id.sum()) == int((rg["world_track_id"] >= 0).sum())
        re_ = _clone(e(fr, timestamps=ts))
        assert g._last.graph is not None and set(rg) - set(rb) == extra and "warm" not in rg
        for k in rb:
            assert torch.equal(rg[k], rb[k]), (f, k)
        for k in rg:
            assert torch.equal(rg[k], re_[k]), (f, k)
        wid = rg["world_track_id"].cpu().numpy()
        n = rg["world_count"].cpu().numpy()
        for gi in range(2):
            assert (wid[gi, n[gi]:] == -1).all() and len(set(wid[gi, :n[gi]][wid[gi, :n[gi]] >= 0])) == (wid[gi, :n[gi]] >= 0).sum()
        wi = rg["world_index"].cpu().numpy()
        tid = rg["track_id"].cpu().numpy()
        for b in range(4):
            want = np.where(wi[b] >= 0, wid[b // 2][np.maximum(wi[b], 0)], -1)
            assert np.array_equal(tid[b], want)
        if f == 1:
            matched = int((wid >= 0).sum())                          # the same frames again: every track is found again
            assert np.array_equal(wid, _prev)
        _prev = wid
    assert matched >= 2
    assert all(torch.equal(a, b) for a, b in zip(g._tracker._state(), e._tracker._state()))
    g.reset(streams=[1])
    st = g._tracker._state()
    assert not st[0][1].any() and st[0][0].any() and int(st[2][1]) == 0 and int(st[2][0]) > 0
    if motion:
        assert np.isnan(g._tracker._last_time[1]) and not np.isnan(g._tracker._last_time[0])
        with pytest.raises(SspError):
            g(frames[0], timestamps=[1.0, 2.0, 3.0, 4.0])            # one per capture, not per frame


def test_world_tracking_refusals(cfg_path):
    """what InstancePosePredictor(rig=...) refuses, WorldTrackingPosePredictor refuses too; its own bad arguments and timestamps
    are refused before any launch; TrackingPosePredictor still takes no rig"""
    from singleshotpose_b200.predict_instances import TrackingPosePredictor, WorldTrackingPosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(False)
    eng = m._engine
    n0 = eng.launches
    for bad in (dict(batch=3), dict(rig=None), dict(rig=KM), dict(match_dist=0.0), dict(match_dist=float("nan")), dict(max_tracks=300),
                dict(max_misses=-1), dict(motion="cv"), dict(gate=0.0), dict(fuse=(4.0, 8.0, 2.0))):
        kw = dict(shape=(416, 416), batch=4, conf_thresh=0.5, rig=rig)
        kw.update(bad)
        with pytest.raises(SspError):
            WorldTrackingPosePredictor(m, {0: CORNERS}, **kw)
    for bad in (dict(K=KM), dict(dist_coeffs=BARREL), dict(pnp="consensus"), dict(meshes={})):     # not its arguments
        with pytest.raises(TypeError):
            WorldTrackingPosePredictor(m, {0: CORNERS}, rig, shape=(416, 416), batch=4, **bad)
    with pytest.raises(TypeError):
        TrackingPosePredictor(m, {0: CORNERS}, None, shape=(416, 416), batch=4, rig=rig)
    assert eng.launches == n0
    pred = WorldTrackingPosePredictor(m, {0: CORNERS}, rig, shape=(416, 416), batch=4, conf_thresh=0.5, motion="constant_velocity")
    n0 = eng.launches
    with pytest.raises(SspError):
        pred(_frames(4, 3), timestamps=[0.0])                                                # G = 2 captures
    assert eng.launches == n0


def test_cli_rig_track_motion_writes_what_the_predictor_returns(cfg_path, tmp_path):
    """predict_instances --rig --track --motion cv on three captures of a two-camera rig: every .npz column equals the flattened
    outputs of WorldTrackingPosePredictor on the same images"""
    from PIL import Image
    from singleshotpose_b200.predict import mesh_corners
    from singleshotpose_b200.predict_instances import MOTION_KEYS, ROW_KEYS as CLI_ROWS, WORLD_KEYS, WorldTrackingPosePredictor, main
    from test_gpu_refine_depth import V, _posed_model
    m = _posed_model(cfg_path)
    wf = str(tmp_path / "posed.weights")
    m.save_weights(wf)
    ply = str(tmp_path / "obj.ply")
    with open(ply, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n" % len(V))
        for v in V:
            f.write("%.17g %.17g %.17g\n" % tuple(v))
    data = tmp_path / "obj.data"
    data.write_text("mesh = %s\nwidth = 640\nheight = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n" % ply)
    rig = _rig2(True)
    rig_path = str(tmp_path / "rig.npz")
    np.savez(rig_path, K=rig.K, R=rig.R, t=rig.t, dist=rig.dist)
    fr = _frames(6, 21)
    paths = []
    for i in range(6):
        paths.append(str(tmp_path / ("img%d.png" % i)))
        Image.fromarray(fr[i]).save(paths[-1])
    out = str(tmp_path / "tracks.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf, "--out", out, "--max-instances", "16", "--rig", rig_path,
          "--track", "--match-dist", "0.7", "--max-tracks", "8", "--motion", "cv", "--keypoint-sigma", "1.5", "--fps", "10"] + paths)
    got = np.load(out)
    pred = WorldTrackingPosePredictor(m, {0: mesh_corners(ply)}, rig, frame_size=(640, 480), batch=2, max_instances=16, match_dist=0.7,
                                      max_tracks=8, motion="constant_velocity", fuse=(40.0, 8.0, 1.5), frame_dt=0.1)
    rows = {k: [] for k in CLI_ROWS + ("world_index", "track_id")}
    world = {k: [] for k in WORLD_KEYS + ("world_track_id",) + MOTION_KEYS}
    for g in range(3):
        r = pred(fr[2 * g:2 * g + 2], to_host=True)
        for b in range(2):
            n = int(r["count"][b])
            for k in rows:
                rows[k].append(r[k][b, :n])
        n = int(r["world_count"][0])
        for k in world:
            world[k].append(r[k][0, :n])
    for k, v in list(rows.items()) + list(world.items()):
        assert np.array_equal(got[k], np.concatenate(v)), k
    ids = got["world_track_id"].reshape(3, -1)                       # the same instances every capture, 8 of them tracked
    assert (ids == ids[0]).all() and sorted(ids[0][ids[0] >= 0]) == list(range(8))
    tracked = got["track_id"] >= 0                                   # a detection is tracked exactly when its world instance is
    assert tracked.sum() > 0 and not tracked[got["world_index"] < 0].any()
