"""GPU checks of the instance fusion across a rig: ssp_fuse_instances against the host harness
(tests/helpers/multiview_instances_host.cpp) on the CPU tests' scenes, and InstancePosePredictor with a rig (per-frame outputs
equal to one single-camera predictor per camera, fused outputs equal to utils.fuse_instances_batched, graph replay equal to eager
launches, one detection per view reducing to utils.fuse_views_batched, the worst case of full slots, the refusals, and the
predict_instances --rig command line against the predictor)."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import utils
from singleshotpose_b200._lib import SspError
from test_fuse_instances_cpu import TABLE, host_instances, ihost, scene, scene_rig  # noqa: F401
from test_gpu_multiview import _frames, _rig2, _same
from test_multiview_cpu import BARREL, KM

pytestmark = pytest.mark.gpu

ROW_KEYS = ("R", "t", "corners_px")


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("n_cams", [1, 2, 4])
def test_kernel_equals_harness(ihost, n_cams, distorted):
    rng = np.random.default_rng(500 + n_cams + distorted)
    rig = scene_rig(rng, n_cams, distorted)
    caps = [scene(rng, rig, M=12) for _ in range(5)]
    uv, cls, count = (np.concatenate([c[i] for c in caps]) for i in range(3))
    d = _host(utils.fuse_instances_batched(TABLE, uv, cls, count, rig))
    h = host_instances(ihost, rig, uv, cls, count)                       # step 1 on the host: within a tolerance
    assert np.abs(d["R"] - h["R"]).max() < 1e-6 and np.abs(d["t"] - h["t"]).max() < 1e-6
    h = host_instances(ihost, rig, uv, cls, count, rows=(d["R"], d["t"]))  # from the device's rows: the fusion bit for bit
    for k in h:
        if k not in ROW_KEYS:
            assert np.array_equal(d[k], h[k]), k
    empty = np.arange(12)[None] >= count[:, None]
    assert (d["R"][empty] == 0).all() and (d["corners_px"][empty] == 0).all()
    assert d["world_count"].sum() >= 5


def test_a_capture_alone_equals_the_batch(ihost):
    rng = np.random.default_rng(9)
    rig = scene_rig(rng, 3, True)
    caps = [scene(rng, rig, M=10) for _ in range(4)]
    uv, cls, count = (np.concatenate([c[i] for c in caps]) for i in range(3))
    d = _host(utils.fuse_instances_batched(TABLE, uv, cls, count, rig))
    for g in (0, 3):
        s = slice(3 * g, 3 * g + 3)
        one = _host(utils.fuse_instances_batched(TABLE, uv[s], cls[s], count[s], rig))
        for k in one:
            want = d[k][s] if one[k].shape[0] == 3 else d[k][g:g + 1]
            assert np.array_equal(one[k], want), (g, k)
    with pytest.raises(SspError):
        utils.fuse_instances_batched(TABLE, uv[:4], cls[:4], count[:4], rig)
    with pytest.raises(SspError):
        utils.fuse_instances_batched(TABLE, uv, cls, count, rig, gate=4.0)


# ---------------------------------------------------------------------------------------------------- the predictor
@pytest.mark.parametrize("distorted", [False, True])
def test_instance_predictor_with_a_rig(cfg_path, distorted):
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(distorted)
    fr = _frames(4, 3)
    kw = dict(shape=(416, 416), batch=4, conf_thresh=0.5, max_instances=32)
    pred = InstancePosePredictor(m, {0: CORNERS}, None, rig=rig, **kw)
    r = _host(pred(fr))
    assert r["count"].min() >= 2
    for c in range(2):                                                    # each row as a single-camera predictor sees it
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        one = _host(InstancePosePredictor(m, {0: CORNERS}, rig.K[c], dist_coeffs=k, **kw)(fr))
        for key in one:
            assert np.array_equal(r[key][c::2], one[key][c::2]), (c, key)
    P9c = np.concatenate([np.zeros((1, 3)), CORNERS[:3].T]).astype(np.float32)[None]
    want = _host(utils.fuse_instances_batched(P9c, r["keypoints_px"], r["cls"], r["count"], rig))
    for key in want:
        assert np.array_equal(r[key], want[key]), key
    assert (r["world_count"] >= 1).all()
    assert _same(_host(InstancePosePredictor(m, {0: CORNERS}, None, rig=rig, graph=False, **kw)(fr)), r)
    # one detection per view: the first world instance is ssp_fuse_views' fused pose
    r1 = _host(InstancePosePredictor(m, {0: CORNERS}, None, rig=rig, **dict(kw, max_instances=1))(fr))
    f = _host(utils.fuse_views_batched(P9c[0], r1["keypoints_px"][:, 0], rig, r1["count"] > 0))
    for g in range(2):
        if f["fuse_status"][g] & 3:
            assert r1["world_count"][g] == 0
            continue
        assert np.array_equal(r1["R_world"][g, 0], f["R_world"][g]) and np.array_equal(r1["t_world"][g, 0], f["t_world"][g])
        assert np.array_equal(r1["world_cov"][g, 0], f["world_cov"][g]) and np.array_equal(r1["members"][g, 0] >= 0, f["views"][g])
        assert r1["fuse_hyp"][g, 0] == f["fuse_hyp"][g]                  # M = 1: c M + m = c


def test_full_slots_of_a_random_network(cfg_multi_path):
    """the worst case: a random multi-object network at conf_thresh 0.02 fills every slot"""
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    objects = {c: utils.get_3D_corners(np.c_[np.random.default_rng(c).normal(0, 0.04, (50, 3)), np.ones((50, 1))].T) for c in (0, 3, 7)}
    rig = _rig2(True)
    fr = _frames(2, 8)
    pred = InstancePosePredictor(m, objects, None, batch=2, conf_thresh=0.02, max_instances=32, rig=rig)
    r = _host(pred(fr))
    assert (r["count"] == 32).all()
    for c in range(2):
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        one = _host(InstancePosePredictor(m, objects, rig.K[c], batch=2, conf_thresh=0.02, max_instances=32, dist_coeffs=k)(fr))
        for key in one:
            assert np.array_equal(r[key][c], one[key][c]), (c, key)
    table = np.zeros((m.num_classes, 9, 3), np.float32)
    for c, corners in objects.items():
        table[c, 1:] = corners[:3].T
    want = _host(utils.fuse_instances_batched(table, r["keypoints_px"], r["cls"], r["count"], rig))
    for key in want:
        assert np.array_equal(r[key], want[key]), key
    assert r["world_count"][0] + r["unfused"][0] <= 64
    assert _same(_host(InstancePosePredictor(m, objects, None, batch=2, conf_thresh=0.02, max_instances=32, rig=rig, graph=False)(fr)), r)


def test_refusals(cfg_path):
    from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(False)
    for bad in (dict(K=KM), dict(dist_coeffs=BARREL), dict(pnp="consensus"), dict(batch=3), dict(meshes={0: (np.zeros((3, 3)), np.zeros((1, 3), int))})):
        kw = dict(K=None, shape=(416, 416), batch=4, conf_thresh=0.5, rig=rig)
        kw.update(bad)
        with pytest.raises(SspError):
            InstancePosePredictor(m, {0: CORNERS}, **kw)
    with pytest.raises(TypeError):
        TrackingPosePredictor(m, {0: CORNERS}, None, shape=(416, 416), batch=4, rig=rig)


def test_cli_rig_writes_what_the_predictor_returns(cfg_path, tmp_path):
    """predict_instances --rig on two captures of a two-camera rig: every .npz column equals the flattened outputs of
    InstancePosePredictor(rig=...) on the same images"""
    from PIL import Image
    from singleshotpose_b200.predict import mesh_corners
    from singleshotpose_b200.predict_instances import ROW_KEYS as CLI_ROWS, WORLD_KEYS, InstancePosePredictor, main
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
    fr = _frames(4, 21)
    paths = []
    for i in range(4):
        paths.append(str(tmp_path / ("img%d.png" % i)))
        Image.fromarray(fr[i]).save(paths[-1])
    out = str(tmp_path / "world.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf, "--out", out, "--max-instances", "16", "--rig", rig_path] + paths)
    got = np.load(out)
    pred = InstancePosePredictor(m, {0: mesh_corners(ply)}, None, frame_size=(640, 480), batch=2, max_instances=16, rig=rig)
    rows = {k: [] for k in CLI_ROWS + ("world_index",)}
    world = {k: [] for k in WORLD_KEYS}
    image, capture = [], []
    for g in range(2):
        r = pred(fr[2 * g:2 * g + 2], to_host=True)
        for b in range(2):
            n = int(r["count"][b])
            image += [2 * g + b] * n
            for k in rows:
                rows[k].append(r[k][b, :n])
        n = int(r["world_count"][0])
        capture += [g] * n
        for k in world:
            world[k].append(r[k][0, :n])
    assert list(got["paths"]) == paths
    assert np.array_equal(got["image"], np.array(image, np.int64)) and np.array_equal(got["capture"], np.array(capture, np.int64))
    assert len(image) >= 4 and len(capture) >= 2
    for k, v in list(rows.items()) + list(world.items()):
        assert np.array_equal(got[k], np.concatenate(v)), k
    assert (got["world_index"] >= 0).any()
