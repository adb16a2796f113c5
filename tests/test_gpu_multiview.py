"""GPU checks of the multi-view fusion: ssp_fuse_views against the host harness (tests/helpers/multiview_host.cpp) on the CPU tests'
rigs, every row's solve and projection against ssp_pnp_batched / ssp_pnp_dist and ssp_project_points(_dist), batch
independence, and PosePredictor / MultiPosePredictor with a rig (per-row outputs equal to one single-camera predictor per camera,
fused outputs equal to utils.fuse_views_batched, graph replay equal to eager launches, the one-camera identity rig)."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import utils
from singleshotpose_b200._lib import SspError
from test_multiview_cpu import BARREL, KM, P9, host, host_fuse, observe, random_object, random_rig  # noqa: F401

pytestmark = pytest.mark.gpu


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


def _scenes(n_cams, distorted, G, seed):
    rng = np.random.default_rng(seed)
    rig = random_rig(rng, n_cams, distorted)
    uv = np.concatenate([observe(rig, *random_object(rng), rng) for _ in range(G)])
    if G > 2:
        uv[n_cams + 1] += 90.0                                              # a shifted view in capture 1
    valid = np.ones(len(uv), bool)
    if G > 3:
        valid[3 * n_cams] = False
    return rig, uv, valid


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("n_cams", [1, 2, 4])
def test_kernel_equals_harness(host, n_cams, distorted):
    rig, uv, valid = _scenes(n_cams, distorted, 8, 100 + n_cams + distorted)
    d = _host(utils.fuse_views_batched(P9, uv, rig, valid))
    h = host_fuse(host, rig, uv, valid)                                   # step 1 on the host: within a tolerance
    assert np.abs(d["R"] - h["R"]).max() < 1e-6 and np.abs(d["t"] - h["t"]).max() < 1e-6
    h = host_fuse(host, rig, uv, valid, rows=(d["R"], d["t"]))            # from the device's rows: the fusion stages bit for bit
    for k in ("R_world", "t_world", "world_cov", "views", "view_err", "fuse_hyp", "fuse_status", "corners_world_px"):
        assert np.array_equal(d[k], h[k]), k
    assert (d["fuse_status"] == 0).sum() >= 7


@pytest.mark.parametrize("distorted", [False, True])
def test_rows_equal_the_single_camera_kernels(distorted):
    n_cams = 3
    rig, uv, valid = _scenes(n_cams, distorted, 4, 7)
    d = _host(utils.fuse_views_batched(P9, uv, rig, valid))
    X = np.concatenate([P9.T, np.ones((1, 9), np.float32)])
    for c in range(n_cams):
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        rows = slice(c, None, n_cams)
        R, t = (x.cpu().numpy() for x in utils.pnp_batched(P9, uv[rows], rig.K[c].astype(np.float32), dist_coeffs=k))
        assert np.array_equal(d["R"][rows], R) and np.array_equal(d["t"][rows], t), c
        px = utils.project_points_batched(X, np.concatenate([R, t[:, :, None]], 2), rig.K[c], dist_coeffs=k).cpu().numpy()
        assert np.array_equal(d["corners_px"][rows], px.transpose(0, 2, 1)), c


def test_a_capture_alone_equals_the_batch():
    rig, uv, valid = _scenes(3, True, 6, 11)
    d = _host(utils.fuse_views_batched(P9, uv, rig, valid))
    for g in (0, 1, 5):
        s = slice(3 * g, 3 * g + 3)
        one = _host(utils.fuse_views_batched(P9, uv[s], rig, valid[s]))
        for k in one:
            want = d[k][s] if k in ("R", "t", "corners_px", "corners_world_px") else d[k][g:g + 1]
            assert np.array_equal(one[k], want), (g, k)
    with pytest.raises(SspError):
        utils.fuse_views_batched(P9, uv[:4], rig)
    with pytest.raises(SspError):
        utils.fuse_views_batched(P9, uv, rig, gate=4.0)


# ---------------------------------------------------------------------------------------------------- the predictors
def _frames(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, 480, 640, 3), dtype=np.uint8)


def _rig2(distorted):
    R1 = utils_so3(np.array([0.0, 1.2, 0.1]))
    return utils.camera_rig([KM, KM * np.array([[1.01, 1, 1], [1, 0.99, 1], [1, 1, 1]])], [np.eye(3), R1], [np.zeros(3), [-0.5, 0.0, 0.3]],
                            [BARREL, None] if distorted else None)


def utils_so3(w):
    from oracle.pose_filter_ref import so3_exp
    return so3_exp(w)


@pytest.mark.parametrize("distorted", [False, True])
def test_pose_predictor_with_a_rig(cfg_path, distorted):
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(distorted)
    fr = _frames(4, 3)
    fr[2:] = fr[:2]                                                       # capture 1 repeats capture 0's frames
    pred = PosePredictor(m, CORNERS, None, shape=(416, 416), batch=4, rig=rig, conf_thresh=0.0)
    r = _host(pred(fr))
    for c in range(2):                                                    # each row as a single-camera predictor sees it
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        one = _host(PosePredictor(m, CORNERS, rig.K[c], shape=(416, 416), batch=4, dist_coeffs=k)(fr))
        for key in one:
            assert np.array_equal(r[key][c::2], one[key][c::2]), (c, key)
    P9c = np.concatenate([np.zeros((1, 3)), CORNERS[:3].T]).astype(np.float32)
    want = _host(utils.fuse_views_batched(P9c, r["keypoints_px"], rig, r["conf"] > 0.0))
    for key in want:
        assert np.array_equal(r[key], want[key]), key
    assert np.array_equal(r["R_world"][0], r["R_world"][1])
    assert _same(_host(PosePredictor(m, CORNERS, None, shape=(416, 416), batch=4, rig=rig, conf_thresh=0.0, graph=False)(fr)), r)
    # a one-camera identity rig: the fused pose is the frame's pose
    ident = utils.camera_rig([KM], [np.eye(3)], [np.zeros(3)])
    r1 = _host(PosePredictor(m, CORNERS, None, shape=(416, 416), batch=2, rig=ident, conf_thresh=0.0)(fr[:2]))
    assert np.array_equal(r1["R_world"], r1["R"]) and np.array_equal(r1["t_world"], r1["t"]) and (r1["fuse_status"] == 0).all()
    for bad in (dict(K=KM, rig=rig), dict(K=None, rig=rig, dist_coeffs=BARREL), dict(K=None, rig=rig, pnp="consensus"),
                dict(K=None, rig=rig, batch=3)):
        kw = dict(shape=(416, 416), batch=4, conf_thresh=0.0)
        kw.update(bad)
        with pytest.raises(SspError):
            PosePredictor(m, CORNERS, **kw)


def _same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


def test_multi_predictor_with_a_rig(cfg_multi_path):
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    objects = {c: utils.get_3D_corners(np.c_[np.random.default_rng(c).normal(0, 0.04, (50, 3)), np.ones((50, 1))].T) for c in (0, 3, 7)}
    rig = _rig2(True)
    fr = _frames(2, 8)
    pred = MultiPosePredictor(m, objects, None, batch=2, conf_thresh=0.02, rig=rig)
    r = _host(pred(fr))
    for c in range(2):
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        one = _host(MultiPosePredictor(m, objects, rig.K[c], batch=2, conf_thresh=0.02, dist_coeffs=k)(fr))
        for key in one:
            assert np.array_equal(r[key][c] if key != "classes" else r[key], one[key][c] if key != "classes" else one[key]), (c, key)
    P3 = np.stack([np.concatenate([np.zeros((1, 3)), objects[c][:3].T]) for c in (0, 3, 7)]).astype(np.float32)
    want = _host(utils.fuse_views_batched(np.broadcast_to(P3, (2, 3, 9, 3)).copy(), r["keypoints_px"], rig, r["detected"]))
    for key in want:
        assert np.array_equal(r[key], want[key]), key
    assert _same(_host(MultiPosePredictor(m, objects, None, batch=2, conf_thresh=0.02, rig=rig, graph=False)(fr)), r)
    with pytest.raises(SspError):
        MultiPosePredictor(m, objects, None, batch=2, conf_thresh=0.02, rig=rig, meshes={})
