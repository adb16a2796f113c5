"""GPU checks of the depth refinement: ssp_refine_depth against the host harness (tests/helpers/refine_depth_host.cpp) on the CPU
tests' rendered scenes, counted groups, batch independence, utils.refine_depth_batched with host and device depth, the three
predictors with meshes (unchanged existing outputs, R_ref / t_ref equal to refine_depth_batched, graph replay, depth sources,
empty slots, argument checks) and the command lines' --depth-dir."""
import os

import numpy as np
import pytest
import torch

from singleshotpose_b200 import synth, utils
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from test_refine_depth_cpu import DIAM, KM, MODEL, SCALE, F, V, host, host_refine, perturb, scene_depth, scene_set  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
NC = 13


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def kernel_refine(depth, R, t, per_group=1, count=None, dist=None, iters=10, gate=(0.5, 0.02), model=MODEL, diam=DIAM):
    """ssp_refine_depth over one class: depth (groups, H, W) uint16, R (n, 3, 3), t (n, 3) -> host arrays"""
    depth = np.ascontiguousarray(depth, np.uint16)
    n, (groups, H, W) = len(R), depth.shape
    D = _d(depth.view(np.int16))
    args = [_d(np.asarray(model, np.float64)), _d(np.array([0, len(model)], np.int32)), _d(np.array([diam]))]
    cls = torch.zeros(n, dtype=torch.int32, device=DEV)
    Rd, td = _d(np.asarray(R, np.float64)), _d(np.asarray(t, np.float64))
    Ro, to = torch.empty_like(Rd), torch.empty_like(td)
    pts, st = torch.empty(n, dtype=torch.int32, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV)
    rmse = torch.empty(n, dtype=torch.float64, device=DEV)
    cnt = None if count is None else _d(np.asarray(count, np.int32))
    kd = None if dist is None else _d(np.asarray(dist, np.float64))
    call("ssp_refine_depth", ptr(D), W, H, SCALE, ptr(_d(KM)), ptr(kd), *map(ptr, args), 1, ptr(cls), groups, per_group, ptr(cnt), ptr(Rd),
         ptr(td), iters, gate[0], gate[1], ptr(Ro), ptr(to), ptr(pts), ptr(rmse), ptr(st), stream_ptr())
    torch.cuda.synchronize()
    return Ro.cpu().numpy(), to.cpu().numpy(), pts.cpu().numpy(), rmse.cpu().numpy(), st.cpu().numpy()


# ---------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("kind", ["plain", "plane", "occluder", "holes"])
def test_kernel_equals_harness(host, kind, distorted):
    """every output bit for bit (sin and cos of so3_exp could in principle round differently in the device's libm; on these
    scenes they do not)"""
    depth, R0, t0, _Rs, _ts, dist = scene_set(kind, distorted)
    h = host_refine(host, depth, MODEL, R0, t0, DIAM, dist=dist)
    k = kernel_refine(depth, R0, t0, dist=dist)
    assert (h[4] == 0).all()
    assert all(np.array_equal(k[j], h[j]) for j in range(5))


def test_counted_groups_and_batch_independence(host):
    depth, R0, t0, _Rs, _ts, _dist = scene_set("plane", False)
    rng = np.random.default_rng(7)
    # 256 problems: each of the 4 frames with 64 perturbed poses of its object
    Rs, ts = synth.object_poses(4, seed=3)
    pairs = [perturb(Rs[i // 64], ts[i // 64], rng) for i in range(256)]
    R, t = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    full = kernel_refine(depth, R, t, per_group=64)
    assert (full[4] == 0).mean() > 0.9
    for i in range(256):
        one = kernel_refine(depth[i // 64:i // 64 + 1], R[i:i + 1], t[i:i + 1])
        assert all(np.array_equal(one[j][0], full[j][i]) for j in range(5)), i
    cnt = kernel_refine(depth, R, t, per_group=64, count=[64, 3, 0, 10])
    for g, c in enumerate([64, 3, 0, 10]):
        sl = slice(64 * g, 64 * g + c)
        assert all(np.array_equal(cnt[j][sl], full[j][sl]) for j in range(5))
        empty = slice(64 * g + c, 64 * (g + 1))
        assert all(not cnt[j][empty].any() for j in range(5))


def test_refine_depth_batched_host_and_device_depth():
    depth, R0, t0, Rs, ts, _dist = scene_set("occluder", False)
    a = utils.refine_depth_batched(depth, V, F, KM, R0, t0)
    b = utils.refine_depth_batched(_d(depth), V, F, KM, _d(R0), _d(t0))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert utils.mesh_diameter(V) == DIAM
    k = kernel_refine(depth, R0, t0, model=np.c_[V, utils.vertex_normals(V, F)])
    assert all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(a, k))
    with pytest.raises(SspError):
        utils.refine_depth_batched(depth.astype(np.int32), V, F, KM, R0, t0)
    with pytest.raises(SspError):
        utils.refine_depth_batched(depth, V, F, KM, R0[:2], t0[:2])
    with pytest.raises(SspError):
        utils.refine_depth_batched(depth, V, F, KM, R0, t0, gate=(0.02, 0.5))


# ---------------------------------------------------------------------------------------------------- the predictors
CORNERS = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
POSE = (synth._rodrigues(np.array([0.3, -0.2, 0.1])), np.array([-0.315, -0.235, 0.6]))


def _posed_model(cfg_path):
    """a single-object network whose constant logits decode, at cell (0, 0), the projection of the mesh's box under POSE (the
    construction of test_gpu_predict.py): the predicted pose is close to POSE, so the refinement has a scene to work on"""
    from singleshotpose_b200.darknet import Darknet
    torch.manual_seed(0)
    m = Darknet(cfg_path)
    last = m.models[30][0]
    R, t = POSE
    P = np.concatenate([np.zeros((3, 1)), CORNERS[:3]], 1)
    cam = KM @ (R @ P + t[:, None])
    uv = cam[:2] / cam[2]
    gx, gy = uv[0] / 640 * 13, uv[1] / 480 * 13
    assert 0 < gx[0] < 1 and 0 < gy[0] < 1
    b = np.zeros(20)
    b[0], b[1] = np.log(gx[0] / (1 - gx[0])), np.log(gy[0] / (1 - gy[0]))
    b[2:18:2], b[3:18:2] = gx[1:], gy[1:]
    b[18] = 2.0
    with torch.no_grad():
        last.weight.zero_()
        last.bias.copy_(torch.from_numpy(b).float())
    return m.cuda().eval()


def _frames(n, seed, w=640, h=480):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


def _same(a, b, keys=None):
    return all(np.array_equal(a[k], b[k]) for k in (keys or a))


def test_pose_predictor_refines(cfg_path):
    from singleshotpose_b200.predict import PosePredictor
    m = _posed_model(cfg_path)
    R, t = POSE
    fr = _frames(2, seed=5)
    depth = np.stack([scene_depth(R, t, plane=True, seed=1), scene_depth(R, t, noise=True, seed=2)])
    plain = _host(PosePredictor(m, CORNERS, KM, shape=(416, 416), batch=2)(fr))
    pred = PosePredictor(m, CORNERS, KM, shape=(416, 416), batch=2, mesh=(V, F))
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys())
    assert set(r) - set(plain) == {"R_ref", "t_ref", "corners_ref_px", "refine_points", "refine_rmse", "refine_status"}
    want = [x.cpu().numpy() for x in utils.refine_depth_batched(depth, V, F, KM, r["R"], r["t"])]
    for k, w in zip(("R_ref", "t_ref", "refine_points", "refine_rmse", "refine_status"), want):
        assert np.array_equal(r[k], w), k
    assert (r["refine_status"] == 0).all() and (r["refine_points"] > 1000).all()
    assert np.abs(r["t_ref"] - t).max() < 2e-3
    X = np.concatenate([np.concatenate([np.zeros((3, 1)), CORNERS[:3]], 1), np.ones((1, 9))]).astype(np.float32)
    for b in range(2):
        Rt = np.c_[r["R_ref"][b], r["t_ref"][b]][None]
        assert np.array_equal(r["corners_ref_px"][b], utils.project_points_batched(X, Rt, KM)[0].cpu().numpy().T)
    # graph replay = eager; host depth = device depth; the depth is read in place on every replay
    eager = _host(PosePredictor(m, CORNERS, KM, shape=(416, 416), batch=2, mesh=(V, F), graph=False)(fr, depth=depth))
    assert _same(eager, r)
    assert _same(_host(pred(torch.from_numpy(fr).to(DEV), depth=_d(depth))), r)
    swapped = _host(pred(fr, depth=depth[::-1].copy()))            # each replay reads the call's own depth
    assert _same(swapped, r, plain.keys()) and not np.array_equal(swapped["refine_rmse"], r["refine_rmse"])
    assert _same(_host(pred(fr, depth=depth)), r)
    # refused before any launch
    for bad in (None, depth[:, :-1], depth.astype(np.int32), depth[:1]):
        with pytest.raises(SspError):
            pred(fr, depth=bad)
    with pytest.raises(SspError):
        PosePredictor(m, CORNERS, KM, shape=(416, 416), batch=2)(fr, depth=depth)


def _meshes():
    out = {}
    for c in range(NC):
        Vc, Fc = synth.closed_mesh(rings=12, segments=20, half_extents=(0.03 + 0.003 * c, 0.04, 0.05 - 0.002 * c), seed=c)
        out[c] = (Vc, Fc)
    return out


def _random_depth(B, seed):
    rng = np.random.default_rng(seed)
    D = rng.integers(500, 1500, size=(B, 480, 640)).astype(np.uint16)
    D[rng.random(D.shape) < 0.3] = 0
    return D


def test_multi_predictor_refines(cfg_multi_path):
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    meshes = _meshes()
    objects = {c: utils.get_3D_corners(np.c_[v, np.ones((len(v), 1))].T) for c, (v, _f) in meshes.items()}
    make = lambda **kw: MultiPosePredictor(m, objects, KM, batch=2, conf_thresh=0.02, **kw)
    fr, depth = _frames(2, seed=9), _random_depth(2, 3)
    plain = _host(make()(fr))
    pred = make(meshes=meshes)
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys())
    assert _same(_host(make(meshes=meshes, graph=False)(fr, depth=depth)), r)
    assert _same(_host(pred(torch.from_numpy(fr).to(DEV), depth=_d(depth))), r)
    for c in range(NC):                                                 # slot c of both frames in one call
        want = utils.refine_depth_batched(depth, *meshes[c], KM, r["R"][:, c], r["t"][:, c])
        for k, w in zip(("R_ref", "t_ref", "refine_points", "refine_rmse", "refine_status"), want):
            assert np.array_equal(r[k][:, c], w.cpu().numpy()), (c, k)
    with pytest.raises(SspError):
        make(meshes={3: meshes[3]})                                  # a mesh for every requested class
    with pytest.raises(SspError):
        pred(fr)


def test_instance_predictor_refines(cfg_path):
    """the posed single-object network lists the same box at every cell, shifted by whole cells; suppression keeps fewer than
    the 256 slots, so empty slots are checked too"""
    from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor
    m = _posed_model(cfg_path)
    R, t = POSE
    make = lambda **kw: InstancePosePredictor(m, {0: CORNERS}, KM, shape=(416, 416), batch=2, conf_thresh=0.5, max_instances=256, **kw)
    fr = _frames(2, seed=5)
    depth = np.stack([scene_depth(R, t, plane=True, seed=1), scene_depth(R, t, occluder=True, seed=2)])
    plain = _host(make()(fr))
    pred = make(meshes={0: (V, F)})
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys())
    assert _same(_host(make(meshes={0: (V, F)}, graph=False)(fr, depth=depth)), r)
    assert _same(_host(pred(torch.from_numpy(fr).to(DEV), depth=_d(depth))), r)
    filled = np.arange(256)[None] < r["count"][:, None]
    assert filled.any() and (~filled).any()
    b, s = np.nonzero(filled)
    want = utils.refine_depth_batched(depth[b], V, F, KM, r["R"][b, s], r["t"][b, s])
    for k, w in zip(("R_ref", "t_ref", "refine_points", "refine_rmse", "refine_status"), want):
        assert np.array_equal(r[k][b, s], w.cpu().numpy()), k
    assert (r["refine_status"][:, 0] == 0).all() and np.abs(r["t_ref"][:, 0] - t).max() < 2e-3      # instance 0 is the object
    for k in ("R_ref", "t_ref", "corners_ref_px", "refine_points", "refine_rmse", "refine_status"):
        assert not r[k][~filled].any(), k
    with pytest.raises(SspError):
        TrackingPosePredictor(m, {0: CORNERS}, KM, shape=(416, 416), conf_thresh=0.5, meshes={0: (V, F)})
    with pytest.raises(SspError):
        utils_multi_tracker({0: CORNERS}, {0: (V, F)})
    with pytest.raises(SspError):
        pred(fr, depth=depth[:, :, :-1])


def utils_multi_tracker(objects, meshes):
    from singleshotpose_b200.utils_multi import InstanceTracker
    return InstanceTracker(objects, KM, 1, 1, (640, 480), meshes=meshes)


# ---------------------------------------------------------------------------------------------------- command line
def test_cli_depth_dir(cfg_path, tmp_path):
    from PIL import Image
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.predict import PosePredictor, main
    m = _posed_model(cfg_path)
    wf = str(tmp_path / "m.weights")
    m.save_weights(wf)
    ply = str(tmp_path / "obj.ply")
    synth.write_ply(ply, V, F)
    data = tmp_path / "obj.data"
    data.write_text("mesh = %s\nwidth = 640\nheight = 480\nfx = %.17g\nfy = %.17g\nu0 = %.17g\nv0 = %.17g\n" % (ply, KM[0, 0], KM[1, 1], KM[0, 2], KM[1, 2]))
    img, ddir = tmp_path / "img", tmp_path / "depth"
    img.mkdir(); ddir.mkdir()
    paths, depths = [], []
    for i in range(2):
        p = str(img / ("%06d.jpg" % i))
        Image.fromarray(_frames(1, seed=30 + i)[0]).save(p, quality=95)
        paths.append(p)
        D = scene_depth(*POSE, plane=i == 1, seed=i)
        Image.fromarray(D).save(str(ddir / ("%06d.png" % i)))
        depths.append(D)
    base = ["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf]
    out0, out1 = str(tmp_path / "p0.npz"), str(tmp_path / "p1.npz")
    main(base + ["--out", out0] + paths)
    main(base + ["--out", out1, "--depth-dir", str(ddir)] + paths)
    g0, g1 = np.load(out0), np.load(out1)
    assert sorted(g0.files) == sorted(["paths", "R", "t", "conf", "keypoints_px", "corners_px"])
    assert sorted(g1.files) == sorted(g0.files + ["R_ref", "t_ref", "corners_ref_px", "refine_points", "refine_rmse", "refine_status"])
    m2 = Darknet(cfg_path)
    m2.load_weights(wf)
    m2.cuda().eval()
    pred = PosePredictor(m2, CORNERS, KM, mesh=(V, F))
    for i, p in enumerate(paths):
        r = pred([open(p, "rb").read()], to_host=True, depth=depths[i][None])
        for k in g1.files:
            if k != "paths":
                assert np.array_equal(g1[k][i], r[k][0]), (p, k)
        for k in g0.files:
            if k != "paths":
                assert np.array_equal(g0[k][i], g1[k][i]), k
    os.remove(str(ddir / "000001.png"))
    with pytest.raises(SspError, match="000001.png"):
        main(base + ["--out", out1, "--depth-dir", str(ddir)] + paths)
    Image.fromarray(depths[1][:-2]).save(str(ddir / "000001.png"))
    with pytest.raises(SspError, match="000001.png"):
        main(base + ["--out", out1, "--depth-dir", str(ddir)] + paths)
