"""GPU checks of the rig refinement: ssp_refine_depth_rig against the host harness (tests/helpers/refine_rig_host.cpp) on the CPU
tests' rendered scenes at 1-4, 9 and 16 cameras, the one-camera identity rig against ssp_refine_depth, batch independence and
repeatability, utils.refine_depth_rig_batched with host and device depth, PosePredictor / MultiPosePredictor with a rig and meshes
(unchanged existing outputs, the refined world poses equal to refine_depth_rig_batched of the predictor's own fused poses,
corners_world_ref_px, graph replay) and the predict --rig --depth-dir command line."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import synth, utils
from singleshotpose_b200._lib import call, ptr, stream_ptr
from test_refine_depth_cpu import DIAM, KM, MODEL, SCALE, F, V, scene_set
from test_refine_rig_cpu import BARREL, BOX, host_refine_rig, make_rig, perturb_world, random_pose, rig_depth, rig_host  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ("R", "t", "points", "rmse", "status", "view_points", "view_rmse", "corners")


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def kernel_refine_rig(rig, depth, R, t, slots=1, count=None, fuse_status=None, iters=10, gate=(0.5, 0.02)):
    """ssp_refine_depth_rig over one class: depth (G C, H, W), R (G S, 3, 3), t (G S, 3) -> dict of host arrays (host_refine_rig's)"""
    Cn = len(rig.K)
    depth = np.ascontiguousarray(depth, np.uint16)
    B, H, W = depth.shape
    G, n = B // Cn, len(R)
    assert n == G * slots
    dd = lambda a, dt=np.float64: _d(np.asarray(a, dt))
    o = dict(R=torch.empty(n, 3, 3, dtype=torch.float64, device=DEV), t=torch.empty(n, 3, dtype=torch.float64, device=DEV),
             points=torch.empty(n, dtype=torch.int32, device=DEV), rmse=torch.empty(n, dtype=torch.float64, device=DEV),
             status=torch.empty(n, dtype=torch.int32, device=DEV), view_points=torch.empty(n, Cn, dtype=torch.int32, device=DEV),
             view_rmse=torch.empty(n, Cn, dtype=torch.float64, device=DEV),
             corners=torch.empty(B, slots, len(BOX), 2, dtype=torch.float32, device=DEV))
    keep = [_d(depth.view(np.int16)), dd(rig.K), None if rig.dist is None else dd(rig.dist), dd(rig.R), dd(rig.t), dd(MODEL),
            dd([0, len(MODEL)], np.int32), dd([DIAM]), dd(BOX, np.float32), torch.zeros(n, dtype=torch.int32, device=DEV),
            None if count is None else dd(count, np.int32), None if fuse_status is None else dd(fuse_status, np.int32), dd(R), dd(t)]
    D, K, Dd, Rr, tr, model, off, dm, table, cls, cnt, fs, Rd, td = keep
    call("ssp_refine_depth_rig", ptr(D), W, H, SCALE, Cn, ptr(K), ptr(Dd), ptr(Rr), ptr(tr), ptr(model), ptr(off), ptr(dm), ptr(table),
         len(BOX), 1, ptr(cls), G, slots, ptr(cnt), ptr(fs), ptr(Rd), ptr(td), iters, gate[0], gate[1], *(ptr(o[k]) for k in KEYS),
         stream_ptr())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


# ---------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("n_cams", [2, 3, 4])
def test_kernel_equals_harness(rig_host, n_cams, distorted):
    """every output bit for bit on every scene problem; the four scenes of one rig run as four captures of one call"""
    rng = np.random.default_rng(50 * n_cams + distorted)
    rig = make_rig(rng, n_cams, distorted)
    truth = [random_pose(rng) for _ in range(4)]
    dep = np.concatenate([rig_depth(rig, R, t, seed=k, **kw) for k, ((R, t), kw) in
                          enumerate(zip(truth, ({}, dict(table=True), dict(table=True, occluder=0.34), dict(holes=True))))])
    starts = [perturb_world(R, t, rng) for R, t in truth]
    R, t = np.stack([p[0] for p in starts]), np.stack([p[1] for p in starts])
    h = host_refine_rig(rig_host, rig, dep, R, t)
    k = kernel_refine_rig(rig, dep, R, t)
    assert (h["status"] == 0).all()
    for key in KEYS:
        assert np.array_equal(k[key], h[key]), key


def test_one_camera(rig_host):
    """C = 1: the harness bit for bit, and with identity extrinsics ssp_refine_depth bit for bit"""
    from test_gpu_refine_depth import kernel_refine
    for distorted in (False, True):
        depth, R0, t0, _Rs, _ts, dist = scene_set("occluder", distorted)
        ident = utils.camera_rig([KM], [np.eye(3)], [np.zeros(3)], None if dist is None else [dist])
        k = kernel_refine_rig(ident, depth, R0, t0)
        h = host_refine_rig(rig_host, ident, depth, R0, t0)
        for key in KEYS:
            assert np.array_equal(k[key], h[key]), key
        one = kernel_refine(depth, R0, t0, dist=dist)
        for j, key in enumerate(("R", "t", "points", "rmse", "status")):
            assert np.array_equal(k[key], one[j]), key
        assert np.array_equal(k["view_points"][:, 0], one[2]) and np.array_equal(k["view_rmse"][:, 0], one[3])


def _big_rig(rng, n_cams):
    """n_cams cameras around the object with every even camera distorted"""
    rig = make_rig(rng, n_cams)
    dist = [BARREL * rng.uniform(0.5, 1.0) if c % 2 == 0 else None for c in range(n_cams)]
    return utils.camera_rig(rig.K, rig.R, rig.t, dist)


@pytest.mark.parametrize("n_cams", [9, 16])
def test_more_cameras_than_ctas(rig_host, n_cams):
    """9 and 16 cameras: a CTA of the 8-CTA cluster takes two cameras.  Bit for bit except that the device's sin and cos in
    so3_exp may round differently from the host's libm: then within 1e-9, with every count equal"""
    rng = np.random.default_rng(n_cams)
    rig = _big_rig(rng, n_cams)
    poses = [random_pose(rng) for _ in range(2)]
    dep = np.concatenate([rig_depth(rig, R, t, table=True, seed=i) for i, (R, t) in enumerate(poses)])
    starts = [perturb_world(R, t, rng) for R, t in poses]
    R, t = np.stack([p[0] for p in starts]), np.stack([p[1] for p in starts])
    h = host_refine_rig(rig_host, rig, dep, R, t)
    k = kernel_refine_rig(rig, dep, R, t)
    assert (h["status"] == 0).all() and (h["view_points"] > 0).sum() >= n_cams
    for key in ("points", "status", "view_points"):
        assert np.array_equal(k[key], h[key]), key
    exact = all(np.array_equal(k[key], h[key]) for key in KEYS)
    print("%d cameras: bit for bit %s" % (n_cams, exact))
    if not exact:
        for key in ("R", "t", "rmse", "view_rmse"):
            assert np.abs(k[key] - h[key]).max() <= 1e-9 * max(np.abs(h[key]).max(), 1e-3), key
        assert np.abs(k["corners"] - h["corners"]).max() <= 1e-3


def test_batch_independence_and_repeatability(rig_host):
    rng = np.random.default_rng(5)
    rig = make_rig(rng, 3, True)
    G, S = 3, 4
    poses = [random_pose(rng) for _ in range(G)]
    dep = np.concatenate([rig_depth(rig, R, t, table=True, seed=g) for g, (R, t) in enumerate(poses)])
    starts = [perturb_world(*poses[i // S], rng) for i in range(G * S)]
    R, t = np.stack([p[0] for p in starts]), np.stack([p[1] for p in starts])
    fs = np.zeros(G * S, np.int32)
    fs[5], fs[6] = 2, 4
    full = kernel_refine_rig(rig, dep, R, t, slots=S, fuse_status=fs)
    again = kernel_refine_rig(rig, dep, R, t, slots=S, fuse_status=fs)
    assert all(np.array_equal(full[k], again[k]) for k in KEYS)
    assert full["status"][5] == 4 and (np.delete(full["status"], 5) == 0).all()
    for i in range(G * S):
        g, s = divmod(i, S)
        one = kernel_refine_rig(rig, dep[3 * g:3 * g + 3], R[i:i + 1], t[i:i + 1], fuse_status=fs[i:i + 1])
        for k in KEYS:
            want = full[k][3 * g:3 * g + 3, s:s + 1] if k == "corners" else full[k][i:i + 1]
            assert np.array_equal(one[k], want), (i, k)
    cnt = kernel_refine_rig(rig, dep, R, t, slots=S, fuse_status=fs, count=[4, 1, 0])
    h = host_refine_rig(rig_host, rig, dep, R, t, slots=S, fuse_status=fs, count=[4, 1, 0])
    assert all(np.array_equal(cnt[k], h[k]) for k in KEYS)


def test_refine_depth_rig_batched_host_and_device_depth():
    rng = np.random.default_rng(9)
    rig = make_rig(rng, 2, True)
    poses = [random_pose(rng) for _ in range(2)]
    dep = np.concatenate([rig_depth(rig, R, t, table=True, seed=g) for g, (R, t) in enumerate(poses)])
    starts = [perturb_world(R, t, rng) for R, t in poses]
    R, t = np.stack([p[0] for p in starts]), np.stack([p[1] for p in starts])
    a = utils.refine_depth_rig_batched(dep, V, F, rig, R, t)
    b = utils.refine_depth_rig_batched(_d(dep), V, F, rig, _d(R), _d(t))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    k = kernel_refine_rig(rig, dep, R, t)
    for x, key in zip(a, KEYS):
        assert np.array_equal(x.cpu().numpy(), k[key]), key
    s = utils.refine_depth_rig_batched(dep, V, F, rig, R[:, None], t[:, None], fuse_status=np.zeros((2, 1)))
    assert s[5].shape == (2, 1, 2) and all(np.array_equal(x[:, 0].cpu().numpy(), y.cpu().numpy()) for x, y in zip(s, a))
    from singleshotpose_b200._lib import SspError
    for bad in (dict(depth=dep[:3]), dict(R=R[:1], t=t[:1]), dict(gate=(0.02, 0.5)), dict(depth=dep.astype(np.int32)),
                dict(fuse_status=np.zeros(3))):
        kw = dict(depth=dep, R=R, t=t)
        kw.update(bad)
        with pytest.raises(SspError):
            utils.refine_depth_rig_batched(kw.pop("depth"), V, F, rig, kw.pop("R"), kw.pop("t"), **kw)


# ---------------------------------------------------------------------------------------------------- the predictors
def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


def _same(a, b, keys=None):
    return all(np.array_equal(a[k], b[k]) for k in (keys or a))


def _predictor_depth(rig, R_world, t_world, B, seed):
    """(B, 480, 640) depth of the mesh at each capture's fused world pose in each camera (random depth where the object is not
    wholly in front of the camera)"""
    Cn = len(rig.K)
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        g, c = divmod(b, Cn)
        Rc, tc = rig.R[c] @ R_world[g], rig.R[c] @ t_world[g] + rig.t[c]
        if np.isfinite(Rc).all() and ((V @ Rc.T + tc)[:, 2] > 0.1).all():
            one = utils.camera_rig(rig.K[c:c + 1], [np.eye(3)], [np.zeros(3)], None if rig.dist is None else rig.dist[c:c + 1])
            out.append(rig_depth(one, Rc, tc, noise=True, seed=b)[0])
        else:
            D = rng.integers(500, 1500, size=(480, 640)).astype(np.uint16)
            D[rng.random(D.shape) < 0.3] = 0
            out.append(D)
    return np.stack(out)


REF_KEYS = {"R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points", "refine_view_rmse",
            "corners_world_ref_px"}


@pytest.mark.parametrize("distorted", [False, True])
def test_pose_predictor_with_a_rig_and_a_mesh(cfg_path, distorted):
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_multiview import _frames, _rig2
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(distorted)
    fr = _frames(4, 3)
    make = lambda **kw: PosePredictor(m, CORNERS, None, shape=(416, 416), batch=4, rig=rig, conf_thresh=0.0, **kw)
    plain = _host(make()(fr))
    depth = _predictor_depth(rig, plain["R_world"], plain["t_world"], 4, 1)
    pred = make(mesh=(V, F))
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys()) and set(r) - set(plain) == REF_KEYS
    want = utils.refine_depth_rig_batched(depth, V, F, rig, r["R_world"], r["t_world"], fuse_status=r["fuse_status"])
    for k, w in zip(("R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points",
                     "refine_view_rmse"), want):
        assert np.array_equal(r[k], w.cpu().numpy()), k
    print("refine_status %s, refine_points %s" % (r["refine_status"], r["refine_points"]))
    bad = np.repeat(r["refine_status"] != 0, 2)                             # per frame
    assert np.array_equal(r["corners_world_ref_px"][bad], r["corners_world_px"][bad])
    assert _same(_host(make(mesh=(V, F), graph=False)(fr, depth=depth)), r)
    assert _same(_host(pred(torch.from_numpy(fr).to(DEV), depth=_d(depth))), r)


def test_multi_predictor_with_a_rig_and_meshes(cfg_multi_path):
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    from test_gpu_multiview import _frames, _rig2
    from test_gpu_refine_depth import _meshes
    torch.manual_seed(0)
    m = Darknet(cfg_multi_path).cuda().eval()
    meshes = {c: v for c, v in _meshes().items() if c in (0, 3, 7)}
    objects = {c: utils.get_3D_corners(np.c_[v, np.ones((len(v), 1))].T) for c, (v, _f) in meshes.items()}
    rig = _rig2(True)
    fr = _frames(2, 8)
    make = lambda **kw: MultiPosePredictor(m, objects, None, batch=2, conf_thresh=0.02, rig=rig, **kw)
    plain = _host(make()(fr))
    rng = np.random.default_rng(4)
    depth = rng.integers(500, 1500, size=(2, 480, 640)).astype(np.uint16)
    depth[rng.random(depth.shape) < 0.3] = 0
    pred = make(meshes=meshes)
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys()) and set(r) - set(plain) == REF_KEYS
    assert _same(_host(make(meshes=meshes, graph=False)(fr, depth=depth)), r)
    for q, c in enumerate(sorted(meshes)):
        want = utils.refine_depth_rig_batched(depth, *meshes[c], rig, r["R_world"][:, q], r["t_world"][:, q], fuse_status=r["fuse_status"][:, q])
        for k, w in zip(("R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points",
                         "refine_view_rmse"), want):
            assert np.array_equal(r[k][:, q], w.cpu().numpy()), (c, k)
    bad = np.repeat(r["refine_status"] != 0, 2, axis=0)
    assert np.array_equal(r["corners_world_ref_px"][bad], r["corners_world_px"][bad])


# ---------------------------------------------------------------------------------------------------- command line
def test_cli_rig_depth_dir(cfg_path, tmp_path):
    from PIL import Image
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.predict import PosePredictor, main
    from test_gpu_multiview import _frames, _rig2
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    wf = str(tmp_path / "m.weights")
    m.save_weights(wf)
    ply = str(tmp_path / "obj.ply")
    synth.write_ply(ply, V, F)
    data = tmp_path / "obj.data"
    data.write_text("mesh = %s\nwidth = 640\nheight = 480\nfx = %.17g\nfy = %.17g\nu0 = %.17g\nv0 = %.17g\n" % (ply, KM[0, 0], KM[1, 1], KM[0, 2], KM[1, 2]))
    rig = _rig2(True)
    rp = str(tmp_path / "rig.npz")
    np.savez(rp, K=rig.K, R=rig.R, t=rig.t, dist=rig.dist)
    img, ddir = tmp_path / "img", tmp_path / "depth"
    img.mkdir()
    ddir.mkdir()
    fr = _frames(4, 12)
    depth = np.random.default_rng(2).integers(500, 1500, size=(4, 480, 640)).astype(np.uint16)
    paths = []
    for i in range(4):
        p = str(img / ("%06d.png" % i))
        Image.fromarray(fr[i]).save(p)
        Image.fromarray(depth[i]).save(str(ddir / ("%06d.png" % i)))
        paths.append(p)
    out = str(tmp_path / "p.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf, "--rig", rp, "--depth-dir", str(ddir), "--out", out] + paths)
    g = np.load(out)
    m2 = Darknet(cfg_path)
    m2.load_weights(wf)
    m2.cuda().eval()
    pred = PosePredictor(m2, CORNERS, None, frame_size=(640, 480), rig=utils_host_rig(rp), batch=2, mesh=(V, F))
    assert REF_KEYS <= set(g.files) and "R_ref" not in g.files
    for cap in range(2):
        r = pred(fr[2 * cap:2 * cap + 2], to_host=True, depth=depth[2 * cap:2 * cap + 2])
        for k in REF_KEYS | {"R_world", "t_world", "corners_world_px"}:
            n = 2 if k.startswith("corners") else 1
            assert np.array_equal(g[k][n * cap:n * cap + n], r[k]), (cap, k)


def utils_host_rig(path):
    from singleshotpose_b200.utils_host import read_rig
    return read_rig(path)
