"""GPU checks of the refinement of a rig's world instances: ssp_refine_instances_rig against the host harness
(tests/helpers/refine_instances_host.cpp) on the CPU tests' piles at 1-4, 9 and 16 cameras and with 256 drawn slots in one capture
(every output, instance_map and view_hidden included, bit for bit but for the last-bit differences of sin and cos), a capture alone against the same capture in a batch, two calls,
InstancePosePredictor with a rig and meshes (eager and captured; the refined outputs equal to utils.refine_instances_rig_batched
of the predictor's own fused outputs, every other output equal to the predictor without meshes) and the predict_instances --rig
--depth-dir command line against the predictor."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import synth, utils
from singleshotpose_b200._lib import call, ptr, stream_ptr
from test_refine_depth_cpu import SCALE, F, V
from test_refine_instances_cpu import KEYS, host_refine_instances, mesh_tables, pile_depth, pile_poses, ri_host  # noqa: F401
from test_refine_rig_cpu import make_rig, perturb_world

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def kernel_refine_instances(rig, depth, cls, R, t, meshes=None, count=None, fuse_status=None, iters=10, gate=(0.5, 0.02), num_classes=1):
    """ssp_refine_instances_rig on the harness's tables -> dict of host arrays (host_refine_instances')"""
    meshes = {0: (V, F)} if meshes is None else meshes
    Cn = len(rig.K)
    depth = np.ascontiguousarray(depth, np.uint16)
    B, H, W = depth.shape
    G, M = np.shape(cls)
    model, off, diam, faces, foff, table = mesh_tables(meshes, num_classes)
    dd = lambda a, dt=np.float64: _d(np.asarray(a, dt))
    keep = [_d(depth.view(np.int16)), dd(rig.K), None if rig.dist is None else dd(rig.dist), dd(rig.R), dd(rig.t), dd(model), dd(off, np.int32),
            dd(diam), dd(faces, np.int32), dd(foff, np.int32), dd(table, np.float32), dd(cls, np.int32),
            None if count is None else dd(count, np.int32), None if fuse_status is None else dd(fuse_status, np.int32), dd(R), dd(t)]
    D, K, Dd, Rr, tr, mo, of, dm, fa, fo, tab, cl, cnt, fs, Rd, td = keep
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device=DEV)
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=DEV)
    o = dict(R=f64(G, M, 3, 3), t=f64(G, M, 3), points=i32(G, M), rmse=f64(G, M), status=i32(G, M), view_points=i32(G, M, Cn),
             view_rmse=f64(G, M, Cn), view_hidden=i32(G, M, Cn), corners=torch.empty(B, M, 9, 2, dtype=torch.float32, device=DEV),
             instance_map=torch.empty(B, H, W, dtype=torch.int16, device=DEV))
    work = torch.empty(utils.refine_instances_work_bytes(G, Cn, M, W, H) // 8, dtype=torch.float64, device=DEV)
    call("ssp_refine_instances_rig", ptr(D), W, H, SCALE, Cn, ptr(K), ptr(Dd), ptr(Rr), ptr(tr), ptr(mo), ptr(of), ptr(dm), ptr(fa), ptr(fo),
         int(np.diff(foff).max()), ptr(tab), 9, num_classes, ptr(cl), G, M, ptr(cnt), ptr(fs), ptr(Rd), ptr(td), iters, gate[0], gate[1],
         *(ptr(o[k]) for k in KEYS), ptr(work), work.numel() * 8, stream_ptr())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _same(a, b, keys=None):
    return all(np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f") for k in (keys or a))


def _check(d, h):
    """the kernel's outputs against the harness's: every count, status and instance_map entry bit for bit; the poses, residuals and
    corners bit for bit but where sin and cos (so3_exp) rounded differently on the device, which leaves a few last-bit differences
    (measured: at most 1e-15 in R, 3e-17 in t and 3e-18 in rmse on 2 of these scenes, and every integer output equal)"""
    for k in ("points", "status", "view_points", "view_hidden", "instance_map"):
        assert np.array_equal(d[k], h[k]), k
    for k, tol in (("R", 1e-13), ("t", 1e-13), ("rmse", 1e-15), ("view_rmse", 1e-15), ("corners", 1e-3)):
        x, y = d[k].astype(np.float64), h[k].astype(np.float64)
        same = (x == y) | (np.isnan(x) & np.isnan(y))
        assert (np.abs(x - y)[~same] <= tol).all(), (k, int((~same).sum()), np.abs(x - y)[~same].max())


def piles(seed, n_cams, groups, n_inst, distorted=False, mesh=(V, F), places=None):
    """one rig and `groups` captures of a pile each -> rig, depth (G C, H, W), truth and starts (G, M, ...)"""
    rng = np.random.default_rng(seed)
    rig = make_rig(rng, n_cams, distorted)
    dep, Rs, ts = [], [], []
    for g in range(groups):
        truth = pile_poses(rng, n_inst) if places is None else [(perturb_world(np.eye(3), p, rng, 0.0, 180.0)[0], p) for p in places]
        dep.append(pile_depth(rig, truth, noise=True, holes=g % 2 == 1, seed=seed + g, mesh=mesh))
        starts = [perturb_world(R, t, rng, move=0.01, angle_deg=3.0) for R, t in truth]
        Rs.append(np.stack([s[0] for s in starts]))
        ts.append(np.stack([s[1] for s in starts]))
    return rig, np.concatenate(dep), np.stack(Rs), np.stack(ts)


# ---------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("n_cams,distorted", [(1, False), (2, True), (3, False), (4, True)])
def test_kernel_equals_harness(ri_host, n_cams, distorted):
    """three captures of 4-6 instances, with an empty slot past the count, an unknown class and a slot without a fused pose"""
    rig, depth, R, t = piles(700 + n_cams, n_cams, 3, 6, distorted)
    cls = np.zeros((3, 6), np.int32)
    cls[1, 4] = -1
    fs = np.zeros((3, 6), np.int32)
    fs[2, 1] = 2
    count = [6, 5, 6]
    h = host_refine_instances(ri_host, rig, depth, cls, R, t, count=count, fuse_status=fs)
    d = kernel_refine_instances(rig, depth, cls, R, t, count=count, fuse_status=fs)
    _check(d, h)
    assert (h["status"] == 0).sum() >= 12 and (h["view_hidden"].sum() > 0 or n_cams == 1)
    assert not d["R"][1, 5].any() and (d["instance_map"] >= 0).sum() > 3000


SMALL = synth.closed_mesh(rings=10, segments=16, half_extents=(0.012, 0.012, 0.015))


@pytest.mark.parametrize("n_cams", [9, 16])
def test_many_cameras(ri_host, n_cams):
    rig, depth, R, t = piles(900 + n_cams, n_cams, 2, 5, mesh=SMALL, places=[np.array([x, y, -0.05]) for x, y in
                                                                              ((-0.02, 0.0), (0.0, 0.0), (0.02, 0.0), (0.0, 0.02), (0.01, 0.01))])
    cls = np.zeros((2, 5), np.int32)
    h = host_refine_instances(ri_host, rig, depth, cls, R, t, meshes={0: SMALL})
    d = kernel_refine_instances(rig, depth, cls, R, t, meshes={0: SMALL})
    _check(d, h)
    assert (h["status"] == 0).sum() >= 5 and h["view_hidden"].sum() > 0


def test_256_drawn_slots(ri_host):
    places = [np.array([0.03 * (i % 16 - 7.5), 0.03 * (i // 16 - 7.5), -0.05 + 0.01 * (i % 3)]) for i in range(256)]
    rig, depth, R, t = piles(256, 2, 1, 256, mesh=SMALL, places=places)
    cls = np.zeros((1, 256), np.int32)
    h = host_refine_instances(ri_host, rig, depth, cls, R, t, meshes={0: SMALL}, iters=4)
    d = kernel_refine_instances(rig, depth, cls, R, t, meshes={0: SMALL}, iters=4)
    _check(d, h)
    assert len(np.unique(d["instance_map"])) > 200 and d["instance_map"].max() >= 250


def test_a_capture_alone_equals_the_batch_and_calls_repeat(ri_host):
    rig, depth, R, t = piles(31, 3, 3, 5, True)
    cls = np.zeros((3, 5), np.int32)
    full = kernel_refine_instances(rig, depth, cls, R, t)
    assert _same(kernel_refine_instances(rig, depth, cls, R, t), full)
    one = kernel_refine_instances(rig, depth[3:6], cls[1:2], R[1:2], t[1:2])
    for k in KEYS:
        want = full[k][3:6] if k in ("corners", "instance_map") else full[k][1:2]
        assert np.array_equal(one[k], want), k


def test_refine_instances_rig_batched_feeds_from_the_fusion():
    """utils.refine_instances_rig_batched on host and device depth, with fuse_instances_batched's dict as it comes"""
    rig, depth, R, t = piles(41, 2, 2, 4)
    fused = dict(world_cls=_d(np.zeros((2, 4), np.int32)), R_world=_d(R), t_world=_d(t), world_count=_d(np.array([4, 3], np.int32)),
                 fuse_status=_d(np.zeros((2, 4), np.int32)))
    a = utils.refine_instances_rig_batched(depth, {0: (V, F)}, rig, fused["world_cls"], fused["R_world"], fused["t_world"],
                                           fused["world_count"], fused["fuse_status"])
    b = utils.refine_instances_rig_batched(_d(depth), {0: (V, F)}, rig, fused["world_cls"], fused["R_world"], fused["t_world"],
                                           fused["world_count"], fused["fuse_status"])
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert len(a) == 10 and a[9].dtype == torch.int16 and tuple(a[9].shape) == depth.shape and not a[0][1, 3].any()
    assert (a[4][0] == 0).all()


# ---------------------------------------------------------------------------------------------------- the predictor
def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items()}


def _instance_depth(rig, r, B, seed):
    """(B, 480, 640): each capture's fused world instances (those wholly in front of every camera) rendered in every camera with
    the table and noise; random depth for a capture without one"""
    Cn = len(rig.K)
    rng = np.random.default_rng(seed)
    out = []
    for g in range(B // Cn):
        poses = []
        for w in range(int(r["world_count"][g])):
            Rw, tw = r["R_world"][g, w], r["t_world"][g, w]
            if all(((V @ (rig.R[c] @ Rw).T + rig.R[c] @ tw + rig.t[c])[:, 2] > 0.1).all() for c in range(Cn)):
                poses.append((Rw, tw + rng.normal(0, 0.003, 3)))
        if poses:
            out.append(pile_depth(rig, poses, table=False, noise=True, seed=g))
        else:
            D = rng.integers(500, 1500, size=(Cn, 480, 640)).astype(np.uint16)
            D[rng.random(D.shape) < 0.3] = 0
            out.append(D)
    return np.concatenate(out)


REF_KEYS = {"R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points", "refine_view_rmse",
            "refine_view_hidden", "corners_world_ref_px", "instance_map"}


@pytest.mark.parametrize("distorted", [False, True])
def test_instance_predictor_with_a_rig_and_meshes(cfg_path, distorted):
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    from test_gpu_multiview import _frames, _rig2
    from test_gpu_refine_depth import CORNERS, _posed_model
    m = _posed_model(cfg_path)
    rig = _rig2(distorted)
    fr = _frames(4, 3)
    make = lambda **kw: InstancePosePredictor(m, {0: CORNERS}, None, shape=(416, 416), batch=4, conf_thresh=0.5, max_instances=16,
                                              rig=rig, **kw)
    plain = _host(make()(fr))
    depth = _instance_depth(rig, plain, 4, 1)
    pred = make(meshes={0: (V, F)})
    r = _host(pred(fr, depth=depth))
    assert _same(r, plain, plain.keys()) and set(r) - set(plain) == REF_KEYS
    want = utils.refine_instances_rig_batched(depth, {0: (V, F)}, rig, r["world_cls"], r["R_world"], r["t_world"], r["world_count"],
                                              r["fuse_status"])
    for k, w in zip(("R_world_ref", "t_world_ref", "refine_points", "refine_rmse", "refine_status", "refine_view_points",
                     "refine_view_rmse", "refine_view_hidden", None, "instance_map"), want):
        if k:
            assert np.array_equal(r[k], w.cpu().numpy(), equal_nan=True), k
    print("world_count %s, refine_status %s, refine_view_hidden %s" % (r["world_count"], r["refine_status"], r["refine_view_hidden"].sum()))
    assert (r["refine_status"][:, :1] == 0).any() and (r["instance_map"] >= 0).any()
    assert _same(_host(make(meshes={0: (V, F)}, graph=False)(fr, depth=depth)), r)
    assert _same(_host(pred(torch.from_numpy(fr).to(DEV), depth=_d(depth))), r)


def test_cli_rig_depth_dir(cfg_path, tmp_path):
    """predict_instances --rig --depth-dir on two captures: the per-world-instance refinement columns equal the predictor's"""
    from PIL import Image
    from singleshotpose_b200.predict import mesh_corners
    from singleshotpose_b200.predict_instances import RIG_REFINE_KEYS, WORLD_KEYS, InstancePosePredictor, main
    from test_gpu_multiview import _frames, _rig2
    from test_gpu_refine_depth import _posed_model
    m = _posed_model(cfg_path)
    wf = str(tmp_path / "posed.weights")
    m.save_weights(wf)
    ply = str(tmp_path / "obj.ply")
    synth.write_ply(ply, V, F)
    data = tmp_path / "obj.data"
    data.write_text("mesh = %s\nwidth = 640\nheight = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n" % ply)
    rig = _rig2(True)
    rig_path = str(tmp_path / "rig.npz")
    np.savez(rig_path, K=rig.K, R=rig.R, t=rig.t, dist=rig.dist)
    fr = _frames(4, 21)
    ddir = tmp_path / "depth"
    ddir.mkdir()
    plain = _host(InstancePosePredictor(m, {0: mesh_corners(ply)}, None, frame_size=(640, 480), batch=4, max_instances=16, rig=rig)(fr))
    depth = _instance_depth(rig, plain, 4, 5)
    paths = []
    for i in range(4):
        paths.append(str(tmp_path / ("img%d.png" % i)))
        Image.fromarray(fr[i]).save(paths[-1])
        Image.fromarray(depth[i]).save(str(ddir / ("img%d.png" % i)))
    out = str(tmp_path / "world.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf, "--out", out, "--max-instances", "16", "--rig", rig_path,
          "--depth-dir", str(ddir)] + paths)
    got = np.load(out)
    from singleshotpose_b200.utils_host import read_ply_mesh
    pred = InstancePosePredictor(m, {0: mesh_corners(ply)}, None, frame_size=(640, 480), batch=2, max_instances=16, rig=rig,
                                 meshes={0: read_ply_mesh(ply)})
    world = {k: [] for k in WORLD_KEYS + RIG_REFINE_KEYS}
    for g in range(2):
        r = pred(fr[2 * g:2 * g + 2], to_host=True, depth=depth[2 * g:2 * g + 2])
        n = int(r["world_count"][0])
        for k in world:
            world[k].append(r[k][0, :n])
    assert sum(len(v) for v in world["R_world_ref"]) >= 2 and "instance_map" not in got.files
    for k, v in world.items():
        assert np.array_equal(got[k], np.concatenate(v), equal_nan=True), k
