"""GPU checks of ssp_calibrate_rig_depth (utils.calibrate_rig_depth_batched): the kernels against the host harness at 2-4 cameras
and at the limits (16 cameras, more than 256 observations, several slots, a reference other than 0), the no-free-camera case
against refine_depth_rig_batched, repeatability and graph capture, the output rig in the rig refinement and PosePredictor, and
the command line against the API."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import utils
from test_calibrate_rig_depth_cpu import cd_host, host_calibrate_depth, perturb_world, scene, start  # noqa: F401
from test_refine_depth_cpu import MODEL, F, V

pytestmark = pytest.mark.gpu

INTS = ("cam_points", "cam_status", "obs_points", "obs_status")
DOUBLES = ("R", "t", "cam_cov", "cam_rmse", "R_world", "t_world", "obs_rmse", "iter_rmse")


def _diam():
    return utils.mesh_diameter(V)


def device(rig, depth, R0, t0, views=None, linked=None, reference=0, cam_status=None, S=1, **kw):
    Cn = len(rig.K)
    G = len(depth) // Cn
    lead = (G, S) if S > 1 else (G,)
    calib = dict(R=rig.R, t=rig.t, cam_status=np.zeros(Cn, np.int32) if cam_status is None else np.asarray(cam_status, np.int32),
                 R_world=np.reshape(R0, lead + (3, 3)), t_world=np.reshape(t0, lead + (3,)),
                 views=np.ones(lead + (Cn,), bool) if views is None else np.reshape(views, lead + (Cn,)).astype(bool),
                 linked=np.ones(lead, bool) if linked is None else np.reshape(linked, lead).astype(bool))
    d = utils.calibrate_rig_depth_batched(depth, V, F, rig.K, calib, dist=None if rig.dist is None else list(rig.dist), reference=reference,
                                          **kw)
    out = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in d.items()}
    for k in ("R_world", "t_world", "obs_points", "obs_rmse", "obs_status"):
        out[k] = out[k].reshape(G * S, *out[k].shape[len(lead):])
    return out


def _same(d, h, tag, tol=1e-12):
    """every count and status equal; the doubles bit for bit, or within tol of the largest magnitude where the device's sin / cos
    round differently.  -> whether every double matched bit for bit"""
    assert d["status"] == h["status"], tag
    for k in INTS:
        assert np.array_equal(d[k], h[k]), (tag, k, d[k], h[k])
    exact = True
    for k in DOUBLES:
        if not np.array_equal(d[k], h[k]):
            exact = False
            err = np.abs(d[k] - h[k]).max()
            assert err <= tol * max(np.abs(h[k]).max(), 1e-300), (tag, k, err)
    print("%s: %s" % (tag, "bit for bit" if exact else "within %g" % tol))
    return exact


@pytest.mark.parametrize("n_cams,distorted", [(2, False), (3, True), (4, False)])
def test_kernel_equals_harness(cd_host, n_cams, distorted):
    _true, rig0, depth, R0, t0, _R, _t = start(20 + n_cams, n_cams, 4, distorted=distorted, noise=True)
    views = np.ones((4, n_cams), np.uint8)
    views[2, 1] = 0
    h = host_calibrate_depth(cd_host, rig0, depth, R0, t0, views=views, diam=_diam())
    d = device(rig0, depth, R0, t0, views=views)
    assert h["status"] == 0 and (h["cam_status"] == 0).all()
    _same(d, h, "C = %d" % n_cams)


def test_limits(cd_host):
    """16 cameras with reference 5 and camera 9 unconnected; then 3 cameras with 130 captures of 2 slots (260 observations: the
    lane partials take more than one observation each) and reference 1"""
    st = np.zeros(16, np.int32)
    st[9] = 1
    _true, rig0, depth, R0, t0, _R, _t = start(91, 16, 2, ref=5)
    h = host_calibrate_depth(cd_host, rig0, depth, R0, t0, reference=5, cam_status=st, diam=_diam())
    d = device(rig0, depth, R0, t0, reference=5, cam_status=st)
    assert h["cam_status"][9] == 1 and h["status"] == 0 and (h["cam_status"] == 0).sum() >= 8      # a few cameras see too little: held
    _same(d, h, "C = 16", tol=1e-8)         # measured 4.9e-11: with 2 captures the 16-camera system is poorly conditioned, and
                                             # the device's sin / cos in so3_exp differ in the last bits
    true, rig0, depth5, R5, t5 = start(92, 3, 5, ref=1)[:5]
    G, S = 130, 2
    depth = np.concatenate([depth5[(g % 5) * 3:(g % 5) * 3 + 3] for g in range(G)])
    rng = np.random.default_rng(92)
    R0, t0 = perturb_world(np.stack([R5[g % 5] for g in range(G) for _s in range(S)]), np.stack([t5[g % 5] for g in range(G) for _s in range(S)]),
                           rng, angle_deg=0.5, move=0.002)
    linked = np.ones(G * S, np.uint8)
    linked[7] = 0
    h = host_calibrate_depth(cd_host, rig0, depth, R0, t0, reference=1, linked=linked, slots=S, diam=_diam())
    d = device(rig0, depth, R0, t0, reference=1, linked=linked, S=S)
    assert G * S > 256 and h["status"] == 0 and (h["cam_status"] == 0).all()
    _same(d, h, "260 observations")


def test_no_free_camera_equals_the_rig_refinement():
    _true, rig0, depth, R0, t0, _R, _t = start(44, 3, 3, ref=2, noise=True)
    views = np.zeros((3, 3), np.uint8)
    views[:, 2] = 1
    d = device(rig0, depth, R0, t0, views=views, reference=2)
    one = utils.camera_rig(rig0.K[2:], [np.eye(3)], [np.zeros(3)])
    r = [a.cpu().numpy() for a in utils.refine_depth_rig_batched(depth[2::3], V, F, one, R0, t0)]
    for k, a in zip(("R_world", "t_world", "obs_points", "obs_rmse", "obs_status"), r[:5]):
        assert np.array_equal(d[k], a), k
    assert np.array_equal(d["R"], rig0.R) and np.array_equal(d["t"], rig0.t) and np.array_equal(d["cam_status"], [2, 2, 0])


def test_two_calls_and_graph_capture(monkeypatch):
    """two calls give the same bits, and the entry point captured in a CUDA graph and replayed gives the eager call's bits"""
    _true, rig0, depth, R0, t0, _R, _t = start(45, 3, 3)
    a, b = device(rig0, depth, R0, t0), device(rig0, depth, R0, t0)
    for k in INTS + DOUBLES:
        assert np.array_equal(a[k], b[k]), k
    call = utils.call

    def captured(name, *args):
        if name != "ssp_calibrate_rig_depth":
            return call(name, *args)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call(name, *args[:-1], utils.stream_ptr())
        g.replay()
        torch.cuda.synchronize()
        return 0

    monkeypatch.setattr(utils, "call", captured)
    c = device(rig0, depth, R0, t0)
    for k in INTS + DOUBLES:
        assert np.array_equal(a[k], c[k]), k
    assert a["status"] == c["status"] == 0


def test_rig_feeds_the_refinement_and_the_predictor(cfg_path):
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_multiview import _frames, _host
    from test_gpu_refine_depth import CORNERS, _posed_model
    true, rig0, depth, R0, t0, R, t = start(46, 3, 4, noise=True)
    d = utils.calibrate_rig_depth_batched(depth, V, F, rig0.K, dict(R=rig0.R, t=rig0.t, cam_status=np.zeros(3, np.int32), R_world=R0,
                                                                     t_world=t0, views=np.ones((4, 3), bool), linked=np.ones(4, bool)))
    rig = d["rig"]
    assert isinstance(rig, utils.CameraRig) and d["status"] == 0
    Rr, tr, pts, _rm, st, _vp, _vr = utils.refine_depth_rig_batched(depth, V, F, rig, R0, t0)
    assert (st.cpu().numpy() == 0).all() and (pts.cpu().numpy() > 1000).all()
    m = _posed_model(cfg_path)
    res = _host(PosePredictor(m, CORNERS, None, shape=(416, 416), batch=3, rig=rig, conf_thresh=0.0)(_frames(3, 3)))
    assert "R_world" in res


def test_cli_writes_the_api_rig(tmp_path):
    """synthetic predict --out files and depth PNGs of a 2-camera rig: calibrate_rig --depth-dir writes the rig the API returns"""
    from PIL import Image
    from oracle.pose_filter_ref import project
    from singleshotpose_b200 import synth
    from singleshotpose_b200.calibrate_rig import main, object_points
    from singleshotpose_b200.utils_host import read_rig
    from test_refine_rig_cpu import make_rig, random_pose, rig_depth
    rng = np.random.default_rng(13)
    n, G = 2, 16
    ply = tmp_path / "mesh.ply"
    ply.write_text("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nelement face %d\n"
                   "property list uchar int vertex_indices\nend_header\n" % (len(V), len(F)) + "".join("%r %r %r\n" % tuple(map(float, np.float32(v))) for v in V)
                   + "".join("3 %d %d %d\n" % tuple(f) for f in F))
    from singleshotpose_b200.predict import read_mesh
    Vm, Fm = read_mesh(str(ply))
    K = synth.intrinsics()
    rig = make_rig(rng, n)._replace(K=np.repeat(K[None], n, 0))
    datas, files = [], []
    P = object_points(str(ply))
    poses = [random_pose(rng) for _ in range(G)]
    kp = np.array([[project(P, rig.R[c] @ R, rig.R[c] @ t + rig.t[c], K) + rng.normal(0, 2.0, (9, 2)) for R, t in poses] for c in range(n)],
                  np.float32)
    depth = np.concatenate([rig_depth(rig, R, t, noise=True, seed=g) for g, (R, t) in enumerate(poses)])
    dirs = []
    for c in range(n):
        p = tmp_path / ("c%d.data" % c)
        p.write_text("fx = %r\nfy = %r\nu0 = %r\nv0 = %r\nwidth = 640\nheight = 480\nmesh = %s\n" % (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]),
                                                                                                 float(K[1, 2]), ply))
        datas.append(str(p))
        dd = tmp_path / ("depth%d" % c)
        dd.mkdir()
        dirs.append(str(dd))
        names = ["frames/cam%d_%03d.jpg" % (c, g) for g in range(G)]
        for g in range(G):
            Image.fromarray(depth[g * n + c]).save(dd / ("cam%d_%03d.png" % (c, g)))
        f = str(tmp_path / ("p%d.npz" % c))
        np.savez(f, keypoints_px=kp[c], conf=np.ones(G), paths=np.array(names))
        files.append(f)
    out = str(tmp_path / "rig.npz")
    main(["--datacfg", *datas, "--poses", *files, "--out", out, "--depth-dir", *dirs])
    got = read_rig(out)
    o = utils.calibrate_rig_batched(P, kp.transpose(1, 0, 2, 3).reshape(G * n, 9, 2), np.repeat(K[None], n, 0))
    d = utils.calibrate_rig_depth_batched(depth, Vm, Fm, np.repeat(K[None], n, 0), o)
    assert np.array_equal(got.R, d["rig"].R) and np.array_equal(got.t, d["rig"].t) and np.array_equal(got.K, d["rig"].K)
