"""GPU checks of ssp_calibrate_rig (csrc/calibrate_rig.cu): step 1 against the host harness and utils.pnp_batched, every later
output bit for bit against the harness started from the device's per-row poses, repeatability, a distorted rig, multi-slot input,
the write_rig / read_rig round trip into PosePredictor(rig=...) and the command line."""
import numpy as np
import pytest
import torch

from singleshotpose_b200 import utils
from singleshotpose_b200.utils_host import read_rig, write_rig
from test_calibrate_rig_cpu import cal, host_calibrate, moving_object, record, relative, rot_err, scene  # noqa: F401
from test_multiview_cpu import P9, random_rig

pytestmark = pytest.mark.gpu
KEYS = ("R", "t", "cam_cov", "cam_obs", "cam_rmse", "tree_parent", "edge_agree", "cam_status", "R_world", "t_world", "views", "view_err",
        "linked")


def device(uv, rig, valid, **kw):
    o = utils.calibrate_rig_batched(P9, uv, rig.K, dist=None if rig.dist is None else list(rig.dist), valid=valid, **kw)
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in o.items()}


def _same(d, h, tag, tol=0.0):
    """every output equal, bit for bit (tol = 0), or the integers and flags exact and the doubles within tol relative: the device's
    sin and cos (so3_exp in the LM updates) may round a last bit differently from the host's"""
    for k in KEYS:
        a, b = np.asarray(d[k]), np.asarray(h[k])
        a = a.reshape(b.shape)
        if tol and a.dtype == np.float64:
            assert np.abs(a - b).max() <= tol * max(np.abs(b).max(), 1e-300), (tag, k, np.abs(a - b).max())
        else:
            assert np.array_equal(a, b), (tag, k, np.argwhere(a != b)[:5])
    assert (d["rounds"], d["iterations"]) == (h["rounds"], h["iterations"]), tag
    assert d["cost"] == h["cost"] if not tol else abs(d["cost"] - h["cost"]) <= tol * h["cost"], tag


# measured on an H100: bit for bit at 2, 3 and 4 cameras; at 8 cameras one LM update's sin / cos rounds differently, and the
# doubles agree within 1e-9 relative
@pytest.mark.parametrize("n_cams,distorted,tol", [(2, False, 0.0), (3, False, 0.0), (4, True, 0.0), (8, False, 1e-8)])
def test_kernel_equals_harness(cal, n_cams, distorted, tol):
    rig, uv, valid = scene(700 + n_cams, n_cams, G=40, distorted=distorted, miss=0.1, wrong=0.1)
    d = device(uv, rig, valid)
    h = host_calibrate(cal, rig.K, rig.dist, uv, valid)
    assert np.abs(d["R_rows"] - h["R_rows"][:, 0]).max() < 1e-6 and np.abs(d["t_rows"] - h["t_rows"][:, 0]).max() < 1e-6
    h = host_calibrate(cal, rig.K, rig.dist, uv, valid, rows=(d["R_rows"], d["t_rows"]))
    _same(d, h, (n_cams, distorted), tol)
    assert (d["cam_status"] == 0).all() and d["rig"] is not None
    # the per-row poses are utils.pnp_batched's with each camera
    for c in range(n_cams):
        k = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        R, t = utils.pnp_batched(P9, uv[c::n_cams], rig.K[c].astype(np.float32), max_iter=30, dist_coeffs=k)
        assert np.array_equal(R.cpu().numpy(), d["R_rows"][c::n_cams]) and np.array_equal(t.cpu().numpy(), d["t_rows"][c::n_cams])
    # two calls give the same bits
    d2 = device(uv, rig, valid)
    _same(d2, d, "repeat")


def test_unconnected_and_reference(cal):
    rng = np.random.default_rng(4)
    rig = random_rig(rng, 3)
    uv, valid = record(rig, moving_object(rng, 30), rng)
    v = valid.reshape(30, 3).copy()
    v[:15, 2] = False
    v[15:, :2] = False
    d = device(uv, rig, v.reshape(-1))
    assert d["cam_status"].tolist() == [0, 0, 1] and d["rig"] is None
    h = host_calibrate(cal, rig.K, None, uv, v.reshape(-1), rows=(d["R_rows"], d["t_rows"]))
    _same(d, h, "unconnected")
    d = device(uv, rig, valid, reference=1)
    assert np.array_equal(d["R"][1], np.eye(3)) and not d["t"][1].any()


def test_multi_slot_equals_one_slot_per_row():
    """S = 13 slots per row give the outputs of the same observations laid out one slot per row"""
    rng = np.random.default_rng(11)
    n, G, S = 3, 4, 13
    rig = random_rig(rng, n)
    uv, valid = record(rig, moving_object(rng, G * S), rng, 2.0, 0.1, 0.1)          # capture q = g S + s
    one = device(uv, rig, valid)
    # slotted: row g C + c, slot s holds capture g S + s in camera c
    uvs = uv.reshape(G, S, n, 9, 2).transpose(0, 2, 1, 3, 4).reshape(G * n, S, 9, 2)
    vs = valid.reshape(G, S, n).transpose(0, 2, 1).reshape(G * n, S)
    many = device(uvs, rig, vs)
    for k in ("R", "t", "cam_cov", "cam_obs", "cam_rmse", "tree_parent", "edge_agree", "cam_status"):
        assert np.array_equal(one[k], many[k]), k
    for k in ("R_world", "t_world", "views", "view_err", "linked"):
        assert np.array_equal(one[k].reshape(G * S, *one[k].shape[1:]), many[k].reshape(G * S, *many[k].shape[2:])), k


def test_round_trip_into_the_predictor(tmp_path, cfg_path):
    """the calibrated rig, written and read back bit for bit, feeds PosePredictor(rig=...) as the rig in memory does"""
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_multiview import _frames, _host
    from test_gpu_refine_depth import CORNERS, _posed_model
    rig, uv, valid = scene(31, 3, G=40, distorted=True)
    d = device(uv, rig, valid)
    p = str(tmp_path / "rig.npz")
    write_rig(p, d["rig"])
    back = read_rig(p)
    for a, b in zip(d["rig"], back):
        assert (a is None and b is None) or np.array_equal(a, b)
    m = _posed_model(cfg_path)
    fr = _frames(3, 3)
    r1 = _host(PosePredictor(m, CORNERS, None, shape=(416, 416), batch=3, rig=back, conf_thresh=0.0)(fr))
    r2 = _host(PosePredictor(m, CORNERS, None, shape=(416, 416), batch=3, rig=d["rig"], conf_thresh=0.0)(fr))
    assert "R_world" in r1
    for key in r1:
        assert np.array_equal(r1[key], r2[key]), key


def test_cli_writes_the_api_rig(tmp_path):
    """synthetic predict --out files of a 3-camera rig: the CLI writes the rig calibrate_rig_batched gives"""
    from singleshotpose_b200 import synth
    from singleshotpose_b200.calibrate_rig import main, object_points
    rng = np.random.default_rng(12)
    n, G = 3, 40
    V = np.array([[x, y, z] for x in (-0.05, 0.05) for y in (-0.04, 0.04) for z in (-0.06, 0.06)])
    ply = tmp_path / "box.ply"
    ply.write_text("ply\nformat ascii 1.0\nelement vertex 8\nproperty float x\nproperty float y\nproperty float z\nelement face 0\n"
                   "property list uchar int vertex_indices\nend_header\n" + "".join("%g %g %g\n" % tuple(v) for v in V))
    K = synth.intrinsics()
    datas = []
    for c in range(n):
        p = tmp_path / ("c%d.data" % c)
        p.write_text("fx = %r\nfy = %r\nu0 = %r\nv0 = %r\nwidth = 640\nheight = 480\nmesh = %s\n" % (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), ply))
        datas.append(str(p))
    P = object_points(str(ply))
    rig = random_rig(rng, n)._replace(K=np.repeat(K[None], n, 0))
    from oracle.pose_filter_ref import project
    poses = moving_object(rng, G)
    kp = np.array([[project(P, rig.R[c] @ R, rig.R[c] @ t + rig.t[c], K) + rng.normal(0, 2.0, (9, 2)) for R, t in poses] for c in range(n)], np.float32)
    conf = rng.uniform(0.05, 1.0, (n, G))
    files = []
    for c in range(n):
        f = str(tmp_path / ("p%d.npz" % c))
        np.savez(f, keypoints_px=kp[c], conf=conf[c], R=np.zeros((G, 3, 3)), t=np.zeros((G, 3)))
        files.append(f)
    out = str(tmp_path / "rig.npz")
    main(["--datacfg", *datas, "--poses", *files, "--out", out])
    got = read_rig(out)
    o = utils.calibrate_rig_batched(P, kp.transpose(1, 0, 2, 3).reshape(G * n, 9, 2), np.repeat(K[None], n, 0),
                                    valid=(conf.T > 0.1).reshape(-1))
    assert np.array_equal(got.R, o["rig"].R) and np.array_equal(got.t, o["rig"].t) and np.array_equal(got.K, o["rig"].K)
    Rt, _tt = relative(rig)
    assert max(rot_err(got.R[c], Rt[c]) for c in range(n)) < 1.0
