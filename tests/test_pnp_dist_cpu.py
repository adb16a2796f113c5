"""CPU checks of PnP and projection with lens distortion: the arithmetic of pnp_core.h / pnp_consensus_core.h with distortion
coefficients, compiled for the host by tests/helpers/pnp_dist_host.cpp, against cv2's goldens (tests/golden/pnp_dist.npz:
cv2.solvePnP(..., distCoeffs) cold and warm, cv2.projectPoints, cv2.undistortPoints); the zero-distortion path of the same core
against pnp_host bit for bit; the argument checks of ssp_pnp_dist, ssp_pnp_consensus_dist and ssp_project_points_dist;
utils.camera_distortion, the reference's pnp.distCoeffs, the .data file's dist entry and --dist.  No device is touched."""
import argparse
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.pnp_dist_ref import corner_problems, dist8
from singleshotpose_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSP_ERR_ARG = -1
CALIBS = ("barrel", "pincushion", "four", "five", "rational")


def _build(tmp_path_factory, name, src, flags):
    so = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
    subprocess.check_call(["g++", *flags, "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", src)])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return _build(tmp_path_factory, "pnpdisthost", "pnp_dist_host.cpp", ["-O2", "-std=c++17", "-ffp-contract=off"])


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "pnp_dist.npz"))


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def host_pnp_dist(lib, P3, uv, K, dist, guess=None, use=None, shared=1):
    P3 = np.ascontiguousarray(P3, np.float32); uv = np.ascontiguousarray(uv, np.float32); K = np.ascontiguousarray(K, np.float32)
    dist = None if dist is None else np.ascontiguousarray(dist, np.float64)
    n, npts = uv.shape[0], uv.shape[1]
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3)); params = np.zeros((n, 6)); w = np.zeros((n, 3), np.int32)
    if guess is not None:
        guess = np.ascontiguousarray(guess, np.float64)
        use = np.ascontiguousarray(np.ones(n) if use is None else use, np.int32)
    assert lib.h_pnp_dist(_p(P3), shared, _p(uv), _p(K), _p(dist), npts, C.c_longlong(n), 20, _p(guess), _p(use), _p(R), _p(t), _p(params),
                          _p(w)) == 0
    return R, t, params, w


def host_consensus_dist(lib, P3, uv, K, dist, masks, thr=8.0):
    P3 = np.ascontiguousarray(P3, np.float32); uv = np.ascontiguousarray(uv, np.float32); K = np.ascontiguousarray(K, np.float32)
    dist = None if dist is None else np.ascontiguousarray(dist, np.float64)
    masks = np.ascontiguousarray(masks, np.uint16)
    n, npts = uv.shape[0], uv.shape[1]
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3)); params = np.zeros((n, 6))
    inl = np.zeros(n, np.int32); hyp = np.zeros(n, np.int32)
    assert lib.h_pnp_consensus_dist(_p(P3), 1, _p(uv), _p(K), _p(dist), npts, C.c_longlong(n), _p(masks), len(masks), C.c_double(thr), 20,
                                    _p(R), _p(t), _p(params), _p(inl), _p(hyp)) == 0
    return R, t, params, inl, hyp


def _ang(a, b):
    return np.degrees(np.arccos(np.clip((np.trace(a @ b.T) - 1) / 2, -1, 1)))


def _rod(r):
    from oracle.pnp_ref import rodrigues_vec2mat
    return rodrigues_vec2mat(np.asarray(r, np.float64))


# ------------------------------------------------------------------------------------------------ the core against cv2
@pytest.mark.parametrize("calib", CALIBS)
def test_undistort_matches_cv2(host, golden, calib):
    uv = np.ascontiguousarray(golden["und_uv"], np.float64)
    xy = np.zeros_like(uv)
    K, dist = np.ascontiguousarray(golden["K"], np.float32), dist8(golden["dist_" + calib])           # kept alive across the call
    assert host.h_undistort(_p(uv), C.c_longlong(len(uv)), _p(K), _p(dist), _p(xy)) == 0
    assert np.abs(xy - golden["und_" + calib]).max() < 1e-12


@pytest.mark.parametrize("npts", [9, 8])
@pytest.mark.parametrize("calib", CALIBS)
def test_cold_solve_matches_cv2_golden(host, golden, calib, npts):
    tag = "%s_p%d" % (calib, npts)
    R, t, params, w = host_pnp_dist(host, golden["P3_%d" % npts], golden["uv_" + tag], golden["K"], dist8(golden["dist_" + calib]))
    ang = np.array([_ang(R[i], golden["R_" + tag][i]) for i in range(len(R))])
    assert ang.max() < 1e-2 and np.abs(t - golden["tvec_" + tag]).max() * 1e3 < 1e-2, (tag, ang.max())
    assert np.array_equal(params[:, 3:], t) and (w[:, 1] >= 1).all() and (w[:, 1] <= 20).all()
    # the goldens cover both regions and every noise level
    assert golden["corner_" + tag].any() and not golden["corner_" + tag].all() and set(golden["sigma_" + tag]) == {0, 1, 5, 20}


@pytest.mark.parametrize("npts", [9, 8])
@pytest.mark.parametrize("calib", CALIBS)
def test_warm_solve_matches_cv2_golden(host, golden, calib, npts):
    tag = "%s_p%d" % (calib, npts)
    uv, guess = golden["warm_uv_" + tag], golden["warm_guess_" + tag]
    R, t, params, w = host_pnp_dist(host, golden["P3_%d" % npts], uv, golden["K"], dist8(golden["dist_" + calib]), guess)
    ang = np.array([_ang(R[i], golden["warm_R_" + tag][i]) for i in range(len(R))])
    assert ang.max() < 1e-2 and np.abs(t - golden["warm_tvec_" + tag]).max() * 1e3 < 1e-2, (tag, ang.max())
    assert np.degrees(np.abs(params[:, :3] - golden["warm_rvec_" + tag])).max() < 1e-2
    assert (w[:, 0] == 0).all()                                          # no DLT for a warm start
    assert golden["warm_perturbed_" + tag].any() and not golden["warm_perturbed_" + tag].all()


@pytest.mark.parametrize("calib", CALIBS)
def test_projection_matches_cv2_golden(host, golden, calib):
    P3 = np.ascontiguousarray(golden["P3_9"], np.float32)
    tag = "%s_p9" % calib
    Rt = np.ascontiguousarray([np.c_[_rod(r), t] for r, t in zip(golden["rvec_true_" + tag], golden["tvec_true_" + tag])])
    Kd = np.ascontiguousarray(golden["K"], np.float64)
    out = np.zeros((len(Rt), 2, 9), np.float32)
    dist = dist8(golden["dist_" + calib])
    assert host.h_project_dist(_p(P3), 9, _p(Rt), _p(Kd), _p(dist), C.c_longlong(len(Rt)), _p(out)) == 0
    assert np.abs(out.transpose(0, 2, 1) - golden["proj_true_" + tag]).max() < 1e-3       # cv2 returns float32 pixels


def test_null_dist_is_the_plain_core_bit_for_bit(host, tmp_path_factory, golden_dir):
    """pnp_solve_one with dist == null is the zero-distortion solve, as tests/helpers/pnp_host.cpp builds it"""
    plain = _build(tmp_path_factory, "pnphostref", "pnp_host.cpp", ["-O2"])
    g = np.load(os.path.join(golden_dir, "pnp.npz"))
    for tag in ("s0", "s1"):
        P3, uv, K = (np.ascontiguousarray(a, np.float32) for a in (g["P3"], g["uv_" + tag], g["K"]))
        n = len(uv)
        R0, t0, w0 = np.zeros((n, 3, 3)), np.zeros((n, 3)), np.zeros((n, 3), np.int32)
        assert plain.h_pnp(_p(P3), 1, _p(uv), _p(K), uv.shape[1], C.c_longlong(n), 20, _p(R0), _p(t0), _p(w0)) == 0
        R, t, _params, w = host_pnp_dist(host, P3, uv, K, None)
        assert np.array_equal(R, R0) and np.array_equal(t, t0) and np.array_equal(w, w0)


def test_distorted_consensus_keeps_the_corner_keypoints(host, golden):
    """near the frame corners, the box 0.3-0.5 m away, one keypoint moved 40-150 px: the distorted consensus finds exactly the 8
    correct keypoints; the consensus that ignores the distortion (8 px threshold) loses correct ones in a share of the problems
    (farther away, 0.6-1 m, the box is small enough that its pose absorbs the distortion and both find them)"""
    from singleshotpose_b200.utils import consensus_subsets
    K, dist, P3 = golden["K"], dist8(golden["dist_barrel"]), golden["P3_9"]
    uv, out, rv, tv = corner_problems(48, 7, K, dist, P3, depth=(0.3, 0.5))
    masks = consensus_subsets(P3)
    R, t, _p6, inl, hyp = host_consensus_dist(host, P3, uv, K, dist, masks)
    want = 0x1FF & ~(1 << out)
    assert np.array_equal(inl, want)
    assert max(_ang(R[i], _rod(rv[i])) for i in range(len(R))) < 1e-3 and np.abs(t - tv).max() < 1e-6
    _R, _t, _p6, inl0, _h = host_consensus_dist(host, P3, uv, K, None, masks)
    assert (inl0 != want).sum() >= len(uv) // 8, (inl0 != want).sum()          # 6 of these 48


# ------------------------------------------------------------------------------------------------ ABI
def test_symbols_are_declared_and_exported():
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        text = f.read()
    for name in ("ssp_pnp_dist", "ssp_pnp_consensus_dist", "ssp_project_points_dist"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
        assert "int %s(" % name in text


def _fake(a):
    return C.c_void_p(0x10000 * a) if a else None


def test_entry_points_reject_bad_arguments():
    lib = _lib.load()

    def pnp(P3=1, uv=1, K=1, dist=1, np_=9, groups=2, per=4, count=0, g=0, use=0, R=1, t=1, params=0, work=0):
        return lib.ssp_pnp_dist(_fake(P3), 0, _fake(uv), _fake(K), _fake(dist), np_, groups, per, _fake(count), _fake(g), _fake(use), 20,
                                _fake(R), _fake(t), _fake(params), _fake(work), None)
    for kw in (dict(P3=0), dict(uv=0), dict(K=0), dict(dist=0), dict(R=0), dict(t=0), dict(np_=5), dict(np_=17), dict(groups=-1),
               dict(per=0), dict(g=1), dict(use=1), dict(g=1, use=1)):
        assert pnp(**kw) == SSP_ERR_ARG, kw
    pnp(dist=0)
    assert b"pnp_dist" in lib.ssp_last_error()
    assert pnp(groups=0) == 0 and pnp(groups=0, count=1, g=1, use=1, params=1, work=1) == 0      # no problem: no launch

    masks = np.array([0b111111, 0b1111110], np.uint16)

    def cons(P3=1, uv=1, K=1, dist=1, np_=9, groups=0, per=1, tab=masks, H=2, thr=8.0, it=20, R=1, t=1, params=1, inl=1, hyp=1, work=1,
             wb=0):
        return lib.ssp_pnp_consensus_dist(_fake(P3), 1, _fake(uv), _fake(K), _fake(dist), np_, groups, per, None, C.c_void_p(tab.ctypes.data),
                                          H, C.c_double(thr), it, _fake(R), _fake(t), _fake(params), _fake(inl), _fake(hyp), _fake(work),
                                          C.c_longlong(wb), None)
    for kw in (dict(P3=0), dict(uv=0), dict(K=0), dict(dist=0), dict(R=0), dict(t=0), dict(params=0), dict(inl=0), dict(hyp=0),
               dict(work=0), dict(np_=6), dict(np_=11), dict(groups=-1), dict(per=0), dict(H=0), dict(tab=np.array([0b111], np.uint16), H=1),
               dict(tab=np.array([0b1111110000], np.uint16), H=1), dict(thr=0.0), dict(thr=float("inf")), dict(thr=float("nan")),
               dict(it=0), dict(groups=1, wb=8)):
        assert cons(**kw) == SSP_ERR_ARG, kw
    assert cons() == 0

    def proj(X=1, rows=4, nv=9, Rt=1, K=1, dist=1, n=2, out=1):
        return lib.ssp_project_points_dist(_fake(X), rows, nv, _fake(Rt), _fake(K), _fake(dist), C.c_longlong(n), _fake(out), None)
    for kw in (dict(X=0), dict(Rt=0), dict(K=0), dict(dist=0), dict(out=0), dict(rows=2), dict(rows=5), dict(nv=-1), dict(n=-1)):
        assert proj(**kw) == SSP_ERR_ARG, kw
    assert proj(n=0) == 0 and proj(nv=0) == 0


# ------------------------------------------------------------------------------------------------ Python surface
def test_camera_distortion():
    from singleshotpose_b200.utils import camera_distortion
    SspError = _lib.SspError
    for none in (None, [], np.zeros((8, 1), np.float32), np.zeros(5), (0, 0, 0, 0)):
        assert camera_distortion(none) is None
    k = camera_distortion([-0.3, 0.12, 1e-3, -5e-4])
    assert k.dtype == np.float64 and k.shape == (8,) and np.array_equal(k, [-0.3, 0.12, 1e-3, -5e-4, 0, 0, 0, 0])
    f32 = np.array([[-0.3, 0.12, 1e-3, -5e-4, -0.02]], np.float32)          # cv2.calibrateCamera's (1, 5); float32 values kept
    assert np.array_equal(camera_distortion(f32), np.r_[f32.reshape(-1).astype(np.float64), np.zeros(3)])
    assert np.array_equal(camera_distortion(np.arange(1, 9.0).reshape(8, 1)), np.arange(1, 9.0))
    for n in (12, 14):
        with pytest.raises(SspError, match="thin-prism / tilted"):
            camera_distortion(np.full(n, 0.1))
    for bad in (np.ones(3), np.ones(6), np.ones(9), [0.1, float("nan"), 0, 0], [float("inf"), 0, 0, 0, 0], ["a", "b", "c", "d"]):
        with pytest.raises(SspError):
            camera_distortion(bad)


def test_pnp_distcoeffs_attributes_are_the_references():
    """utils.pnp and utils_multi.pnp are two functions, as in the reference: each reads its own pnp.distCoeffs"""
    from singleshotpose_b200 import utils, utils_multi
    assert utils.pnp is not utils_multi.pnp
    assert not hasattr(utils.pnp, "distCoeffs") and not hasattr(utils_multi.pnp, "distCoeffs")
    try:
        utils.pnp.distCoeffs = np.ones(5)
        assert not hasattr(utils_multi.pnp, "distCoeffs")
    finally:
        del utils.pnp.distCoeffs


def _args(argv, datacfg):
    from singleshotpose_b200.predict import add_dist_arg
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    add_dist_arg(ap)
    ap.add_argument("images", nargs="+")
    a = ap.parse_args(argv)
    a.datacfg = str(datacfg)
    return a


def test_dist_flag_and_data_file_entry(tmp_path):
    from singleshotpose_b200.predict import camera_dist
    cam = "fx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\nwidth = 640\nheight = 480\n"
    plain, withd = tmp_path / "plain.data", tmp_path / "dist.data"
    plain.write_text(cam)
    withd.write_text(cam + "dist = -0.3 0.12 0.001 -0.0005 -0.02\n")
    assert camera_dist(_args(["a.png"], plain)) is None                                    # neither: no distortion
    assert np.array_equal(camera_dist(_args(["a.png"], withd)), [-0.3, 0.12, 0.001, -0.0005, -0.02, 0, 0, 0])
    a = _args(["--dist", "-0.2", "0.05", "0", "0.001", "--", "a.png", "b.png"], withd)          # the flag overrides the file
    assert a.images == ["a.png", "b.png"] and np.array_equal(camera_dist(a), [-0.2, 0.05, 0, 0.001, 0, 0, 0, 0])
    a = _args(["--dist", "1", "2", "3", "4", "5", "6", "7", "8", "--out", "o.npz", "a.png"], plain)
    assert a.out == "o.npz" and np.array_equal(camera_dist(a), np.arange(1, 9.0))
    assert camera_dist(_args(["--dist", "0", "0", "0", "0", "--", "a.png"], withd)) is None      # all zeros: none
    for text in ("dist = 0.1 0.2 0.3\n", "dist = 0.1 x 0.3 0.4\n", "dist = 1 2 3 4 5 6 7 8 9 10 11 12\n"):
        bad = tmp_path / "bad.data"
        bad.write_text(cam + text)
        with pytest.raises(_lib.SspError):
            camera_dist(_args(["a.png"], bad))
    comma = tmp_path / "comma.data"
    comma.write_text(cam + "dist = -0.3, 0.12, 0.001, -0.0005\n")
    assert np.array_equal(camera_dist(_args(["a.png"], comma)), [-0.3, 0.12, 0.001, -0.0005, 0, 0, 0, 0])


def test_cli_dist_parsing():
    from singleshotpose_b200.predict_instances import parse_args
    base = ["--datacfg", "d.data", "--modelcfg", "m.cfg", "--weightfile", "w"]
    assert parse_args(base + ["a.png"]).dist is None
    a = parse_args(base + ["--dist", "-0.3", "0.12", "0.001", "-0.0005", "-0.02", "--", "a.png"])
    assert a.dist == [-0.3, 0.12, 0.001, -0.0005, -0.02] and a.images == ["a.png"]
    for bad in (["--dist", "0.1", "0.2", "--", "a.png"], ["--dist"] + ["0.1"] * 12 + ["--", "a.png"]):
        with pytest.raises(_lib.SspError):
            parse_args(base + bad)
    for mod in ("predict", "predict_multi", "predict_instances"):              # every command line has the flag
        import importlib
        m = importlib.import_module("singleshotpose_b200." + mod)
        with pytest.raises(SystemExit):
            m.main(["--help"])
