"""GPU checks of PnP and projection with lens distortion (csrc/pnp_dist.cu): ssp_pnp_dist against cv2's goldens
(tests/golden/pnp_dist.npz) cold, warm and counted; ssp_project_points_dist against cv2.projectPoints; ssp_pnp_consensus_dist on
corner problems against the host harness (tests/helpers/pnp_dist_host.cpp); utils.pnp with pnp.distCoeffs; and the four predictors
with dist_coeffs (the same solve and projection as the batched entry points, graph replay, all-zero coefficients)."""
import numpy as np
import pytest
import torch

from oracle.pnp_dist_ref import corner_problems, dist8
from singleshotpose_b200 import synth, utils
from singleshotpose_b200._lib import call, ptr, stream_ptr
from singleshotpose_b200.utils import consensus_subsets, pnp_batched, pnp_consensus_batched, project_points_batched

from test_pnp_dist_cpu import CALIBS, _ang, _build, _rod, host_consensus_dist

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32
BARREL = (-0.3, 0.12, 1e-3, -5e-4, -0.02)


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "pnp_dist.npz"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return _build(tmp_path_factory, "pnpdisthostg", "pnp_dist_host.cpp", ["-O2", "-std=c++17", "-ffp-contract=off"])


def _check(R, t, Rg, tg):
    R, t = R.cpu().numpy(), t.cpu().numpy()
    ang = np.array([_ang(R[i], Rg[i]) for i in range(len(R))])
    assert ang.max() < 1e-2 and np.abs(t - tg).max() * 1e3 < 1e-2, (ang.max(), np.abs(t - tg).max())


# ------------------------------------------------------------------------------------------------ kernels against cv2
@pytest.mark.parametrize("npts", [9, 8])
@pytest.mark.parametrize("calib", CALIBS)
def test_cold_solve_meets_the_cv2_golden(golden, calib, npts):
    tag = "%s_p%d" % (calib, npts)
    R, t = pnp_batched(golden["P3_%d" % npts], golden["uv_" + tag], golden["K"], dist_coeffs=golden["dist_" + calib])
    _check(R, t, golden["R_" + tag], golden["tvec_" + tag])


def _pnp_dist(P3, uv, K, dist, groups, per, count=None, guess=None, use=None):
    n = groups * per
    P3, uv = (torch.as_tensor(np.ascontiguousarray(a, F32)).to(DEV) for a in (P3, uv))
    Kd, dd = torch.as_tensor(np.asarray(K, F32)).to(DEV), torch.as_tensor(dist8(dist)).to(DEV)
    R = torch.full((n, 3, 3), 7.0, dtype=torch.float64, device=DEV)
    t = torch.full((n, 3), 7.0, dtype=torch.float64, device=DEV)
    params = torch.full((n, 6), 7.0, dtype=torch.float64, device=DEV)
    work = torch.full((n, 3), 7, dtype=torch.int32, device=DEV)
    cnt = None if count is None else torch.as_tensor(np.asarray(count, np.int32)).to(DEV)
    g = None if guess is None else torch.as_tensor(np.asarray(guess, np.float64)).to(DEV)
    u = None if use is None else torch.as_tensor(np.asarray(use, np.int32)).to(DEV)
    call("ssp_pnp_dist", ptr(P3), 0, ptr(uv), ptr(Kd), ptr(dd), uv.shape[1], groups, per, ptr(cnt), ptr(g), ptr(u), 20, ptr(R), ptr(t),
         ptr(params), ptr(work), stream_ptr())
    return R, t, params, work


@pytest.mark.parametrize("calib", ["barrel", "rational"])
def test_warm_and_counted_solves_meet_the_cv2_golden(golden, calib):
    tag = "%s_p9" % calib
    uv, guess = golden["warm_uv_" + tag], golden["warm_guess_" + tag]
    n = len(uv)
    P3 = np.repeat(golden["P3_9"][None], n, 0)
    R, t, params, work = _pnp_dist(P3, uv, golden["K"], golden["dist_" + calib], n, 1, guess=guess, use=np.ones(n))
    _check(R, t, golden["warm_R_" + tag], golden["warm_tvec_" + tag])
    assert (work[:, 0] == 0).all() and torch.equal(params[:, 3:], t)
    # counted groups of 3 slots: count[g] = g % 4 (0..3, 3 fills the group), problem (g, m) = warm problem g*3+m, warm in every other slot
    groups = n // 3
    count = np.arange(groups) % 4
    use = (np.arange(groups * 3) % 2).astype(np.int32)
    R, t, params, work = _pnp_dist(P3[:groups * 3], uv[:groups * 3], golden["K"], golden["dist_" + calib], groups, 3, count, guess[:groups * 3], use)
    solved = (np.arange(groups * 3) % 3) < np.repeat(count, 3)
    empty = torch.from_numpy(~solved).to(DEV)
    assert not R[empty].any() and not t[empty].any() and not params[empty].any() and not work[empty].any()
    warm = solved & (use == 1)
    _check(R[torch.from_numpy(warm).to(DEV)], t[torch.from_numpy(warm).to(DEV)], golden["warm_R_" + tag][:groups * 3][warm],
           golden["warm_tvec_" + tag][:groups * 3][warm])
    cold = solved & (use == 0)                                       # cold slots are ssp_pnp_dist's plain solve, bit for bit
    Rc, tc = pnp_batched(golden["P3_9"], uv[:groups * 3][cold], golden["K"], dist_coeffs=golden["dist_" + calib])
    assert torch.equal(R[torch.from_numpy(cold).to(DEV)], Rc) and torch.equal(t[torch.from_numpy(cold).to(DEV)], tc)


@pytest.mark.parametrize("calib", CALIBS)
def test_projection_meets_cv2(golden, calib):
    tag = "%s_p9" % calib
    Rt = np.array([np.c_[_rod(r), t] for r, t in zip(golden["rvec_true_" + tag], golden["tvec_true_" + tag])])
    X = np.ascontiguousarray(golden["P3_9"].T)
    px = project_points_batched(X, Rt, golden["K"].astype(np.float64), dist_coeffs=golden["dist_" + calib]).cpu().numpy()
    assert np.abs(px.transpose(0, 2, 1) - golden["proj_true_" + tag]).max() < 1e-3
    Xh = np.concatenate([X, np.ones((1, 9), F32)])                     # homogeneous rows give the same pixels
    assert torch.equal(project_points_batched(Xh, Rt, golden["K"].astype(np.float64), dist_coeffs=golden["dist_" + calib]).cpu(),
                       torch.from_numpy(px))


def test_consensus_on_corner_problems(golden, host):
    K, dist, P3 = golden["K"], dist8(golden["dist_barrel"]), golden["P3_9"]
    uv, out, rv, tv = corner_problems(48, 7, K, dist, P3, depth=(0.3, 0.5))
    masks = consensus_subsets(P3)
    want = torch.from_numpy(np.array([[j != o for j in range(9)] for o in out])).to(DEV)
    R, t, _p, inl, hyp = pnp_consensus_batched(P3, uv, K, subsets=masks, dist_coeffs=dist)
    assert torch.equal(inl, want)
    _R, _t, _p, inl0, _h = pnp_consensus_batched(P3, uv, K, subsets=masks)
    assert (inl0 != want).any(1).sum() >= len(uv) // 8
    Rh, th, _ph, inlh, hyph = host_consensus_dist(host, P3, uv, K, dist, masks)
    bits = (inl.cpu().numpy() * (1 << np.arange(9))).sum(1)
    assert np.array_equal(bits, inlh) and np.array_equal(hyp.cpu().numpy(), hyph)
    assert np.abs(R.cpu().numpy() - Rh).max() < 1e-9 and np.abs(t.cpu().numpy() - th).max() < 1e-9


def test_utils_pnp_reads_pnp_distcoeffs(golden):
    tag = "barrel_p9"
    P3, uv, K = golden["P3_9"], golden["uv_" + tag], golden["K"]
    R0, t0 = utils.pnp(P3, uv[0], K)                                  # unset: the zero-distortion solve, bit for bit
    Rb, tb = pnp_batched(P3, uv[:1], K)
    assert np.array_equal(R0, Rb[0].cpu().numpy()) and np.array_equal(t0, tb[0].cpu().numpy().reshape(3, 1))
    utils.pnp.distCoeffs = np.asarray(golden["dist_barrel"], F32).reshape(5, 1)        # as a user sets it for the reference
    try:
        for i in range(0, len(uv), 5):
            R, t = utils.pnp(P3, uv[i], K)
            assert _ang(R, golden["R_" + tag][i]) < 1e-2 and np.abs(t.reshape(3) - golden["tvec_" + tag][i]).max() * 1e3 < 1e-2
    finally:
        del utils.pnp.distCoeffs


# ------------------------------------------------------------------------------------------------ predictors
CORNERS = synth.box_points(with_center=False).T.astype(np.float64)
KM = synth.intrinsics()


def _frames(n, seed, w=640, h=480):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _clone(r):
    return {k: v.clone() for k, v in r.items()}


def _P9(corners):
    return np.concatenate([np.zeros((1, 3)), corners.T]).astype(F32)


def _expect(kp, P3, dist, pnp="plain", subsets=None):
    """R, t, corners of keypoints kp (n, 9, 2) with PnP points P3 (n, 9, 3)"""
    if pnp == "consensus":
        R, t, _p, _i, _h = pnp_consensus_batched(P3, kp, KM.astype(F32), subsets=subsets, dist_coeffs=dist)
    else:
        R, t = pnp_batched(P3, kp, KM.astype(F32), dist_coeffs=dist)
    return R, t


def _corners_of(P3, R, t, dist):
    X = np.concatenate([P3.T, np.ones((1, 9))]).astype(F32)
    return project_points_batched(X, torch.cat([R, t.unsqueeze(2)], 2), KM, dist_coeffs=dist).transpose(1, 2)


@pytest.fixture(scope="module")
def single_model(cfg_path):
    from singleshotpose_b200 import Darknet
    torch.manual_seed(0)
    return Darknet(cfg_path).cuda().eval()


@pytest.fixture(scope="module")
def multi_model(cfg_multi_path):
    from singleshotpose_b200.darknet_multi import Darknet
    torch.manual_seed(0)
    return Darknet(cfg_multi_path).cuda().eval()


@pytest.mark.parametrize("pnp", ["plain", "consensus"])
def test_pose_predictor(single_model, pnp):
    from singleshotpose_b200.predict import PosePredictor
    fr = _frames(2, 1)
    g = PosePredictor(single_model, CORNERS, KM, batch=2, pnp=pnp, dist_coeffs=BARREL)
    e = PosePredictor(single_model, CORNERS, KM, batch=2, pnp=pnp, dist_coeffs=BARREL, graph=False)
    r, re_ = _clone(g(fr)), _clone(e(fr))
    assert g._last.graph is not None and all(torch.equal(r[k], re_[k]) for k in r)
    P3 = np.repeat(_P9(CORNERS)[None], 2, 0)
    R, t = _expect(r["keypoints_px"].cpu().numpy(), P3, BARREL, pnp, consensus_subsets(P3[:1]))
    assert torch.equal(r["R"], R) and torch.equal(r["t"], t)
    assert torch.equal(r["corners_px"], _corners_of(P3[0], R, t, BARREL))
    plain = PosePredictor(single_model, CORNERS, KM, batch=2, pnp=pnp)
    zero = PosePredictor(single_model, CORNERS, KM, batch=2, pnp=pnp, dist_coeffs=np.zeros(8))
    rp, rz = _clone(plain(fr)), _clone(zero(fr))
    assert all(torch.equal(rp[k], rz[k]) for k in rp)
    assert not torch.equal(rp["corners_px"], r["corners_px"])


def test_multi_pose_predictor(multi_model):
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    objs = {c: CORNERS * (1.0 + 0.1 * c) for c in (0, 4, 9)}
    fr = _frames(2, 2)
    for pnp in ("plain", "consensus"):
        p = MultiPosePredictor(multi_model, objs, KM, batch=2, conf_thresh=0.02, pnp=pnp, dist_coeffs=BARREL)
        r = _clone(p(fr))
        re_ = _clone(MultiPosePredictor(multi_model, objs, KM, batch=2, conf_thresh=0.02, pnp=pnp, dist_coeffs=BARREL, graph=False)(fr))
        assert all(torch.equal(r[k], re_[k]) for k in r)
        P3c = np.stack([_P9(objs[c]) for c in sorted(objs)])
        P3 = np.tile(P3c, (2, 1, 1))
        R, t = _expect(r["keypoints_px"].reshape(-1, 9, 2).cpu().numpy(), P3, BARREL, pnp, consensus_subsets(P3c))
        assert torch.equal(r["R"].reshape(-1, 3, 3), R) and torch.equal(r["t"].reshape(-1, 3), t)
        for i in range(len(P3)):
            assert torch.equal(r["corners_px"].reshape(-1, 9, 2)[i], _corners_of(P3[i], R[i:i + 1], t[i:i + 1], BARREL)[0])


def test_instance_and_tracking_predictors(multi_model):
    from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor
    objs = {c: CORNERS * (1.0 + 0.1 * c) for c in (0, 4, 7, 11)}
    kw = dict(batch=2, conf_thresh=0.02, max_instances=32, dist_coeffs=BARREL)
    ip = InstancePosePredictor(multi_model, objs, KM, **kw)
    tp = TrackingPosePredictor(multi_model, objs, KM, **kw)
    rng = np.random.default_rng(3)
    f0 = rng.integers(0, 256, size=(2, 480, 640, 3)).astype(np.int16)
    warm_seen = 0
    for f in range(3):
        fr = np.clip(f0 + rng.integers(-6, 7, size=f0.shape), 0, 255).astype(np.uint8)
        ri, rt = _clone(ip(fr)), _clone(tp(fr))
        n = ri["count"].cpu().numpy()
        assert n.sum() > 0
        for b in range(2):
            m = int(n[b])
            cls = ri["cls"][b, :m].cpu().numpy()
            P3 = np.stack([_P9(objs[c]) for c in cls]) if m else np.zeros((0, 9, 3), F32)
            R, t = _expect(ri["keypoints_px"][b, :m].cpu().numpy(), P3, BARREL)
            assert torch.equal(ri["R"][b, :m], R) and torch.equal(ri["t"][b, :m], t)
            for i in range(m):
                assert torch.equal(ri["corners_px"][b, i], _corners_of(P3[i], R[i:i + 1], t[i:i + 1], BARREL)[0])
            assert not ri["R"][b, m:].any() and not ri["corners_px"][b, m:].any()
        # tracking: the frame's solve is ssp_pnp_dist over the slots with the tracker's guesses
        c = tp._last
        R, t, params, _w = _pnp_dist(c.P3.reshape(-1, 9, 3).cpu().numpy(), c.kp.reshape(-1, 9, 2).cpu().numpy(), KM, BARREL, 2, 32,
                                     c.count.cpu().numpy(), c.guess.reshape(-1, 6).cpu().numpy(), c.use_guess.reshape(-1).cpu().numpy())
        assert torch.equal(rt["R"].reshape(-1, 3, 3), R) and torch.equal(rt["t"].reshape(-1, 3), t)
        warm_seen += int(rt["warm"].sum())
    assert warm_seen > 0


def test_cli_dist_from_the_data_file_and_the_flag(cfg_path, tmp_path):
    from singleshotpose_b200 import Darknet
    from singleshotpose_b200.predict import PosePredictor, main
    listfile, _bgs = synth.write_linemod_like(str(tmp_path), n=2, fmt="jpg")
    paths = open(listfile).read().split()
    V = np.random.default_rng(0).normal(size=(40, 3)) * 0.03
    ply = str(tmp_path / "obj.ply")
    with open(ply, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n" % len(V))
        for v in V:
            f.write("%.17g %.17g %.17g\n" % tuple(v))
    data = tmp_path / "obj.data"
    data.write_text("mesh = %s\nwidth = 640\nheight = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n"
                    "dist = -0.3 0.12 0.001 -0.0005 -0.02\n" % ply)
    torch.manual_seed(4)
    wf = str(tmp_path / "m.weights")
    Darknet(cfg_path).save_weights(wf)
    m = Darknet(cfg_path)
    m.load_weights(wf)
    m.cuda().eval()
    corners = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    P9 = np.concatenate([np.zeros((1, 3)), corners[:3].T]).astype(F32)
    flag = (-0.2, 0.05, 0.0, 0.001)
    for extra, dist in (([], BARREL), (["--dist", *map(str, flag), "--"], flag)):
        out = str(tmp_path / "poses.npz")
        main(["--datacfg", str(data), "--modelcfg", cfg_path, "--weightfile", wf, "--out", out] + extra + paths)
        got = np.load(out)
        pred = PosePredictor(m, corners, Km, dist_coeffs=dist)
        for i, p in enumerate(paths):
            r = pred([open(p, "rb").read()], to_host=True)
            for k in ("R", "t", "keypoints_px", "corners_px"):
                assert np.array_equal(got[k][i], r[k][0]), (p, k)
        R, t = pnp_batched(P9, got["keypoints_px"], Km.astype(F32), dist_coeffs=dist)
        assert np.array_equal(got["R"], R.cpu().numpy()) and np.array_equal(got["t"], t.cpu().numpy())
