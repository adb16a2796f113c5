"""GPU checks of the consensus PnP (ssp_pnp_consensus, rule: singleshotpose_b200/csrc/pnp_consensus_core.h): the kernels against the
host harness (tests/helpers/pnp_consensus_host.cpp) on the cv2 golden and on 10^4 random problems, the invariant against
ssp_pnp_batched bit for bit, determinism and batch independence, counted empty slots, the three predictors with
pnp="consensus", the evaluation tails against a host loop over the oracle (oracle/pnp_consensus_ref.py) and the command line."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle.pnp_consensus_ref import consensus_ref
from singleshotpose_b200 import synth, utils
from singleshotpose_b200._lib import SspError, call, ptr, stream_ptr
from singleshotpose_b200.utils import consensus_subsets, consensus_work_bytes, pnp_batched, pnp_consensus_batched

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KM = synth.intrinsics()
F32 = np.float32
BORDER = 1e-4


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pnpchost") / "libpnpchost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "pnp_consensus_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _ang(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.einsum("...ij,...ij->...", Ra, Rb) - 1) / 2, -1, 1)))


def host_run(host, P3, uv, K, thr, subsets):
    """the harness: result and the smallest |e2 - thr^2| over every hypothesis in front of the camera (how close to a flip)"""
    uv = np.ascontiguousarray(uv, F32); P3 = np.ascontiguousarray(P3, F32); K = np.ascontiguousarray(K, F32)
    subsets = np.ascontiguousarray(subsets, np.uint16)
    n, npts = uv.shape[:2]
    H1 = len(subsets) + 1
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3)); params = np.zeros((n, 6)); inl = np.zeros(n, np.int32); hyp = np.zeros(n, np.int32)
    assert host.h_pnp_consensus(_p(P3), 1, _p(uv), _p(K), npts, C.c_longlong(n), _p(subsets), len(subsets), C.c_double(thr), 20, _p(R),
                                _p(t), _p(params), _p(inl), _p(hyp)) == 0
    slots = np.zeros((n, H1, 15)); hm = np.zeros((n, H1), np.uint32)
    assert host.h_consensus_hyps(_p(P3), 1, _p(uv), _p(K), npts, C.c_longlong(n), _p(subsets), len(subsets), C.c_double(thr), 20,
                                 _p(slots), _p(hm)) == 0
    Pc = np.einsum("nhij,pj->nhpi", slots[..., :9].reshape(n, H1, 3, 3), P3.astype(np.float64)) + slots[:, :, None, 12:]
    with np.errstate(divide="ignore", invalid="ignore"):
        e2 = ((K[0, 0] * Pc[..., 0] / Pc[..., 2] + K[0, 2] - uv[:, None, :, 0]) ** 2
              + (K[1, 1] * Pc[..., 1] / Pc[..., 2] + K[1, 2] - uv[:, None, :, 1]) ** 2)
    front = (Pc[..., 2] > 0).all(-1, keepdims=True)
    gap = np.where(front, np.abs(e2 - thr * thr), np.inf).min((1, 2))
    return dict(R=R, t=t, params=params, mask=inl, hyp=hyp, gap=gap)


def _dev_run(P3, uv, K, thr, subsets):
    R, t, params, inl, hyp = pnp_consensus_batched(P3, uv, K, thr, subsets=subsets)
    bits = (inl.cpu().numpy() * (1 << np.arange(uv.shape[1]))).sum(1)
    return dict(R=R.cpu().numpy(), t=t.cpu().numpy(), params=params.cpu().numpy(), mask=bits, hyp=hyp.cpu().numpy())


def _assert_agree(d, h, firm, what):
    bad = firm & ((d["hyp"] != h["hyp"]) | (d["mask"] != h["mask"]))
    assert not bad.any(), (what, np.nonzero(bad)[0][:10])
    ang = _ang(d["R"], h["R"])
    dt = np.abs(d["t"] - h["t"]).max(1) * 1e3
    off = firm & ((ang >= 1e-2) | (dt >= 1e-2))
    # the device contracts the LM's multiply-adds (the harness does not): an ill-conditioned refinement can amplify that, as the
    # plain solve's goldens see at large noise; at most 1 problem in 2000 may leave the tolerance
    assert off.sum() <= len(off) // 2000, (what, np.nonzero(off)[0][:10], ang[off][:5], dt[off][:5])


def outlier_problems(n, seed, with_center=True):
    pr = synth.pnp_problems(n, sigma=1.0, seed=seed, with_center=with_center)
    rng = np.random.default_rng(seed)
    uv = pr["uv"].astype(np.float64)
    npts = uv.shape[1]
    for i in range(n):
        k = int(rng.integers(0, 4))
        bad = rng.choice(npts, k, replace=False)
        ang, rad = rng.uniform(0, 2 * np.pi, k), rng.uniform(40, 150, k)
        uv[i, bad] += np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
    return pr["P3"], uv.astype(F32), pr["K"]


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("npts", [9, 8])
def test_kernels_match_harness_on_the_golden(host, golden_dir, npts):
    g = np.load(os.path.join(golden_dir, "pnp_consensus.npz"))
    tag = "_p%d" % npts
    P3, subsets = g["P3" + tag], g["subsets" + tag]
    for thr in np.unique(g["thr" + tag]):
        sel = g["thr" + tag] == thr
        uv = g["uv" + tag][sel]
        d = _dev_run(P3, uv, g["K"], float(thr), subsets)
        h = host_run(host, P3, uv, g["K"], float(thr), subsets)
        firm = g["gap" + tag][sel] > BORDER
        _assert_agree(d, h, firm, "golden thr %g" % thr)
        assert (d["hyp"][firm] == g["hyp" + tag][sel][firm]).all() and (d["mask"][firm] == g["mask" + tag][sel][firm]).all()
        assert _ang(d["R"][firm], g["R" + tag][sel][firm]).max() < 1e-2


@pytest.mark.parametrize("npts", [9, 8])
def test_kernels_match_harness_on_random_problems(host, npts):
    n = 10000 if npts == 9 else 3000
    P3, uv, K = outlier_problems(n, seed=40 + npts, with_center=npts == 9)
    subsets = consensus_subsets(P3)
    d = _dev_run(P3, uv, K, 8.0, subsets)
    h = host_run(host, P3, uv, K, 8.0, subsets)
    firm = h["gap"] > BORDER
    assert firm.mean() > 0.99
    _assert_agree(d, h, firm, "random")


@pytest.mark.parametrize("npts", [9, 8])
def test_all_inliers_is_bit_identical_to_the_plain_kernel(npts):
    pr = synth.pnp_problems(2000, sigma=1.0, seed=50, with_center=npts == 9)
    R, t, params, inl, hyp = pnp_consensus_batched(pr["P3"], pr["uv"], pr["K"])
    Rp, tp = pnp_batched(pr["P3"], pr["uv"], pr["K"])
    full = (hyp == 0) & inl.all(1)
    assert int(full.sum()) >= 1900
    assert torch.equal(R[full], Rp[full]) and torch.equal(t[full], tp[full])
    assert torch.equal(params[:, 3:], t)


def test_deterministic_and_independent_of_batch_and_position():
    P3, uv, K = outlier_problems(1000, seed=60)
    a = pnp_consensus_batched(P3, uv, K)
    b = pnp_consensus_batched(P3, uv, K)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    perm = np.random.default_rng(0).permutation(1000)[:137]
    c = pnp_consensus_batched(P3, uv[perm], K)
    idx = torch.from_numpy(perm).to(DEV)
    assert all(torch.equal(x[idx], y) for x, y in zip(a, c))
    P3n = np.repeat(P3[None], 1000, 0)                                  # per-problem points give the same bits as shared ones
    e = pnp_consensus_batched(P3n, uv, K)
    assert all(torch.equal(x, y) for x, y in zip(a, e))


def test_counted_empty_slots_are_zero():
    groups, per = 5, 7
    P3, uv, K = outlier_problems(groups * per, seed=70)
    subsets = consensus_subsets(P3)
    count = torch.tensor([0, 3, 7, 1, 5], dtype=torch.int32, device=DEV)
    n = groups * per
    P3d = torch.from_numpy(np.repeat(P3[None], n, 0)).to(DEV)
    uvd, Kd = torch.from_numpy(uv).to(DEV), torch.from_numpy(K).to(DEV)
    R = torch.full((n, 3, 3), 7.0, dtype=torch.float64, device=DEV)
    t, params = torch.full((n, 3), 7.0, dtype=torch.float64, device=DEV), torch.full((n, 6), 7.0, dtype=torch.float64, device=DEV)
    inl, hyp = torch.full((n,), 7, dtype=torch.int32, device=DEV), torch.full((n,), 7, dtype=torch.int32, device=DEV)
    wb = consensus_work_bytes(9, len(subsets), n)
    work = torch.empty(wb // 8, dtype=torch.float64, device=DEV)
    call("ssp_pnp_consensus", ptr(P3d), 0, ptr(uvd), ptr(Kd), 9, groups, per, ptr(count), subsets.ctypes.data, len(subsets), 8.0, 20, ptr(R),
         ptr(t), ptr(params), ptr(inl), ptr(hyp), ptr(work), wb, stream_ptr())
    full = pnp_consensus_batched(P3, uv, K)
    live = (torch.arange(per, device=DEV)[None] < count[:, None]).reshape(-1)
    for got, want in zip((R, t, params, inl, hyp), full[:3] + ((full[3].int() << torch.arange(9, device=DEV, dtype=torch.int32)).sum(1).int(), full[4])):
        assert torch.equal(got[live], want[live])
        assert not got[~live].any()


def test_bad_arguments_raise():
    P3, uv, K = outlier_problems(4, seed=80)
    for kw in (dict(reproj_thresh=0.0), dict(reproj_thresh=float("nan")), dict(subsets=np.array([0b111111 << 4], np.uint16))):
        with pytest.raises(SspError):
            pnp_consensus_batched(P3, uv, K, **kw)
    with pytest.raises(SspError):
        pnp_consensus_batched(P3[:6], uv[:, :6], K)


# ---------------------------------------------------------------------------------------------------- predictors
def _frames(n, seed, w=640, h=480):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _clone(r):
    return {k: v.clone() for k, v in r.items()}


def _corners(c):
    s = 1.0 + 0.1 * c
    return synth.box_points((0.038 * s, 0.039 * s, 0.046 * (2.0 - 0.05 * c)), with_center=False).T.astype(np.float64)


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


def _p3(corners):
    return np.concatenate([np.zeros((1, 3)), np.asarray(corners)[:3].T]).astype(F32)


@pytest.mark.parametrize("B", [1, 3])
def test_pose_predictor_consensus(single_model, B):
    from singleshotpose_b200.predict import PosePredictor
    corners = _corners(0)
    g = PosePredictor(single_model, corners, KM, batch=B, pnp="consensus")
    e = PosePredictor(single_model, corners, KM, batch=B, pnp="consensus", graph=False)
    plain = PosePredictor(single_model, corners, KM, batch=B)
    for seed in (1, 2):
        fr = _frames(B, seed)
        rg, re_, rp = _clone(g(fr)), _clone(e(fr)), _clone(plain(fr))
        assert g._last.graph is not None and all(torch.equal(rg[k], re_[k]) for k in rg)
        assert set(rg) == set(rp) | {"inliers", "hyp"} and torch.equal(rg["keypoints_px"], rp["keypoints_px"])
        R, t, params, inl, hyp = pnp_consensus_batched(_p3(corners), rg["keypoints_px"], KM)
        assert torch.equal(rg["R"], R) and torch.equal(rg["t"], t) and torch.equal(rg["inliers"], inl) and torch.equal(rg["hyp"], hyp)
        full = (hyp == 0) & inl.all(1)
        assert torch.equal(rg["R"][full], rp["R"][full])


def test_multi_pose_predictor_consensus(multi_model):
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    objs = {c: _corners(c) for c in (0, 4, 9)}
    kw = dict(batch=2, conf_thresh=0.02, pnp="consensus", reproj_thresh=6.0)
    g = MultiPosePredictor(multi_model, objs, KM, **kw)
    e = MultiPosePredictor(multi_model, objs, KM, graph=False, **kw)
    fr = _frames(2, 3)
    rg, re_ = _clone(g(fr)), _clone(e(fr))
    assert all(torch.equal(rg[k], re_[k]) for k in rg)
    P3 = np.repeat(np.stack([_p3(objs[c]) for c in sorted(objs)])[None], 2, 0).reshape(-1, 9, 3)
    R, t, params, inl, hyp = pnp_consensus_batched(P3, rg["keypoints_px"].reshape(-1, 9, 2), KM, 6.0)
    assert torch.equal(rg["R"].reshape(-1, 3, 3), R) and torch.equal(rg["inliers"].reshape(-1, 9), inl)
    assert torch.equal(rg["hyp"].reshape(-1), hyp) and rg["inliers"].shape == (2, 3, 9)


def test_instance_predictor_consensus_and_tracker_refusal(multi_model):
    from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor
    objs = {c: _corners(c) for c in (0, 4, 7, 11)}
    kw = dict(batch=2, conf_thresh=0.02, max_instances=16, pnp="consensus")
    g = InstancePosePredictor(multi_model, objs, KM, **kw)
    e = InstancePosePredictor(multi_model, objs, KM, graph=False, **kw)
    fr = _frames(2, 4)
    rg, re_ = _clone(g(fr)), _clone(e(fr))
    assert all(torch.equal(rg[k], re_[k]) for k in rg)
    count = rg["count"].cpu().numpy()
    assert count.sum() > 0
    for b in range(2):
        n = int(count[b])
        if n == 0:
            continue
        P3 = np.stack([_p3(objs[int(c)]) for c in rg["cls"][b, :n].cpu().numpy()])
        R, t, params, inl, hyp = pnp_consensus_batched(P3, rg["keypoints_px"][b, :n], KM)
        assert torch.equal(rg["R"][b, :n], R) and torch.equal(rg["inliers"][b, :n], inl) and torch.equal(rg["hyp"][b, :n], hyp)
        assert not rg["R"][b, n:].any() and not rg["inliers"][b, n:].any() and not rg["hyp"][b, n:].any()
    with pytest.raises(SspError, match="warm guess"):
        TrackingPosePredictor(multi_model, objs, KM, pnp="consensus")


# ---------------------------------------------------------------------------------------------------- evaluation tails
def test_evaluate_poses_batched_consensus_matches_oracle_loop():
    gen = torch.Generator().manual_seed(31)
    B = 6
    pr = synth.pnp_problems(B, sigma=0.0, seed=12)
    out = torch.randn(B, 20, 13, 13, generator=gen) * 0.3
    tgt = torch.zeros(B, 21)
    for b in range(B):                                   # plant noisy true keypoints in one confident cell; corner 3 wrong in odd frames
        uvn = pr["uv"][b] / np.array([640.0, 480.0], F32) + np.random.default_rng(b).normal(size=(9, 2)).astype(F32) * 1e-3
        if b % 2:
            uvn[3] += 0.12
        cx, cy = min(max(int(uvn[0, 0] * 13), 0), 12), min(max(int(uvn[0, 1] * 13), 0), 12)
        for k in range(9):
            vx, vy = uvn[k, 0] * 13 - cx, uvn[k, 1] * 13 - cy
            if k == 0:
                vx, vy = (np.log(np.clip(v, 1e-3, 1 - 1e-3) / (1 - np.clip(v, 1e-3, 1 - 1e-3))) for v in (vx, vy))
            out[b, 2 * k, cy, cx] = float(vx); out[b, 2 * k + 1, cy, cx] = float(vy)
        out[b, 18, cy, cx] = 6.0
        tgt[b, 1:19] = torch.from_numpy((pr["uv"][b] / np.array([640.0, 480.0], F32)).reshape(-1))
    verts = np.concatenate([np.random.default_rng(3).uniform(-0.04, 0.04, size=(3, 500)), np.ones((1, 500))])
    plain = utils.evaluate_poses_batched(out.cuda(), tgt, verts, pr["P3"], KM)
    res = utils.evaluate_poses_batched(out.cuda(), tgt, verts, pr["P3"], KM, pnp="consensus", reproj_thresh=8.0)
    assert torch.equal(res["R_gt"], plain["R_gt"]) and torch.equal(res["t_gt"], plain["t_gt"])
    subsets = consensus_subsets(pr["P3"])
    pr2d = (res["boxes"][:, :18].reshape(B, 9, 2) * torch.tensor([640.0, 480.0], device=DEV)).cpu().numpy()
    for b in range(B):
        o = consensus_ref(pr["P3"], pr2d[b], KM.astype(F32), 8.0, subsets)
        if o["gap"] <= BORDER:
            continue
        assert int(res["hyp"][b]) == o["hyp"] and np.array_equal(res["inliers"][b].cpu().numpy(), [(o["mask"] >> i) & 1 == 1 for i in range(9)])
        assert _ang(res["R_pr"][b].cpu().numpy(), o["R"]) < 1e-2 and np.abs(res["t_pr"][b].cpu().numpy() - o["t"]).max() * 1e3 < 1e-2
    odd = torch.arange(B, device=DEV) % 2 == 1
    assert not res["inliers"][odd, 3].any() and (res["angle_err_deg"][odd] < plain["angle_err_deg"][odd]).all()
    acc_p, acc_c = utils.pose_accuracy(plain, 0.1), utils.pose_accuracy(res, 0.1)
    assert acc_c["mean_angle_err"] < acc_p["mean_angle_err"]


def test_evaluate_multi_poses_batched_consensus_matches_oracle_loop():
    from singleshotpose_b200.utils_multi import evaluate_multi_poses_batched, get_3D_corners
    B, NC, NA = 3, 13, 5
    out = torch.randn(B, (19 + NC) * NA, 13, 13, generator=torch.Generator().manual_seed(5)).cuda()
    tgt = synth.targets_multi(B, seed=2)
    rng = np.random.default_rng(0)
    V = np.c_[rng.uniform(-1, 1, (200, 3)) * [0.038, 0.039, 0.046], np.ones(200)].T
    corners = get_3D_corners(V)
    plain = evaluate_multi_poses_batched(out, tgt, 0.05, NC, 9, NA, V, corners, KM)
    res = evaluate_multi_poses_batched(out, tgt, 0.05, NC, 9, NA, V, corners, KM, pnp="consensus")
    G = res["box"].shape[0]
    assert G > 0 and res["inliers"].shape == (G, 9)
    for k in ("box", "R_gt", "t_gt"):
        assert torch.equal(res[k], plain[k]), k
    P3 = np.concatenate([np.zeros((1, 3)), corners[:3].T]).astype(F32)
    subsets = consensus_subsets(P3)
    pr2d = (res["box"][:, :18].reshape(G, 9, 2) * torch.tensor([640.0, 480.0], device=DEV)).cpu().numpy()
    checked = 0
    for i in range(G):
        o = consensus_ref(P3, pr2d[i], KM.astype(F32), 8.0, subsets)
        if o["gap"] <= BORDER or not np.abs(o["t"]).max() < 10.0:
            continue
        assert int(res["hyp"][i]) == o["hyp"] and int((res["inliers"][i].int() << torch.arange(9, device=DEV, dtype=torch.int32)).sum()) == o["mask"]
        assert _ang(res["R_pr"][i].cpu().numpy(), o["R"]) < 1e-2 and np.abs(res["t_pr"][i].cpu().numpy() - o["t"]).max() * 1e3 < 1e-2
        checked += 1
    assert checked >= G - 1


# ---------------------------------------------------------------------------------------------------- command line
def test_cli_writes_inliers(cfg_multi_path, tmp_path):
    import glob
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import InstancePosePredictor, main
    from singleshotpose_b200.utils_multi import get_3D_corners
    root = str(tmp_path)
    synth.write_linemod_multi_like(root, n=2)
    paths = sorted(glob.glob(os.path.join(root, "LINEMOD", "*", "JPEGImages", "*.png")))[:3]
    V = np.random.default_rng(0).normal(size=(40, 3)) * 0.03
    ply = str(tmp_path / "obj.ply")
    with open(ply, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n" % len(V))
        for v in V:
            f.write("%.17g %.17g %.17g\n" % tuple(v))
    data = tmp_path / "occlusion.data"
    data.write_text("im_width = 640\nim_height = 480\nfx = 572.4114\nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    torch.manual_seed(4)
    wf = str(tmp_path / "m.weights")
    Darknet(cfg_multi_path).save_weights(wf)
    out = str(tmp_path / "det.npz")
    main(["--datacfg", str(data), "--modelcfg", cfg_multi_path, "--weightfile", wf, "--out", out, "--max-instances", "8",
          "--pnp", "consensus", "--reproj-thresh", "8", "--object", "0=%s" % ply] + paths)
    got = np.load(out)
    assert "inliers" in got.files and "hyp" in got.files and got["inliers"].shape == (len(got["cls"]), 9)
    m = Darknet(cfg_multi_path)
    m.load_weights(wf)
    m.cuda().eval()
    Km = np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]])
    pred = InstancePosePredictor(m, {0: get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)}, Km, max_instances=8, pnp="consensus")
    from PIL import Image
    rows = {k: [] for k in ("R", "inliers", "hyp")}
    for p in paths:
        r = pred(np.asarray(Image.open(p).convert("RGB"))[None], to_host=True)
        for k in rows:
            rows[k].append(r[k][0, :int(r["count"][0])])
    for k in rows:
        assert np.array_equal(got[k], np.concatenate(rows[k])), k
