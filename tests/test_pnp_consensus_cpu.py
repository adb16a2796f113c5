"""CPU checks of the consensus PnP (singleshotpose_b200/csrc/pnp_consensus_core.h): the rule compiled for the host by
tests/helpers/pnp_consensus_host.cpp and its numpy restatement (oracle/pnp_consensus_ref.py) against cv2 (tests/golden/
pnp_consensus.npz), the invariant against the plain solve, recovery from wrong keypoints, the depth rule, the subset table, the
argument checks of the C entry points and the command lines.  No device is touched."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from oracle.pnp_consensus_ref import consensus_ref
from singleshotpose_b200 import _lib, synth
from singleshotpose_b200.utils import check_pnp_args, consensus_subsets, consensus_work_bytes

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSP_ERR_ARG = -1
F32 = np.float32
BORDER = 1e-4        # px^2: a problem whose chosen hypothesis has an error this close to thr^2 may flip between implementations


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pnpchost") / "libpnpchost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "pnp_consensus_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host_consensus(host, P3, uv, K, thr=8.0, subsets=None):
    """-> R (n,3,3), t (n,3), params (n,6), inlier masks (n,), hyp (n,) of the harness; P3 (P,3) shared or (n,P,3)"""
    uv = np.ascontiguousarray(uv, F32)
    n, npts = uv.shape[:2]
    P3 = np.ascontiguousarray(P3, F32)
    subsets = np.ascontiguousarray(consensus_subsets(P3) if subsets is None else subsets, np.uint16)
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3)); params = np.zeros((n, 6)); inl = np.zeros(n, np.int32); hyp = np.zeros(n, np.int32)
    assert host.h_pnp_consensus(_p(P3), int(P3.ndim == 2), _p(uv), _p(np.ascontiguousarray(K, F32)), npts, C.c_longlong(n), _p(subsets),
                                len(subsets), C.c_double(thr), 20, _p(R), _p(t), _p(params), _p(inl), _p(hyp)) == 0
    return R, t, params, inl, hyp


def host_plain(host, P3, uv, K):
    uv = np.ascontiguousarray(uv, F32)
    n, npts = uv.shape[:2]
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3))
    assert host.h_pnp_plain(_p(np.ascontiguousarray(P3, F32)), 1, _p(uv), _p(np.ascontiguousarray(K, F32)), npts, C.c_longlong(n), 20,
                            _p(R), _p(t)) == 0
    return R, t


def _ang(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.einsum("...ij,...ij->...", Ra, Rb) - 1) / 2, -1, 1)))


def outlier_problems(n, k, sigma=1.0, seed=0, with_center=True):
    """seeded problems (synth.pnp_problems) with k keypoints moved by 40-150 px; -> problems dict, (n,) mask of the good points"""
    pr = synth.pnp_problems(n, sigma=sigma, seed=100 + seed, with_center=with_center)
    rng = np.random.default_rng(seed)
    npts = pr["uv"].shape[1]
    uv = pr["uv"].astype(np.float64)
    good = np.zeros(n, np.int64)
    for i in range(n):
        bad = rng.choice(npts, k, replace=False)
        ang, rad = rng.uniform(0, 2 * np.pi, k), rng.uniform(40, 150, k)
        uv[i, bad] += np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
        good[i] = sum(1 << j for j in range(npts) if j not in bad)
    pr["uv"] = uv.astype(F32)
    return pr, good


# ------------------------------------------------------------------------------------------------ against cv2
@pytest.mark.parametrize("npts", [9, 8])
def test_harness_matches_cv2_golden(host, golden_dir, npts):
    g = np.load(os.path.join(golden_dir, "pnp_consensus.npz"))
    tag = "_p%d" % npts
    uv, thr = g["uv" + tag], g["thr" + tag]
    assert np.array_equal(g["subsets" + tag], consensus_subsets(g["P3" + tag]))
    firm = g["gap" + tag] > BORDER
    assert firm.sum() >= len(firm) - 2
    hyp = g["hyp" + tag]
    assert (hyp == -1).any() and (hyp == 0).any() and (hyp > 0).any()
    n_few = 0
    for i in range(len(uv)):
        R, t, params, inl, h = host_consensus(host, g["P3" + tag], uv[i:i + 1], g["K"], thr[i], g["subsets" + tag])
        if not firm[i]:
            continue
        assert h[0] == hyp[i] and inl[0] == g["mask" + tag][i], (i, h[0], hyp[i], inl[0], g["mask" + tag][i])
        assert _ang(R[0], g["R" + tag][i]) < 1e-2 and np.abs(t[0] - g["t" + tag][i]).max() * 1e3 < 1e-2, i
        assert np.array_equal(params[0, 3:], t[0])
        n_few += 0 < bin(int(inl[0])).count("1") < 6
    assert n_few > 0                                                  # the unrefined branch is covered too


@pytest.mark.parametrize("npts", [9, 8])
def test_oracle_matches_cv2_golden(golden_dir, npts):
    g = np.load(os.path.join(golden_dir, "pnp_consensus.npz"))
    tag = "_p%d" % npts
    for i in range(0, len(g["uv" + tag]), 3):                         # every third problem: the numpy LM is slow
        o = consensus_ref(g["P3" + tag], g["uv" + tag][i], g["K"], g["thr" + tag][i], g["subsets" + tag])
        if g["gap" + tag][i] <= BORDER:
            continue
        assert o["hyp"] == g["hyp" + tag][i] and o["mask"] == g["mask" + tag][i], i
        assert _ang(o["R"], g["R" + tag][i]) < 1e-2 and np.abs(o["t"] - g["t" + tag][i]).max() * 1e3 < 1e-2, i


# ------------------------------------------------------------------------------------------------ the rule
@pytest.mark.parametrize("npts", [9, 8])
def test_all_inliers_is_bit_identical_to_the_plain_solve(host, npts):
    pr = synth.pnp_problems(200, sigma=1.0, seed=21, with_center=npts == 9)
    R, t, params, inl, hyp = host_consensus(host, pr["P3"], pr["uv"], pr["K"])
    Rp, tp = host_plain(host, pr["P3"], pr["uv"], pr["K"])
    full = (hyp == 0) & (inl == (1 << npts) - 1)
    assert full.sum() >= 190
    assert R[full].tobytes() == Rp[full].tobytes() and t[full].tobytes() == tp[full].tobytes()


@pytest.mark.parametrize("k,need", [(1, 145), (2, 140)])
def test_recovers_from_wrong_keypoints(host, k, need):
    pr, good = outlier_problems(150, k, seed=k)
    R, t, params, inl, hyp = host_consensus(host, pr["P3"], pr["uv"], pr["K"])
    err = _ang(R, pr["R"])
    assert ((inl == good) & (err <= 5)).sum() >= need, ((inl == good) & (err <= 5)).sum()
    Rp, _tp = host_plain(host, pr["P3"], pr["uv"], pr["K"])
    assert np.median(_ang(Rp, pr["R"])) > 30                          # the plain solve fails on the same problems


def test_depth_rule_keeps_the_pose_in_front_of_the_camera(host):
    pr, good = outlier_problems(150, 1, seed=7)
    P3, K = pr["P3"], pr["K"]
    subsets = np.ascontiguousarray(consensus_subsets(P3), np.uint16)
    n, H1 = len(pr["uv"]), len(subsets) + 1
    slots = np.zeros((n, H1, 15)); hmask = np.zeros((n, H1), np.uint32)
    assert host.h_consensus_hyps(_p(P3), 1, _p(pr["uv"]), _p(K), 9, C.c_longlong(n), _p(subsets), len(subsets), C.c_double(8.0), 20,
                                 _p(slots), _p(hmask)) == 0
    R, t, params, inl, hyp = host_consensus(host, P3, pr["uv"], K)
    found = 0
    for i in range(n):
        Rh, th = slots[i, :, :9].reshape(H1, 3, 3), slots[i, :, 12:]
        Pc = np.einsum("hij,pj->hpi", Rh, P3.astype(np.float64)) + th[:, None]
        e2 = ((K[0, 0] * Pc[..., 0] / Pc[..., 2] + K[0, 2] - pr["uv"][i, :, 0]) ** 2
              + (K[1, 1] * Pc[..., 1] / Pc[..., 2] + K[1, 2] - pr["uv"][i, :, 1]) ** 2)
        counts = (e2 <= 64.0).sum(1)                                   # the scores without the depth rule
        behind = (Pc[..., 2] <= 0).any(1)
        assert not hmask[i][behind].any()                              # the rule: no inliers behind the camera
        best = int(np.argmax(counts))                                 # the selection without the rule (lower index on a tie)
        if behind[best]:
            found += 1
            z = P3.astype(np.float64) @ R[i].T + t[i]
            assert (z[:, 2] > 0).all() and hyp[i] >= 0 and not behind[hyp[i]]
    assert found >= 1


def _dlt_nullity(P, K):
    """nullity of the DLT system of an exact projection of the points P (n, 3) under a generic pose"""
    r = np.array([0.3, -0.5, 0.2]); th = np.linalg.norm(r); u = r / th
    ux = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]])
    R = np.cos(th) * np.eye(3) + (1 - np.cos(th)) * np.outer(u, u) + np.sin(th) * ux
    Pc = P @ R.T + np.array([0.05, -0.02, 0.9])
    x, y = Pc[:, 0] / Pc[:, 2], Pc[:, 1] / Pc[:, 2]
    L = np.zeros((2 * len(P), 12))
    for i, X in enumerate(np.c_[P, np.ones(len(P))]):
        L[2 * i, :4] = X; L[2 * i, 8:] = -x[i] * X
        L[2 * i + 1, 4:8] = X; L[2 * i + 1, 8:] = -y[i] * X
    s = np.linalg.svd(L, compute_uv=False)
    return int((s < 1e-9 * s[0]).sum()) + (12 - len(s))


@pytest.mark.parametrize("npts,kept", [(9, 60), (8, 28)])
def test_consensus_subsets(npts, kept):
    P = synth.box_points(with_center=npts == 9).astype(np.float64)
    tab = consensus_subsets(P)
    assert tab.dtype == np.uint16 and len(tab) == kept
    allm = [sum(1 << i for i in S) for S in itertools.combinations(range(npts), 6)]
    assert list(tab) == [m for m in allm if m in set(tab.tolist())]   # lexicographic order
    assert all(bin(int(m)).count("1") == 6 for m in tab)
    for m in allm:
        idx = [i for i in range(npts) if (m >> i) & 1]
        assert _dlt_nullity(P[idx], synth.intrinsics()) == (1 if m in set(tab.tolist()) else 2), idx
    assert np.array_equal(consensus_subsets([P, P * 2.0]), tab)       # the boxes of several classes share the table


# ------------------------------------------------------------------------------------------------ ABI and command line
def test_symbols_are_declared_and_exported():
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        text = f.read()
    assert "int ssp_pnp_consensus(" in text and "int ssp_pnp_consensus_work_bytes(" in text
    lib = _lib.load()
    for name in ("ssp_pnp_consensus", "ssp_pnp_consensus_work_bytes"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)


def _fake(a):
    return C.c_void_p(0x10000 * a) if a else None


def test_entry_points_reject_bad_arguments():
    lib = _lib.load()
    good = np.array(consensus_subsets(synth.box_points()), np.uint16)
    wb = consensus_work_bytes(9, len(good), 8)
    assert wb == 8 * 61 * (15 * 8 + 4)
    out = C.c_longlong(0)
    for args in ((6, 60, 8), (11, 60, 8), (9, 0, 8), (9, 211, 8), (9, 60, -1)):
        assert lib.ssp_pnp_consensus_work_bytes(*args, C.byref(out)) == SSP_ERR_ARG, args
    assert lib.ssp_pnp_consensus_work_bytes(9, 60, 8, None) == SSP_ERR_ARG

    def run(P3=1, uv=1, K=1, np_=9, groups=2, per=4, count=0, tab=good, thr=8.0, it=20, R=1, t=1, params=1, inl=1, hyp=1, work=1,
            wbytes=wb):
        tab = np.ascontiguousarray(tab, np.uint16)
        return lib.ssp_pnp_consensus(_fake(P3), 0, _fake(uv), _fake(K), np_, groups, per, _fake(count), C.c_void_p(tab.ctypes.data),
                                     len(tab), thr, it, _fake(R), _fake(t), _fake(params), _fake(inl), _fake(hyp), _fake(work), wbytes,
                                     None)
    bad_tabs = [good[:0], np.tile(good, 4)[:211], np.array([0b111111 << 4], np.uint16), np.array([0b11111], np.uint16),
                np.array([0b1111111], np.uint16)]
    for kw in (dict(P3=0), dict(uv=0), dict(K=0), dict(R=0), dict(t=0), dict(params=0), dict(inl=0), dict(hyp=0), dict(work=0),
               dict(np_=6), dict(np_=11), dict(groups=-1), dict(per=0), dict(thr=0.0), dict(thr=-1.0), dict(thr=float("nan")),
               dict(thr=float("inf")), dict(it=0), dict(wbytes=wb - 1)) + tuple(dict(tab=b) for b in bad_tabs):
        assert run(**kw) == SSP_ERR_ARG, kw
    run(tab=bad_tabs[2])
    assert b"subset table" in lib.ssp_last_error()
    assert run(np_=8, tab=bad_tabs[2][:0]) == SSP_ERR_ARG
    eight = np.array(consensus_subsets(synth.box_points(with_center=False)), np.uint16)
    assert run(np_=8, tab=good) == SSP_ERR_ARG                        # masks with bit 8 for 8 points
    assert run(groups=0, np_=8, tab=eight, wbytes=0) == 0             # nothing to solve: no launch


def test_pnp_argument_checks():
    assert check_pnp_args("consensus", 8) == ("consensus", 8.0)
    for pnp, thr in (("ransac", 8.0), ("plain", 0.0), ("consensus", -1.0), ("consensus", float("nan")), ("consensus", float("inf"))):
        with pytest.raises(_lib.SspError):
            check_pnp_args(pnp, thr)
    with pytest.raises(_lib.SspError):
        consensus_subsets(synth.box_points()[:6])


def test_cli_pnp_checks():
    from singleshotpose_b200 import predict, predict_multi
    from singleshotpose_b200.predict_instances import parse_args
    base = ["--datacfg", "d.data", "--modelcfg", "m.cfg", "--weightfile", "w"]
    a = parse_args(base + ["a.png"])
    assert a.pnp == "plain" and a.reproj_thresh == 8.0
    a = parse_args(base + ["--pnp", "consensus", "--reproj-thresh", "4", "a.png"])
    assert a.pnp == "consensus" and a.reproj_thresh == 4.0
    for bad in (["--reproj-thresh", "0"], ["--reproj-thresh", "-2"], ["--reproj-thresh", "nan"]):
        with pytest.raises(_lib.SspError):
            parse_args(base + ["--pnp", "consensus"] + bad + ["a.png"])
    with pytest.raises(_lib.SspError, match="warm guess"):
        parse_args(base + ["--track", "--pnp", "consensus", "a.png"])
    with pytest.raises(SystemExit):
        parse_args(base + ["--pnp", "ransac", "a.png"])
    for main in (predict.main, predict_multi.main):                   # checked before the .data file is read
        extra = ["--object", "0=x.ply"] if main is predict_multi.main else []
        with pytest.raises(_lib.SspError, match="reproj_thresh"):
            main(base + extra + ["--pnp", "consensus", "--reproj-thresh", "0", "a.png"])


def test_tracker_refuses_consensus():
    from singleshotpose_b200.predict_instances import TrackingPosePredictor
    with pytest.raises(_lib.SspError, match="warm guess"):
        TrackingPosePredictor(None, synth.box_points(with_center=False).T, synth.intrinsics(), pnp="consensus")
