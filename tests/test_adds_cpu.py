"""CPU tests of the ADD-S / ADD / diameter rules (singleshotpose_b200/csrc/adds_core.h) and of utils.pose_accuracy:
  * the rules compiled for the host by tests/helpers/adds_host.cpp, in the kernels' order, against the reference's adi,
    ADD and calc_pts_diameter through the committed golden (tests/golden/adds.npz, written by tests/golden/make_golden_adds.py):
    the diameter bit for bit, ADD-S and ADD within rtol 1e-12;
  * pose_accuracy against the summary figures of the reference's valid.py, exactly;
  * the argument checks of ssp_adds_batched, ssp_adds_work_bytes and ssp_mesh_diameter."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from singleshotpose_b200 import _lib, synth, utils, utils_host

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_SYM = 4          # make_golden_adds.py: the exact symmetric pairs are rows [-2 N_SYM, -N_SYM) of mesh_s


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "adds.npz"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("addshost") / "libaddshost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "adds_host.cpp")])
    lib = C.CDLL(so)
    lib.h_mesh_diameter.restype = C.c_double
    lib.h_mesh_diameter.argtypes = [C.c_void_p, C.c_int]
    lib.h_adds_batched.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host_adds(host, X, Rt_est, Rt_gt):
    X = np.ascontiguousarray(X, np.float64)
    E, G = np.ascontiguousarray(Rt_est, np.float64), np.ascontiguousarray(Rt_gt, np.float64)
    adds, add = np.zeros(len(E)), np.zeros(len(E))
    assert host.h_adds_batched(_p(X), len(X), _p(E), _p(G), len(E), _p(adds), _p(add)) == 0
    return adds, add


# ------------------------------------------------------------------------------------------------ host build vs reference golden
@pytest.mark.parametrize("mesh", ["a", "s"])
def test_host_diameter_is_bit_identical_to_reference(golden, host, mesh):
    X = np.ascontiguousarray(golden["mesh_" + mesh])
    d = host.h_mesh_diameter(_p(X), len(X))
    assert d.hex() == float(golden["diam_" + mesh]).hex()


@pytest.mark.parametrize("mesh", ["a", "s"])
def test_host_adds_matches_reference_golden(golden, host, mesh):
    adds, add = host_adds(host, golden["mesh_" + mesh], golden["Rt_est_" + mesh], golden["Rt_gt_" + mesh])
    want_adds, want_add = golden["adds_" + mesh], golden["add_" + mesh]
    sym = np.zeros(len(adds), bool)
    if mesh == "s":
        sym[-2 * N_SYM:-N_SYM] = True
    # exact symmetric pairs: both sides are rounding noise (about 1e-17 m), no relative comparison is meaningful
    np.testing.assert_allclose(adds[~sym], want_adds[~sym], rtol=1e-12, atol=0)
    assert (np.abs(adds[sym]) < 1e-12).all() and (np.abs(want_adds[sym]) < 1e-12).all()
    np.testing.assert_allclose(add, want_add, rtol=1e-12, atol=0)
    assert (want_add[sym] > 0.05).all()                                # the symmetric pose is a miss under ADD


def test_host_adds_matches_scipy_small_and_odd_sizes(host):
    rng = np.random.default_rng(5)
    for nv in (1, 7, 1025):                                            # one vertex, one partial tile, one vertex past a query block
        X = rng.uniform(-0.05, 0.05, size=(nv, 3))
        R = synth._rodrigues(rng.normal(size=(3, 3)))
        t = rng.uniform(-0.1, 0.1, size=(3, 3)) + np.array([0, 0, 0.8])
        Rt = np.concatenate([R, t[:, :, None]], 2)
        E, G = Rt[:2], Rt[1:]
        adds, add = host_adds(host, X, E, G)
        for p in range(2):
            Xh = np.c_[X, np.ones(nv)].T
            pe, pg = (E[p] @ Xh).T, (G[p] @ Xh).T
            assert adds[p] == pytest.approx(utils_host.adi(pe, pg), rel=1e-12)
            assert add[p] == pytest.approx(np.linalg.norm(pg - pe, axis=1).mean(), rel=1e-12)


# ------------------------------------------------------------------------------------------------ pose_accuracy
def _golden_results(golden, split=None):
    keys = dict(pixel_err="errs_2d", vertex_dist="errs_3d", trans_err="errs_trans", angle_err_deg="errs_angle", corner_err_px="errs_corner2D")
    adds = golden["adds_s"][golden["summary_idx"]]
    res = dict({k: torch.from_numpy(golden[v]) for k, v in keys.items()}, adds_dist=torch.from_numpy(adds))
    if split is None:
        return res
    return [{k: v[:split] for k, v in res.items()}, {k: v[split:] for k, v in res.items()}]


FIGURES = ("acc", "acc3d10", "acc5cm5deg", "corner_acc", "mean_err_2d", "mean_vertex_err", "mean_corner_err_2d", "mean_trans_err",
           "mean_angle_err", "mean_pixel_err", "acc_adds10")


@pytest.mark.parametrize("split", [None, 7])
def test_pose_accuracy_equals_reference_summary(golden, split):
    acc = utils.pose_accuracy(_golden_results(golden, split), float(golden["diam_s"]))
    for k in FIGURES:
        assert acc[k] == golden[k][()], k
    assert golden["acc_adds10"] > golden["acc3d10"]                    # the near-symmetric poses pass ADD-S only
    printed = "\n".join(golden["printed"])
    assert "= {:.2f}%".format(acc["acc"]) in printed and "Mean vertex error is %f" % acc["mean_vertex_err"] in printed
    assert "angle error: %f degree" % acc["mean_angle_err"] in printed


def test_pose_accuracy_without_adds_and_threshold(golden):
    res = _golden_results(golden)
    del res["adds_dist"]
    acc = utils.pose_accuracy(res, float(golden["diam_s"]), px_threshold=10)
    assert "acc_adds10" not in acc
    e = golden["errs_2d"]
    assert acc["acc"] == len(np.where(e <= 10)[0]) * 100. / (len(e) + 1e-5)


# ------------------------------------------------------------------------------------------------ the C ABI
def test_adds_abi_rejects_bad_arguments():
    d, n0 = C.c_void_p(1), None
    call = lambda *a: _lib.call("ssp_adds_batched", *a)
    ok = lambda nv=100, n=4, wb=1 << 20: (d, nv, d, d, n, d, d, d, wb, n0)
    for args in ((n0,) + ok()[1:], ok()[:2] + (n0,) + ok()[3:], ok()[:5] + (n0,) + ok()[6:], ok()[:7] + (n0,) + ok()[8:]):
        with pytest.raises(_lib.SspError, match="bad argument"):
            call(*args)
    with pytest.raises(_lib.SspError, match="bad argument"):
        call(*ok(nv=0))
    with pytest.raises(_lib.SspError, match="bad argument"):
        call(*ok(n=-1))
    with pytest.raises(_lib.SspError, match="SSP_ADDS_MAX_VERTICES"):
        call(*ok(nv=(1 << 20) + 1))
    with pytest.raises(_lib.SspError, match="work buffer"):
        call(*ok(wb=_lib.load().ssp_adds_work_bytes(100, 4) - 8))
    assert call(*ok(n=0)) == 0                                         # n = 0: returns before any device access
    lib = _lib.load()
    assert lib.ssp_adds_work_bytes(1 << 20, 4) == 2 * 4 * 1024 * 8 and lib.ssp_adds_work_bytes(100000, 1) > 0
    assert lib.ssp_adds_work_bytes(0, 4) < 0 and lib.ssp_adds_work_bytes((1 << 20) + 1, 4) < 0 and lib.ssp_adds_work_bytes(10, -1) < 0


def test_mesh_diameter_abi_rejects_bad_arguments():
    d = C.c_void_p(1)
    for args in ((None, 10, d, None), (d, 10, None, None), (d, 0, d, None)):
        with pytest.raises(_lib.SspError, match="bad argument"):
            _lib.call("ssp_mesh_diameter", *args)
    with pytest.raises(_lib.SspError, match="SSP_ADDS_MAX_VERTICES"):
        _lib.call("ssp_mesh_diameter", d, (1 << 20) + 1, d, None)
