"""GPU tests of ADD-S, ADD and the mesh diameter (utils.adi_batched, utils.mesh_diameter, ssp_adds_batched, ssp_mesh_diameter)
against the reference's adi / calc_pts_diameter through tests/golden/adds.npz, against scipy (utils_host.adi) and against the
host build of the same rules (tests/helpers/adds_host.cpp), plus the adds=True paths of both evaluation tails."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from singleshotpose_b200 import synth, utils, utils_host, utils_multi

pytestmark = pytest.mark.gpu
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
    lib.h_adds_batched.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    return lib


def _poses(rng, n, deg=5.0, sigma_t=0.01):
    """(est, gt) (n, 3, 4) fp64: random poses 0.6-1.1 m away, the estimate rotated by `deg` and shifted by ~sigma_t"""
    R = synth._rodrigues(rng.normal(size=(n, 3)))
    t = np.stack([rng.uniform(-.1, .1, n), rng.uniform(-.07, .07, n), rng.uniform(.6, 1.1, n)], 1)
    ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    dR = synth._rodrigues(ax * np.deg2rad(deg))
    est = np.concatenate([dR @ R, (t + rng.normal(0, sigma_t, (n, 3)))[:, :, None]], 2)
    return est, np.concatenate([R, t[:, :, None]], 2)


def _scipy_adi(X, Re, Rg):
    Xh = np.c_[X, np.ones(len(X))].T
    return utils_host.adi(utils.compute_transformation(Xh, Re).T, utils.compute_transformation(Xh, Rg).T)


def _add(X, Re, Rg):
    Xh = np.c_[X, np.ones(len(X))].T
    return np.mean(np.linalg.norm(utils.compute_transformation(Xh, Rg) - utils.compute_transformation(Xh, Re), axis=0))


# ------------------------------------------------------------------------------------------------ against the reference golden
@pytest.mark.parametrize("mesh", ["a", "s"])
def test_matches_reference_golden(golden, host, mesh):
    X, E, G = golden["mesh_" + mesh], golden["Rt_est_" + mesh], golden["Rt_gt_" + mesh]
    adds, add = (v.cpu().numpy() for v in utils.adi_batched(X, E, G, with_add=True))
    want = golden["adds_" + mesh]
    sym = np.zeros(len(want), bool)
    if mesh == "s":
        sym[-2 * N_SYM:-N_SYM] = True
        assert (adds[sym] < 1e-9).all() and (add[sym] > 0.05).all()   # symmetric pose: ADD-S about 0, ADD large
    np.testing.assert_allclose(adds[~sym], want[~sym], rtol=1e-12, atol=0)
    np.testing.assert_allclose(add, golden["add_" + mesh], rtol=1e-12, atol=0)
    # the host build of adds_core.h, in the kernel's order, gives the same bits
    h_adds, h_add = np.zeros(len(E)), np.zeros(len(E))
    Xc, Ec, Gc = (np.ascontiguousarray(a, np.float64) for a in (X, E, G))
    assert host.h_adds_batched(Xc.ctypes.data, len(Xc), Ec.ctypes.data, Gc.ctypes.data, len(Ec), h_adds.ctypes.data, h_add.ctypes.data) == 0
    np.testing.assert_array_equal(adds, h_adds)
    np.testing.assert_array_equal(add, h_add)
    # the diameter, bit for bit, from either vertex layout and from float64 tensors
    assert utils.mesh_diameter(X).hex() == float(golden["diam_" + mesh]).hex()
    assert utils.mesh_diameter(torch.from_numpy(X).cuda()).hex() == float(golden["diam_" + mesh]).hex()
    # (4, Nv) homogeneous vertices as valid.py holds them give the same ADD-S
    Xh = np.c_[X, np.ones(len(X))].T
    assert torch.equal(utils.adi_batched(Xh, E, G).cpu(), torch.from_numpy(adds))


# ------------------------------------------------------------------------------------------------ against scipy
@pytest.mark.parametrize("nv", [1, 1000, 20000])
def test_matches_scipy(nv):
    """one vertex; a size that fills neither a tile (256) nor a query block (1024); a large mesh"""
    rng = np.random.default_rng(nv)
    X = rng.uniform(-0.05, 0.05, size=(nv, 3))
    n = 3 if nv > 10000 else 8
    E, G = _poses(rng, n)
    adds, add = (v.cpu().numpy() for v in utils.adi_batched(X.T, E, G, with_add=True))
    for p in range(n):
        assert adds[p] == pytest.approx(_scipy_adi(X, E[p], G[p]), rel=1e-12)
        assert add[p] == pytest.approx(_add(X, E[p], G[p]), rel=1e-12)
    assert utils.mesh_diameter(X) == utils_host.calc_pts_diameter(X)


def test_float32_vertices_are_converted_on_the_device():
    rng = np.random.default_rng(3)
    X = rng.uniform(-0.05, 0.05, size=(700, 3)).astype(np.float32)
    E, G = _poses(rng, 4)
    got = utils.adi_batched(torch.from_numpy(X).cuda(), E, G)
    want = utils.adi_batched(X.astype(np.float64), E, G)
    assert got.dtype == torch.float64 and torch.equal(got, want)
    assert utils.mesh_diameter(X) == utils_host.calc_pts_diameter(X.astype(np.float64))


# ------------------------------------------------------------------------------------------------ determinism and n = 0
def test_bit_identical_across_batches_and_launches():
    rng = np.random.default_rng(11)
    X = rng.uniform(-0.05, 0.05, size=(3000, 3))
    E, G = _poses(rng, 40, deg=10.0)
    full = utils.adi_batched(X, E, G)
    for _ in range(3):
        assert torch.equal(utils.adi_batched(X, E, G), full)
    rev = utils.adi_batched(X, E[::-1].copy(), G[::-1].copy())
    assert torch.equal(rev.flip(0), full)
    for p in (0, 17, 39):
        assert torch.equal(utils.adi_batched(X, E[p:p + 1], G[p:p + 1]), full[p:p + 1])
        assert torch.equal(utils.adi_batched(X, E[p], G[p]), full[p:p + 1])


def test_empty_batch_is_a_no_op():
    X = np.random.default_rng(0).uniform(-0.05, 0.05, size=(100, 3))
    adds, add = utils.adi_batched(X, np.zeros((0, 3, 4)), np.zeros((0, 3, 4)), with_add=True)
    assert adds.shape == (0,) and add.shape == (0,) and adds.is_cuda and adds.dtype == torch.float64


# ------------------------------------------------------------------------------------------------ the evaluation tails
def _planted_single(B, seed, noise=3e-3):
    """network outputs with the (noisy) true keypoints planted in one confident cell per image, as test_gpu_heads.py does"""
    gen = torch.Generator().manual_seed(seed)
    pr = synth.pnp_problems(B, sigma=0.0, seed=seed)
    out = torch.randn(B, 20, 13, 13, generator=gen) * 0.3
    tgt = torch.zeros(B, 21)
    for b in range(B):
        uvn = pr["uv"][b] / np.array([640.0, 480.0], np.float32) + np.random.default_rng(b).normal(size=(9, 2)).astype(np.float32) * noise
        cx, cy = min(max(int(uvn[0, 0] * 13), 0), 12), min(max(int(uvn[0, 1] * 13), 0), 12)
        for k in range(9):
            vx, vy = uvn[k, 0] * 13 - cx, uvn[k, 1] * 13 - cy
            if k == 0:
                vx, vy = (np.log(np.clip(v, 1e-3, 1 - 1e-3) / (1 - np.clip(v, 1e-3, 1 - 1e-3))) for v in (vx, vy))
            out[b, 2 * k, cy, cx] = float(vx); out[b, 2 * k + 1, cy, cx] = float(vy)
        out[b, 18, cy, cx] = 6.0
        tgt[b, 1:19] = torch.from_numpy((pr["uv"][b] / np.array([640.0, 480.0], np.float32)).reshape(-1))
    return out, tgt, pr["P3"]


def _check_against_loop(res, X, n):
    Rt_gt = torch.cat([res["R_gt"], res["t_gt"].unsqueeze(2)], 2).cpu().numpy()
    Rt_pr = torch.cat([res["R_pr"], res["t_pr"].unsqueeze(2)], 2).cpu().numpy()
    adds = res["adds_dist"].cpu().numpy()
    assert adds.shape == (n,) and res["adds_dist"].dtype == torch.float64
    for i in range(n):
        assert adds[i] == pytest.approx(_scipy_adi(X, Rt_pr[i], Rt_gt[i]), rel=1e-12)
    return Rt_gt, Rt_pr


def test_evaluate_poses_batched_adds():
    out, tgt, P3 = _planted_single(6, 21)
    rng = np.random.default_rng(3)
    X = rng.uniform(-0.04, 0.04, size=(1500, 3))
    verts = np.c_[X, np.ones(len(X))].T
    Kc = synth.intrinsics()
    base = utils.evaluate_poses_batched(out.cuda(), tgt, verts, P3, Kc)
    res = utils.evaluate_poses_batched(out.cuda(), tgt, verts, P3, Kc, adds=True)
    assert set(res) == set(base) | {"adds_dist"} and "adds_dist" not in base
    for k in base:
        assert torch.equal(res[k], base[k]), k
    _check_against_loop(res, X, 6)
    assert (res["adds_dist"] <= res["vertex_dist"] + 1e-6).all()      # the nearest vertex is never farther than the same vertex


def test_evaluate_multi_poses_batched_adds():
    gen = torch.Generator().manual_seed(70)
    B, NC, K, NA = 6, 13, 9, 5
    out = torch.randn(B, (2 * K + 1 + NC) * NA, 13, 13, generator=gen)
    out[:, [18 + 32 * a for a in range(NA)]] += 1.0
    tgt = synth.targets_multi(B, seed=71, num_classes=4, max_gts=3)
    tgt[2] = 0                                                          # an image without ground truths
    rng = np.random.default_rng(5)
    X = np.concatenate([synth.box_points(with_center=False).astype(np.float64), rng.uniform(-1, 1, (992, 3)) * np.array([0.038, 0.039, 0.046])])
    V = np.c_[X, np.ones(len(X))].T
    corners = utils_multi.get_3D_corners(V)
    run = lambda **kw: utils_multi.evaluate_multi_poses_batched(out.cuda(), tgt, 0.05, NC, K, NA, V, corners, synth.intrinsics(), **kw)
    base, res = run(), run(adds=True)
    assert set(res) == set(base) | {"adds_dist", "vertex_dist"} and "adds_dist" not in base
    for k in base:
        assert torch.equal(res[k], base[k]), k
    G = res["pixel_err"].shape[0]
    assert G > 3
    Rt_gt, Rt_pr = _check_against_loop(res, X, G)
    vd = res["vertex_dist"].cpu().numpy()
    assert res["vertex_dist"].dtype == torch.float64
    for i in range(G):
        assert vd[i] == pytest.approx(_add(X, Rt_pr[i], Rt_gt[i]), rel=1e-12)
    empty = utils_multi.evaluate_multi_poses_batched(out[2:3].cuda(), tgt[2:3], 0.05, NC, K, NA, V, corners, synth.intrinsics(), adds=True)
    assert empty["adds_dist"].shape == (0,) and empty["vertex_dist"].shape == (0,)
