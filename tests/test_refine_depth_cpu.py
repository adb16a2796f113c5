"""CPU checks of the depth refinement (singleshotpose_b200/csrc/refine_depth_core.h), compiled for the host by
tests/helpers/refine_depth_host.cpp: the harness against the numpy oracle (oracle/refine_depth_ref.py) on rendered scenes, the
Jacobian against central differences, outward vertex normals of either winding, the status edges, and what the refinement is
worth on perturbed poses.  No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.pose_filter_ref import so3_exp
from oracle.refine_depth_ref import add_error, refine_ref, render_depth_ref
from singleshotpose_b200 import synth
from singleshotpose_b200.utils import check_refine_args, vertex_normals
from singleshotpose_b200._lib import SspError

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KM = synth.intrinsics()
W, H, SCALE = 640, 480, 0.001
BARREL = np.array([-0.3, 0.12, 1e-3, -5e-4, -0.02, 0, 0, 0])          # the distortion tests' barrel calibration (pnp_dist.npz)
V, F = synth.closed_mesh()
N = vertex_normals(V, F)
MODEL = np.ascontiguousarray(np.concatenate([V, N], 1))
DIAM = float(max(np.linalg.norm(V[i] - V, axis=1).max() for i in range(len(V))))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rdhost") / "librdhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "refine_depth_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def host_refine(lib, depth, model, R, t, diam, iters=10, gate=(0.5, 0.02), dist=None, K=KM, count=None, per_group=1):
    """h_refine_depth over n problems of one class: depth (groups, H, W), R (n, 3, 3), t (n, 3)"""
    depth = np.ascontiguousarray(depth, np.uint16)
    R, t = np.ascontiguousarray(R, np.float64).reshape(-1, 9), np.ascontiguousarray(t, np.float64).reshape(-1, 3)
    n, groups = len(R), depth.shape[0]
    assert n == groups * per_group
    off = np.array([0, len(model)], np.int32)
    dm = np.array([diam])
    cls = np.zeros(n, np.int32)
    cnt = None if count is None else np.ascontiguousarray(count, np.int32)
    Ro, to, pts, rmse, st = np.zeros((n, 9)), np.zeros((n, 3)), np.zeros(n, np.int32), np.zeros(n), np.zeros(n, np.int32)
    d = None if dist is None else np.ascontiguousarray(dist, np.float64)
    rc = lib.h_refine_depth(_p(depth), depth.shape[2], depth.shape[1], C.c_double(SCALE), _p(np.ascontiguousarray(K, np.float64)), _p(d),
                            _p(np.ascontiguousarray(model)), _p(off), _p(dm), 1, _p(cls), groups, per_group, _p(cnt), _p(R), _p(t), iters,
                            C.c_double(gate[0]), C.c_double(gate[1]), _p(Ro), _p(to), _p(pts), _p(rmse), _p(st))
    assert rc == 0
    return Ro.reshape(n, 3, 3), to, pts, rmse, st


# ---------------------------------------------------------------------------------------------------- scenes
def scene_depth(R, t, plane=False, occluder=False, holes=False, noise=False, dist=None, seed=0):
    """the rendered depth (H, W) uint16 of the mesh at (R, t), optionally with a table plane 6 cm behind its centre, an occluder
    10 cm in front of it over the left third of its silhouette, holes (about 20 % of the pixels and a block) and +-1 unit noise"""
    Pc = [V @ R.T + t]
    Fs = [F]
    nv = len(V)
    if plane:
        z = t[2] + 0.06
        Pc.append(np.array([[-2.0, -2.0, z], [2.0, -2.0, z], [2.0, 2.0, z], [-2.0, 2.0, z]]))
        Fs.append(np.array([[0, 1, 2], [0, 2, 3]]) + nv)
        nv += 4
    if occluder:
        z = t[2] - 0.10
        x0, x1 = (t[0] - 0.2) * z / t[2], (t[0] - 0.015) * z / t[2]
        y0, y1 = (t[1] - 0.2) * z / t[2], (t[1] + 0.2) * z / t[2]
        Pc.append(np.array([[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]))
        Fs.append(np.array([[0, 1, 2], [0, 2, 3]]) + nv)
    D = render_depth_ref(np.concatenate(Pc), np.concatenate(Fs), KM, W, H, SCALE, dist)
    rng = np.random.default_rng(1000 + seed)
    if holes:
        D[rng.random(D.shape) < 0.2] = 0
        u, v = np.flatnonzero(D.any(0)), np.flatnonzero(D.any(1))
        D[v[len(v) // 3]:v[len(v) // 3] + 12, u[len(u) // 2]:u[len(u) // 2] + 12] = 0
    if noise:
        D = np.where(D > 0, D.astype(np.int64) + rng.integers(-1, 2, D.shape), 0).astype(np.uint16)
    return D


def perturb(R, t, rng, along=0.03, lateral=0.005, angle_deg=5.0):
    """(R, t) moved by up to `along` along the viewing ray, up to `lateral` across it and turned by up to angle_deg"""
    ray = t / np.linalg.norm(t)
    side = np.cross(ray, rng.normal(size=3))
    side /= np.linalg.norm(side)
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    dR = so3_exp(ax * np.radians(rng.uniform(0, angle_deg)))
    return dR @ R, t + ray * rng.uniform(-along, along) + side * rng.uniform(0, lateral)


SCENES = {"plain": {}, "plane": dict(plane=True), "occluder": dict(occluder=True, plane=True), "holes": dict(holes=True)}


def scene_set(kind, distorted, n=4, seed=3):
    Rs, ts = synth.object_poses(n, seed=seed)
    rng = np.random.default_rng(seed)
    dist = BARREL if distorted else None
    depth = np.stack([scene_depth(Rs[i], ts[i], dist=dist, seed=i, **SCENES[kind]) for i in range(n)])
    R0, t0 = zip(*(perturb(Rs[i], ts[i], rng) for i in range(n)))
    return depth, np.stack(R0), np.stack(t0), Rs, ts, dist


# ---------------------------------------------------------------------------------------------------- harness = oracle
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("kind", sorted(SCENES))
def test_harness_equals_oracle(host, kind, distorted):
    depth, R0, t0, Rs, ts, dist = scene_set(kind, distorted)
    R, t, pts, rmse, st = host_refine(host, depth, MODEL, R0, t0, DIAM, dist=dist)
    for i in range(len(R0)):
        Ro, to, po, ro, so = refine_ref(depth[i], V, N, KM, R0[i], t0[i], DIAM, SCALE, 10, (0.5, 0.02), dist)
        assert st[i] == so == 0 and pts[i] == po > 500, (i, st[i], so, pts[i], po)
        assert np.abs(R[i] - Ro).max() < 1e-9 and np.abs(t[i] - to).max() < 1e-9
        assert abs(rmse[i] - ro) <= 1e-9 * max(ro, 1e-3)


def test_one_iteration_and_the_gate(host):
    """iters = 1 runs at the gate d * s; a narrow gate drops the pairs of a pose 3 cm off along the ray"""
    depth, R0, t0, Rs, ts, _d = scene_set("plain", False, n=2)
    for gate in ((0.5, 0.02), (0.05, 0.05)):
        R, t, pts, rmse, st = host_refine(host, depth, MODEL, R0, t0, DIAM, iters=1, gate=gate)
        for i in range(2):
            Ro, to, po, ro, so = refine_ref(depth[i], V, N, KM, R0[i], t0[i], DIAM, SCALE, 1, gate)
            assert st[i] == so and pts[i] == po and np.abs(t[i] - to).max() < 1e-9
    far = ts + 0.03 * ts / np.linalg.norm(ts, axis=1, keepdims=True)
    _R, _t, pts, _r, st = host_refine(host, depth, MODEL, Rs, far, DIAM, iters=1, gate=(0.5, 0.5))
    _R, _t, pts2, _r, st2 = host_refine(host, depth, MODEL, Rs, far, DIAM, iters=1, gate=(0.2, 0.2))
    assert (st == 0).all() and (pts > 1000).all() and (st2 == 1).all() and (pts2 < 50).all()


# ---------------------------------------------------------------------------------------------------- the Jacobian
@pytest.mark.parametrize("distorted", [False, True])
def test_jacobian_against_central_differences(host, distorted):
    depth, R0, t0, _Rs, _ts, dist = scene_set("plain", distorted, n=1)
    d = None if dist is None else np.ascontiguousarray(dist)
    R, t = np.ascontiguousarray(R0[0]), np.ascontiguousarray(t0[0])
    D = np.ascontiguousarray(depth[0])
    checked = 0
    for i in range(0, len(V), 97):
        x6 = np.ascontiguousarray(MODEL[i])
        r, J, q = C.c_double(), np.zeros(6), np.zeros(3)
        if not host.h_point_pair(_p(x6), _p(R), _p(t), _p(D), W, H, C.c_double(SCALE), _p(np.ascontiguousarray(KM)), _p(d),
                                 C.c_double(1.0), C.byref(r), _p(J), _p(q)):
            continue
        res = lambda e: (so3_exp(e[:3]) @ R @ x6[3:]) @ (so3_exp(e[:3]) @ R @ x6[:3] + t + e[3:] - q)
        assert abs(res(np.zeros(6)) - r.value) < 1e-15
        h = 1e-6
        Jn = np.array([(res(h * np.eye(6)[j]) - res(-h * np.eye(6)[j])) / (2 * h) for j in range(6)])
        assert np.abs(Jn - J).max() <= 1e-6 * np.abs(J).max(), (i, Jn, J)
        checked += 1
    assert checked > 20


# ---------------------------------------------------------------------------------------------------- normals
def test_vertex_normals_are_outward_for_either_winding():
    N1 = vertex_normals(V, F)
    N2 = vertex_normals(V, F[:, ::-1].copy())
    assert np.abs(N1 - N2).max() < 1e-12                               # the same normals, up to the order of the sums
    centred = V - V.mean(0)
    assert ((N1 * centred).sum(1) > 0).mean() > 0.99 and np.allclose(np.linalg.norm(N1, axis=1), 1.0)
    # a vertex no face uses gets a zero normal
    Nz = vertex_normals(np.concatenate([V, [[1.0, 2.0, 3.0]]]), F)
    assert not Nz[-1].any() and np.array_equal(Nz[:-1], N1)
    with pytest.raises(SspError):
        vertex_normals(V, F + len(V))


# ---------------------------------------------------------------------------------------------------- status edges
def _assert_unchanged(out, R0, t0, bit):
    R, t, _pts, _rmse, st = out
    assert (st == bit).all() and np.array_equal(R, R0.reshape(R.shape)) and np.array_equal(t, t0.reshape(t.shape), equal_nan=True)


def test_status_edges_return_the_input_pose(host):
    depth, R0, t0, _Rs, _ts, _d = scene_set("plain", False, n=1)
    off = t0.copy()
    off[0, 0] += 3.0                                                    # the object off the frame: no pairs
    out = host_refine(host, depth, MODEL, R0, off, DIAM)
    _assert_unchanged(out, R0, off, 1)
    assert out[2][0] == 0
    for bad in (np.array([[0.0, 0.0, -0.8]]), np.array([[0.0, 0.0, 0.0]]), np.array([[0.0, np.nan, 0.8]])):
        _assert_unchanged(host_refine(host, depth, MODEL, R0, bad, DIAM), R0, bad, 4)
    # a planar patch facing the camera: rotation about its normal and the in-plane translations are free
    g = np.linspace(-0.05, 0.05, 21)
    X, Y = np.meshgrid(g, g)
    Vp = np.c_[X.reshape(-1), Y.reshape(-1), np.zeros(X.size)]
    idx = np.arange(X.size).reshape(X.shape)
    a, b, c, e = idx[:-1, :-1].reshape(-1), idx[:-1, 1:].reshape(-1), idx[1:, :-1].reshape(-1), idx[1:, 1:].reshape(-1)
    Fp = np.concatenate([np.c_[a, c, b], np.c_[b, c, e]])
    Np = vertex_normals(Vp, Fp)
    assert np.allclose(Np, [0, 0, -1])                                 # toward a camera on -z of the patch
    Rp, tp = np.eye(3), np.array([0.01, -0.02, 0.8])
    Dp = render_depth_ref(Vp + tp, Fp, KM, W, H, SCALE)[None]
    out = host_refine(host, Dp, np.c_[Vp, Np], Rp[None], tp[None], 0.14)
    _assert_unchanged(out, Rp, tp, 2)
    assert out[2][0] >= 50
    assert refine_ref(Dp[0], Vp, Np, KM, Rp, tp, 0.14)[4] == 2


def test_counted_groups_and_arguments(host):
    depth, R0, t0, _Rs, _ts, _d = scene_set("plain", False, n=2)
    Rb, tb = np.repeat(R0, 3, 0), np.repeat(t0, 3, 0)
    R, t, pts, rmse, st = host_refine(host, depth, MODEL, Rb, tb, DIAM, count=[1, 3], per_group=3)
    assert not R[1:3].any() and not t[1:3].any() and not pts[1:3].any() and not rmse[1:3].any() and not st[1:3].any()
    R1, t1, *_ = host_refine(host, depth[1:], MODEL, R0[1:], t0[1:], DIAM)
    assert np.array_equal(R[3:], np.repeat(R1, 3, 0)) and np.array_equal(t[0], host_refine(host, depth[:1], MODEL, R0[:1], t0[:1], DIAM)[1][0])
    for bad in ((0.0, 1, (0.5, 0.02)), (np.inf, 1, (0.5, 0.02)), (0.001, 0, (0.5, 0.02)), (0.001, 101, (0.5, 0.02)),
                (0.001, 10, (0.02, 0.5)), (0.001, 10, (0.5, 0.0)), (0.001, 10, (np.inf, 0.1)), (0.001, 2.5, (0.5, 0.02))):
        with pytest.raises(SspError):
            check_refine_args(*bad)
    assert check_refine_args(0.001, 10, (0.5, 0.02)) == (0.001, 10, (0.5, 0.02))


# ---------------------------------------------------------------------------------------------------- what it is worth
VALUE_N = 200


def _value(host, gates, **scene):
    """ADD of 200 perturbed poses (along the ray up to 3 cm, across it up to 5 mm, up to 5 degrees) before and after the
    refinement at each gate range, against depth rendered at the true pose"""
    Rs, ts = synth.object_poses(VALUE_N, seed=11)
    rng = np.random.default_rng(11)
    before, after, status = np.zeros(VALUE_N), np.zeros((len(gates), VALUE_N)), np.zeros((len(gates), VALUE_N), np.int32)
    for i in range(VALUE_N):
        D = scene_depth(Rs[i], ts[i], seed=i, **scene)[None]
        R0, t0 = perturb(Rs[i], ts[i], rng)
        before[i] = add_error(V, R0, t0, Rs[i], ts[i])
        for g, gate in enumerate(gates):
            R, t, _pts, _rmse, st = host_refine(host, D, MODEL, R0[None], t0[None], DIAM, gate=gate)
            after[g, i], status[g, i] = add_error(V, R[0], t[0], Rs[i], ts[i]), st[0]
    for g, gate in enumerate(gates):
        print("%s gate %s: ADD median %.2f mm -> %.3f mm, p90 %.3f mm, <= 1 mm in %d, better in %d of %d, status 0 in %d"
              % (scene, gate, 1e3 * np.median(before), 1e3 * np.median(after[g]), 1e3 * np.percentile(after[g], 90),
                 (after[g] <= 1e-3).sum(), (after[g] < before).sum(), VALUE_N, (status[g] == 0).sum()))
    return before, after


def test_value_on_exact_depth(host):
    _before, after = _value(host, [(0.5, 0.02)])
    assert (after[0] <= 1e-3).sum() >= 190


def test_value_with_table_occluder_and_noise(host):
    """The occluder stands 10 cm in front of the object's centre, about 5.5 cm in front of its nearest surface.  A pose 3 cm too
    near brings it within the default first gate (0.5 x the 10.3 cm diameter), and the first iterations pair the occluder: at
    the default gate 164 of 200 poses improve.  A first gate below the occluder's distance (0.3 x the diameter) separates it:
    195 of 200 improve."""
    before, after = _value(host, [(0.5, 0.02), (0.3, 0.02)], plane=True, occluder=True, noise=True)
    assert (after[0] < before).sum() >= 160
    assert (after[1] < before).sum() >= 190
