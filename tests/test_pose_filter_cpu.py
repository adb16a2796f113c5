"""CPU checks of the pose covariance and the constant-velocity pose filter (singleshotpose_b200/csrc/pose_filter_core.h), compiled for
the host by tests/helpers/pose_filter_host.cpp, against cv2's empirical covariance (tests/golden/pose_cov.npz), central differences,
the batch MAP estimate of the linear case and the numpy oracle (oracle/pose_filter_ref.py); the filter on noisy PnP of a moving box;
association on predicted rectangles (tests/helpers/track_host.cpp's rule); the argument checks of the entry points and the CLI.
No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.pose_filter_ref import FilterRef, pose_covariance, pose_jacobian, process_noise, project, so3_exp, so3_log
from singleshotpose_b200 import _lib, synth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSP_ERR_ARG = -1
FD = 163
KM = synth.intrinsics()
P3 = synth.box_points((0.038, 0.039, 0.046)).astype(np.float32)            # the 9 box points of an ape-sized box


def _build(tmp_path_factory, name, src):
    so = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", src)])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return _build(tmp_path_factory, "pfhost", "pose_filter_host.cpp")


@pytest.fixture(scope="module")
def pnp_host(tmp_path_factory):
    return _build(tmp_path_factory, "pfpnphost", "pnp_dist_host.cpp")


@pytest.fixture(scope="module")
def track_host(tmp_path_factory):
    return _build(tmp_path_factory, "pftrackhost", "track_host.cpp")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "pose_cov.npz"))


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _c(a, dt=np.float64):
    return np.ascontiguousarray(a, dt)


def host_cov(lib, P, R, t, K, sigma, dist=None):
    P, K, R, t = _c(P, np.float32), _c(K, np.float32), _c(R).reshape(-1, 9), _c(t).reshape(-1, 3)
    dist = None if dist is None else _c(dist)
    n = len(R)
    cov, st = np.zeros((n, 6, 6)), np.zeros(n, np.int32)
    assert lib.h_pose_covariance(_p(P), 1, _p(K), _p(dist), len(P), C.c_longlong(n), _p(R), _p(t), C.c_double(sigma), _p(cov), _p(st)) == 0
    return cov, st


def _close(a, b, rel):
    """|a - b| <= rel x the largest |b| of the array (a covariance mixes rad^2 and m^2 entries of one scale per block)"""
    return np.abs(np.asarray(a) - np.asarray(b)).max() <= rel * max(np.abs(b).max(), 1e-300)


# ------------------------------------------------------------------------------------------------ covariance
@pytest.mark.parametrize("tag", ["plain", "barrel"])
def test_covariance_meets_cv2_golden(host, golden, tag):
    K = golden["K"].astype(np.float64)
    dist = None if tag == "plain" else golden["dist_barrel"]
    hc, hs = host_cov(host, golden["P3"], golden["R_" + tag], golden["t_" + tag], golden["K"], float(golden["sigma"]), dist)
    for i in range(len(hc)):
        S, st = pose_covariance(golden["P3"], golden["R_" + tag][i], golden["t_" + tag][i], K, float(golden["sigma"]), dist)
        ratio = np.diag(S) / np.diag(golden["cov_" + tag][i])
        assert st == 0 and hs[i] == 0 and np.abs(ratio - 1).max() < 0.10, (i, ratio)        # sampling error about 3 %
        assert _close(hc[i], S, 1e-12)
    if dist is not None:                              # the distortion matters at these poses
        S0, _ = pose_covariance(golden["P3"], golden["R_" + tag][0], golden["t_" + tag][0], K, 1.0, None)
        assert np.abs(np.diag(S0) / np.diag(golden["cov_" + tag][0]) - 1).max() > 0.10


@pytest.mark.parametrize("tag", ["plain", "barrel"])
def test_jacobian_against_central_differences(host, golden, tag):
    K = golden["K"].astype(np.float64)
    dist = None if tag == "plain" else _c(golden["dist_barrel"])
    P = golden["P3"].astype(np.float64)
    for i in range(len(golden["R_" + tag])):
        R, t = golden["R_" + tag][i], golden["t_" + tag][i]
        Jn = np.zeros((18, 6))
        for j in range(6):
            h = 1e-6
            e = np.zeros(6); e[j] = h
            up = project(P, so3_exp(e[:3]) @ R, t + e[3:], K, dist)
            dn = project(P, so3_exp(-e[:3]) @ R, t - e[3:], K, dist)
            Jn[:, j] = ((up - dn) / (2 * h)).reshape(-1)
        J = np.zeros((9, 2, 6))
        for k in range(9):
            assert host.h_pose_jacobian(_p(_c(P[k])), _p(_c(R)), _p(_c(t)), C.c_double(K[0, 0]), C.c_double(K[1, 1]), _p(dist), _p(J[k])) == 0
        assert _close(J.reshape(18, 6), Jn, 1e-6)
        assert _close(pose_jacobian(P, R, t, K, dist), Jn, 1e-6)


def test_unusable_covariances(host):
    R, t = np.eye(3), np.array([0.0, 0.0, 0.5])
    coplanar = np.array([[x, 0.0, 0.0] for x in (-0.04, 0.0, 0.02, 0.04)], np.float32)      # collinear: the roll about the line is free
    cov, st = host_cov(host, coplanar, R, t, KM, 2.0)
    assert st[0] == 1 and not cov.any()
    behind = P3.copy(); behind[:, 2] -= 0.6
    cov, st = host_cov(host, behind, R, t, KM, 2.0)
    assert st[0] & 2 and not cov.any()
    assert pose_covariance(coplanar, R, t, KM, 2.0)[1] == 1 and pose_covariance(behind, R, t, KM, 2.0)[1] == 2


# ------------------------------------------------------------------------------------------------ the filter, exact cases
class HostSlot:
    """one stream with one track slot, driven through h_track_predict / h_track_filter_update"""

    def __init__(self, lib, acc, v0, gate=22.46):
        self.lib, self.acc, self.v0, self.gate = lib, acc, v0, gate
        self.f = np.zeros(FD)
        self.tracks = np.array([1, 0, 0, 0, 1], np.int32)

    def predict(self, dt):
        pp, pr = np.zeros(6), np.zeros(4, np.float32)
        assert self.lib.h_track_predict(1, 1, _p(self.tracks), _p(np.zeros(4, np.float32)), _p(np.zeros(6)), _p(self.f), _p(np.array([dt])),
                                        _p(P3), 1, _p(_c(KM)), None, C.c_double(self.acc[0]), C.c_double(self.acc[1]), _p(pp), _p(pr)) == 0
        return pp, pr

    def update(self, R, t, S, matched=True, status=0):
        out = [np.zeros(9), np.zeros(3), np.zeros(36), np.zeros(6), np.zeros(1, np.int32)]
        assert self.lib.h_track_filter_update(1, 1, 1, _p(np.ones(1, np.int32)), _p(np.zeros(1, np.int32)), _p(np.array([int(matched)], np.int32)),
                                              _p(_c(R)), _p(_c(t)), _p(_c(S)), _p(np.array([status], np.int32)), _p(self.f),
                                              C.c_double(self.v0[0]), C.c_double(self.v0[1]), C.c_double(self.gate), *map(_p, out)) == 0
        return out

    @property
    def P(self):
        return self.f[18:162].reshape(12, 12)


def _block_cov(rng, rot=1e-4, trans=1e-5):
    A, B = rng.normal(size=(3, 3)), rng.normal(size=(3, 3))
    S = np.zeros((6, 6))
    S[:3, :3] = rot * (A @ A.T + np.eye(3)); S[3:, 3:] = trans * (B @ B.T + np.eye(3))
    return S


def test_linear_case_equals_batch_map(host):
    """rotation fixed (w = 0, rotation measurements equal to it, block-diagonal Sigma_m): the translation part is a linear Gaussian
    system, and the filter's last (t, v) and their covariance are the batch MAP estimate of prior + dynamics + measurements"""
    rng = np.random.default_rng(3)
    acc, v0, N = (0.3, 0.2), (0.5, 0.4), 12
    dts = rng.uniform(0.02, 0.05, N)
    ms = [np.array([0.1, -0.05, 0.7]) + 0.02 * k + rng.normal(0, 3e-3, 3) for k in range(N + 1)]
    Ss = [_block_cov(rng) for _ in range(N + 1)]
    hs, ref = HostSlot(host, acc, v0, gate=1e12), FilterRef(acc, v0, gate=1e12)
    hs.update(np.eye(3), ms[0], Ss[0], matched=False)
    ref.init(np.eye(3), ms[0], Ss[0])
    for k in range(N):
        hs.predict(dts[k]); ref.predict(dts[k])
        hs.update(np.eye(3), ms[k + 1], Ss[k + 1]); ref.update(np.eye(3), ms[k + 1], Ss[k + 1])
    # batch: unknowns x_k = (t_k, v_k), k = 0..N; whitened rows of the prior, the dynamics and the measurements
    n = 6 * (N + 1)
    rows, rhs = [], []

    def add(A, b, cov):
        Li = np.linalg.inv(np.linalg.cholesky(cov))
        rows.append(Li @ A); rhs.append(Li @ b)
    A = np.zeros((6, n)); A[:, :6] = np.eye(6)
    add(A, np.r_[ms[0], np.zeros(3)], np.block([[Ss[0][3:, 3:], np.zeros((3, 3))], [np.zeros((3, 3)), v0[1] ** 2 * np.eye(3)]]))
    for k in range(N):
        dt = dts[k]
        F = np.block([[np.eye(3), dt * np.eye(3)], [np.zeros((3, 3)), np.eye(3)]])
        Q = process_noise(dt, acc)[np.ix_([3, 4, 5, 9, 10, 11], [3, 4, 5, 9, 10, 11])]
        A = np.zeros((6, n)); A[:, 6 * k:6 * k + 6] = -F; A[:, 6 * k + 6:6 * k + 12] = np.eye(6)
        add(A, np.zeros(6), Q)
        A = np.zeros((3, n)); A[:, 6 * k + 6:6 * k + 9] = np.eye(3)
        add(A, ms[k + 1], Ss[k + 1][3:, 3:])
    A, b = np.vstack(rows), np.concatenate(rhs)
    x = np.linalg.lstsq(A, b, rcond=None)[0]
    Pb = np.linalg.inv(A.T @ A)[-6:, -6:]
    idx = [3, 4, 5, 9, 10, 11]
    for t, v, P in ((ref.t, ref.v, ref.P), (hs.f[9:12], hs.f[15:18], hs.P)):
        assert np.abs(np.r_[t, v] - x[-6:]).max() < 1e-9 * np.abs(x[-6:]).max()
        assert _close(P[np.ix_(idx, idx)], Pb, 1e-9)
    assert np.allclose(hs.f[:9], np.eye(3).reshape(-1), atol=0) and not hs.f[12:15].any()


def test_noise_free_prediction(host):
    w, R0, dt, N = np.array([0.3, -0.5, 0.2]), so3_exp([0.4, 0.1, -0.7]), 1 / 30, 60
    hs, ref = HostSlot(host, (1.0, 1.0), (1.0, 1.0)), FilterRef((1.0, 1.0), (1.0, 1.0))
    hs.update(R0, [0.0, 0.0, 0.8], 1e-4 * np.eye(6), matched=False)
    ref.init(R0, [0.0, 0.0, 0.8], 1e-4 * np.eye(6))
    hs.f[12:15] = w; ref.w = w.copy()
    for _ in range(N):
        hs.predict(dt); ref.predict(dt)
    want = so3_exp(N * dt * w) @ R0
    assert np.abs(hs.f[:9] - want.reshape(-1)).max() < 1e-12 and np.abs(ref.R - want).max() < 1e-12
    assert _close(hs.P, ref.P, 1e-12)


def test_update_with_the_prediction_changes_nothing_but_shrinks_p(host):
    rng = np.random.default_rng(8)
    hs = HostSlot(host, (0.5, 0.2), (1.0, 0.5))
    R0, t0 = so3_exp([0.2, 0.3, -0.1]), np.array([0.05, 0.02, 0.6])
    S = _block_cov(rng)
    hs.update(R0, t0, S, matched=False)
    hs.f[12:18] = [0.1, -0.2, 0.3, 0.05, 0.0, -0.02]
    hs.predict(1 / 30)
    before, Pb = hs.f[:18].copy(), hs.P.copy()
    R_f, t_f, _cov, vel, reinit = hs.update(hs.f[:9].reshape(3, 3), hs.f[9:12], S)
    assert reinit[0] == 0 and np.array_equal(hs.f[:18], before)
    assert np.linalg.eigvalsh(Pb - hs.P).min() > -1e-15 * np.abs(Pb).max()


def test_predicted_rectangle_with_and_without_distortion(host):
    """the predicted corner rectangle is the oracle's projection of the 8 corners under the predicted pose, distorted with the barrel
    coefficients when they are given; near a frame corner the two differ by pixels"""
    barrel = np.array([-0.3, 0.12, 1e-3, -5e-4, -0.02, 0, 0, 0])
    R0, t0, w, v, dt = so3_exp([0.3, -0.4, 0.2]), np.array([-0.28, -0.2, 0.6]), np.array([0.2, 0.1, -0.3]), np.array([0.05, -0.02, 0.1]), 0.04
    rects = {}
    for dist in (None, barrel):
        f = np.zeros(FD)
        f[:9], f[9:12], f[12:15], f[15:18], f[162] = R0.reshape(-1), t0, w, v, 1.0
        pp, pr = np.zeros(6), np.zeros(4, np.float32)
        assert host.h_track_predict(1, 1, _p(np.array([1, 0, 0, 0, 1], np.int32)), _p(np.zeros(4, np.float32)), _p(np.zeros(6)), _p(f),
                                    _p(np.array([dt])), _p(P3), 1, _p(_c(KM)), _p(None if dist is None else _c(dist)), C.c_double(1.0),
                                    C.c_double(1.0), _p(pp), _p(pr)) == 0
        uv = project(P3[1:], so3_exp(w * dt) @ R0, t0 + v * dt, KM, dist).astype(np.float32)
        want = np.r_[uv.min(0), uv.max(0)][[0, 1, 2, 3]]
        assert np.abs(pr - want).max() <= 1e-3, (pr, want)
        assert np.abs(so3_exp(pp[:3]) - so3_exp(w * dt) @ R0).max() < 1e-12 and np.abs(pp[3:] - (t0 + v * dt)).max() < 1e-15
        rects[dist is None] = pr
    assert np.abs(rects[True] - rects[False]).max() > 5.0


def _slot_ref(refs, b, s, acc, v0, gate):
    return refs.setdefault((b, s), FilterRef(acc, v0, gate))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_harness_equals_oracle_on_sequences(host, seed):
    """births, updates, coasts, gate re-initialisations (a flipped pose), unusable covariances and deaths on B = 2 streams of
    T = 4 slots, M = 3 detection slots; every output to 1e-12 of its array's scale"""
    rng = np.random.default_rng(seed)
    B, T, M, acc, v0, gate = 2, 4, 3, (0.8, 0.3), (1.0, 0.5), 22.46
    filt = np.zeros((B, T, FD))
    tracks = np.zeros((B, T, 5), np.int32)
    refs = {}
    truth = {(b, s): (so3_exp(rng.normal(size=3)), np.array([rng.uniform(-.2, .2), rng.uniform(-.1, .1), rng.uniform(.5, 1.)]),
                      rng.normal(0, 0.5, 3), rng.normal(0, 0.1, 3)) for b in range(B) for s in range(T)}
    seen = dict(born=0, updated=0, reinit=0, coast=0)
    for f in range(30):
        dt = rng.uniform(0.02, 0.05, B)
        pp, pr = np.zeros((B, T, 6)), np.zeros((B, T, 4), np.float32)
        rects, poses = rng.uniform(0, 400, (B, T, 4)).astype(np.float32), rng.normal(size=(B, T, 6))
        tracks[..., 2] = 0
        assert host.h_track_predict(B, T, _p(tracks), _p(rects), _p(poses), _p(filt), _p(dt), _p(P3), 1, _p(_c(KM)), None, C.c_double(acc[0]),
                                    C.c_double(acc[1]), _p(pp), _p(pr)) == 0
        for b in range(B):
            for s in range(T):
                r = refs.get((b, s))
                if tracks[b, s, 0] and r is not None and r.valid:
                    r.predict(dt[b])
                    assert np.abs(pp[b, s, 3:] - r.t).max() <= 1e-12 * np.abs(r.t).max() and np.abs(so3_log(so3_exp(pp[b, s, :3]) @ r.R.T)).max() < 1e-12
                    seen["coast"] += 1
                else:
                    assert np.array_equal(pp[b, s], poses[b, s]) and np.array_equal(pr[b, s], rects[b, s])
        count = rng.integers(0, M + 1, B).astype(np.int32)
        slot = np.full((B, M), -1, np.int32); use = np.zeros((B, M), np.int32)
        Rm, tm, Sm, st = np.zeros((B, M, 9)), np.zeros((B, M, 3)), np.zeros((B, M, 36)), np.zeros((B, M), np.int32)
        for b in range(B):
            free = list(rng.permutation(T))[:count[b]]
            for m, s in enumerate(free):
                if rng.random() < 0.15:
                    continue                                              # untracked
                slot[b, m] = s
                use[b, m] = int(tracks[b, s, 0] and rng.random() < 0.85)
                tracks[b, s, 0] = 1
                R0, t0, w, v = truth[(b, s)]
                Rt, tt = so3_exp(w * 0.03 * f) @ R0, t0 + v * 0.03 * f
                noise = rng.normal(0, 1e-3, 6)
                Rt, tt = so3_exp(noise[:3]) @ Rt, tt + noise[3:]
                if rng.random() < 0.1:                                    # a flipped solution
                    Rt = so3_exp([np.pi * 0.9, 0, 0]) @ Rt
                Rm[b, m], tm[b, m] = Rt.reshape(-1), tt
                A = rng.normal(size=(6, 6)) * np.r_[np.full(3, 3e-3), np.full(3, 1e-3)][:, None]
                S = A @ A.T + np.diag(np.r_[np.full(3, 1e-5), np.full(3, 1e-6)])      # rotation and translation correlated
                Sm[b, m] = S.reshape(-1)
                st[b, m] = 1 if rng.random() < 0.05 else 0
        outs = [np.zeros((B, M, 9)), np.zeros((B, M, 3)), np.zeros((B, M, 36)), np.zeros((B, M, 6)), np.zeros((B, M), np.int32)]
        assert host.h_track_filter_update(B, T, M, _p(count), _p(slot), _p(use), _p(Rm), _p(tm), _p(Sm), _p(st), _p(filt), C.c_double(v0[0]),
                                          C.c_double(v0[1]), C.c_double(gate), *map(_p, outs)) == 0
        for b in range(B):
            for m in range(M):
                s = slot[b, m] if m < count[b] else -1
                if s < 0:
                    assert not any(o[b, m].any() for o in outs)
                    continue
                r = _slot_ref(refs, b, s, acc, v0, gate)
                S = Sm[b, m].reshape(6, 6)
                if use[b, m]:
                    ok = r.update(Rm[b, m].reshape(3, 3), tm[b, m], S, st[b, m] == 0)
                else:
                    r.init(Rm[b, m].reshape(3, 3), tm[b, m], S, st[b, m] == 0); ok = False
                seen["updated" if ok else ("reinit" if use[b, m] else "born")] += 1
                assert outs[4][b, m] == (not ok)
                assert np.abs(outs[0][b, m] - r.R.reshape(-1)).max() < 1e-12 and np.abs(outs[1][b, m] - r.t).max() <= 1e-12 * np.abs(r.t).max()
                assert _close(outs[2][b, m], r.P[:6, :6].reshape(-1), 1e-12)
                assert _close(outs[3][b, m], np.r_[r.w, r.v], 1e-10) if np.abs(np.r_[r.w, r.v]).max() > 0 else not outs[3][b, m].any()
        if f % 7 == 6:                                                    # deaths: a freed slot is born again later
            b, s = rng.integers(0, B), rng.integers(0, T)
            tracks[b, s, 0] = 0
            refs.pop((b, s), None)
    assert all(v > 0 for v in seen.values()), seen


# ------------------------------------------------------------------------------------------------ the filter on noisy PnP
def _pnp(lib, uv, guess):
    R, t, prm, w = np.zeros((1, 3, 3)), np.zeros((1, 3)), np.zeros((1, 6)), np.zeros((1, 3), np.int32)
    g = np.ascontiguousarray(guess[None])
    assert lib.h_pnp_dist(_p(P3), 1, _p(_c(uv, np.float32)), _p(_c(KM, np.float32)), None, 9, C.c_longlong(1), 20, _p(g),
                          _p(np.ones(1, np.int32)), _p(R), _p(t), _p(prm), _p(w)) == 0
    return R[0], t[0]


def _moving_box(host, pnp_host, seed, accel_sigma):
    """0.5 rad/s about a random axis and 0.3 m/s, constant, 30 fps, 200 frames, sigma = 2 px keypoint noise; each PnP warm-started
    from the filter's prediction, as the tracker does.  -> (filtered / raw RMS rotation error, the same for translation, mean NEES
    of the filtered pose with its covariance), all over the frames after frame 20"""
    rng = np.random.default_rng(seed)
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    w = 0.5 * ax
    d = np.array([0.28, 0.05, 0.1]); v = 0.3 * d / np.linalg.norm(d)
    R0, t0, dt, sigma = so3_exp(rng.normal(size=3)), np.array([-0.9, -0.1, 0.6]), 1 / 30, 2.0
    hs = HostSlot(host, accel_sigma, (1.0, 1.0))
    guess = None
    ef, em, nees = [], [], []
    for k in range(200):
        R, t = so3_exp(w * k * dt) @ R0, t0 + v * k * dt
        uv = project(P3, R, t, KM) + rng.normal(0, sigma, (9, 2))
        if k:
            guess, _ = hs.predict(dt)
        Rm, tm = _pnp(pnp_host, uv, np.r_[so3_log(R), t] if guess is None else guess)
        S, st = host_cov(host, P3, Rm, tm, KM, sigma)
        hs.update(Rm, tm, S[0], matched=k > 0, status=int(st[0]))
        Rf, tf = hs.f[:9].reshape(3, 3), hs.f[9:12]
        if k >= 20:
            e = np.r_[so3_log(R @ Rf.T), t - tf]
            ef.append(e); em.append(np.r_[so3_log(R @ Rm.T), t - tm])
            nees.append(e @ np.linalg.solve(hs.P[:6, :6], e))
    ef, em = np.array(ef), np.array(em)
    rms = lambda e: np.sqrt((e ** 2).sum(1).mean())
    return rms(ef[:, :3]) / rms(em[:, :3]), rms(ef[:, 3:]) / rms(em[:, 3:]), float(np.mean(nees))


def test_filter_is_consistent_and_beats_raw_pnp_on_a_moving_box(host, pnp_host):
    """The truth moves at constant velocity, so the filter is told to expect (almost) no acceleration: accel_sigma = 1e-6.  Then the
    mean NEES is 6 (chi^2 with 6 degrees of freedom) in expectation.  The filtered errors of consecutive frames are strongly
    correlated, so one sequence's mean NEES spreads far wider than a band for independent frames would say; the check is on the
    mean over SEEDS sequences, whose spread across seeds gives its own standard error.  With a process noise the truth does not have
    (accel_sigma = 0.01) the filter expects more error than it makes, and the NEES falls below 6."""
    runs = np.array([_moving_box(host, pnp_host, seed, (1e-6, 1e-6)) for seed in range(SEEDS)])
    for rot, trans, nees in runs:
        assert rot < 0.5 and trans < 0.5, runs
    m, se = runs[:, 2].mean(), runs[:, 2].std(ddof=1) / np.sqrt(SEEDS)
    print("filtered / raw RMS rotation %.3f-%.3f translation %.3f-%.3f; mean NEES %.2f +/- %.2f over %d seeds (per seed %.2f-%.2f)"
          % (runs[:, 0].min(), runs[:, 0].max(), runs[:, 1].min(), runs[:, 1].max(), m, se, SEEDS, runs[:, 2].min(), runs[:, 2].max()))
    assert abs(m - 6.0) < max(3 * se, 0.3), (m, se)
    noisy = np.array([_moving_box(host, pnp_host, seed, (0.01, 0.01))[2] for seed in range(4)])
    assert noisy.mean() < m - 0.5, (noisy, m)                                 # too much process noise: a conservative filter


SEEDS = 40


# ------------------------------------------------------------------------------------------------ association on predictions
def test_predicted_rectangles_keep_a_fast_box_tracked(host, track_host):
    """a box about 95 px wide that speeds up to 55 px per frame sideways (IoU of consecutive rectangles about 0.27 < match_iou 0.3): with the
    last rectangles the box gets new ids again and again (the perspective widens its rectangle off-centre, so not on every frame); with the predicted ones the id stays, also across a 3-frame gap with
    max_misses = 5.  The velocity is learnt while the box is still slow: a track that is never matched has no velocity."""
    z = 0.66
    Rb = so3_exp([0.2, -0.3, 0.1])
    px = lambda k: 30.0 * k if k < 3 else 60.0 + 55.0 * (k - 2)          # image x offset: 0, 30, 60, then +55 px per frame
    frames = [k for k in range(16) if k not in (9, 10, 11)]            # a 3-frame gap
    T, M = 16, 2

    def run(motion):
        tracks, rects, poses, nid = np.zeros((1, T, 5), np.int32), np.zeros((1, T, 4), np.float32), np.zeros((1, T, 6)), np.zeros(1, np.int32)
        filt = np.zeros((1, T, FD))
        ids, last = [], None
        for k in range(16):
            t = np.array([-0.25 + px(k) * z / KM[0, 0], 0.0, z])
            uv = project(P3, Rb, t, KM).astype(np.float32)
            present = k in frames
            count = np.array([1 if present else 0], np.int32)
            cls = np.zeros((1, M), np.int32)
            kp = np.zeros((1, M, 9, 2), np.float32); kp[0, 0] = uv
            pr, pp = rects, poses
            if motion:
                pp, pr = np.zeros((1, T, 6)), np.zeros((1, T, 4), np.float32)
                dt = np.array([0.0 if last is None else (k - last) / 30.0])
                host.h_track_predict(1, T, _p(tracks), _p(rects), _p(poses), _p(filt), _p(dt), _p(P3), 1, _p(_c(KM)), None, C.c_double(20.0),
                                     C.c_double(2.0), _p(pp), _p(pr))
            last = k
            slot, tid, use = np.zeros((1, M), np.int32), np.zeros((1, M), np.int32), np.zeros((1, M), np.int32)
            guess = np.zeros((1, M, 6))
            assert track_host.h_track_associate(1, T, M, _p(count), _p(cls), _p(kp), C.c_float(0.3), 5, _p(tracks), _p(pr), _p(pp), _p(nid),
                                                _p(slot), _p(tid), _p(guess), _p(use)) == 0
            params = np.zeros((1, M, 6)); params[0, 0] = np.r_[so3_log(Rb), t]
            track_host.h_track_commit(1, T, M, _p(count), _p(kp), _p(slot), _p(params), _p(tracks), _p(rects), _p(poses))
            if motion and present:
                S, st = host_cov(host, P3, Rb, t, KM, 2.0)
                Rm, tm = np.zeros((1, M, 9)), np.zeros((1, M, 3)); Rm[0, 0], tm[0, 0] = Rb.reshape(-1), t
                Sm = np.zeros((1, M, 36)); Sm[0, 0] = S[0].reshape(-1)
                outs = [np.zeros((1, M, 9)), np.zeros((1, M, 3)), np.zeros((1, M, 36)), np.zeros((1, M, 6)), np.zeros((1, M), np.int32)]
                host.h_track_filter_update(1, T, M, _p(count), _p(slot), _p(use), _p(Rm), _p(tm), _p(Sm), _p(np.zeros((1, M), np.int32)), _p(filt),
                                           C.c_double(1.0), C.c_double(1.0), C.c_double(22.46), *map(_p, outs))
            if present:
                ids.append(int(tid[0, 0]))
        return ids
    w = np.ptp(project(P3, Rb, np.array([0, 0, z]), KM)[1:, 0])
    assert 90 < w < 100
    last_ids, pred_ids = run(False), run(True)
    assert pred_ids == [0] * len(frames), pred_ids
    assert len(set(last_ids)) >= 5, last_ids                           # the last rectangles lose the box again and again


# ------------------------------------------------------------------------------------------------ ABI and Python checks
def test_symbols_are_declared_and_exported():
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        text = f.read()
    for name in ("ssp_pose_covariance", "ssp_track_predict", "ssp_track_filter_update"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
        assert "int %s(" % name in text
    assert _lib.CONSTANTS["SSP_FILTER_DOUBLES"] == FD and _lib.CONSTANTS["SSP_POSE_COV_SINGULAR"] == 1 and _lib.CONSTANTS["SSP_POSE_COV_DEPTH"] == 2


def _fake(a):
    return C.c_void_p(0x10000 * a) if a else None


def test_entry_points_reject_bad_arguments():
    lib = _lib.load()
    nan, inf = float("nan"), float("inf")

    def cov(P3=1, K=1, np_=9, groups=2, per=3, R=1, t=1, sigma=2.0, out=1, st=1):
        return lib.ssp_pose_covariance(_fake(P3), 0, _fake(K), None, np_, groups, per, None, _fake(R), _fake(t), C.c_double(sigma), _fake(out),
                                       _fake(st), None)
    for kw in (dict(P3=0), dict(K=0), dict(R=0), dict(t=0), dict(out=0), dict(st=0), dict(np_=2), dict(np_=17), dict(groups=-1), dict(per=0),
               dict(sigma=0.0), dict(sigma=-1.0), dict(sigma=nan), dict(sigma=inf)):
        assert cov(**kw) == SSP_ERR_ARG, kw
    assert cov(groups=0) == 0
    assert b"pose_covariance" in (cov(sigma=0.0), lib.ssp_last_error())[1]

    def pred(B=0, T=4, tr=1, rc=1, po=1, fi=1, dt=1, tab=1, ncls=2, K=1, ar=1.0, at=1.0, pp=1, pr=1):
        return lib.ssp_track_predict(B, T, _fake(tr), _fake(rc), _fake(po), _fake(fi), _fake(dt), _fake(tab), ncls, _fake(K), None, C.c_double(ar),
                                     C.c_double(at), _fake(pp), _fake(pr), None)
    for kw in (dict(tr=0), dict(rc=0), dict(po=0), dict(fi=0), dict(dt=0), dict(tab=0), dict(K=0), dict(pp=0), dict(pr=0), dict(B=-1), dict(T=0),
               dict(T=257), dict(ncls=0), dict(ar=0.0), dict(at=-1.0), dict(ar=nan), dict(at=inf)):
        assert pred(**kw) == SSP_ERR_ARG, kw
    assert pred() == 0

    def upd(B=0, T=4, M=8, null=None, vr=1.0, vt=1.0, gate=22.46):
        ptrs = [_fake(1)] * 14
        if null is not None:
            ptrs[null] = None
        c, sl, ug, R, t, cv, cs, fi, Rf, tf, pc, ve, ri = ptrs[:13]
        return lib.ssp_track_filter_update(B, T, M, c, sl, ug, R, t, cv, cs, fi, C.c_double(vr), C.c_double(vt), C.c_double(gate), Rf, tf, pc,
                                           ve, ri, None)
    for kw in [dict(null=i) for i in range(13)] + [dict(B=-1), dict(T=0), dict(T=257), dict(M=0), dict(M=257), dict(vr=0.0), dict(vt=nan),
                                                   dict(gate=0.0), dict(gate=inf)]:
        assert upd(**kw) == SSP_ERR_ARG, kw
    assert upd() == 0


def test_motion_argument_checks():
    from singleshotpose_b200.utils_multi import check_motion_args
    ok = check_motion_args("constant_velocity", 2, (1, 0.5), [0.3, 0.2], 22.46, 1 / 30)
    assert ok == ("constant_velocity", 2.0, (1.0, 0.5), (0.3, 0.2), 22.46, 1 / 30)
    assert check_motion_args(None, 2.0, (1, 1), (1, 1), 1.0, 0.1)[0] is None
    bad = [dict(motion="cv"), dict(motion="imu"), dict(keypoint_sigma=0), dict(keypoint_sigma=float("nan")), dict(accel_sigma=(1,)),
           dict(accel_sigma=(1, -1)), dict(accel_sigma="ab"), dict(init_velocity_sigma=(float("inf"), 1)), dict(gate=0), dict(gate=-3),
           dict(frame_dt=0), dict(frame_dt=float("inf")), dict(keypoint_sigma="x")]
    base = dict(motion="constant_velocity", keypoint_sigma=2.0, accel_sigma=(1, 1), init_velocity_sigma=(1, 1), gate=22.46, frame_dt=0.1)
    for kw in bad:
        with pytest.raises(_lib.SspError):
            check_motion_args(**dict(base, **kw))


def test_cli_motion_checks():
    from singleshotpose_b200.predict_instances import parse_args
    base = ["--datacfg", "d.data", "--modelcfg", "m.cfg", "--weightfile", "w"]
    a = parse_args(base + ["--track", "--motion", "cv", "--keypoint-sigma", "1.5", "--fps", "15", "a.png"])
    assert a.motion == "cv" and a.keypoint_sigma == 1.5 and a.fps == 15.0
    assert parse_args(base + ["--track", "a.png"]).motion is None
    for bad in (["--motion", "cv", "a.png"], ["--track", "--motion", "cv", "--fps", "0", "a.png"],
                ["--track", "--motion", "cv", "--keypoint-sigma", "-1", "a.png"]):
        with pytest.raises(_lib.SspError):
            parse_args(base + bad)
    with pytest.raises(SystemExit):
        parse_args(base + ["--track", "--motion", "imu", "a.png"])
