"""CPU checks of the instance fusion across a rig (singleshotpose_b200/csrc/multiview_instances_core.h), compiled for the host by
tests/helpers/multiview_instances_host.cpp: the harness against the numpy oracle (oracle/fuse_instances_ref.py), the reduction to
ssp_fuse_views' rule (tests/helpers/multiview_host.cpp) with at most one detection per class per view, the one-camera identity
rig, the order of detections within a view, the reuse of scores, the association and accuracy on seeded multi-instance scenes and
the command line's refusals.  No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.fuse_instances_ref import fuse_instances_ref
from oracle.pose_filter_ref import project, so3_exp
from singleshotpose_b200.utils import camera_rig
from test_multiview_cpu import BARREL, KM, P9, host, host_fuse, look_at, oracle_rig  # noqa: F401

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF1 = np.array([0.03, 0.07, 0.04])
P9B = np.concatenate([np.zeros((1, 3)), np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)]) * HALF1]).astype(np.float32)
TABLE = np.stack([P9, P9B])                                             # class 0 and class 1
DIAM = 2 * max(np.linalg.norm(P9[1]), np.linalg.norm(P9B[1]))


@pytest.fixture(scope="module")
def ihost(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mvihost") / "libmvihost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "multiview_instances_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def host_instances(lib, rig, uv, cls, count, table=TABLE, gate=40.0, thr=8.0, sigma=2.0, max_iter=20, rows=None, rescore_all=False):
    """h_fuse_instances: uv (B, M, P, 2), cls (B, M), count (B,) -> dict; rows = (R, t) per (row, slot) skips step 1"""
    Cn = len(rig.K)
    uv = np.ascontiguousarray(uv, np.float32)
    B, M, npts = uv.shape[:3]
    G = B // Cn
    cls, count = np.ascontiguousarray(cls, np.int32), np.ascontiguousarray(count, np.int32)
    table = np.ascontiguousarray(table, np.float32)
    K32, K64 = np.ascontiguousarray(rig.K, np.float32), np.ascontiguousarray(rig.K, np.float64)
    D = None if rig.dist is None else np.ascontiguousarray(rig.dist)
    Rr, tr = np.ascontiguousarray(rig.R), np.ascontiguousarray(rig.t)
    i32 = lambda *s: np.zeros(s, np.int32)
    o = dict(R=np.zeros((B, M, 3, 3)), t=np.zeros((B, M, 3)), corners_px=np.zeros((B, M, npts, 2), np.float32), world_count=i32(G),
             unfused=i32(G), world_cls=i32(G, M), R_world=np.zeros((G, M, 3, 3)), t_world=np.zeros((G, M, 3)), world_cov=np.zeros((G, M, 6, 6)),
             members=i32(G, M, Cn), view_err=np.zeros((G, M, Cn)), fuse_hyp=i32(G, M), fuse_status=i32(G, M), world_index=i32(B, M),
             corners_world_px=np.zeros((B, M, npts, 2), np.float32))
    if rows is not None:
        o["R"][:], o["t"][:] = rows
    rc = lib.h_fuse_instances(_p(table), len(table), _p(uv), _p(cls), _p(count), npts, G, Cn, M, _p(K32), _p(K64), _p(D), _p(Rr), _p(tr),
                              C.c_double(gate), C.c_double(thr), C.c_double(sigma), max_iter, int(rows is not None), int(rescore_all),
                              *(_p(v) for v in o.values()))
    if rc != 0:
        raise ValueError("h_fuse_instances refused its arguments")
    return o


# ---------------------------------------------------------------------------------------------------- scenes
def scene_rig(rng, n_cams, distorted=False):
    """n_cams cameras 1.4-1.8 m from the origin, each 45-135 degrees from camera 0's viewing direction"""
    d0 = rng.normal(size=3)
    d0 /= np.linalg.norm(d0)
    dirs = [d0]
    while len(dirs) < n_cams:
        ax = np.cross(d0, rng.normal(size=3))
        ax /= np.linalg.norm(ax)
        dirs.append(so3_exp(ax * np.radians(rng.uniform(45, 135))) @ d0)
    Rs, ts = [], []
    for d in dirs:
        pos = d * rng.uniform(1.4, 1.8)
        Rs.append(look_at(pos))
        ts.append(-Rs[-1] @ pos)
    dist = [BARREL * 0.5 if (distorted and c % 2 == 0) else None for c in range(n_cams)]
    return camera_rig([KM] * n_cams, Rs, ts, dist if distorted else None)


def scene(rng, rig, n_per_class=(1, 5), M=16, miss=0.1, spurious=0.3, noise=2.0, shuffle=True):
    """instances of classes 0 and 1 (n_per_class range each) at least 1.5 diameters apart, seen by every camera with `noise` px,
    each detection missed with probability `miss`, a spurious detection per view with probability `spurious` -> (uv (C, M, 9, 2),
    cls (C, M), count (C,), truth (C, M) instance id or -1, poses [(cls, R, t)])"""
    Cn = len(rig.K)
    poses = []
    for k in (0, 1):
        for _ in range(rng.integers(n_per_class[0], n_per_class[1] + 1)):
            for _try in range(200):
                t = rng.uniform(-0.35, 0.35, 3)
                if all(np.linalg.norm(t - q[2]) >= 1.5 * DIAM for q in poses):
                    break
            else:
                raise AssertionError("no place 1.5 diameters from the other instances: shrink n_per_class")
            ax = rng.normal(size=3)
            poses.append((k, so3_exp(ax / np.linalg.norm(ax) * rng.uniform(0, np.pi)), t))
    uv = np.zeros((Cn, M, 9, 2), np.float32)
    cls = -np.ones((Cn, M), np.int32)
    truth = -np.ones((Cn, M), np.int64)
    count = np.zeros(Cn, np.int32)
    for c in range(Cn):
        kd = None if rig.dist is None or not rig.dist[c].any() else rig.dist[c]
        dets = []
        for j, (k, R, t) in enumerate(poses):
            if rng.random() < miss:
                continue
            dets.append((k, project(TABLE[k], rig.R[c] @ R, rig.R[c] @ t + rig.t[c], rig.K[c], kd) + rng.normal(0, noise, (9, 2)), j))
        if rng.random() < spurious:
            k = int(rng.integers(2))
            ax = rng.normal(size=3)
            R = so3_exp(ax / np.linalg.norm(ax) * rng.uniform(0, np.pi))
            t = rng.uniform(-0.35, 0.35, 3)
            dets.append((k, project(TABLE[k], rig.R[c] @ R, rig.R[c] @ t + rig.t[c], rig.K[c], kd), -1))
        order = rng.permutation(len(dets)) if shuffle else np.arange(len(dets))
        dets = [dets[i] for i in order][:M]
        count[c] = len(dets)
        for m, (k, kp, j) in enumerate(dets):
            uv[c, m], cls[c, m], truth[c, m] = kp, k, j
    return uv, cls, count, truth, poses


# ---------------------------------------------------------------------------------------------------- harness = oracle
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("n_cams", [2, 3])
def test_harness_equals_oracle(ihost, n_cams, distorted):
    rng = np.random.default_rng(20 * n_cams + distorted)
    for trial in range(3):
        rig = scene_rig(rng, n_cams, distorted)
        uv, cls, count, _truth, _poses = scene(rng, rig, n_per_class=(1, 3), M=8)
        o = host_instances(ihost, rig, uv, cls, count)
        ref, unfused = fuse_instances_ref(oracle_rig(rig), TABLE, uv, cls, count, o["R"], o["t"])
        assert o["world_count"][0] == len(ref) and o["unfused"][0] == unfused, (trial, o["world_count"], len(ref))
        for w, r in enumerate(ref):
            assert o["world_cls"][0, w] == r["cls"] and o["fuse_hyp"][0, w] == r["hyp"] and o["fuse_status"][0, w] == r["status"], (trial, w)
            assert np.array_equal(o["members"][0, w], r["members"]), (trial, w)
            assert np.abs(o["R_world"][0, w] - r["R"]).max() < 1e-7 and np.abs(o["t_world"][0, w] - r["t"]).max() < 1e-7      # LM rounding
            scale = np.abs(r["cov"]).max()
            assert np.abs(o["world_cov"][0, w] - r["cov"]).max() <= 1e-6 * scale
        assert (o["world_cls"][0, len(ref):] == -1).all() and (o["R_world"][0, len(ref):] == 0).all()
        assert (o["members"][0, len(ref):] == -1).all() and (o["corners_world_px"][:, len(ref):] == 0).all()


# ---------------------------------------------------------------------------------------------------- the reduction to ssp_fuse_views
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("n_cams", [1, 2, 3, 4])
def test_one_detection_per_class_reduces_to_fuse_views(ihost, host, n_cams, distorted):
    rng = np.random.default_rng(300 + 10 * n_cams + distorted)
    M = 6
    for trial in range(8):
        rig = scene_rig(rng, n_cams, distorted)
        uv, cls, count, _truth, _poses = scene(rng, rig, n_per_class=(1, 1), M=M, miss=0.25, spurious=0.0)
        if trial % 2:                                   # a shifted view
            uv[rng.integers(n_cams), 0] += 70.0
        o = host_instances(ihost, rig, uv, cls, count)
        for k in (0, 1):
            mine = [w for w in range(o["world_count"][0]) if o["world_cls"][0, w] == k]
            slot = {c: m for c in range(n_cams) for m in range(count[c]) if cls[c, m] == k}
            valid = np.array([c in slot for c in range(n_cams)])
            if not valid.any():
                assert not mine
                continue
            kv = np.stack([uv[c, slot.get(c, 0)] for c in range(n_cams)])
            rows = (np.stack([o["R"][c, slot.get(c, 0)] for c in range(n_cams)]), np.stack([o["t"][c, slot.get(c, 0)] for c in range(n_cams)]))
            f = host_fuse(host, rig, kv, valid, P3=TABLE[k], rows=rows)
            if f["fuse_status"][0] & 3:
                assert not mine, (trial, k)
                continue
            w = mine[0]
            assert np.array_equal(o["R_world"][0, w], f["R_world"][0]) and np.array_equal(o["t_world"][0, w], f["t_world"][0]), (trial, k)
            assert np.array_equal(o["world_cov"][0, w], f["world_cov"][0]) and o["fuse_status"][0, w] == f["fuse_status"][0]
            assert np.array_equal(o["members"][0, w] >= 0, f["views"][0]), (trial, k)
            assert o["fuse_hyp"][0, w] // M == f["fuse_hyp"][0]


def test_one_camera_identity_rig(ihost):
    """one camera at the world frame: every well-separated detection is a world instance with its own pose's bits"""
    rig = camera_rig([KM], [np.eye(3)], [np.zeros(3)])
    rng = np.random.default_rng(5)
    for trial in range(4):
        poses = [(k, so3_exp(rng.normal(0, 0.5, size=3)), np.array([x, y, 1.2])) for k, (x, y) in enumerate([(-0.25, -0.1), (0.25, 0.1)] * 2)]
        poses = [(k % 2, R, t + [0, 0.0, 0.3 * (k // 2)]) for k, (_, R, t) in enumerate(poses)]
        M = 6
        uv = np.zeros((1, M, 9, 2), np.float32)
        cls = -np.ones((1, M), np.int32)
        for m, (k, R, t) in enumerate(poses):
            uv[0, m] = project(TABLE[k], R, t, rig.K[0], None) + rng.normal(0, 0.5, (9, 2))
            cls[0, m] = k
        o = host_instances(ihost, rig, uv, cls, np.array([len(poses)]))
        assert o["world_count"][0] == len(poses) and o["unfused"][0] == 0
        for w in range(len(poses)):
            m = o["fuse_hyp"][0, w]
            assert o["members"][0, w, 0] == m and o["world_index"][0, m] == w
            assert np.array_equal(o["R_world"][0, w], o["R"][0, m]) and np.array_equal(o["t_world"][0, w], o["t"][0, m])
            assert np.array_equal(o["corners_world_px"][0, w], o["corners_px"][0, m])


# ---------------------------------------------------------------------------------------------------- order and reuse
def test_order_within_a_view_changes_nothing(ihost):
    rng = np.random.default_rng(77)
    for trial in range(6):
        rig = scene_rig(rng, 3, trial % 2 == 1)
        uv, cls, count, _truth, _poses = scene(rng, rig, M=12)
        o = host_instances(ihost, rig, uv, cls, count)
        perm = [np.concatenate([rng.permutation(count[c]), np.arange(count[c], 12)]) for c in range(3)]
        uv2 = np.stack([uv[c, perm[c]] for c in range(3)])
        cls2 = np.stack([cls[c, perm[c]] for c in range(3)])
        p = host_instances(ihost, rig, uv2, cls2, count)
        assert p["world_count"][0] == o["world_count"][0]
        back = lambda mem: [perm[c][m] if m >= 0 else -1 for c, m in enumerate(mem)]
        want = {tuple(o["members"][0, w]): w for w in range(o["world_count"][0])}
        for w in range(p["world_count"][0]):
            v = want[tuple(back(p["members"][0, w]))]
            assert np.abs(p["R_world"][0, w] - o["R_world"][0, v]).max() < 1e-9 and np.abs(p["t_world"][0, w] - o["t_world"][0, v]).max() < 1e-9


def reuse_check(lib, rig, uv, cls, count, R_rows, t_rows):
    """h_reuse_check over one capture -> (pairs changed without touched(), pairs changed, pairs changed by a refit-only argmin)"""
    Cn, M = cls.shape
    changed, refit_only = C.c_int(), C.c_int()
    D = None if rig.dist is None else np.ascontiguousarray(rig.dist)
    bad = lib.h_reuse_check(_p(np.ascontiguousarray(TABLE, np.float32)), len(TABLE), _p(np.ascontiguousarray(uv, np.float32)),
                            _p(np.ascontiguousarray(cls, np.int32)), _p(np.ascontiguousarray(count, np.int32)), 9, Cn, M,
                            _p(np.ascontiguousarray(rig.K, np.float32)), _p(D), _p(np.ascontiguousarray(rig.R)), _p(np.ascontiguousarray(rig.t)),
                            _p(np.ascontiguousarray(R_rows)), _p(np.ascontiguousarray(t_rows)), C.c_double(40.0), C.c_double(8.0), 20,
                            C.byref(changed), C.byref(refit_only))
    return bad, changed.value, refit_only.value


def refit_scene(shift, noise=0.5):
    """one object seen by four cameras; camera 0's detection solved `shift` m off along camera 0's ray, and in camera 1 a
    second detection of the class where that wrong pose projects.  Camera 0's hypothesis first takes the decoy in camera 1 (the
    gate's argmin), and the fit, pinned by cameras 2 and 3, then takes the true detection (the refit's argmin)
    -> (rig, uv, cls, count, R, tw): camera 0's wrong world pose is (R, tw)"""
    rng = np.random.default_rng(0)
    pos = [np.array([1.6, 0, 0]), np.array([0, 1.6, 0.2]), np.array([0.2, 0.3, 1.6]), np.array([0.3, -1.2, -1.0])]
    Rs = [look_at(q) for q in pos]
    rig = camera_rig([KM] * 4, Rs, [-R @ q for R, q in zip(Rs, pos)])
    R, t = so3_exp(np.array([0.3, -0.5, 0.2])), np.array([0.01, -0.02, 0.0])
    tw = t + shift * pos[0] / np.linalg.norm(pos[0])
    px = lambda c, t: project(TABLE[0], rig.R[c] @ R, rig.R[c] @ t + rig.t[c], rig.K[c], None)
    uv = np.zeros((4, 4, 9, 2), np.float32)
    cls = -np.ones((4, 4), np.int32)
    for c in range(4):
        uv[c, 0], cls[c, 0] = px(c, t) + rng.normal(0, noise, (9, 2)), 0
    uv[1, 1], cls[1, 1] = px(1, tw), 0
    count = np.array([1, 2, 1, 1], np.int32)
    return rig, uv, cls, count, R, tw


def test_score_reuse_is_exact(ihost):
    """rescoring only the touched hypotheses gives the bits of rescoring all of them, and touched() is exact pair by pair"""
    # the refit's argmin: removing the true detection that only the refit chose changes camera 0's hypothesis
    for shift in (0.03, 0.05):
        rig, uv, cls, count, R, tw = refit_scene(shift)
        o = host_instances(ihost, rig, uv, cls, count)
        R_rows, t_rows = o["R"].copy(), o["t"].copy()
        R_rows[0, 0], t_rows[0, 0] = rig.R[0] @ R, rig.R[0] @ tw + rig.t[0]
        bad, changed, refit_only = reuse_check(ihost, rig, uv, cls, count, R_rows, t_rows)
        assert bad == 0 and refit_only >= 1, (shift, bad, changed, refit_only)
        a = host_instances(ihost, rig, uv, cls, count, rows=(R_rows, t_rows))
        b = host_instances(ihost, rig, uv, cls, count, rows=(R_rows, t_rows), rescore_all=True)
        assert all(np.array_equal(a[k], b[k]) for k in a)
    # seeded scenes: every pair, and whole extractions
    rng = np.random.default_rng(1000)
    pairs = 0
    for trial in range(VALUE_N):
        rig = scene_rig(rng, int(rng.integers(2, 5)), bool(rng.integers(2)))
        uv, cls, count, _truth, _poses = scene(rng, rig)
        o = host_instances(ihost, rig, uv, cls, count)
        a = host_instances(ihost, rig, uv, cls, count, rescore_all=True)
        for k in o:
            assert np.array_equal(o[k], a[k]), (trial, k)
        if trial < 30:
            bad, changed, _r = reuse_check(ihost, rig, uv, cls, count, o["R"], o["t"])
            assert bad == 0, trial
            pairs += changed
    assert pairs > 100


# ---------------------------------------------------------------------------------------------------- what association is worth
VALUE_N = 120


def _t_err(R, t, truth):
    return np.linalg.norm(t - truth[2])


def _r_err(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def association_stats(ihost, n=VALUE_N, seed=1000):
    rng = np.random.default_rng(seed)
    emitted = exact = pure = spurious = 0
    t_f, t_b, r_f, r_b = [], [], [], []
    for _ in range(n):
        rig = scene_rig(rng, int(rng.integers(2, 5)), bool(rng.integers(2)))
        uv, cls, count, truth, poses = scene(rng, rig)
        o = host_instances(ihost, rig, uv, cls, count)
        Cn = len(rig.K)
        wi = -np.ones((Cn, cls.shape[1]), int)
        for w in range(o["world_count"][0]):
            for c, m in enumerate(o["members"][0, w]):
                if m >= 0:
                    assert wi[c, m] == -1                 # a detection joins one world instance at most
                    wi[c, m] = w
        assert np.array_equal(wi, o["world_index"])
        for w in range(o["world_count"][0]):
            mem = o["members"][0, w]
            ids = {truth[c, m] for c, m in enumerate(mem) if m >= 0}
            emitted += 1
            if ids == {-1}:                             # spurious detections alone: no true instance to be exact about
                spurious += 1
                continue
            if len(ids) != 1 or -1 in ids:
                continue
            pure += 1
            j = ids.pop()
            full = {c: m for c in range(Cn) for m in range(count[c]) if truth[c, m] == j}
            exact += full == {c: m for c, m in enumerate(mem) if m >= 0}
            if len(full) < 2:
                continue
            singles = [(rig.R[c].T @ o["R"][c, m], rig.R[c].T @ (o["t"][c, m] - rig.t[c])) for c, m in full.items()]
            t_f.append(_t_err(o["R_world"][0, w], o["t_world"][0, w], poses[j]))
            t_b.append(min(_t_err(R, t, poses[j]) for R, t in singles))
            r_f.append(_r_err(o["R_world"][0, w], poses[j][1]))
            r_b.append(min(_r_err(R, poses[j][1]) for R, t in singles))
    return dict(emitted=emitted - spurious, spurious=spurious, pure=pure, exact=exact, t_fused=np.median(t_f), t_best=np.median(t_b), r_fused=np.median(r_f),
                r_best=np.median(r_b), n_err=len(t_f))


def test_value_on_seeded_scenes(ihost):
    s = association_stats(ihost)
    print("\nassociation: %(emitted)d world instances with a true detection (and %(spurious)d of spurious ones alone), %(pure)d of one true instance, %(exact)d exactly its detections; median "
          "translation %(t_fused).5f m fused vs %(t_best).5f m best single view, rotation %(r_fused).3f vs %(r_best).3f deg over "
          "%(n_err)d instances" % s)
    assert s["pure"] >= 0.95 * s["emitted"]
    assert s["exact"] >= 0.95 * s["emitted"]
    assert s["t_fused"] < 0.8 * s["t_best"]


# ---------------------------------------------------------------------------------------------------- the command line
@pytest.mark.parametrize("extra", [["--track"], ["--dist", "0.1", "0", "0", "0", "--"], ["--depth-dir", "d"], ["--pnp", "consensus"], []])
def test_cli_rig_refusals(tmp_path, extra):
    from singleshotpose_b200._lib import SspError
    from singleshotpose_b200.predict_instances import main
    from singleshotpose_b200.utils_host import read_rig  # noqa: F401
    rig = str(tmp_path / "rig.npz")
    np.savez(rig, K=np.stack([KM, KM]), R=np.stack([np.eye(3)] * 2), t=np.zeros((2, 3)))
    imgs = ["a.png", "b.png", "c.png"] if not extra else ["a.png", "b.png"]
    with pytest.raises(SspError):
        main(["--datacfg", "no.data", "--modelcfg", "no.cfg", "--weightfile", "no.weights", "--rig", rig] + extra + imgs)
