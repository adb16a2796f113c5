"""CPU checks of tracking the world instances of a rig over time (singleshotpose_b200/csrc/world_track_core.h), compiled for the host
by tests/helpers/world_track_host.cpp: the harness against the numpy oracle (oracle/world_track_ref.py) on seeded random state
sequences, the value of the tracks on seeded moving scenes fused by the instance-fusion harness (id consistency with and without
motion, what prediction is worth for fast objects, the filter's smoothing), and the argument and command-line checks.  No device
is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.pose_filter_ref import project, so3_exp
from oracle.world_track_ref import class_size, world_track_step
from test_fuse_instances_cpu import DIAM, TABLE, host_instances, ihost, scene_rig  # noqa: F401

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FD = 163
SIZE = class_size(TABLE)
CV = ((2.0, 1.0), (1.0, 0.5), 22.46)                # accel_sigma, init_velocity_sigma, gate: the tracker's defaults


@pytest.fixture(scope="module")
def whost(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wthost") / "libwthost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "world_track_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def new_state(G, T, motion, params=CV):
    st = dict(tracks=np.zeros((G, T, 5), np.int32), poses=np.zeros((G, T, 12)), next_id=np.zeros(G, np.int32))
    if motion:
        st.update(filter=np.zeros((G, T, FD)), params=params)
    return st


def host_step(lib, st, fused, match_dist=0.5, max_misses=5, dt=None, size=SIZE):
    """one capture through h_world_track_associate and h_world_track_commit; st (new_state) is updated in place -> outputs"""
    G, T = st["tracks"].shape[:2]
    M = fused["world_cls"].shape[1]
    Cn = fused["world_index"].shape[0] // G
    f = {k: np.ascontiguousarray(v, np.int32 if k in ("world_count", "world_cls", "fuse_status", "world_index") else np.float64)
         for k, v in fused.items()}
    motion = "filter" in st
    filt = st["filter"] if motion else None
    dtv = np.ascontiguousarray(dt, np.float64) if motion else None
    accel, v0, gate = st["params"] if motion else CV
    i32 = lambda *s: np.zeros(s, np.int32)
    o = dict(wslot=i32(G, M), world_track_id=i32(G, M), matched=i32(G, M), track_id=i32(G * Cn, M))
    sz = np.ascontiguousarray(size, np.float64)
    rc = lib.h_world_track_associate(G, Cn, T, M, _p(f["world_count"]), _p(f["world_cls"]), _p(f["t_world"]), _p(f["world_index"]), _p(sz),
                                     len(sz), C.c_double(match_dist), max_misses, _p(st["tracks"]), _p(st["poses"]), _p(filt), _p(dtv),
                                     C.c_double(accel[0]), C.c_double(accel[1]), _p(st["next_id"]), _p(o["wslot"]), _p(o["world_track_id"]),
                                     _p(o["matched"]), _p(o["track_id"]))
    if rc != 0:
        raise ValueError("h_world_track_associate refused its arguments")
    mo = [np.zeros((G, M) + s) for s in ((3, 3), (3,), (6, 6), (6,))] + [i32(G, M)] if motion else [None] * 5
    rc = lib.h_world_track_commit(G, T, M, _p(f["world_count"]), _p(f["R_world"]), _p(f["t_world"]), _p(f["world_cov"]), _p(f["fuse_status"]),
                                  _p(o["wslot"]), _p(o["matched"]), _p(st["tracks"]), _p(st["poses"]), _p(filt), C.c_double(v0[0]),
                                  C.c_double(v0[1]), C.c_double(gate), *map(_p, mo))
    if rc != 0:
        raise ValueError("h_world_track_commit refused its arguments")
    if motion:
        o.update(zip(("R_filt", "t_filt", "pose_cov", "velocity", "reinit"), mo))
    return o


# ---------------------------------------------------------------------------------------------------- harness = oracle
def random_fused(rng, G, Cn, M, prev_t, nC=2):
    """world instances near the last ones (so tracks match), some far, some of an unknown class, some singular"""
    wc = rng.integers(0, M + 1, G).astype(np.int32)
    cls = -np.ones((G, M), np.int32)
    R, t, cov = np.zeros((G, M, 3, 3)), np.zeros((G, M, 3)), np.zeros((G, M, 6, 6))
    st = np.zeros((G, M), np.int32)
    for g in range(G):
        for w in range(wc[g]):
            cls[g, w] = rng.integers(0, nC) if rng.random() > 0.05 else 7
            base = prev_t[rng.integers(len(prev_t))] if len(prev_t) and rng.random() < 0.7 else rng.uniform(-0.3, 0.3, 3)
            t[g, w] = base + rng.normal(0, 0.02, 3)
            R[g, w] = so3_exp(rng.normal(0, 1.0, 3))
            A = rng.normal(size=(6, 6))
            cov[g, w] = 1e-6 * (A @ A.T + np.eye(6))
            st[g, w] = 4 if rng.random() < 0.05 else 0
    wi = -np.ones((G * Cn, M), np.int32)
    for b in range(G * Cn):
        n = int(wc[b // Cn])
        for m in range(M):
            wi[b, m] = rng.integers(-1, n) if n and rng.random() < 0.7 else -1
    return dict(world_count=wc, world_cls=cls, R_world=R, t_world=t, world_cov=cov, fuse_status=st, world_index=wi)


@pytest.mark.parametrize("motion", [None, "constant_velocity"])
def test_harness_equals_oracle(whost, motion):
    rng = np.random.default_rng(11 if motion else 12)
    G, Cn, T, M = 3, 2, 6, 5
    st = new_state(G, T, motion, ((2.0, 3.0), (1.0, 2.0), 22.46))
    ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}
    prev, born, matched, died, reinit = [], 0, 0, 0, 0
    for step in range(40):
        fused = random_fused(rng, G, Cn, M, prev)
        dt = rng.uniform(0.02, 0.05, G)
        alive0 = st["tracks"][..., 0].copy()
        ref = dict({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()})      # go on from the harness's state
        o = host_step(whost, st, fused, match_dist=0.8, max_misses=2, dt=dt)
        ref, r = world_track_step(ref, fused, SIZE, 0.8, 2, motion, dt)
        for k in ("wslot", "world_track_id", "matched", "track_id"):
            assert np.array_equal(o[k], r[k]), (step, k)
        assert np.array_equal(st["tracks"], ref["tracks"]) and np.array_equal(st["next_id"], ref["next_id"]), step
        assert np.array_equal(st["poses"], ref["poses"]), step                     # stored, not computed
        if motion:
            assert np.array_equal(o["reinit"] != 0, r["reinit"]), step
            for k in ("R_filt", "t_filt", "pose_cov", "velocity"):
                assert np.allclose(o[k], r[k], rtol=1e-9, atol=1e-12 * max(np.abs(r[k]).max(), 1e-300)), (step, k)
            assert np.allclose(st["filter"], ref["filter"], rtol=1e-9, atol=1e-15), step
            reinit += int(((o["reinit"] != 0) & (o["matched"] != 0)).sum())
        born += int(((o["world_track_id"] >= 0) & (o["matched"] == 0)).sum())
        matched += int(o["matched"].sum())
        died += int(((alive0 != 0) & (st["tracks"][..., 0] == 0)).sum())
        prev = [fused["t_world"][g, w] for g in range(G) for w in range(fused["world_count"][g])]
    assert born > 20 and matched > 20 and died > 5, (born, matched, died)
    assert (st["next_id"] > T).any()                                                 # slots were reused
    if motion:
        assert reinit > 0


def test_rule_details(whost):
    """strict radius, the nearest track, the lower slot on a tie, an unknown class untracked, no free slot untracked"""
    G, Cn, T, M = 1, 1, 3, 4
    st = new_state(G, T, None)

    def fused(ts, cls):
        n = len(ts)
        f = dict(world_count=np.array([n]), world_cls=-np.ones((1, M), np.int32), R_world=np.zeros((1, M, 3, 3)), t_world=np.zeros((1, M, 3)),
                 world_cov=np.zeros((1, M, 6, 6)), fuse_status=np.zeros((1, M), np.int32), world_index=-np.ones((1, M), np.int32))
        for w, (t, k) in enumerate(zip(ts, cls)):
            f["world_cls"][0, w], f["t_world"][0, w], f["R_world"][0, w] = k, t, np.eye(3)
            f["world_index"][0, w] = w
        return f
    r = 0.5 * SIZE[0]
    o = host_step(whost, st, fused([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], [0, 0, 5, 0]))
    assert list(o["world_track_id"][0]) == [0, 1, -1, 2] and list(o["track_id"][0]) == [0, 1, -1, 2]      # class 5 untracked
    o = host_step(whost, st, fused([[0, 0, 0], [0, 0, 0]], [0, 0]))                  # slots full: the second is untracked
    assert list(o["world_track_id"][0, :2]) == [0, -1] and o["matched"][0, 0] == 1
    st = new_state(G, T, None)
    host_step(whost, st, fused([[-r / 2, 0, 0], [r / 2, 0, 0]], [0, 0]))               # two tracks r apart
    o = host_step(whost, st, fused([[0, 0, 0]], [0]))                                  # equidistant: the lower slot
    assert o["world_track_id"][0, 0] == 0
    st = new_state(G, T, None)
    host_step(whost, st, fused([[0, 0, 0]], [0]))
    o = host_step(whost, st, fused([[r, 0, 0]], [0]))                                  # exactly r away: not within
    assert o["world_track_id"][0, 0] == 1 and o["matched"][0, 0] == 0
    o = host_step(whost, st, fused([[r * 0.999, 0, 0]], [0]))                          # nearest of tracks 0 (r 0.999) and 1 (r 0.001)
    assert o["world_track_id"][0, 0] == 1


# ---------------------------------------------------------------------------------------------------- moving scenes
def trajectories(rng, n_per_class, n_caps, speed, ramp=0, sep=1.2, reach=0.7):
    """[(cls, R (n_caps, 3, 3), t (n_caps, 3))]: each instance at constant velocity (speed: box diagonals per capture, a range) with
    a small random acceleration and a constant spin, at least sep diagonals from every other instance at every capture and within
    reach of the origin; with ramp > 0 the speed grows from a quarter over the first ramp captures"""
    counts = rng.integers(n_per_class[0], n_per_class[1] + 1, 2)
    for _try in range(2000):
        out = []
        for k in (0, 1):
            for _ in range(counts[k]):
                d = rng.normal(size=3)
                v = d / np.linalg.norm(d) * rng.uniform(*speed) * SIZE[k]
                scale = np.minimum(1.0, (np.arange(n_caps) + 1.0) / ramp) if ramp else np.ones(n_caps)
                steps = scale[:, None] * v + rng.normal(0, 0.02 * SIZE[k], (n_caps, 3)).cumsum(0) * 0.1
                t = np.concatenate([[np.zeros(3)], steps[:-1].cumsum(0)])
                t += rng.uniform(-0.3, 0.3, 3) - t.mean(0)
                w = rng.normal(0, 0.5, 3) / 30.0                                 # rad per capture
                R0 = so3_exp(rng.normal(size=3))
                out.append((k, np.stack([so3_exp(w * f) @ R0 for f in range(n_caps)]), t))
        ts = np.stack([o[2] for o in out])
        far = np.linalg.norm(ts, axis=2).max() <= reach
        gaps = np.linalg.norm(ts[:, None] - ts[None], axis=3) + np.eye(len(out))[:, :, None] * 1e9
        if far and gaps.min() >= sep * DIAM:
            return out
    raise AssertionError("no trajectories apart from each other: fewer instances or a smaller speed")


def detections(rng, rig, poses, M=16, miss=0.1, spurious=0.3, noise=2.0):
    """test_fuse_instances_cpu.scene's detections of the given instances [(cls, R, t)] -> (uv (C, M, 9, 2), cls, count, truth)"""
    Cn = len(rig.K)
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
        dets = [dets[i] for i in rng.permutation(len(dets))][:M]
        count[c] = len(dets)
        for m, (k, kp, j) in enumerate(dets):
            uv[c, m], cls[c, m], truth[c, m] = kp, k, j
    return uv, cls, count, truth


def run_sequence(ihost, whost, rng, n_caps, speed, ramp=0, n_per_class=(1, 5), motions=(None, "constant_velocity"), params=CV):
    """one seeded moving scene of 2-4 cameras fused capture by capture and tracked with each motion -> per motion: ids
    {instance: [(capture, world_track_id)]} over the captures where a world instance holds a true detection of the instance (the
    one holding most of them, the first emitted on a tie), and with motion the filtered and raw pose errors over captures >= 10"""
    rig = scene_rig(rng, int(rng.integers(2, 5)), bool(rng.integers(2)))
    traj = trajectories(rng, n_per_class, n_caps, speed, ramp)
    states = {m: new_state(1, 64, m, params) for m in motions}
    res = {m: dict(ids={j: [] for j in range(len(traj))}, t_f=[], t_r=[], r_f=[], r_r=[]) for m in motions}
    for f in range(n_caps):
        poses = [(k, R[f], t[f]) for k, R, t in traj]
        uv, cls, count, truth = detections(rng, rig, poses)
        o = host_instances(ihost, rig, uv, cls, count)
        fused = {k: o[k] for k in ("world_count", "world_cls", "R_world", "t_world", "world_cov", "fuse_status", "world_index")}
        for m in motions:
            out = host_step(whost, states[m], fused, dt=np.array([0.0 if f == 0 else 1 / 30.0]))
            for j, (k, R, t) in enumerate(poses):
                held = [o["world_index"][c, s] for c in range(len(rig.K)) for s in range(count[c]) if truth[c, s] == j and o["world_index"][c, s] >= 0]
                if not held:
                    continue
                w = min(held, key=lambda x: (-held.count(x), x))       # most of its detections, then the first emitted
                res[m]["ids"][j].append((f, int(out["world_track_id"][0, w])))
                if m and f >= 10 and out["world_track_id"][0, w] >= 0:
                    res[m]["t_f"].append(np.linalg.norm(out["t_filt"][0, w] - t))
                    res[m]["t_r"].append(np.linalg.norm(o["t_world"][0, w] - t))
                    res[m]["r_f"].append(_angle(out["R_filt"][0, w], R))
                    res[m]["r_r"].append(_angle(o["R_world"][0, w], R))
    return res


def _angle(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def kept(ids):
    """instances whose observed id never changed (an untracked capture, -1, counts as a change)"""
    out = []
    for seq in ids.values():
        if seq:
            vals = [i for _f, i in seq]
            out.append(all(v == vals[0] for v in vals) and vals[0] >= 0)
    return out


def value_stats(ihost, whost, n_seq, n_caps, speed, ramp=0, n_per_class=(1, 5), params=CV, seed=0):
    rng = np.random.default_rng(seed)
    keep = {None: [], "constant_velocity": []}
    err = dict(t_f=[], t_r=[], r_f=[], r_r=[])
    for _ in range(n_seq):
        res = run_sequence(ihost, whost, rng, n_caps, speed, ramp, n_per_class, params=params)
        for m in keep:
            keep[m] += kept(res[m]["ids"])
        for k in err:
            err[k] += res["constant_velocity"][k]
    out = dict(n=len(keep[None]), plain=float(np.mean(keep[None])), cv=float(np.mean(keep["constant_velocity"])))
    if err["t_f"]:
        out.update(t_ratio=float(np.median(err["t_f"]) / np.median(err["t_r"])), r_ratio=float(np.median(err["r_f"]) / np.median(err["r_r"])),
                   t_raw=float(np.median(err["t_r"])), r_raw=float(np.median(err["r_r"])))
    return out


def test_value_slow_scenes_keep_ids_and_smooth(ihost, whost):
    """30 captures at 30 fps, up to 0.2 box diagonals per capture: ids kept with and without motion; the filter smooths"""
    s = value_stats(ihost, whost, n_seq=12, n_caps=30, speed=(0.0, 0.2), n_per_class=(1, 3), seed=1)
    print("\nslow: %(n)d instances, ids kept %(plain).3f without motion, %(cv).3f with; filtered / raw median error over captures "
          "10-30: translation %(t_ratio).3f (raw %(t_raw).5f m), rotation %(r_ratio).3f (raw %(r_raw).3f deg)" % s)
    assert s["n"] >= 40
    assert s["plain"] >= 0.6 and s["cv"] >= 0.6
    assert s["t_ratio"] < 1.0 and s["r_ratio"] < 1.0


FAST = ((2.0, 40.0), (1.0, 10.0), 22.46)            # accel_sigma for objects that speed up by ~40 m/s^2, a 10 m/s velocity prior


def test_value_fast_scenes_need_prediction(ihost, whost):
    """0.6-1.0 box diagonals per capture, reached over the first 4 captures (a track needs two measurements before it has a
    velocity): without motion the ids are lost, with the constant-velocity filter they are kept"""
    s = value_stats(ihost, whost, n_seq=16, n_caps=8, speed=(0.6, 1.0), ramp=4, n_per_class=(1, 2), params=FAST, seed=2)
    print("\nfast: %(n)d instances, ids kept %(plain).3f without motion, %(cv).3f with" % s)
    assert s["n"] >= 30
    assert s["plain"] <= 0.2
    assert s["cv"] >= 0.75


# ---------------------------------------------------------------------------------------------------- arguments and command line
def test_harness_refusals(whost):
    st = new_state(1, 4, None)
    f = random_fused(np.random.default_rng(0), 1, 1, 3, [])
    for kw in (dict(match_dist=0.0), dict(match_dist=float("nan")), dict(max_misses=-1)):
        with pytest.raises(ValueError):
            host_step(whost, st, f, **kw)


def test_tracker_arguments():
    from singleshotpose_b200._lib import SspError
    from singleshotpose_b200.utils import camera_rig
    from singleshotpose_b200.utils_multi import WorldInstanceTracker
    from test_multiview_cpu import KM
    rig = camera_rig([KM] * 2, [np.eye(3)] * 2, [np.zeros(3)] * 2)
    corners = TABLE[0, 1:].T.astype(np.float64)
    for kw in (dict(match_dist=0.0), dict(match_dist=-1.0), dict(match_dist=float("inf")), dict(max_tracks=0), dict(max_tracks=257),
               dict(max_misses=-1), dict(groups=0), dict(motion="cv"), dict(gate=0.0), dict(rig=np.eye(3))):
        args = dict(objects={0: corners}, rig=rig, num_classes=2, groups=1)
        args.update(kw)
        with pytest.raises(SspError):
            WorldInstanceTracker(**args)


@pytest.mark.parametrize("argv,ok", [(["--track"], True), (["--track", "--motion", "cv", "--match-dist", "0.7"], True),
                                     (["--match-dist", "0.5"], True), (["--track", "--match-dist", "-1"], False),
                                     (["--track", "--match-dist", "nan"], False)])
def test_cli_accepts_track_with_rig(tmp_path, argv, ok):
    from singleshotpose_b200._lib import SspError
    from singleshotpose_b200.predict_instances import parse_args
    from test_multiview_cpu import KM
    rig = str(tmp_path / "rig.npz")
    np.savez(rig, K=np.stack([KM, KM]), R=np.stack([np.eye(3)] * 2), t=np.zeros((2, 3)))
    base = ["--datacfg", "x.data", "--modelcfg", "x.cfg", "--weightfile", "x.weights", "--rig", rig]
    if ok:
        a = parse_args(base + argv + ["a.png", "b.png"])
        assert a.rig_cams is not None and len(a.rig_cams.K) == 2
    else:
        with pytest.raises(SspError):
            parse_args(base + argv + ["a.png", "b.png"])


def test_cli_match_dist_needs_a_rig():
    from singleshotpose_b200._lib import SspError
    from singleshotpose_b200.predict_instances import parse_args
    with pytest.raises(SspError):
        parse_args(["--datacfg", "x.data", "--modelcfg", "x.cfg", "--weightfile", "x.weights", "--track", "--match-dist", "0.5", "a.png"])
