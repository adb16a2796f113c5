"""CPU checks of the rig rules at the sizes their kernels are declared for, where the kernel-only code (strided loops, warp
arg-mins, ballots over 32-wide chunks, lane partials, the subsampled pair hypotheses) runs more than one pass: the host harnesses
against the numpy oracles with 16 cameras, 33 and 256 track and world slots, and more than 256 co-observations per camera pair,
and the calibration of a 16-camera rig from noise-free keypoints against the true rig.  Each case asserts the size it is there
for.  The scenes are shared with tests/test_gpu_rig_limits.py, which holds the kernels to these harnesses.  No device is touched."""
import numpy as np
import pytest

from oracle.calibrate_rig_ref import MAX_PAIR_HYP, calibrate_ref
from oracle.fuse_instances_ref import fuse_instances_ref
from oracle.multiview_ref import fuse_ref
from oracle.pose_filter_ref import so3_exp
from oracle.world_track_ref import world_track_step
from test_calibrate_rig_cpu import cal, host_calibrate, moving_object, record, relative, scene as cal_scene  # noqa: F401
from test_fuse_instances_cpu import TABLE, host_instances, ihost, scene as inst_scene, scene_rig  # noqa: F401
from test_multiview_cpu import P9, host, host_fuse, observe, oracle_rig, random_object, random_rig  # noqa: F401
from test_world_track_cpu import SIZE, host_step, new_state, whost  # noqa: F401

WARP = 32


def co_observations(valid, n_cams):
    """the number of captures both cameras of each pair see: {(a, b): n}"""
    v = np.asarray(valid, bool).reshape(-1, n_cams)
    return {(a, b): int((v[:, a] & v[:, b]).sum()) for a in range(n_cams) for b in range(a + 1, n_cams)}


# ---------------------------------------------------------------------------------------------------- calibration
def subsample_picks(n, div=MAX_PAIR_HYP):
    """the co-observations a pair of n > 256 takes as hypotheses: floor(i n / 256), i < 256"""
    return set((np.arange(MAX_PAIR_HYP) * n) // div)


def planted_subsample_scene(seed, n_cams, distorted, G=262):
    """G captures of every camera (so G co-observations per pair), 2 px noise and 10 % wrong views, except one capture without
    noise or wrong view: the last index floor(i G / 256) takes that neither floor(i G / 257) nor the first 256 take -> (rig, uv,
    valid, planted capture)"""
    rng = np.random.default_rng(seed)
    rig = random_rig(rng, n_cams, distorted)
    poses = moving_object(rng, G)
    uv, valid = record(rig, poses, rng, 2.0, 0.0, 0.1)
    j = max(subsample_picks(G) - subsample_picks(G, MAX_PAIR_HYP + 1) - set(range(MAX_PAIR_HYP)))
    uv[j * n_cams:(j + 1) * n_cams] = record(rig, poses[j:j + 1], rng, noise=0.0)[0]
    return rig, uv, valid, j


def planted_hypothesis_won(o, n_cams, j):
    """whether the tree rig is capture j's relative poses, R_c = R_j,c R_j,0^T: every pair's winning hypothesis was the planted one"""
    Rr = o["R_rows"][:, 0].reshape(-1, n_cams, 3, 3)
    return np.abs(o["R"] - np.einsum("cij,kj->cik", Rr[j], Rr[j, 0])).max() < 1e-9


# C = 2 and C = 3 past MAX_PAIR_HYP co-observations: each pair's hypotheses are the co-observations at floor(i n / 256).  At
# n = 262 that index differs from floor(i n / 257), or from the first 256, in only 5 picks, which noisy views seldom tell apart,
# so the one noise-free capture sits at an index only the rule takes, and its hypothesis must win every pair: the planted
# capture has the lowest cost among the hypotheses of the most agreements (in some seeds a noisy hypothesis admits one more view
# and wins; the test asserts that the planted one did).  The oracle takes ~30 s per pair here, so distortion is covered at C = 2
# (one pair) and the three pairs of C = 3 run without it
@pytest.mark.parametrize("n_cams,distorted,seed", [(2, True, 4103), (3, False, 4102)])
def test_calibration_subsample_harness_equals_oracle(cal, n_cams, distorted, seed):
    G = 262
    rig, uv, valid, j = planted_subsample_scene(seed, n_cams, distorted, G)
    co = co_observations(valid, n_cams)
    assert min(co.values()) > MAX_PAIR_HYP, co                          # every pair takes the subsample branch
    assert j >= MAX_PAIR_HYP and j in subsample_picks(G) and j not in subsample_picks(G, MAX_PAIR_HYP + 1)
    tree = host_calibrate(cal, rig.K, rig.dist, uv, valid, tree_only=True)
    assert planted_hypothesis_won(tree, n_cams, j)
    o = host_calibrate(cal, rig.K, rig.dist, uv, valid)
    sh = lambda a: np.asarray(a).reshape(G, n_cams, *np.shape(a)[1:])
    ref = calibrate_ref(rig.K, rig.dist, np.repeat(P9[None, None], G, 0).repeat(n_cams, 1), sh(uv), sh(valid), sh(o["R_rows"][:, 0]),
                        sh(o["t_rows"][:, 0]))
    for k in ("tree_parent", "edge_agree", "cam_status", "cam_obs"):
        assert np.array_equal(o[k], ref[k]), (k, o[k], ref[k])
    assert np.array_equal(o["views"], ref["views"]) and np.array_equal(o["linked"], ref["linked"])
    assert o["rounds"] == ref["rounds"]
    assert np.abs(o["R"] - ref["R"]).max() < 1e-9 and np.abs(o["t"] - ref["t"]).max() < 1e-9
    assert np.abs(o["R_world"] - ref["R_world"]).max() < 1e-8 and np.abs(o["t_world"] - ref["t_world"]).max() < 1e-8
    assert np.abs(o["cam_rmse"] - ref["cam_rmse"]).max() < 1e-6
    assert np.abs(o["cam_cov"] - ref["cam_cov"]).max() <= 1e-6 * np.abs(ref["cam_cov"]).max()
    assert abs(o["cost"] - ref["cost"]) <= 1e-6 * max(ref["cost"], 1e-12)
    assert (o["cam_status"] == 0).all() and (o["edge_agree"][1:] >= 3).all()
    # the initial tree rig is the winning subsampled pair hypotheses' (the bundle adjustment forgets which ones won)
    assert np.abs(tree["R"] - ref["R_tree"]).max() < 1e-12 and np.abs(tree["t"] - ref["t_tree"]).max() < 1e-12


@pytest.mark.parametrize("distorted", [False, True])
def test_sixteen_cameras_from_noise_free_keypoints(cal, distorted):
    """16 cameras (n = 90 unknowns in the bundle adjustment), 40 captures without keypoint noise: the true rig within 1e-7 rad and
    1e-7 m, as at 2 and 4 cameras (the fp32 keypoints bound it)"""
    rig, uv, valid = cal_scene(60 + distorted, 16, G=40, distorted=distorted, noise=0.0)
    o = host_calibrate(cal, rig.K, rig.dist, uv, valid)
    Rt, tt = relative(rig)
    assert len(rig.K) == 16 and (o["cam_status"] == 0).all() and o["linked"].all()
    assert np.abs(o["R"] - Rt).max() < 1e-7 and np.abs(o["t"] - tt).max() < 1e-7, (np.abs(o["R"] - Rt).max(), np.abs(o["t"] - tt).max())


# ---------------------------------------------------------------------------------------------------- world tracking
TIE_D = 0.0625                                      # the planted ties: tracks at p -+ TIE_D along x, exact in binary


def tie_slots(T, M):
    """(lower slot in another lane, lower slot in the same lane, upper slot >= 32) of the ties planted in streams 0 and 1"""
    b = 37 if min(T, M) > 37 else 32
    return 6, b % WARP, b


def _grid(i):
    return 0.25 * np.array([i % 16, i // 16 % 16, i // 256], np.float64) - 2.0


def limit_frames(T, M, G=3, Cn=3, n_frames=5, seed=0):
    """synthesised outputs of ssp_fuse_instances for G streams of a Cn-camera rig, n_frames captures -> (list of fused dicts,
    list of planted ties (frame, stream, world slot, lower slot, upper slot)).

    Capture 0 gives every stream new objects of classes 0 and 1 on a 0.25 m grid, so instance w is born in slot w; streams 0 and
    1 see M instances (T = 33 cannot hold them all: a full table).  Later captures give the world counts 31, 32, 33 and M in turn,
    re-emit about 80 % of the last capture's objects 0-5 mm from where they were (matches; the others miss and, with
    max_misses = 1, die), then new objects (births, 5 % of an unknown class).  In capture 1 streams 0 and 1 lead with an instance
    of class 0 at exactly TIE_D from the tracks born in the tie slots (6 and b; b % 32 and b), which capture 0 placed there."""
    rng = np.random.default_rng(seed)
    lo_other, lo_same, hi = tie_slots(T, M)
    p = np.array([2.5, 2.5, 2.5])
    fused_all, ties = [], []
    pos = [dict() for _ in range(G)]
    cls_of = [dict() for _ in range(G)]
    last = [[] for _ in range(G)]
    fresh = [0] * G
    for f in range(n_frames):
        wc = np.zeros(G, np.int32)
        cls = -np.ones((G, M), np.int32)
        R, t, cov = np.zeros((G, M, 3, 3)), np.zeros((G, M, 3)), np.zeros((G, M, 6, 6))
        st = np.zeros((G, M), np.int32)
        for g in range(G):
            n = M if f == 0 and g < 2 else (31 if f == 0 else [31, 32, 33, M][(f - 1 + g) % 4])
            n = min(n, M)
            ids = []
            if f == 1 and g < 2:
                ids.append(("tie", g))
            if f > 0:
                keep = [j for j in last[g] if rng.random() < 0.8 and j not in (("obj", lo_other), ("obj", lo_same), ("obj", hi))]
                ids += [keep[i] for i in rng.permutation(len(keep))][:n - len(ids)]
            while len(ids) < n:
                j = ("obj", fresh[g])
                fresh[g] += 1
                pos[g][j] = _grid(j[1] + 1)
                cls_of[g][j] = int(rng.random() < 0.5) if f == 0 or rng.random() > 0.05 else 7
                ids.append(j)
            if f == 0 and g < 2:                                            # the tracks of the tie, born in its slots
                lo = lo_other if g == 0 else lo_same
                pos[g][ids[lo]], pos[g][ids[hi]] = p - [TIE_D, 0, 0], p + [TIE_D, 0, 0]
                cls_of[g][ids[lo]] = cls_of[g][ids[hi]] = 0
            if f == 1 and g < 2:
                pos[g][("tie", g)], cls_of[g][("tie", g)] = p.copy(), 0
                ties.append((f, g, 0, lo_other if g == 0 else lo_same, hi))
            wc[g] = n
            for w, j in enumerate(ids):
                cls[g, w] = cls_of[g][j]
                jitter = rng.uniform(0, 0.005) * rng.normal(size=3) / np.sqrt(3) if f > 0 and j[0] == "obj" else 0.0
                t[g, w] = pos[g][j] + jitter
                R[g, w] = so3_exp(rng.normal(0, 1.0, 3))
                A = rng.normal(size=(6, 6))
                cov[g, w] = 1e-6 * (A @ A.T + np.eye(6))
                st[g, w] = 4 if rng.random() < 0.05 else 0
            last[g] = [j for j in ids if j[0] == "obj"]
        wi = -np.ones((G * Cn, M), np.int32)
        for b in range(G * Cn):
            k = int(wc[b // Cn])
            wi[b] = np.where(rng.random(M) < 0.7, rng.integers(-1, k, M), -1)
        fused_all.append(dict(world_count=wc, world_cls=cls, R_world=R, t_world=t, world_cov=cov, fuse_status=st, world_index=wi))
    return fused_all, ties


def track_positions(st, g, motion):
    """each slot's position before a capture's prediction: the started filter's t, else the last pose's t"""
    pos = st["poses"][g, :, 9:12].copy()
    if motion:
        started = st["filter"][g, :, 162] == 1.0
        pos[started] = st["filter"][g, started, 9:12]
    return pos


def check_tie(st, tie, fused, motion):
    """the planted tie is exact: both tracks alive, of the class, at the same squared distance, and (with motion) without velocity"""
    _f, g, w, lo, hi = tie
    pos = track_positions(st, g, motion)
    tw = fused["t_world"][g, w]
    d2 = [((tw - pos[s]) ** 2).sum() for s in (lo, hi)]
    assert st["tracks"][g, lo, 0] and st["tracks"][g, hi, 0] and st["tracks"][g, lo, 2] == st["tracks"][g, hi, 2] == fused["world_cls"][g, w]
    assert d2[0] == d2[1] and d2[0] < (0.5 * SIZE[0]) ** 2, d2
    if motion:
        assert not st["filter"][g, [lo, hi], 12:18].any()
    return lo // WARP != hi // WARP and lo % WARP == hi % WARP, lo % WARP != hi % WARP


def tally(o, st, alive0, fused):
    """births, matches, deaths, full tables (more unmatched instances than free slots), matches in a slot >= 32"""
    born = int(((o["world_track_id"] >= 0) & (o["matched"] == 0)).sum())
    matched = int((o["matched"] != 0).sum())
    died = int(((alive0 != 0) & (st["tracks"][..., 0] == 0)).sum())
    untracked = [int(((o["world_track_id"][g, :fused["world_count"][g]] < 0) & (fused["world_cls"][g, :fused["world_count"][g]] < 2)).sum())
                 for g in range(len(alive0))]
    high = int(((o["matched"] != 0) & (o["wslot"] >= WARP)).sum())
    return np.array([born, matched, died, sum(u > 0 for u in untracked), high])


@pytest.mark.parametrize("motion", [None, "constant_velocity"])
@pytest.mark.parametrize("T,M", [(33, 33), (33, 256), (256, 33), (256, 256)])
def test_world_track_harness_equals_oracle_at_the_limits(whost, T, M, motion):
    G = 3
    frames, ties = limit_frames(T, M, G)
    counts = {int(n) for fr in frames for n in fr["world_count"]}
    assert {31, 32, 33, M} <= counts and T > WARP and M > WARP, counts
    st = new_state(G, T, motion, ((2.0, 3.0), (1.0, 2.0), 22.46))
    total = np.zeros(5, int)
    kinds = set()
    for f, fused in enumerate(frames):
        dt = np.full(G, 1 / 32)
        for tie in (x for x in ties if x[0] == f):
            kinds.add(check_tie(st, tie, fused, motion))
        ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}
        alive0 = st["tracks"][..., 0].copy()
        o = host_step(whost, st, fused, match_dist=0.5, max_misses=1, dt=dt)
        ref, r = world_track_step(ref, fused, SIZE, 0.5, 1, motion, dt)
        for k in ("wslot", "world_track_id", "matched", "track_id"):
            assert np.array_equal(o[k], r[k]), (f, k, np.argwhere(o[k] != r[k])[:5])
        assert np.array_equal(st["tracks"], ref["tracks"]) and np.array_equal(st["next_id"], ref["next_id"]), f
        assert np.array_equal(st["poses"], ref["poses"]), f
        if motion:
            assert np.array_equal(o["reinit"] != 0, r["reinit"]), f
            for k in ("R_filt", "t_filt", "pose_cov", "velocity"):
                assert np.allclose(o[k], r[k], rtol=1e-9, atol=1e-12 * max(np.abs(r[k]).max(), 1e-300)), (f, k)
            assert np.allclose(st["filter"], ref["filter"], rtol=1e-9, atol=1e-15), f
        for tie in (x for x in ties if x[0] == f):                      # the lower slot wins the tie
            _f, g, w, lo, _hi = tie
            assert o["wslot"][g, w] == lo and o["matched"][g, w], (tie, o["wslot"][g, w])
        total += tally(o, st, alive0, fused)
    born, matched, died, full, high = total
    assert born > 50 and matched > 50 and died > 0 and high > 0, total
    assert kinds == {(True, False), (False, True)}                      # a tie within a lane and a tie across lanes
    if T < M or T == 33:
        assert full > 0, total


# ---------------------------------------------------------------------------------------------------- fusion at 16 cameras
def test_fuse_views_sixteen_cameras_harness_equals_oracle(host):
    """16 cameras, the even ones distorted: an undisturbed capture, one with a view shifted 60-120 px and one with an invalid view"""
    rng = np.random.default_rng(1600)
    rig = random_rig(rng, 16, True)
    assert len(rig.K) == 16 and rig.dist[::2].any(1).all() and not rig.dist[1::2].any()
    for trial in range(3):
        R, t = random_object(rng)
        uv = observe(rig, R, t, rng)
        valid = np.ones(16, bool)
        if trial == 1:
            uv[5] += rng.uniform(60, 120, 2).astype(np.float32)
        if trial == 2:
            valid[10] = False
        o = host_fuse(host, rig, uv, valid)
        ref = fuse_ref(oracle_rig(rig), np.repeat(P9[None], 16, 0), uv, valid, o["R"], o["t"])
        assert o["fuse_status"][0] == ref["status"] == 0 and o["fuse_hyp"][0] == ref["hyp"], (trial, o["fuse_status"], ref["status"])
        assert np.array_equal(o["views"][0], ref["views"]) and o["views"][0].sum() >= 12, (trial, o["views"], ref["views"])
        assert np.abs(o["R_world"][0] - ref["R"]).max() < 1e-9 and np.abs(o["t_world"][0] - ref["t"]).max() < 1e-9
        assert np.abs(o["view_err"][0] - ref["view_err"]).max() < 1e-6
        assert np.abs(o["world_cov"][0] - ref["cov"]).max() <= 1e-6 * np.abs(ref["cov"]).max()


def sixteen_camera_instances(seed, n_captures):
    """captures of a 16-camera rig (the even cameras distorted) holding 5-6 instances of each class, 16 slots per view -> (rig,
    list of (uv, cls, count, truth, poses))"""
    rng = np.random.default_rng(seed)
    rig = scene_rig(rng, 16, True)
    return rig, [inst_scene(rng, rig, n_per_class=(5, 6), M=16) for _ in range(n_captures)]


def test_fuse_instances_sixteen_cameras_harness_equals_oracle(ihost):
    """a capture of more than 128 hypotheses, more than one 128-thread CTA takes in one pass (the oracle rescores every one of
    them every round: ~50 s)"""
    rig, caps = sixteen_camera_instances(1616, 1)
    for i, (uv, cls, count, _truth, _poses) in enumerate(caps):
        assert count.sum() > 128, count.sum()
        o = host_instances(ihost, rig, uv, cls, count)
        ref, unfused = fuse_instances_ref(oracle_rig(rig), TABLE, uv, cls, count, o["R"], o["t"])
        assert o["world_count"][0] == len(ref) and o["unfused"][0] == unfused, (i, o["world_count"], len(ref))
        for w, r in enumerate(ref):
            assert o["world_cls"][0, w] == r["cls"] and o["fuse_hyp"][0, w] == r["hyp"] and o["fuse_status"][0, w] == r["status"], (i, w)
            assert np.array_equal(o["members"][0, w], r["members"]), (i, w)
            assert np.abs(o["R_world"][0, w] - r["R"]).max() < 1e-7 and np.abs(o["t_world"][0, w] - r["t"]).max() < 1e-7
            assert np.abs(o["world_cov"][0, w] - r["cov"]).max() <= 1e-6 * np.abs(r["cov"]).max()
        assert (o["world_cls"][0, len(ref):] == -1).all() and (o["members"][0, len(ref):] == -1).all()
        assert len(ref) >= 8
