"""CPU checks of tracking across frames (singleshotpose_b200/csrc/track_core.h): the rule compiled for the host by
tests/helpers/track_host.cpp against the numpy oracle (oracle/track_ref.py), the warm-started PnP of pnp_core.h against
cv2.solvePnP(..., useExtrinsicGuess=True) (tests/golden/pnp_guess.npz), the argument checks of ssp_track_associate,
ssp_track_commit and ssp_pnp_batched_guess, and the command line's --track checks.  No device is touched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.track_ref import StreamRef
from singleshotpose_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSP_ERR_ARG = -1
F32 = np.float32


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("trackhost") / "libtrackhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "track_host.cpp")])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


class HostTracker:
    """the harness's state arrays (the layout of ssp_track_associate) and one frame = associate + given LM vectors + commit"""

    def __init__(self, lib, B, T, M):
        self.lib, self.B, self.T, self.M = lib, B, T, M
        self.tracks = np.zeros((B, T, 5), np.int32)
        self.rects = np.zeros((B, T, 4), F32)
        self.poses = np.zeros((B, T, 6))
        self.next_id = np.zeros(B, np.int32)

    def step(self, count, cls, uv, params_of, match_iou, max_misses):
        """count (B,), cls (B, M), uv (B, M, 9, 2); params_of(guess, use_guess) -> (B, M, 6) LM vectors of the frame's solves"""
        B, T, M = self.B, self.T, self.M
        count = np.ascontiguousarray(count, np.int32)
        cls = np.ascontiguousarray(cls, np.int32)
        uv = np.ascontiguousarray(uv, F32)
        slot = np.zeros((B, M), np.int32); tid = np.zeros((B, M), np.int32)
        guess = np.zeros((B, M, 6)); use = np.zeros((B, M), np.int32)
        assert self.lib.h_track_associate(B, T, M, _p(count), _p(cls), _p(uv), C.c_float(match_iou), max_misses, _p(self.tracks),
                                          _p(self.rects), _p(self.poses), _p(self.next_id), _p(slot), _p(tid), _p(guess), _p(use)) == 0
        params = np.ascontiguousarray(params_of(guess, use), np.float64)
        assert self.lib.h_track_commit(B, T, M, _p(count), _p(uv), _p(slot), _p(params), _p(self.tracks), _p(self.rects),
                                       _p(self.poses)) == 0
        return dict(slot=slot, track_id=tid, guess=guess, use_guess=use, params=params)


def _oracle_step(refs, count, cls, uv, params, match_iou, max_misses):
    out = []
    for b, ref in enumerate(refs):
        n = int(count[b])
        slot, tid, warm, guess = ref.associate(cls[b, :n], uv[b, :n], match_iou, max_misses)
        ref.commit(uv[b, :n], slot, params[b, :n])
        out.append((slot, tid, warm, guess))
    return out


def _assert_same(ht, refs, got, want, count):
    M = ht.M
    for b, ref in enumerate(refs):
        n = int(count[b])
        slot, tid, warm, guess = want[b]
        assert np.array_equal(got["slot"][b, :n], slot) and (got["slot"][b, n:] == -1).all()
        assert np.array_equal(got["track_id"][b, :n], tid) and (got["track_id"][b, n:] == -1).all()
        assert np.array_equal(got["use_guess"][b, :n] != 0, warm) and not got["use_guess"][b, n:].any()
        assert np.array_equal(got["guess"][b, :n], guess) and not got["guess"][b, n:].any()
        st = ht.tracks[b]
        assert np.array_equal(st[:, 0] != 0, ref.alive)
        for k, f in enumerate((ref.id, ref.cls, ref.misses, ref.hits), 1):
            assert np.array_equal(st[:, k], f), k
        assert ht.rects[b].tobytes() == ref.rect.tobytes() and np.array_equal(ht.poses[b], ref.pose)
        assert ht.next_id[b] == ref.next_id
    assert M == got["slot"].shape[1]


def _uv_of(rects, rng=None):
    """(n, 4) rectangles -> (n, 9, 2) fp32 keypoints whose corners 1..8 span exactly each rectangle (and a centroid inside)"""
    r = np.asarray(rects, F32).reshape(-1, 4)
    uv = np.zeros((len(r), 9, 2), F32)
    xs = np.stack([r[:, 0], r[:, 2]], 1)
    ys = np.stack([r[:, 1], r[:, 3]], 1)
    for k in range(8):
        uv[:, 1 + k, 0] = xs[:, k & 1]
        uv[:, 1 + k, 1] = ys[:, (k >> 1) & 1]
    if rng is not None:                                             # interior corners move: the rectangle stays the same
        for k in range(4, 8):
            a = rng.random(len(r)).astype(F32)
            uv[:, 1 + k, 0] = r[:, 0] + a * (r[:, 2] - r[:, 0])
    uv[:, 0] = (uv[:, 1] + uv[:, 8]) * F32(0.5)
    return uv


def _frame(rng, objs, B, M, nC, t):
    """a frame of B streams: each stream's objects (x, y, w, h, cls, vx, vy, period) move and blink; plus clutter"""
    count = np.zeros(B, np.int32); cls = np.full((B, M), -1, np.int32); uv = np.zeros((B, M, 9, 2), F32)
    for b in range(B):
        rows = []
        for (x, y, w, h, c, vx, vy, period) in objs[b]:
            if period and (t // period) % 3 == 2:                    # absent one period in three
                continue
            j = rng.normal(size=4) * 0.6
            rows.append(([x + vx * t + j[0], y + vy * t + j[1], x + vx * t + w + j[2], y + vy * t + h + j[3]], c))
        for _ in range(rng.integers(0, 4)):
            x, y = rng.random(2) * 600
            rows.append(([x, y, x + 10 + rng.random() * 60, y + 10 + rng.random() * 60], int(rng.integers(0, nC))))
        order = rng.permutation(len(rows))[:M]
        count[b] = len(order)
        for m, i in enumerate(order):
            cls[b, m] = rows[i][1]
            uv[b, m] = _uv_of([rows[i][0]], rng)[0]
    return count, cls, uv


def _objects(rng, B, n, nC):
    return [[(rng.random() * 500, rng.random() * 400, 20 + rng.random() * 80, 20 + rng.random() * 80, int(rng.integers(0, nC)),
              rng.normal() * 3, rng.normal() * 3, int(rng.integers(0, 6))) for _ in range(n)] for _ in range(B)]


def _params(rng):
    def f(guess, use):
        noise = rng.normal(size=guess.shape)
        return np.where(use[..., None] != 0, guess + 1e-3 * noise, noise)
    return f


def _run(host, seed, B, T, M, nC, nobj, frames, match_iou, max_misses):
    rng = np.random.default_rng(seed)
    objs = _objects(rng, B, nobj, nC)
    ht = HostTracker(host, B, T, M)
    refs = [StreamRef(T) for _ in range(B)]
    stats = dict(warm=0, born=0, untracked=0)
    pr = _params(rng)
    for t in range(frames):
        count, cls, uv = _frame(rng, objs, B, M, nC, t)
        got = ht.step(count, cls, uv, pr, match_iou, max_misses)
        want = _oracle_step(refs, count, cls, uv, got["params"], match_iou, max_misses)
        _assert_same(ht, refs, got, want, count)
        for b in range(B):
            n = int(count[b])
            stats["warm"] += int(got["use_guess"][b, :n].sum())
            stats["untracked"] += int((got["slot"][b, :n] < 0).sum())
        stats["born"] = int(ht.next_id.sum())
    return stats


# ------------------------------------------------------------------------------------------------ harness against the oracle
@pytest.mark.parametrize("seed,B,T,M,nC,nobj,match_iou,max_misses", [
    (0, 1, 64, 32, 13, 6, 0.3, 5), (1, 3, 16, 32, 3, 10, 0.3, 2), (2, 2, 4, 16, 2, 8, 0.1, 0), (3, 1, 256, 256, 13, 40, 0.5, 3),
    (4, 2, 1, 8, 1, 3, 0.0, 1), (5, 3, 8, 8, 4, 12, 1.0, 4)])
def test_harness_equals_oracle_on_random_sequences(host, seed, B, T, M, nC, nobj, match_iou, max_misses):
    s = _run(host, seed, B, T, M, nC, nobj, 60, match_iou, max_misses)
    if match_iou < 1.0:
        assert s["warm"] > 0
    assert s["born"] > 0
    if T <= 4:
        assert s["untracked"] > 0                                    # a full table was met


def _single(host, T=8, M=8):
    return HostTracker(host, 1, T, M), [StreamRef(T)]


def _step(ht, refs, dets, match_iou=0.3, max_misses=2, params=None):
    """dets: list of (rect, cls) for stream 0 -> the harness outputs (checked against the oracle) for the first len(dets) slots"""
    M = ht.M
    count = np.array([len(dets)], np.int32)
    cls = np.full((1, M), -1, np.int32); uv = np.zeros((1, M, 9, 2), F32)
    for m, (r, c) in enumerate(dets):
        cls[0, m] = c
        uv[0, m] = _uv_of([r])[0]
    pf = (lambda g, u: np.where(u[..., None] != 0, g + 1.0, 0.5)) if params is None else params
    got = ht.step(count, cls, uv, pf, match_iou, max_misses)
    want = _oracle_step(refs, count, cls, uv, got["params"], match_iou, max_misses)
    _assert_same(ht, refs, got, want, count)
    n = len(dets)
    return got["track_id"][0, :n].tolist(), got["slot"][0, :n].tolist(), (got["use_guess"][0, :n] != 0).tolist()


def test_misses_boundary_births_and_deaths(host):
    ht, refs = _single(host)
    A = ([100, 100, 150, 160], 3)
    assert _step(ht, refs, [A], max_misses=2) == ([0], [0], [False])
    for _ in range(2):                                                # absent max_misses frames: still alive
        assert _step(ht, refs, [], max_misses=2) == ([], [], [])
    assert ht.tracks[0, 0, 0] == 1 and ht.tracks[0, 0, 3] == 2
    assert _step(ht, refs, [A], max_misses=2) == ([0], [0], [True])  # seen again at misses == max_misses: the same id
    assert ht.tracks[0, 0, 3] == 0 and ht.tracks[0, 0, 4] == 2
    for _ in range(3):                                                # absent max_misses + 1 frames: dies
        _step(ht, refs, [], max_misses=2)
    assert ht.tracks[0, 0, 0] == 0
    assert _step(ht, refs, [A], max_misses=2) == ([1], [0], [False])  # comes back with a new id in the freed slot
    ht0, refs0 = _single(host)
    _step(ht0, refs0, [A], max_misses=0)
    _step(ht0, refs0, [], max_misses=0)                               # max_misses 0: one missed frame kills
    assert ht0.tracks[0, 0, 0] == 0


def test_no_cross_class_match_and_strict_threshold(host):
    ht, refs = _single(host)
    r = [0, 0, 2, 2]
    assert _step(ht, refs, [(r, 1)]) == ([0], [0], [False])
    assert _step(ht, refs, [(r, 2)]) == ([1], [1], [False])          # same place, other class: a new track
    assert _step(ht, refs, [(r, 2), (r, 1)]) == ([1, 0], [1, 0], [True, True])
    at = float(F32(2) / F32(6))                                        # IoU([0,0,2,2], [1,0,3,2]) = 2/6 exactly in fp32
    ht2, refs2 = _single(host)
    _step(ht2, refs2, [([0, 0, 2, 2], 0)], match_iou=at)
    assert _step(ht2, refs2, [([1, 0, 3, 2], 0)], match_iou=at) == ([1], [1], [False])      # IoU == match_iou: no match
    ht3, refs3 = _single(host)
    below = float(np.nextafter(F32(at), F32(0)))
    _step(ht3, refs3, [([0, 0, 2, 2], 0)], match_iou=below)
    assert _step(ht3, refs3, [([1, 0, 3, 2], 0)], match_iou=below) == ([0], [0], [True])


def test_equal_ious_take_the_lower_slot_and_the_best_iou_wins(host):
    ht, refs = _single(host)
    # slot 0 gets id 2 and slot 1 id 1 (slot 0 freed and reused), so the lower slot is not the lower id
    _step(ht, refs, [([0, 0, 2, 2], 0), ([100, 0, 102, 2], 5)], max_misses=0)
    _step(ht, refs, [([100, 0, 102, 2], 5), ([2, 0, 4, 2], 0)], max_misses=0)   # id 0 dies, [2,0,4,2] is born in slot 0
    _step(ht, refs, [([100, 0, 102, 2], 5), ([2, 0, 4, 2], 0), ([0, 0, 2, 2], 0)], max_misses=0)
    assert ht.tracks[0, :3, 1].tolist() == [2, 1, 3] and ht.tracks[0, 2, 2] == 0
    # [1, 0, 3, 2] overlaps slot 0 ([2,0,4,2]) and slot 2 ([0,0,2,2]) with the same IoU 1/3: slot 0 wins
    ids, slots, warm = _step(ht, refs, [([1, 0, 3, 2], 0), ([0, 0, 2, 2], 0)], max_misses=0)
    assert slots == [0, 2] and ids == [2, 3] and warm == [True, True]
    # a higher IoU beats a lower slot; the second detection takes what is left
    ids, slots, warm = _step(ht, refs, [([0.25, 0, 2.25, 2], 0), ([1, 0, 3, 2], 0)], max_misses=0)    # IoU 0.45 (slot 0), 0.78 (slot 2)
    assert slots == [2, 0] and ids == [3, 2]


def test_full_table_untracked_and_slots_freed_in_the_same_frame(host):
    ht, refs = _single(host, T=2, M=4)
    a, b, c, d = ([0, 0, 10, 10], 0), ([50, 0, 60, 10], 0), ([100, 0, 110, 10], 0), ([200, 0, 210, 10], 0)
    assert _step(ht, refs, [a, b, c], max_misses=0) == ([0, 1, -1], [0, 1, -1], [False, False, False])
    assert ht.next_id[0] == 2                                         # an untracked detection takes no id
    # b is missed (dies: max_misses 0); its slot is reused in the same frame by the first unmatched detection
    assert _step(ht, refs, [a, c, d], max_misses=0) == ([0, 2, -1], [0, 1, -1], [True, False, False])
    assert ht.tracks[0, 1, 2] == 0 and ht.tracks[0, 1, 4] == 1


def test_reset_and_streams_never_interact(host):
    rng = np.random.default_rng(9)
    B, T, M = 3, 8, 16
    objs = _objects(rng, B, 6, 3)
    frames = [_frame(rng, objs, B, M, 3, t) for t in range(25)]
    pr = lambda g, u: np.where(u[..., None] != 0, g + 0.25, 1.5)
    ht = HostTracker(host, B, T, M)
    alone = [HostTracker(host, 1, T, M) for _ in range(B)]
    for t, (count, cls, uv) in enumerate(frames):
        got = ht.step(count, cls, uv, pr, 0.3, 2)
        for b in range(B):
            one = alone[b].step(count[b:b + 1], cls[b:b + 1], uv[b:b + 1], pr, 0.3, 2)
            for k in got:
                assert np.array_equal(got[k][b], one[k][0]), (t, b, k)
            assert np.array_equal(ht.tracks[b], alone[b].tracks[0]) and np.array_equal(ht.poses[b], alone[b].poses[0])
    # reset = zero the state in place: the next frames equal a fresh tracker's
    ht.tracks[:] = 0; ht.rects[:] = 0; ht.poses[:] = 0; ht.next_id[:] = 0
    fresh = HostTracker(host, B, T, M)
    for count, cls, uv in frames[:10]:
        a, f = ht.step(count, cls, uv, pr, 0.3, 2), fresh.step(count, cls, uv, pr, 0.3, 2)
        assert all(np.array_equal(a[k], f[k]) for k in a)
    assert np.array_equal(ht.tracks, fresh.tracks) and np.array_equal(ht.next_id, fresh.next_id)


# ------------------------------------------------------------------------------------------------ warm PnP against cv2
def _ang(a, b):
    return np.degrees(np.arccos(np.clip((np.trace(a @ b.T) - 1) / 2, -1, 1)))


def _rod(r):
    from oracle.pnp_ref import rodrigues_vec2mat
    return rodrigues_vec2mat(r)


def host_pnp_guess(host, P3, uv, K, guess, use):
    n, npts = uv.shape[:2]
    P3n = np.ascontiguousarray(np.repeat(np.asarray(P3, F32)[None], n, 0))
    uv = np.ascontiguousarray(uv, F32); K = np.ascontiguousarray(K, F32)
    guess = np.ascontiguousarray(guess, np.float64); use = np.ascontiguousarray(use, np.int32)
    R = np.zeros((n, 3, 3)); t = np.zeros((n, 3)); params = np.zeros((n, 6)); w = np.zeros((n, 3), np.int32)
    assert host.h_pnp_guess(_p(P3n), _p(uv), _p(K), npts, C.c_longlong(n), 20, _p(guess), _p(use), _p(R), _p(t), _p(params), _p(w)) == 0
    return R, t, params, w


@pytest.mark.parametrize("npts", [9, 8])
@pytest.mark.parametrize("sigma", [0, 1, 5, 20, 80])
def test_warm_pnp_matches_cv2_golden(host, golden_dir, npts, sigma):
    g = np.load(os.path.join(golden_dir, "pnp_guess.npz"))
    tag = "p%d_s%d" % (npts, sigma)
    uv, guess = g["uv_" + tag], g["guess_" + tag]
    R, t, params, w = host_pnp_guess(host, g["P3_%d" % npts], uv, g["K"], guess, np.ones(len(uv)))
    ang = np.array([_ang(R[i], g["R_" + tag][i]) for i in range(len(R))])
    assert ang.max() < 1e-2 and np.abs(t - g["tvec_" + tag]).max() * 1e3 < 1e-2, (tag, ang.max(), np.abs(t - g["tvec_" + tag]).max())
    assert np.degrees(np.abs(params[:, :3] - g["rvec_" + tag])).max() < 1e-2 and np.abs(params[:, 3:] - g["tvec_" + tag]).max() * 1e3 < 1e-2
    assert np.array_equal(params[:, 3:], t)                           # t is the LM vector's translation
    assert max(np.abs(_rod(params[i, :3]) - R[i]).max() for i in range(len(R))) < 1e-12     # R is the Rodrigues matrix of the LM vector
    assert (w[:, 0] == 0).all() and (w[:, 1] >= 1).all() and (w[:, 1] <= 20).all()      # no DLT for a warm start
    assert g["perturbed_" + tag].any() and not g["perturbed_" + tag].all()


def test_cold_slots_of_the_guess_solve_are_the_plain_solve(host, golden_dir):
    g = np.load(os.path.join(golden_dir, "pnp_guess.npz"))
    uv, guess = g["uv_p9_s5"], g["guess_p9_s5"]
    use = (np.arange(len(uv)) % 3 == 0).astype(np.int32)
    R, t, params, w = host_pnp_guess(host, g["P3_9"], uv, g["K"], guess, use)
    Rc, tc, pc, wc = host_pnp_guess(host, g["P3_9"], uv, g["K"], guess, np.zeros(len(uv)))
    cold = use == 0
    assert np.array_equal(R[cold], Rc[cold]) and np.array_equal(t[cold], tc[cold]) and np.array_equal(params[cold], pc[cold])
    assert (w[cold, 0] != 0).all() and (w[~cold, 0] == 0).all()


# ------------------------------------------------------------------------------------------------ ABI and command line
def test_symbols_are_declared_and_exported():
    with open(os.path.join(REPO, "include", "ssp_b200.h")) as f:
        text = f.read()
    for name in ("ssp_track_associate", "ssp_track_commit", "ssp_pnp_batched_guess"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
        assert "int %s(" % name in text


def _fake(a):
    return C.c_void_p(0x10000 * a) if a else None


def test_track_entry_points_reject_bad_arguments():
    lib = _lib.load()

    def assoc(B=1, T=8, M=8, count=1, cls=1, uv=1, iou=0.3, misses=5, tracks=1, rects=1, poses=1, nid=1, slot=1, tid=1, guess=1, use=1):
        return lib.ssp_track_associate(B, T, M, _fake(count), _fake(cls), _fake(uv), C.c_float(iou), misses, _fake(tracks), _fake(rects),
                                       _fake(poses), _fake(nid), _fake(slot), _fake(tid), _fake(guess), _fake(use), None)
    for kw in (dict(count=0), dict(cls=0), dict(uv=0), dict(tracks=0), dict(rects=0), dict(poses=0), dict(nid=0), dict(slot=0),
               dict(tid=0), dict(guess=0), dict(use=0), dict(B=-1), dict(T=0), dict(T=257), dict(M=0), dict(M=257), dict(iou=-0.01),
               dict(iou=1.01), dict(iou=float("nan")), dict(misses=-1)):
        assert assoc(**kw) == SSP_ERR_ARG, kw
    assoc(iou=2.0)
    assert b"match_iou" in lib.ssp_last_error()
    assert assoc(B=0) == 0                                              # no stream: no launch

    def commit(B=1, T=8, M=8, count=1, uv=1, slot=1, params=1, tracks=1, rects=1, poses=1):
        return lib.ssp_track_commit(B, T, M, _fake(count), _fake(uv), _fake(slot), _fake(params), _fake(tracks), _fake(rects), _fake(poses),
                                    None)
    for kw in (dict(count=0), dict(uv=0), dict(slot=0), dict(params=0), dict(tracks=0), dict(rects=0), dict(poses=0), dict(B=-1),
               dict(T=0), dict(T=257), dict(M=0), dict(M=257)):
        assert commit(**kw) == SSP_ERR_ARG, kw
    assert commit(B=0) == 0

    def guess(P3=1, uv=1, K=1, np_=9, groups=2, per=4, count=1, g=1, use=1, R=1, t=1, params=1):
        return lib.ssp_pnp_batched_guess(_fake(P3), _fake(uv), _fake(K), np_, groups, per, _fake(count), _fake(g), _fake(use), 20,
                                         _fake(R), _fake(t), _fake(params), None, None)
    for kw in (dict(P3=0), dict(uv=0), dict(K=0), dict(count=0), dict(g=0), dict(use=0), dict(R=0), dict(t=0), dict(params=0),
               dict(np_=5), dict(np_=17), dict(groups=-1), dict(per=0)):
        assert guess(**kw) == SSP_ERR_ARG, kw
    assert guess(groups=0) == 0


def test_cli_track_checks():
    from singleshotpose_b200.predict_instances import parse_args
    base = ["--datacfg", "d.data", "--modelcfg", "m.cfg", "--weightfile", "w"]
    a = parse_args(base + ["a.png"])
    assert not a.track and a.match_iou == 0.3 and a.max_misses == 5 and a.max_tracks == 64
    a = parse_args(base + ["--track", "--match-iou", "0", "--max-misses", "0", "--max-tracks", "256", "a.png", "b.png"])
    assert a.track and a.match_iou == 0.0 and a.max_misses == 0 and a.max_tracks == 256
    for bad in (["--match-iou", "1.5"], ["--match-iou", "-0.1"], ["--max-misses", "-1"], ["--max-tracks", "0"], ["--max-tracks", "257"]):
        with pytest.raises(_lib.SspError):
            parse_args(base + ["--track"] + bad + ["a.png"])
