"""Oracle of tracking the world instances of a camera rig over time (singleshotpose_b200/csrc/world_track_core.h) in numpy, with whole
arrays where the core loops.  TEST INFRASTRUCTURE ONLY.

Each capture stream owns T slots (alive, id, cls, misses, hits), each track's last fused world pose (R, t), a next_id counter and,
with motion, a pose filter per slot (oracle/pose_filter_ref.py's FilterRef, in world axes).  Per capture, with the world instances
in slot order:
  1. predict: every alive slot whose filter has started moves by dt; a slot's position is its started filter's t, else its last t;
  2. match: instance w of class k takes the alive, not yet taken track of class k with the smallest |t_w - position|^2 < r_k^2,
     r_k = match_dist * class_size[k] (the lower slot on ties);
  3. age: unmatched alive tracks get misses += 1 and die when misses > max_misses;
  4. birth: unmatched instances, in order, take the lowest free slot and id = next_id++; none free -> untracked (-1);
  5. commit: matched and born tracks store the instance's R, t, misses 0, hits + 1; the filter of a born track starts from the
     instance, a matched one is updated (usable when fuse_status lacks the singular bit 4)."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import FilterRef

SINGULAR = 4
FILTER_DOUBLES = 163


def _to_ref(f, fr):
    fr.R, fr.t, fr.w, fr.v = f[:9].reshape(3, 3).copy(), f[9:12].copy(), f[12:15].copy(), f[15:18].copy()
    fr.P, fr.valid = f[18:162].reshape(12, 12).copy(), f[162] == 1.0
    return fr


def _from_ref(fr):
    return np.concatenate([fr.R.reshape(9), fr.t, fr.w, fr.v, fr.P.reshape(144), [1.0 if fr.valid else 0.0]])


def class_size(table):
    """d_k (num_classes,) fp64: the largest distance between two of each class's 8 box corners table[k, 1:9] (fp32 values)"""
    c = np.asarray(table, np.float32).astype(np.float64)[:, 1:9]
    return np.sqrt((((c[:, :, None] - c[:, None, :]) ** 2).sum(-1)).max((1, 2)))


def world_track_step(state, fused, class_size, match_dist, max_misses, motion=None, dt=None):
    """one capture of every stream.  state: dict tracks (G, T, 5) int, poses (G, T, 12), next_id (G,), and with motion filter
    (G, T, 163) and params = (accel_sigma, init_velocity_sigma, gate); fused: world_count (G,), world_cls (G, M), R_world (G, M, 3, 3),
    t_world (G, M, 3), world_cov (G, M, 6, 6), fuse_status (G, M), world_index (G C, M).  -> (new state, outputs: wslot,
    world_track_id, matched (G, M), track_id (G C, M), and with motion R_filt, t_filt, pose_cov, velocity, reinit per world slot)"""
    st = {k: np.array(v, copy=True) for k, v in state.items() if k != "params"}
    tracks, poses, next_id = st["tracks"], st["poses"], st["next_id"]
    G, T, _ = tracks.shape
    M = fused["world_cls"].shape[1]
    C = fused["world_index"].shape[0] // max(G, 1)
    out = dict(wslot=-np.ones((G, M), np.int64), world_track_id=-np.ones((G, M), np.int64), matched=np.zeros((G, M), bool),
               track_id=-np.ones((G * C, M), np.int64))
    if motion:
        accel, v0, gate = state["params"]
        out.update(R_filt=np.zeros((G, M, 3, 3)), t_filt=np.zeros((G, M, 3)), pose_cov=np.zeros((G, M, 6, 6)), velocity=np.zeros((G, M, 6)),
                   reinit=np.zeros((G, M), bool))
    nC = len(class_size)
    for g in range(G):
        n = int(np.clip(fused["world_count"][g], 0, M))
        alive, cls = tracks[g, :, 0] != 0, tracks[g, :, 2]
        pos = poses[g, :, 9:12].copy()
        if motion:
            for s in np.flatnonzero(alive & (st["filter"][g, :, 162] == 1.0)):
                fr = _to_ref(st["filter"][g, s], FilterRef(accel, v0, gate))
                fr.predict(dt[g])
                st["filter"][g, s] = _from_ref(fr)
            started = st["filter"][g, :, 162] == 1.0
            pos[started] = st["filter"][g, started, 9:12]
        taken = np.zeros(T, bool)
        wcls = fused["world_cls"][g, :n]
        ok_cls = (wcls >= 0) & (wcls < nC)
        sl = -np.ones(n, np.int64)
        for w in range(n):
            if not ok_cls[w]:
                continue
            tw = fused["t_world"][g, w]
            diff = tw[None] - pos
            d2 = diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1] + diff[:, 2] * diff[:, 2]
            r2 = (match_dist * class_size[wcls[w]]) ** 2
            ok = alive & ~taken & (cls == wcls[w]) & (d2 < r2)
            if ok.any():
                s = int(np.flatnonzero(ok & (d2 == d2[ok].min()))[0])
                taken[s], sl[w] = True, s
        age = alive & ~taken
        tracks[g, age, 3] += 1
        tracks[g, age & (tracks[g, :, 3] > max_misses), 0] = 0
        hit = sl >= 0
        ids = np.where(hit, tracks[g, np.maximum(sl, 0), 1], -1)
        for w in np.flatnonzero(~hit & ok_cls):
            free = np.flatnonzero(tracks[g, :, 0] == 0)
            if len(free) == 0:
                continue
            s = int(free[0])
            tracks[g, s] = (1, next_id[g], wcls[w], 0, 0)
            sl[w], ids[w] = s, next_id[g]
            next_id[g] += 1
        out["wslot"][g, :n], out["world_track_id"][g, :n], out["matched"][g, :n] = sl, ids, hit
        wi = fused["world_index"][g * C:(g + 1) * C]
        out["track_id"][g * C:(g + 1) * C] = np.where((wi >= 0) & (wi < n), np.concatenate([ids, [-1]])[np.where(wi < n, wi, n)], -1)
        for w in np.flatnonzero(sl >= 0):
            s = sl[w]
            R, t = fused["R_world"][g, w], fused["t_world"][g, w]
            poses[g, s, :9], poses[g, s, 9:] = R.reshape(9), t
            tracks[g, s, 3] = 0
            tracks[g, s, 4] += 1
            if not motion:
                continue
            fr = _to_ref(st["filter"][g, s], FilterRef(accel, v0, gate))
            usable = not fused["fuse_status"][g, w] & SINGULAR
            if hit[w]:
                folded = fr.update(R, t, fused["world_cov"][g, w], usable)
            else:
                fr.init(R, t, fused["world_cov"][g, w], usable)
                folded = False
            st["filter"][g, s] = _from_ref(fr)
            out["R_filt"][g, w], out["t_filt"][g, w], out["pose_cov"][g, w] = fr.R, fr.t, fr.P[:6, :6]
            out["velocity"][g, w], out["reinit"][g, w] = np.concatenate([fr.w, fr.v]), not folded
    if motion:
        st["params"] = state["params"]
    return st, out
