"""Oracle of tracking instances across frames (singleshotpose_b200/csrc/track_core.h) in numpy, and of the warm-started PnP
(cv2.solvePnP(..., SOLVEPNP_ITERATIVE, useExtrinsicGuess=True)).  TEST INFRASTRUCTURE ONLY.

Each stream owns T slots and a next_id counter.  Per frame, with the detections in detector order:
  1. match: detection m takes the alive, not yet taken track of its class with the highest IoU(track rect, rect_m) > match_iou
     (the lower slot on ties);
  2. age: unmatched alive tracks get misses += 1 and die when misses > max_misses;
  3. birth: unmatched detections, in order, take the lowest free slot and id = next_id++; none free -> untracked (-1);
  4. matched detections start LM from their track's pose (warm), the others get the DLT + LM (cold);
  5. commit: matched and born tracks take the detection's rectangle and the solve's final LM vector, misses 0, hits + 1.
The rectangles and IoU are those of oracle/detect_ref.py (fp32, every operation rounded on its own).

The warm PnP restates cvFindExtrinsicCameraParams2 with useExtrinsicGuess: the given (rvec, t) replace the DLT, then the same
CvLevMarq schedule as oracle/pnp_ref.py."""
from __future__ import annotations

import numpy as np

from .detect_ref import corner_rects, iou_ref
from .pnp_ref import FLT_EPSILON, project, rodrigues_vec2mat

F32 = np.float32


class StreamRef:
    """the state of one stream: T slots of alive, id, cls, misses, hits, rect (4,) fp32, pose (6,) fp64, and next_id"""

    def __init__(self, T):
        self.T = T
        self.reset()

    def reset(self):
        T = self.T
        self.alive = np.zeros(T, bool)
        self.id = np.zeros(T, np.int64)
        self.cls = np.zeros(T, np.int64)
        self.misses = np.zeros(T, np.int64)
        self.hits = np.zeros(T, np.int64)
        self.rect = np.zeros((T, 4), F32)
        self.pose = np.zeros((T, 6), np.float64)
        self.next_id = 0

    def associate(self, cls, uv, match_iou, max_misses):
        """steps 1-3 for the frame's n detections (cls (n,), uv (n, 9, 2) fp32 pixels) -> (slot (n,), track_id (n,), warm (n,) bool,
        guess (n, 6)); slot and track_id are -1 for an untracked detection"""
        n = len(cls)
        rects = corner_rects(uv) if n else np.zeros((0, 4), F32)
        slot = np.full(n, -1, np.int64)
        warm = np.zeros(n, bool)
        taken = np.zeros(self.T, bool)
        for m in range(n):
            v = iou_ref(rects[m], self.rect) if self.T else np.zeros(0, F32)
            ok = self.alive & ~taken & (self.cls == int(cls[m])) & (v > F32(match_iou))
            if ok.any():
                s = int(np.flatnonzero(ok & (v == v[ok].max()))[0])
                taken[s], slot[m], warm[m] = True, s, True
        age = self.alive & ~taken
        self.misses[age] += 1
        self.alive[age & (self.misses > max_misses)] = False
        track_id = np.where(warm, self.id[np.maximum(slot, 0)], -1)
        guess = np.where(warm[:, None], self.pose[np.maximum(slot, 0)], 0.0)
        for m in range(n):
            if warm[m]:
                continue
            free = np.flatnonzero(~self.alive)
            if len(free) == 0:
                continue
            s = int(free[0])
            self.alive[s], self.id[s], self.cls[s], self.misses[s], self.hits[s] = True, self.next_id, int(cls[m]), 0, 0
            slot[m], track_id[m] = s, self.next_id
            self.next_id += 1
        return slot, track_id, warm, guess

    def commit(self, uv, slot, params):
        """step 5: every detection with slot >= 0 stores its rectangle and its solve's LM vector params (n, 6)"""
        for m, s in enumerate(slot):
            if s < 0:
                continue
            self.rect[s] = corner_rects(np.asarray(uv, F32)[m:m + 1])[0]
            self.pose[s] = params[m]
            self.misses[s] = 0
            self.hits[s] += 1


def solve_pnp_guess(points_3D, points_2D, K, rvec, tvec, max_iter=20):
    """cv2.solvePnP(points_3D, points_2D, K, None, rvec, tvec, useExtrinsicGuess=True, flags=SOLVEPNP_ITERATIVE): the CvLevMarq
    refinement of oracle/pnp_ref.py started from (rvec, tvec) -> (rvec (3,), tvec (3,)) fp64"""
    M = np.asarray(points_3D, np.float64).reshape(-1, 3)
    m = np.asarray(points_2D, np.float64).reshape(-1, 2)
    K = np.asarray(K, np.float64)
    p = np.concatenate([np.asarray(rvec, np.float64).reshape(3), np.asarray(tvec, np.float64).reshape(3)])
    lam_lg10, iters = -3, 0

    def step(JtJ, Jte, prev, lg):
        A = JtJ.copy()
        A[np.diag_indices(6)] *= 1.0 + np.exp(lg * np.log(10.0))
        return prev - np.linalg.lstsq(A, Jte, rcond=None)[0]

    while True:
        uv, J = project(M, p[:3], p[3:], K, jac=True)
        err = (uv - m).reshape(-1)
        JtJ, Jte = J.T @ J, J.T @ err
        prev = p.copy()
        p = step(JtJ, Jte, prev, lam_lg10)
        if iters == 0:
            prev_err = np.linalg.norm(err)
        while True:
            e = np.linalg.norm((project(M, p[:3], p[3:], K) - m).reshape(-1))
            if e > prev_err:
                lam_lg10 += 1
                if lam_lg10 <= 16:
                    p = step(JtJ, Jte, prev, lam_lg10)
                    continue
            break
        lam_lg10 = max(lam_lg10 - 1, -16)
        iters += 1
        if iters >= max_iter or np.linalg.norm(p - prev) / np.linalg.norm(prev) < FLT_EPSILON:
            break
        prev_err = e
    return p[:3].copy(), p[3:].copy()


def pnp_guess_ref(points_3D, points_2D, K, rvec, tvec):
    """-> R (3, 3), t (3, 1) of solve_pnp_guess, as oracle/pnp_ref.py's pnp_ref returns them"""
    r, t = solve_pnp_guess(points_3D, np.asarray(points_2D)[:, :2], K, rvec, tvec)
    return rodrigues_vec2mat(r), t.reshape(3, 1)
