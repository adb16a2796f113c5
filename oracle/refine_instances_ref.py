"""Oracle of the refinement of a rig's world instances (singleshotpose_b200/csrc/refine_instances_core.h) in numpy, written from the
rule's text: whole arrays per camera and iteration, numpy's summation order where the core sums per virtual thread, by a halving
tree and in camera order.

The rule per iteration k of one capture: the drawing set is every slot w < count of a known class whose input pose is finite and
whose fusion status has neither NO_VALID nor NO_VIEW, at its current pose (its input pose once a status bit has stopped it).  In
camera c each drawn face (every vertex at camera depth z > 0 and within +-2^20 px, fp32 pixels of the camera pose's projection with
the fp64 K and coefficients, computed in the kernel's order of operations) is rasterised with render_ref's snapping, top-left rule
and pixel centres, at the depth 1 / ((l_0 / z_0 + l_1 / z_1) + l_2 / z_2) of its clockwise vertices (l_i the edge value opposite
vertex i over the doubled area, as render_depth_ref weighs them); the owner of a pixel is the minimum of the keys
bits((float)z) << 32 | w.  Each running slot then pairs as refine_rig_ref does, dropping the pairs whose pixel another slot owns
(counted per camera as view_hidden), and solves; the instance map is the owners under the output poses, -1 where nobody."""
from __future__ import annotations

import numpy as np

from .pose_filter_ref import chol_ok, so3_exp
from .refine_depth_ref import BAD_POSE, FEW_POINTS, MIN_POINTS, SINGULAR, terms, undistort
from .refine_rig_ref import FUSE_NONE
from .render_ref import GUARD, snap

NOBODY = np.uint64(0xFFFFFFFFFFFFFFFF)


def camera_pose(Rc, tc, R, t):
    """(Rc R, Rc t + tc), every product and sum in ssp_mv::to_camera's order"""
    Rw, tw = np.empty((3, 3)), np.empty(3)
    for i in range(3):
        for j in range(3):
            Rw[i, j] = Rc[i, 0] * R[0, j] + Rc[i, 1] * R[1, j] + Rc[i, 2] * R[2, j]
        tw[i] = Rc[i, 0] * t[0] + Rc[i, 1] * t[1] + Rc[i, 2] * t[2] + tc[i]
    return Rw, tw


def draw_vertices(Rw, tw, X, K, k=None):
    """fp32 pixels (u, v) and fp64 camera depth z of the points X (n, 3) under the camera pose (Rw, tw), in ssp_mv::project's order"""
    x, y, z = (Rw[i, 0] * X[:, 0] + Rw[i, 1] * X[:, 1] + Rw[i, 2] * X[:, 2] + tw[i] for i in range(3))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if k is None:
            px = K[0, 0] * x + K[0, 1] * y + K[0, 2] * z
            py = K[1, 0] * x + K[1, 1] * y + K[1, 2] * z
            pz = K[2, 0] * x + K[2, 1] * y + K[2, 2] * z
            u, v = px / pz, py / pz
        else:
            iz = 1.0 / z
            xn, yn = x * iz, y * iz
            r2 = xn * xn + yn * yn
            r4 = r2 * r2
            r6 = r4 * r2
            a1, a2, a3 = 2 * xn * yn, r2 + 2 * xn * xn, r2 + 2 * yn * yn
            cd = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6
            ic = 1.0 / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6)
            u = (xn * cd * ic + k[2] * a1 + k[3] * a2) * K[0, 0] + K[0, 2]
            v = (yn * cd * ic + k[2] * a3 + k[3] * a1) * K[1, 1] + K[1, 2]
        return u.astype(np.float32), v.astype(np.float32), z


def draw_keys(owner, u, v, z, faces, w):
    """rasterise the faces (f, 3) of one instance with vertex pixels (u, v) and depths z into the flat key buffer owner (H, W)"""
    H, W = owner.shape
    F = np.asarray(faces, np.int64)
    with np.errstate(invalid="ignore"):
        good = (z > 0) & (np.abs(u) <= GUARD) & (np.abs(v) <= GUARD)
    F = F[good[F].all(1)]
    s = snap(np.stack([u, v]))
    a, b, c = F[:, 0], F[:, 1], F[:, 2]
    area = (s[0, b] - s[0, a]) * (s[1, c] - s[1, a]) - (s[1, b] - s[1, a]) * (s[0, c] - s[0, a])
    keep = area != 0
    a, b, c, area = a[keep], b[keep], c[keep], area[keep]
    flip = area < 0
    b, c = np.where(flip, c, b), np.where(flip, b, c)
    area = np.abs(area)
    V = np.stack([a, b, c], 1)                                         # clockwise on screen
    X, Y = s[0, V], s[1, V]
    x0 = np.maximum(-((-X.min(1)) // 256), 0); x1 = np.minimum(X.max(1) // 256, W - 1)
    y0 = np.maximum(-((-Y.min(1)) // 256), 0); y1 = np.minimum(Y.max(1) // 256, H - 1)
    keep = (x0 <= x1) & (y0 <= y1)
    V, X, Y, area, x0, x1, y0, y1 = V[keep], X[keep], Y[keep], area[keep], x0[keep], x1[keep], y0[keep], y1[keep]
    iz = 1.0 / z
    w_, h_ = x1 - x0 + 1, y1 - y0 + 1
    cnt = w_ * h_
    flat = owner.reshape(-1)
    for lo in range(0, len(V), 4096):
        sl = slice(lo, lo + 4096)
        tri = np.repeat(np.arange(len(V))[sl], cnt[sl])
        off = np.arange(cnt[sl].sum()) - np.repeat(np.cumsum(cnt[sl]) - cnt[sl], cnt[sl])
        xx, yy = x0[tri] + off % w_[tri], y0[tri] + off // w_[tri]
        px, py = xx * 256, yy * 256
        inside = np.ones(len(tri), bool)
        lam = np.zeros((len(tri), 3))
        for i, j in ((0, 1), (1, 2), (2, 0)):
            ax, ay = X[tri, i], Y[tri, i]
            dx, dy = X[tri, j] - ax, Y[tri, j] - ay
            e = dx * (py - ay) - dy * (px - ax)
            top_left = ((dy == 0) & (dx > 0)) | (dy < 0)
            inside &= (e > 0) | ((e == 0) & top_left)
            lam[:, 3 - i - j] = e / area[tri]                          # the weight of the vertex opposite edge (i, j)
        tri, xx, yy, lam = tri[inside], xx[inside], yy[inside], lam[inside]
        izv = iz[V[tri]]
        zz = 1.0 / ((lam[:, 0] * izv[:, 0] + lam[:, 1] * izv[:, 1]) + lam[:, 2] * izv[:, 2])
        keys = (zz.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(w)
        np.minimum.at(flat, yy * W + xx, keys)


def draw_owners(meshes, Ks, ks, Rr, tr, W, H, drawn, cls, R, t):
    """(C, H, W) uint64 owner keys of the slots `drawn` (M,) bool at the world poses R (M, 3, 3), t (M, 3)"""
    O = np.full((len(Ks), H, W), NOBODY, np.uint64)
    for c in range(len(Ks)):
        for w in np.flatnonzero(drawn):
            X, _N, faces, _d = meshes[int(cls[w])]
            Rw, tw = camera_pose(Rr[c], tr[c], R[w], t[w])
            u, v, z = draw_vertices(Rw, tw, X, np.asarray(Ks[c], np.float64), ks[c])
            draw_keys(O[c], u, v, z, faces, w)
    return O


def instance_map(O):
    """int16 owner slots of owner keys, -1 where nobody"""
    return np.where(O == NOBODY, -1, (O & np.uint64(0xFFFFFFFF)).astype(np.int64)).astype(np.int16)


def key_depth(O):
    """the fp32 depth each owner key holds (inf where nobody)"""
    return np.where(O == NOBODY, np.inf, (O >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64))


def owned_pairs(depth, owner, w, X, N, R, t, K, tau, depth_scale, k=None):
    """refine_depth_ref.pairs under (R, t) with the pixel each pair read -> (a, m, p, q, owned by nobody or w)"""
    depth = np.asarray(depth)
    H, W = depth.shape
    a, m = X @ R.T, N @ R.T
    p = a + t
    ok = ((m * p).sum(1) < 0) & (p[:, 2] > 0)
    a, m, p = a[ok], m[ok], p[ok]
    x, y = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    if k is not None:
        r2 = x * x + y * y
        g = (1 + k[0] * r2 + k[1] * r2 ** 2 + k[4] * r2 ** 3) / (1 + k[5] * r2 + k[6] * r2 ** 2 + k[7] * r2 ** 3)
        x, y = x * g + 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x), y * g + k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y
    u, v = K[0, 0] * x + K[0, 2], K[1, 1] * y + K[1, 2]
    fu, fv = np.floor(u + 0.5), np.floor(v + 0.5)
    ok = (fu >= 0) & (fu < W) & (fv >= 0) & (fv < H)
    a, m, p, fu, fv = a[ok], m[ok], p[ok], fu[ok], fv[ok]
    iu, iv = fu.astype(np.int64), fv.astype(np.int64)
    D = depth[iv, iu].astype(np.float64)
    z = D * depth_scale
    ok = (D > 0) & (np.abs(p[:, 2] - z) <= tau)
    a, m, p, fu, fv, z, iu, iv = a[ok], m[ok], p[ok], fu[ok], fv[ok], z[ok], iu[ok], iv[ok]
    if k is None:
        xh, yh = (fu - K[0, 2]) / K[0, 0], (fv - K[1, 2]) / K[1, 1]
    else:
        xh, yh = undistort(k, fu, fv, K)
    key = owner[iv, iu]
    mine = (key == NOBODY) | ((key & np.uint64(0xFFFFFFFF)) == np.uint64(w))
    return a, m, p, np.stack([z * xh, z * yh, z], 1), mine


def refine_instances_ref(depths, meshes, Ks, dists, Rr, tr, cls, R, t, count=None, fuse_status=None, depth_scale=0.001, iters=10,
                         gate=(0.5, 0.02)):
    """one capture: depths (C, H, W); meshes {class: (X (n, 3), N (n, 3), faces (f, 3), diam)}; Ks (C, 3, 3), dists None or (C, 8)
    (a zero row: pinhole), Rr (C, 3, 3), tr (C, 3); cls (M,), R (M, 3, 3), t (M, 3) the world slots, count (default M),
    fuse_status (M,) or None -> dict R, t, points, rmse, status, view_points, view_rmse, view_hidden, instance_map (C, H, W), owner"""
    Cn, H, W = np.asarray(depths).shape
    M = len(cls)
    count = M if count is None else int(count)
    fs = np.zeros(M, np.int64) if fuse_status is None else np.asarray(fuse_status)
    ks = [None if dists is None or not np.any(dists[c]) else np.asarray(dists[c], np.float64) for c in range(Cn)]
    R0, t0 = np.asarray(R, np.float64).copy(), np.asarray(t, np.float64).copy()
    known = np.array([int(c) in meshes for c in cls])
    out = np.arange(M) >= count
    usable = np.array([np.isfinite(R0[w]).all() and np.isfinite(t0[w]).all() and not (fs[w] & FUSE_NONE) for w in range(M)])
    drawn = ~out & known & usable
    o = dict(R=np.where(out[:, None, None], 0.0, R0), t=np.where(out[:, None], 0.0, t0), points=np.zeros(M, np.int64), rmse=np.zeros(M),
             status=np.where(out | usable, 0, BAD_POSE), view_points=np.zeros((M, Cn), np.int64), view_rmse=np.zeros((M, Cn)),
             view_hidden=np.zeros((M, Cn), np.int64))
    s, e = gate
    for it in range(iters):
        O = draw_owners(meshes, Ks, ks, Rr, tr, W, H, drawn, cls, o["R"], o["t"])
        for w in np.flatnonzero(~out & (o["status"] == 0)):
            X, N, _faces, diam = meshes[int(cls[w])] if known[w] else (np.zeros((0, 3)), np.zeros((0, 3)), None, 0.0)
            tau = diam * (s if iters == 1 else s * (e / s) ** (it / (iters - 1)))
            Rw, tw = o["R"][w], o["t"][w]
            rs, Js = [], []
            for c in range(Cn):
                Kc = np.asarray(Ks[c], np.float64)
                a, m, p, q, mine = owned_pairs(depths[c], O[c], w, X, N, Rr[c] @ Rw, Rr[c] @ tw + tr[c], Kc, tau, depth_scale, ks[c])
                a, m, p, q = a[mine], m[mine], p[mine], q[mine]
                r, J = terms(a @ Rr[c], m @ Rr[c], a @ Rr[c] + tw, (q - tr[c]) @ Rr[c])
                rs.append(r)
                Js.append(J)
                o["view_points"][w, c], o["view_hidden"][w, c] = len(r), int((~mine).sum())
                o["view_rmse"][w, c] = np.sqrt((r @ r) / len(r)) if len(r) else 0.0
            r, J = np.concatenate(rs), np.concatenate(Js)
            n = len(r)
            o["points"][w], o["rmse"][w] = n, (float(np.sqrt((r @ r) / n)) if n else 0.0)
            if n < MIN_POINTS:
                o["status"][w] = FEW_POINTS
            elif not chol_ok(J.T @ J):
                o["status"][w] = SINGULAR
            else:
                delta = -np.linalg.solve(J.T @ J, J.T @ r)
                o["R"][w], o["t"][w] = so3_exp(delta[:3]) @ Rw, tw + delta[3:]
                continue
            o["R"][w], o["t"][w] = R0[w], t0[w]
    O = draw_owners(meshes, Ks, ks, Rr, tr, W, H, drawn, cls, o["R"], o["t"])
    o["owner"], o["instance_map"] = O, instance_map(O)
    return o
