"""numpy restatement of the silhouette-mask rules (singleshotpose_b200/csrc/render_core.h), written from the rules' text and
not from that header: vertex coordinates snapped to 1/256 px with round-half-even, edge functions in int64, a pixel centre
(x, y) covered when it lies inside a non-degenerate triangle of either winding, a centre on an edge counted for top and left
edges only (Direct3D's rule), 255 / 0 bytes, and the status bits (1: a vertex at camera depth <= 0, 2: a projected coordinate
that is not finite or outside +-2^20 px, 4: a face index outside [0, nv)); a pose with a status bit gets an all-zero mask.

The camera depth here is a plain fp64 dot product, where the kernel uses FMAs: the two can disagree on the sign only for a
vertex within rounding of the camera plane, which the tests do not produce."""
import numpy as np

GUARD = 2.0 ** 20


def status_ref(X, faces, Rt, uv):
    """X (3|4, nv); faces (nf, 3) int; Rt (n, 3, 4); uv (n, 2, nv) float32 -> (n,) int32"""
    X = np.asarray(X, np.float64)
    Xh = X if X.shape[0] == 4 else np.concatenate([X, np.ones((1, X.shape[1]))])
    nv = X.shape[1]
    z = np.einsum("nk,kv->nv", np.asarray(Rt, np.float64)[:, 2, :], Xh)
    st = np.where((z > 0).all(axis=1), 0, 1)
    with np.errstate(invalid="ignore"):
        ok = (np.abs(uv) <= GUARD).all(axis=(1, 2))
    st |= np.where(ok, 0, 2)
    faces = np.asarray(faces)
    if ((faces < 0) | (faces >= nv)).any():
        st |= 4
    return st.astype(np.int32)


def snap(uv):
    """round-half-even(u * 256) of float32 coordinates, as int64"""
    return np.rint(np.asarray(uv, np.float32) * np.float32(256)).astype(np.int64)


def raster_ref(s, faces, W, H):
    """s (2, nv) int64 snapped coordinates of one pose; faces (nf, 3) in range -> (H, W) uint8 mask"""
    a, b, c = (s[:, faces[:, k]].T for k in range(3))                  # (nf, 2) each
    area = (b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0])
    keep = area != 0
    a, b, c, area = a[keep], b[keep], c[keep], area[keep]
    flip = area < 0                                                     # make every triangle clockwise on screen (y down)
    b, c = np.where(flip[:, None], c, b), np.where(flip[:, None], b, c)
    P = np.stack([a, b, c], 1)                                          # (T, 3, 2)
    lo, hi = P.min(1), P.max(1)
    x0 = np.maximum(-((-lo[:, 0]) // 256), 0); x1 = np.minimum(hi[:, 0] // 256, W - 1)
    y0 = np.maximum(-((-lo[:, 1]) // 256), 0); y1 = np.minimum(hi[:, 1] // 256, H - 1)
    keep = (x0 <= x1) & (y0 <= y1)
    P, x0, x1, y0, y1 = P[keep], x0[keep], x1[keep], y0[keep], y1[keep]
    mask = np.zeros((H, W), np.uint8)
    if not len(P):
        return mask
    w, h = x1 - x0 + 1, y1 - y0 + 1
    cnt = w * h
    tri = np.repeat(np.arange(len(P)), cnt)
    off = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    xx, yy = x0[tri] + off % w[tri], y0[tri] + off // w[tri]
    px, py = xx * 256, yy * 256
    inside = np.ones(len(tri), bool)
    for i, j in ((0, 1), (1, 2), (2, 0)):
        ax, ay = P[tri, i, 0], P[tri, i, 1]
        dx, dy = P[tri, j, 0] - ax, P[tri, j, 1] - ay
        e = dx * (py - ay) - dy * (px - ax)
        top_left = ((dy == 0) & (dx > 0)) | (dy < 0)
        inside &= (e > 0) | ((e == 0) & top_left)
    mask[yy[inside], xx[inside]] = 255
    return mask


def render_masks_ref(X, faces, Rt, uv, W, H):
    """-> masks (n, H, W) uint8, status (n,) int32 for projected coordinates uv (n, 2, nv) float32 of X under Rt"""
    faces = np.asarray(faces, np.int64)
    st = status_ref(X, faces, Rt, uv)
    masks = np.zeros((len(st), H, W), np.uint8)
    for p in np.flatnonzero(st == 0):
        masks[p] = raster_ref(snap(uv[p]), faces, W, H)
    return masks, st
