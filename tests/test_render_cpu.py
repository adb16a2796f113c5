"""CPU tests of the training-set maker's pieces:
  * the silhouette rules of singleshotpose_b200/csrc/render_core.h compiled for the host (tests/helpers/render_host.cpp)
    against their numpy int64 restatement (oracle/render_ref.py): masks and status equal, on the synthetic closed mesh, partly
    off-screen poses, single-pixel and image-sized triangles, degenerate faces, depth <= 0, the guard band and bad indices;
  * the restatement itself against geometry it does not share: the convex hull of a convex mesh (scipy) and the tie rule on
    a two-triangle square;
  * label rows against the reference's own get_3D_corners / compute_projection / fill_truth_detection (tests/golden/labels.npz,
    written by tests/golden/make_golden_labels.py);
  * read_ply_mesh, the make_dataset command line's checks, and the ABI of ssp_render_masks / ssp_render_work_bytes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from oracle.render_ref import render_masks_ref, snap
from singleshotpose_b200 import _lib, make_dataset, synth, utils, utils_host

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("renderhost") / "librenderhost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(REPO, "tests", "helpers", "render_host.cpp")])
    lib = C.CDLL(so)
    lib.h_render_masks.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong,
                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def host_render(host, X, faces, Rt, uv, W, H):
    """X (3|4, nv) float32; faces (nf, 3); Rt (n, 3, 4); uv (n, 2, nv) float32 -> masks, status"""
    X = np.ascontiguousarray(X, np.float32)
    F = np.ascontiguousarray(faces, np.int32)
    T = np.ascontiguousarray(Rt, np.float64)
    U = np.ascontiguousarray(uv, np.float32)
    n = len(T)
    masks = np.full((n, H, W), 7, np.uint8)
    status = np.full(n, -1, np.int32)
    assert host.h_render_masks(X.ctypes.data, X.shape[0], X.shape[1], F.ctypes.data, len(F), T.ctypes.data, U.ctypes.data, n, W, H,
                               masks.ctypes.data, status.ctypes.data) == 0
    return masks, status


def project(X, Rt, K):
    """(n, 2, nv) float32 pixel coordinates (compute_projection per pose)"""
    Xh = np.r_[np.asarray(X, np.float64)[:3], np.ones((1, X.shape[1]))]
    return np.stack([utils.compute_projection(Xh, T, K) for T in Rt])


def poses_rt(R, t):
    return np.concatenate([R, t[:, :, None]], 2)


def check_equal(host, X, faces, Rt, uv, W, H):
    m, s = host_render(host, X, faces, Rt, uv, W, H)
    mr, sr = render_masks_ref(X, faces, Rt, uv, W, H)
    np.testing.assert_array_equal(s, sr)
    for p in range(len(m)):
        assert np.array_equal(m[p], mr[p]), (p, int((m[p] != mr[p]).sum()))
    assert set(np.unique(m)) <= {0, 255}
    return m, s


@pytest.fixture(scope="module")
def mesh():
    V, F = synth.closed_mesh(seed=1)
    return V.T.astype(np.float32), F


# ------------------------------------------------------------------------------------------------ host build vs numpy restatement
def test_mesh_size_is_linemod_like(mesh):
    X, F = mesh
    assert 5000 < X.shape[1] < 8000 and 10000 < len(F) < 15000
    edges = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), axis=1)
    _, cnt = np.unique(edges, axis=0, return_counts=True)
    assert (cnt == 2).all()                                             # closed: every edge has two faces


def test_random_poses_match_oracle(host, mesh):
    X, F = mesh
    R, t = synth.object_poses(6, seed=3)
    Rt = poses_rt(R, t)
    uv = project(X, Rt, synth.intrinsics())
    m, s = check_equal(host, X, F, Rt, uv, 640, 480)
    assert (s == 0).all() and all(1000 < (mm > 0).sum() < 640 * 480 // 4 for mm in m)


def test_partly_off_screen_poses_match_oracle(host, mesh):
    X, F = mesh
    R, _ = synth.object_poses(4, seed=4)
    t = np.array([[0.34, 0.0, 0.6], [-0.34, 0.1, 0.6], [0.05, 0.26, 0.6], [-0.3, -0.25, 0.55]])
    Rt = poses_rt(R, t)
    uv = project(X, Rt, synth.intrinsics())
    m, s = check_equal(host, X, F, Rt, uv, 640, 480)
    for p in range(4):                                                  # each pose leaves the image on one side
        assert (uv[p, 0] < 0).any() or (uv[p, 0] > 639).any() or (uv[p, 1] < 0).any() or (uv[p, 1] > 479).any()
        assert m[p].any()


def test_odd_size_and_handmade_triangles_match_oracle(host):
    rng = np.random.default_rng(11)
    W, H = 37, 23
    pts = [
        [5.0, 5.0], [5.25, 6.0], [4.75, 6.0],                  # covers no centre ... or one, depending on the tie rule
        [10.0, 10.0], [10.5, 9.5], [10.5, 10.5],              # one-pixel triangle with a vertex on a centre
        [-40.0, -40.0], [120.0, -40.0], [-40.0, 120.0],       # bigger than the image
        [2.0, 2.0], [6.0, 2.0], [6.0, 6.0], [2.0, 6.0],       # a square with corners on centres
        [20.0, 3.0], [25.0, 3.0], [30.0, 3.0],                # collinear: degenerate
    ]
    # coordinates on the 1/256 grid, on half steps of it (round-half-even ties) and anywhere
    rnd = rng.uniform(-3, W + 3, size=(60, 2))
    rnd[:20] = np.round(rnd[:20] * 256) / 256
    rnd[20:40] = (np.floor(rnd[20:40] * 256) + 0.5) / 256
    uv = np.concatenate([np.array(pts), rnd]).T.astype(np.float32)
    nv = uv.shape[1]
    faces = [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11], [9, 11, 12], [13, 14, 15], [13, 13, 14]]
    faces += [[16 + 3 * i, 17 + 3 * i, 18 + 3 * i] for i in range(20)]
    X = np.vstack([np.zeros((2, nv)), np.ones((1, nv))]).astype(np.float32)          # depth 1 for every vertex
    Rt = np.array([np.c_[np.eye(3), np.zeros(3)]])
    faces = np.array(faces)
    for sub in (faces[6:7], faces[:6], faces):
        check_equal(host, X, sub, Rt, uv[None], W, H)
    m, _ = host_render(host, X, faces[2:3], Rt, uv[None], W, H)
    assert (m == 255).all()                                             # the image-sized triangle covers every pixel
    m, _ = host_render(host, X, faces[5:7], Rt, uv[None], W, H)
    assert not m.any()                                                  # degenerate faces cover nothing


def test_status_bits_match_oracle(host, mesh):
    X, F = mesh
    R, t = synth.object_poses(5, seed=5)
    t[1, 2] = 0.0                                                       # pose 1: the mesh straddles the camera plane
    Rt = poses_rt(R, t)
    uv = project(X, Rt, synth.intrinsics())
    uv[2, 0, 17] = 2.0 ** 20 + 1                                        # pose 2: outside the guard band
    uv[3, 1, 5] = np.nan                                                # pose 3: not finite
    uv[4, 0, 9] = -np.inf
    m, s = check_equal(host, X, F, Rt, uv, 640, 480)
    assert s.tolist() == [0, s[1], 2, 2, 2] and s[1] & 1
    assert m[0].any() and not m[1:].any()
    Fb = F.copy()
    Fb[7, 1] = X.shape[1]
    m, s = check_equal(host, X, Fb, Rt[:1], uv[:1], 640, 480)
    assert s.tolist() == [4] and not m.any()
    Fb[7, 1] = -1
    assert host_render(host, X, Fb, Rt[:1], uv[:1], 640, 480)[1].tolist() == [4]
    uv[0, 0, 3] = 2.0 ** 20                                             # exactly on the guard: allowed
    assert host_render(host, X, F, Rt[:1], uv[:1], 640, 480)[1].tolist() == [0]


# ------------------------------------------------------------------------------------------------ the restatement, independently
def test_convex_mesh_equals_hull_of_snapped_vertices(mesh):
    from scipy.spatial import ConvexHull
    V, F = synth.closed_mesh(bumps=0.0, seed=2)
    X = V.T.astype(np.float32)
    R, t = synth.object_poses(3, seed=6)
    Rt = poses_rt(R, t)
    uv = project(X, Rt, synth.intrinsics())
    masks, st = render_masks_ref(X, F, Rt, uv, 640, 480)
    assert (st == 0).all()
    yy, xx = np.mgrid[0:480, 0:640]
    P = np.stack([xx.ravel(), yy.ravel()], 1).astype(np.float64)
    for p in range(3):
        S = snap(uv[p]).T / 256.0
        hull = ConvexHull(S)
        d = (P @ hull.equations[:, :2].T + hull.equations[:, 2]).max(1)   # signed distance to the hull (< 0 inside)
        far = np.abs(d) >= 1 / 128
        inside = (d < 0).reshape(480, 640)
        got = masks[p] == 255
        assert np.array_equal(got.ravel()[far], inside.ravel()[far]) and got.sum() > 1000


@pytest.mark.parametrize("diagonal", ["main", "anti"])
@pytest.mark.parametrize("reverse", [False, True])
def test_square_tie_rule(diagonal, reverse):
    sq = np.array([[2.0, 2.0], [6.0, 2.0], [6.0, 6.0], [2.0, 6.0]]).T.astype(np.float32)   # corners on pixel centres
    F = np.array([[0, 1, 2], [0, 2, 3]] if diagonal == "main" else [[0, 1, 3], [1, 2, 3]])
    if reverse:
        F = F[:, ::-1]
    X = np.vstack([np.zeros((2, 4)), np.ones((1, 4))])
    Rt = np.array([np.c_[np.eye(3), np.zeros(3)]])
    m, _ = render_masks_ref(X, F, Rt, sq[None], 10, 9)
    want = np.zeros((9, 10), np.uint8)
    want[2:6, 2:6] = 255                 # top edge y = 2 and left edge x = 2 covered; bottom y = 6 and right x = 6 not
    assert np.array_equal(m[0], want)   # the diagonal's centres, shared by both triangles, included


# ------------------------------------------------------------------------------------------------ label rows
@pytest.fixture(scope="module")
def labels(golden_dir):
    return np.load(os.path.join(golden_dir, "labels.npz"))


def test_label_rows_equal_reference(labels):
    rows = utils_host.label_rows_from_projection(labels["px"], int(labels["width"]), int(labels["height"]), int(labels["class_id"]))
    assert rows.dtype == np.float64 and np.array_equal(rows, labels["rows"])


def test_written_label_reads_back_as_reference(labels, tmp_path):
    for p, row in enumerate(labels["rows"]):
        lab = str(tmp_path / ("%06d.txt" % p))
        np.savetxt(lab, row[None])                                      # make_dataset's writer
        assert np.array_equal(utils_host.read_truths(lab)[0], labels["readback"][p])
        assert np.array_equal(utils_host.read_truths_args(lab), labels["readback"][p][:19])


def test_label_corners_are_get_3D_corners(labels):
    V, _ = synth.closed_mesh(seed=1)
    assert np.array_equal(utils.get_3D_corners(np.c_[V, np.ones(len(V))].T), labels["corners3D"])


# ------------------------------------------------------------------------------------------------ read_ply_mesh
def test_read_ply_mesh_parses_faces(tmp_path, mesh):
    V, F = synth.closed_mesh(seed=1)
    path = str(tmp_path / "m.ply")
    synth.write_ply(path, V, F)
    V2, F2 = utils_host.read_ply_mesh(path)
    assert np.array_equal(V2, V) and F2.dtype == np.int32 and np.array_equal(F2, F)
    assert np.array_equal(utils_host.read_ply_vertices(path), V)


def _ply(path, faces_lines, nv=4, fmt="ascii"):
    with open(path, "w") as f:
        f.write("ply\nformat %s 1.0\ncomment x\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "property uchar red\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n" % (fmt, nv, len(faces_lines)))
        for i in range(nv):
            f.write("%d.5 %d %d 200\n" % (i, 2 * i, -i))
        f.write("".join(s + "\n" for s in faces_lines))
    return path


def test_read_ply_mesh_refuses_quads_bad_indices_and_binary(tmp_path):
    ok = _ply(str(tmp_path / "ok.ply"), ["3 0 1 2", "3 0 2 3"])
    V, F = utils_host.read_ply_mesh(ok)
    assert V.shape == (4, 3) and F.tolist() == [[0, 1, 2], [0, 2, 3]] and V[1].tolist() == [1.5, 2.0, -1.0]
    with pytest.raises(ValueError, match="triangulate the mesh first"):
        utils_host.read_ply_mesh(_ply(str(tmp_path / "q.ply"), ["3 0 1 2", "4 0 1 2 3"]))
    for bad in ("3 0 1 4", "3 -1 1 2"):
        with pytest.raises(ValueError, match="outside"):
            utils_host.read_ply_mesh(_ply(str(tmp_path / "b.ply"), ["3 0 1 2", bad]))
    with pytest.raises(ValueError, match="ASCII PLY only"):
        utils_host.read_ply_mesh(_ply(str(tmp_path / "bin.ply"), ["3 0 1 2"], fmt="binary_little_endian"))


def test_read_ply_vertices_unchanged_on_meshes_with_faces(tmp_path):
    p = _ply(str(tmp_path / "v.ply"), ["4 0 1 2 3", "3 0 1 9"])          # faces read_ply_mesh refuses
    V = utils_host.read_ply_vertices(p)
    assert V.shape == (4, 3) and V[3].tolist() == [3.5, 6.0, -3.0]


# ------------------------------------------------------------------------------------------------ make_dataset's checks
def _tree(tmp_path, names, sizes=None):
    d = tmp_path / "obj" / "JPEGImages"
    d.mkdir(parents=True, exist_ok=True)
    paths = []
    for i, nm in enumerate(names):
        w, h = (sizes or {}).get(i, (64, 48))
        p = str(d / nm)
        Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(p)
        paths.append(p)
    return paths


def test_cli_parses_arguments():
    a = make_dataset.parse_args(["--mesh", "m.ply", "--poses", "p.npz", "--fx", "572.4", "--fy", "573.5", "--u0", "325.2", "--v0", "242.0",
                                 "--name", "obj", "--data-out", "cfg/obj.data"])
    assert (a.mesh, a.poses, a.fx, a.fy, a.u0, a.v0, a.name, a.class_id, a.test_list, a.data_out) == \
        ("m.ply", "p.npz", 572.4, 573.5, 325.2, 242.0, "obj", 0, None, "cfg/obj.data")
    a = make_dataset.parse_args(["--mesh", "m", "--poses", "p", "--fx", "1", "--fy", "1", "--u0", "0", "--v0", "0", "--name", "o",
                                 "--class-id", "4", "--test-list", "t.txt", "--data-out", "d"])
    assert a.class_id == 4 and a.test_list == "t.txt"
    with pytest.raises(SystemExit):
        make_dataset.parse_args(["--mesh", "m.ply"])


def test_cli_refuses_colliding_paths(tmp_path):
    paths = _tree(tmp_path, ["001.jpg", "1.jpg"])                     # both map to mask/1.png
    with pytest.raises(make_dataset.DatasetError, match="1.jpg.*mask"):
        make_dataset.check_images(paths)
    paths = _tree(tmp_path / "images", ["000123.jpg"]) + _tree(tmp_path / "labels", ["000123.jpg"])
    with pytest.raises(make_dataset.DatasetError, match="both map to the label file"):   # .../labels/obj/labels/000123.txt
        make_dataset.check_images(paths)
    assert make_dataset.check_images(_tree(tmp_path, ["000001.jpg", "000002.jpg"])) == (64, 48)


def test_cli_refuses_mixed_sizes_and_missing_images(tmp_path):
    paths = _tree(tmp_path, ["000001.png", "000002.png"], sizes={1: (64, 50)})
    with pytest.raises(make_dataset.DatasetError, match="000002.png is 64 x 50"):
        make_dataset.check_images(paths)
    with pytest.raises(make_dataset.DatasetError, match="000009.png: no such image"):
        make_dataset.check_images(paths[:1] + [paths[0].replace("000001", "000009")])
    with pytest.raises(make_dataset.DatasetError, match="JPEGImages"):
        make_dataset.check_images([str(tmp_path / "x.png")])


def test_cli_refuses_before_touching_the_device(tmp_path):
    paths = _tree(tmp_path, ["001.jpg", "1.jpg"])
    np.savez(str(tmp_path / "p.npz"), paths=np.array(paths), R=np.stack([np.eye(3)] * 2), t=np.ones((2, 3)))
    with pytest.raises(SystemExit, match="make_dataset: .*both map to the mask file"):
        make_dataset.main(["--mesh", "m.ply", "--poses", str(tmp_path / "p.npz"), "--fx", "1", "--fy", "1", "--u0", "0", "--v0", "0",
                           "--name", "o", "--data-out", str(tmp_path / "o.data")])
    assert not (tmp_path / "obj" / "labels").exists() and not (tmp_path / "o.data").exists()
    np.savez(str(tmp_path / "q.npz"), paths=np.array(paths), R=np.stack([np.eye(3)] * 2))
    with pytest.raises(make_dataset.DatasetError, match="no 't' array"):
        make_dataset.load_poses(str(tmp_path / "q.npz"))


# ------------------------------------------------------------------------------------------------ the C ABI
def test_render_symbols_are_declared_and_exported():
    for name in ("ssp_render_masks", "ssp_render_work_bytes"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)


def test_render_work_bytes_rejects_bad_sizes():
    wb = _lib.load().ssp_render_work_bytes
    assert wb(6002, 12000, 1, 640, 480) > 0 and wb(6002, 12000, 0, 640, 480) == 0
    assert wb(6002, 12000, 1024, 640, 480) >= 1024 * (6002 * 8 + 12000 * 32)
    for args in ((2, 10, 1, 64, 64), (10, 0, 1, 64, 64), (10, 10, -1, 64, 64), (10, 10, 1, 0, 64), (10, 10, 1, 64, 16385),
                 (10, 10, 1, 16385, 64), (10, 10, 1, 64, 0), (10, 10, 1 << 62, 64, 64)):
        assert wb(*args) < 0, args


def test_render_masks_abi_rejects_bad_arguments():
    d = C.c_void_p(256)
    wb = _lib.load().ssp_render_work_bytes(10, 4, 2, 64, 48)

    def args(**kw):
        a = dict(X=d, rows=3, nv=10, faces=d, nf=4, Rt=d, K=d, n=2, W=64, H=48, masks=d, status=d, work=d, wb=wb, stream=None)
        a.update(kw)
        return list(a.values())
    for k in ("X", "faces", "Rt", "K", "masks", "status", "work"):
        with pytest.raises(_lib.SspError, match="null pointer"):
            _lib.call("ssp_render_masks", *args(**{k: None}))
    for kw in (dict(rows=2), dict(rows=5), dict(nv=2), dict(nf=0), dict(n=-1), dict(W=0), dict(W=16385), dict(H=0), dict(H=16385)):
        with pytest.raises(_lib.SspError, match="bad argument"):
            _lib.call("ssp_render_masks", *args(**kw))
    with pytest.raises(_lib.SspError, match="work buffer"):
        _lib.call("ssp_render_masks", *args(wb=wb - 1))
    assert _lib.call("ssp_render_masks", *args(n=0, wb=0)) == 0          # n = 0: returns before any device access
