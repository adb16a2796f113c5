"""GPU tests of the silhouette masks and the training-set maker (ssp_render_masks, utils.render_masks, utils.pose_label_rows,
python -m singleshotpose_b200.make_dataset):
  * device masks and status bit-identical to the host build of render_core.h (tests/helpers/render_host.cpp) fed with the
    device's own projected coordinates, at 640 x 480 and an odd size, for n = 1 and n = 1000;
  * each pose's mask the same whatever the batch and the chunking; the coordinates the kernel used are project_points_batched's;
  * label rows against the reference's (tests/golden/labels.npz);
  * end to end: make_dataset on synthetic images and poses writes a tree that listDataset + GpuCollate load, whose labels are
    pose_label_rows, from whose keypoints PnP recovers the poses, and whose .data file holds calc_pts_diameter."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest
import torch
from PIL import Image

from singleshotpose_b200 import _lib, synth, utils, utils_host

pytestmark = pytest.mark.gpu
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


@pytest.fixture(scope="module")
def mesh():
    V, F = synth.closed_mesh(seed=1)
    return V, F


def _poses(n, seed, bad=True):
    """n poses; with bad=True a few have a vertex behind the camera or straddle the image border"""
    R, t = synth.object_poses(n, seed=seed)
    if bad and n > 10:
        t[3, 2] = 0.01                       # the mesh crosses the camera plane
        t[5, :2] = [0.35, -0.27]             # partly off-screen
        t[7, 2] = 0.06                       # close: projections far outside the image, but finite
    return np.concatenate([R, t[:, :, None]], 2)


def _render_raw(X4, F, Rt, K, W, H):
    """ssp_render_masks called directly -> (masks, status, the projected coordinates the launch used)"""
    n, nv = len(Rt), X4.shape[1]
    Xd = torch.from_numpy(np.ascontiguousarray(X4, np.float32)).cuda()
    Fd = torch.from_numpy(np.ascontiguousarray(F, np.int32)).cuda()
    Td = torch.from_numpy(np.ascontiguousarray(Rt, np.float64)).cuda()
    Kd = torch.from_numpy(np.ascontiguousarray(K, np.float64)).cuda()
    wb = int(_lib.load().ssp_render_work_bytes(nv, len(F), n, W, H))
    work = torch.zeros(wb, dtype=torch.uint8, device="cuda")
    masks = torch.full((n, H, W), 7, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    _lib.call("ssp_render_masks", _lib.ptr(Xd), Xd.shape[0], nv, _lib.ptr(Fd), len(F), _lib.ptr(Td), _lib.ptr(Kd), n, W, H,
              _lib.ptr(masks), _lib.ptr(status), _lib.ptr(work), wb, _lib.stream_ptr())
    uv = work[:n * 2 * nv * 4].view(torch.float32).view(n, 2, nv)
    return masks.cpu().numpy(), status.cpu().numpy(), uv


def _host(host, X4, F, Rt, uv, W, H):
    X = np.ascontiguousarray(X4, np.float32)
    Fc, T, U = np.ascontiguousarray(F, np.int32), np.ascontiguousarray(Rt, np.float64), np.ascontiguousarray(uv, np.float32)
    n = len(T)
    masks, status = np.zeros((n, H, W), np.uint8), np.zeros(n, np.int32)
    assert host.h_render_masks(X.ctypes.data, X.shape[0], X.shape[1], Fc.ctypes.data, len(Fc), T.ctypes.data, U.ctypes.data, n, W, H,
                               masks.ctypes.data, status.ctypes.data) == 0
    return masks, status


@pytest.mark.parametrize("size", [(640, 480), (333, 251)])
@pytest.mark.parametrize("n", [1, 1000])
def test_device_masks_equal_host_build(host, mesh, size, n):
    V, F = mesh
    W, H = size
    X4 = np.r_[V.T, np.ones((1, len(V)))]
    K = synth.intrinsics()
    Rt = _poses(n, seed=n + W)
    m, s, uv = _render_raw(X4, F, Rt, K, W, H)
    uvh = uv.cpu().numpy()
    assert torch.equal(uv, utils.project_points_batched(X4, Rt, K))        # the coordinates of project_points_batched
    hm, hs = _host(host, X4, F, Rt, uvh, W, H)
    np.testing.assert_array_equal(s, hs)
    bad = [p for p in range(n) if not np.array_equal(m[p], hm[p])]
    assert not bad, (bad[:10], len(bad))
    assert set(np.unique(m)) <= {0, 255}
    if n > 10:
        assert s[3] & 1 and not m[3].any() and s[5] == 0 and s[7] == 0 and m[7].any()
        assert m[5].any() or W < 640                                    # partly in a 640 x 480 view, outside a smaller one
        assert (s == 0).sum() >= n - 3


def test_mask_independent_of_batch_and_chunking(mesh, monkeypatch):
    V, F = mesh
    K = synth.intrinsics()
    Rt = _poses(300, seed=9)
    full, st = utils.render_masks(V, F, Rt, K, 640, 480)
    part, st_part = utils.render_masks(V, F, Rt[100:117], K, 640, 480)
    assert torch.equal(full[100:117], part) and torch.equal(st[100:117], st_part)
    per_pose = int(_lib.load().ssp_render_work_bytes(len(V), len(F), 1, 640, 480))
    monkeypatch.setattr(utils, "RENDER_CHUNK_BYTES", 7 * per_pose)           # chunks of 7 poses
    chunked, st_chunked = utils.render_masks(V, F, Rt, K, 640, 480)
    assert torch.equal(full, chunked) and torch.equal(st, st_chunked)
    one, _ = utils.render_masks(V.T, F, Rt[250], K, 640, 480)                # (3, Nv) vertices, a single (3, 4) pose
    assert torch.equal(one[0], full[250])


def test_render_masks_zero_poses_and_bad_face(mesh):
    V, F = mesh
    m, s = utils.render_masks(V, F, np.zeros((0, 3, 4)), synth.intrinsics(), 64, 48)
    assert m.shape == (0, 48, 64) and s.shape == (0,)
    Fb = F.copy()
    Fb[10, 2] = len(V)
    m, s = utils.render_masks(V, Fb, _poses(2, seed=1, bad=False), synth.intrinsics(), 640, 480)
    assert s.tolist() == [4, 4] and not m.any()


def test_pose_label_rows_match_reference(labels_golden):
    g = labels_golden
    rows = utils.pose_label_rows(g["corners3D"], g["Rt"], g["K"], int(g["width"]), int(g["height"]), int(g["class_id"]))
    np.testing.assert_allclose(rows, g["rows"], rtol=0, atol=1e-6)      # fp32 projections, to within an ulp of the pixel
    px = utils.project_points_batched(np.c_[np.zeros(3), g["corners3D"][:3]], g["Rt"], g["K"]).cpu().numpy()
    assert np.array_equal(rows, utils_host.label_rows_from_projection(px, int(g["width"]), int(g["height"]), int(g["class_id"])))


@pytest.fixture(scope="module")
def labels_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "labels.npz"))


def test_make_dataset_end_to_end(mesh, tmp_path):
    from singleshotpose_b200 import dataset as D, make_dataset
    V, F = mesh
    W, H, n = 640, 480, 6
    root = tmp_path / "custom" / "obj"
    (root / "JPEGImages").mkdir(parents=True)
    paths = []
    for i in range(n):
        img = synth.photo_sample(300 + i, W, H, 8, 8)[0]
        p = str(root / "JPEGImages" / ("%06d.jpg" % i))
        Image.fromarray(img).save(p, quality=95)
        paths.append(p)
    bg = str(tmp_path / "bg.png")
    Image.fromarray(synth.photo_sample(7, 8, 8, 200, 150)[2]).save(bg)
    mesh_path = str(tmp_path / "obj.ply")
    synth.write_ply(mesh_path, V, F)
    Rt = _poses(n, seed=21, bad=False)
    np.savez(str(tmp_path / "poses.npz"), paths=np.array(paths), R=Rt[:, :, :3], t=Rt[:, :, 3])
    test_list = str(tmp_path / "test_images.txt")
    with open(test_list, "w") as f:
        f.write(paths[1] + "\n" + paths[4] + "\n")
    K = synth.intrinsics()
    data = str(tmp_path / "cfg" / "obj.data")
    make_dataset.main(["--mesh", mesh_path, "--poses", str(tmp_path / "poses.npz"), "--fx", str(K[0, 0]), "--fy", str(K[1, 1]),
                       "--u0", str(K[0, 2]), "--v0", str(K[1, 2]), "--name", "obj", "--class-id", "2", "--test-list", test_list,
                       "--data-out", data])
    opts = utils_host.read_data_cfg(data)
    assert float(opts["diam"]) == utils_host.calc_pts_diameter(V)
    assert (int(opts["width"]), int(opts["height"])) == (W, H) and float(opts["fx"]) == K[0, 0] and float(opts["v0"]) == K[1, 2]
    assert utils_host.file_lines(opts["train"]) == 4 and utils_host.file_lines(opts["valid"]) == 2
    # masks: the rendered silhouettes, as 8-bit PNG at the reference's mask paths
    want_masks, st = utils.render_masks(V, F, Rt, K, W, H)
    assert (st == 0).all()
    for i, p in enumerate(paths):
        m = np.asarray(Image.open(D.mask_path(p)))
        assert m.dtype == np.uint8 and m.shape == (H, W) and np.array_equal(m, want_masks[i].cpu().numpy())
    # the test split through the loader: label targets equal pose_label_rows
    rows = utils.pose_label_rows(utils.get_3D_corners(np.c_[V, np.ones(len(V))].T), Rt, K, W, H, 2)
    dt = D.listDataset(opts["valid"], shape=(416, 416), shuffle=False, train=False, num_workers=1)
    data_t, target = D.GpuCollate("cuda")([dt[i] for i in range(len(dt))])
    assert data_t.shape == (2, 3, 416, 416)
    assert torch.equal(target[:, :19], torch.from_numpy(rows[[1, 4], :19]).float())
    # the training split through the augmenting loader (mask compositing onto a background)
    random.seed(3)
    ds = D.listDataset(opts["train"], shape=(416, 416), shuffle=False, train=True, num_workers=1, batch_size=4, bg_file_names=[bg])
    data_tr, target_tr = D.GpuCollate("cuda")([ds[i] for i in range(4)])
    assert data_tr.shape == (4, 3, 416, 416) and torch.isfinite(data_tr).all() and target_tr[:, 0].eq(2).all()
    # PnP on every image's label keypoints recovers its pose
    P3 = np.r_[np.zeros((1, 3)), utils.get_3D_corners(np.c_[V, np.ones(len(V))].T)[:3].T]
    uv = np.stack([utils_host.read_truths_args(D.label_path(p))[1:19].reshape(9, 2) * [W, H] for p in paths])
    R, t = utils.pnp_batched(P3, uv, K)
    R, t = R.cpu().numpy(), t.cpu().numpy()
    for i in range(n):
        ang = np.degrees(np.arccos(np.clip((np.trace(R[i] @ Rt[i, :, :3].T) - 1) / 2, -1, 1)))
        assert ang < 1e-2 and np.abs(t[i] - Rt[i, :, 3]).max() * 1e3 < 1e-2, (i, ang, t[i] - Rt[i, :, 3])
