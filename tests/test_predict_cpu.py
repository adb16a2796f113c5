"""CPU checks of the pose predictor's pieces: the split-K ABI (symbols, argument checks, the split rule), the PLY reader and the
command line's .data parsing.  No device is touched."""
import ctypes as C
import os

import numpy as np
import pytest

from singleshotpose_b200 import _lib
from singleshotpose_b200.cfg import parse_cfg
from singleshotpose_b200.engine import build_plan
from singleshotpose_b200.utils_host import read_ply_vertices

NEW = ("ssp_conv_gemm_splitk", "ssp_conv_splitk_count", "ssp_bn_apply_splitk")
H100_SMS = 132


def test_new_symbols_are_declared_and_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.SIGNATURES
        assert hasattr(lib, name)


def _fake(addr):
    return C.c_void_p(addr)


def _gemm(splits=2, partial=0x10000, slab=None, ld=1024, N=1, H=13, W=13, taps=9, cin=1024, cout=1024):
    lib = _lib.load()
    rows = _lib.flat_alloc_rows(N, H, W)
    slab = rows * ld if slab is None else slab
    a, b = _fake(0x20000), _fake(0x40000)
    return lib.ssp_conv_gemm_splitk(a, a, rows, cin, cin, b, b, cout, taps * cin, N, H, W, taps, cout, splits,
                                    _fake(partial) if partial else None, slab, ld, None)


def test_conv_gemm_splitk_argument_checks():
    assert _gemm(splits=0) == -1
    assert _gemm(splits=-3) == -1
    assert _gemm(splits=9 * 16 + 1) == -1                 # more splits than k-blocks (9 taps x 16)
    assert _gemm(partial=0) == -1                         # no workspace
    assert _gemm(partial=0x10004) == -1                   # not 16-B aligned
    assert _gemm(ld=1022) == -1                           # partial_ld % 4
    assert _gemm(ld=512) == -1                            # partial_ld < cout
    rows = _lib.flat_alloc_rows(1, 13, 13)
    assert _gemm(slab=rows * 1024 - 4) == -1              # a slab smaller than rows x ld: workspace under splits x that
    assert _gemm(slab=rows * 1024 + 2) == -1              # slabs must keep 16-B alignment
    assert _gemm(splits=2, taps=3) == -1                  # taps must be 1 or 9


def _bn(splits=2, partial=0x10000, slab=None, ld=1024, C_=1024, N=1, H=13, W=13):
    lib = _lib.load()
    slab = _lib.flat_alloc_rows(N, H, W) * ld if slab is None else slab
    d = _fake(0x80000)
    return lib.ssp_bn_apply_splitk(_fake(partial) if partial else None, splits, slab, ld, _fake(0x1000), _fake(0x2000), N, C_, H, W,
                                   C.c_float(0.1), d, d, ld, 0, _lib.ROUTE_DIRECT, None, None, 0, 0, _lib.ROUTE_NONE, None)


def test_bn_apply_splitk_argument_checks():
    assert _bn(splits=0) == -1
    assert _bn(partial=0) == -1
    assert _bn(partial=0x10008) == -1
    assert _bn(ld=1022) == -1
    assert _bn(ld=1020, C_=1024) == -1
    rows = _lib.flat_alloc_rows(1, 13, 13)
    assert _bn(slab=rows * 1024 - 4) == -1
    assert _bn(C_=1022, ld=1024) == -1                    # channels in groups of 4


def _layers(cfg_path):
    return build_plan(parse_cfg(cfg_path))


def _rule(N, h, w, L):
    """the split rule restated from the tile geometry: 128-row tiles of N(h+1)(w+1) rows x N tiles of 32 / 64 / 128 channels"""
    bn = 128 if L.cout > 64 else (L.cout + 31) // 32 * 32
    tiles = -(-N * (h + 1) * (w + 1) // 128) * -(-L.cout // bn)
    kb = L.taps * -(-L.cin // 64)
    s = min(H100_SMS // tiles, kb // 8)
    return s if s >= 2 else 1


@pytest.mark.parametrize("size", [416, 672])
@pytest.mark.parametrize("N", [1, 8, 64])
def test_splitk_count_of_gemm_layers_follows_the_tile_table(cfg_path, N, size):
    lib = _lib.load()
    got = {}
    for L in _layers(cfg_path)[1:]:                       # the GEMM layers (layer 0 is the fused unit of blocks 0-1)
        h, w = L.H * size // 416, L.W * size // 416
        s = lib.ssp_conv_splitk_count(N, h, w, L.taps, L.cin, L.cout, H100_SMS)
        assert s == _rule(N, h, w, L), (L.block_ind, N, size)
        got[L.block_ind] = s
    if N == 64:
        assert set(got.values()) == {1}                   # a full batch fills the machine: no layer is split
    if (N, size) == (1, 416):
        # 13x13 3x3 layers: 16 tiles, 72 / 144 / 180 k-blocks -> min(132 // 16, kb // 8) = 8
        for blk in (18, 20, 22, 23, 24, 29):
            assert got[blk] == 8, blk
        assert got[19] == got[21] == 2                    # 13x13 1x1: 8 tiles, 16 k-blocks
        assert got[12] == got[14] == got[16] == 4         # 26x26 3x3: 24 tiles, 36 k-blocks
        assert got[8] == got[10] == 2                     # 52x52 3x3: 44 tiles
    if (N, size) == (1, 672):
        for blk in (18, 23, 29):
            assert got[blk] == 4                          # 21x21: 32 tiles


def test_splitk_count_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.ssp_conv_splitk_count(0, 13, 13, 9, 512, 1024, 132) == -1
    assert lib.ssp_conv_splitk_count(1, 13, 13, 4, 512, 1024, 132) == -1
    assert lib.ssp_conv_splitk_count(1, 13, 13, 9, 512, 1024, 0) == -1


def _write_ply(path, V, faces=((0, 1, 2),), extra_elem=False, fmt="ascii"):
    with open(path, "w") as f:
        f.write("ply\nformat %s 1.0\ncomment written by a test\n" % fmt)
        if extra_elem:
            f.write("element camera 1\nproperty float view_px\nproperty float view_py\n")
        f.write("element vertex %d\nproperty float x\nproperty float y\nproperty float z\nproperty float nx\nproperty uchar red\n" % len(V))
        f.write("element face %d\nproperty list uchar int vertex_indices\nend_header\n" % len(faces))
        if extra_elem:
            f.write("0.5 0.25\n")
        for v in V:
            f.write("%r %r %r 0.0 255\n" % tuple(float(x) for x in v))
        for fc in faces:
            f.write("%d %s\n" % (len(fc), " ".join(map(str, fc))))


@pytest.mark.parametrize("extra_elem", [False, True])
def test_read_ply_vertices_matches_numpy(tmp_path, extra_elem):
    V = np.random.default_rng(0).normal(size=(57, 3)) * 0.05
    p = str(tmp_path / "m.ply")
    _write_ply(p, V, extra_elem=extra_elem)
    got = read_ply_vertices(p)
    assert got.shape == (57, 3) and got.dtype == np.float64
    assert np.array_equal(got, V)


def test_read_ply_vertices_refuses_binary(tmp_path):
    p = str(tmp_path / "b.ply")
    with open(p, "wb") as f:
        f.write(b"ply\nformat binary_little_endian 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\nend_header\n")
        f.write(np.zeros(3, dtype="<f4").tobytes())
    with pytest.raises(ValueError, match="ASCII"):
        read_ply_vertices(p)
    q = str(tmp_path / "n.ply")
    with open(q, "w") as f:
        f.write("not a ply\n")
    with pytest.raises(ValueError):
        read_ply_vertices(q)


def test_cli_data_cfg_parsing(tmp_path):
    from singleshotpose_b200.predict import SIZE_KEYS, main, read_camera
    p = tmp_path / "ape.data"
    p.write_text("train  = LINEMOD/ape/train.txt\nmesh = LINEMOD/ape/ape.ply\nname = ape\ndiam = 0.103\nwidth = 640\nheight = 480\n"
                 "fx = 572.4114 \nfy = 573.5704\nu0 = 325.2611\nv0 = 242.0489\n")
    mesh, K, size = read_camera(str(p), SIZE_KEYS)
    assert mesh == "LINEMOD/ape/ape.ply" and size == (640, 480)
    assert np.array_equal(K, np.array([[572.4114, 0, 325.2611], [0, 573.5704, 242.0489], [0, 0, 1]]))
    q = tmp_path / "bad.data"
    q.write_text("mesh = m.ply\nwidth = 640\n")
    with pytest.raises(_lib.SspError, match="height|fx"):
        read_camera(str(q), SIZE_KEYS)
    with pytest.raises(SystemExit):
        main(["--datacfg", str(p)])                       # model cfg, weights and images are required
