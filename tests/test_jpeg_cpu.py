"""CPU tests of the JPEG decode rules (singleshotpose_b200/csrc/jpeg_core.h):
  * the rules compiled for the host by tests/helpers/jpeg_host.cpp, driven like the kernels, byte-equal to the installed
    Pillow on the whole matrix of tests/helpers/jpeg_cases.py, with the kernels' subsequence length and with a tiny one that
    forces many candidate links and serial decodes;
  * the same against the committed golden (tests/golden/jpeg.npz, Pillow 12.2 on libjpeg-turbo 3.1), so that another Pillow
    cannot silently move the target;
  * the declines and their reasons; malformed streams under AddressSanitizer / UBSan: every result flagged, declined or
    byte-equal to Pillow;
  * read_jpeg_size, and the argument checks of the C ABI."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from singleshotpose_b200 import _lib
from singleshotpose_b200.jpeg import read_jpeg_size

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "tests", "helpers"))
import jpeg_cases as JC  # noqa: E402

SRC = os.path.join(REPO, "tests", "helpers", "jpeg_host.cpp")
KERNEL_SUB_BITS = 1024       # kSubBits of csrc/jpeg.cu
TINY_SUB_BITS = 24


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("jpeghost") / "libjpeghost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, SRC])
    lib = C.CDLL(so)
    lib.h_parse.argtypes = [C.c_char_p, C.c_longlong, C.c_void_p]
    lib.h_decode.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p]
    lib.h_reason.restype = C.c_char_p
    return lib


@pytest.fixture(scope="module")
def cases():
    return JC.matrix()


def host_decode(host, data, sub_bits):
    info = np.zeros(6, np.int32)
    rc = host.h_parse(data, len(data), info.ctypes.data)
    if rc:
        return -rc, None, None
    out = np.zeros((info[1], info[0], 3), np.uint8)
    stats = np.zeros(2, np.int64)
    st = host.h_decode(data, len(data), sub_bits, out.ctypes.data, stats.ctypes.data)
    return st, out, stats


@pytest.mark.parametrize("sub_bits", [KERNEL_SUB_BITS, TINY_SUB_BITS])
def test_host_decode_matches_pillow_on_matrix(host, cases, sub_bits):
    bad, serial = [], 0
    if sub_bits == TINY_SUB_BITS:               # nearly every subsequence decodes serially: the tiny length on the smaller files only
        cases = [(n, b) for n, b in cases if len(b) < 40000]
    for name, data in cases:
        st, out, stats = host_decode(host, data, sub_bits)
        if st != 0 or not np.array_equal(out, JC.pillow_rgb(data)):
            bad.append((name, st))
        else:
            serial = max(serial, int(stats[0]))
    assert not bad, bad
    assert len(cases) >= 120
    if sub_bits == TINY_SUB_BITS:
        assert serial >= 2                     # the tiny length really exercises the serial part of the walk


def test_matrix_covers_every_sampling_and_restart_option(host, cases):
    seen = set()
    for name, data in cases:
        info = np.zeros(6, np.int32)
        assert host.h_parse(data, len(data), info.ctypes.data) == 0, name
        seen.add((int(info[2]), int(info[3]), int(info[4])))
        if "rst" in name:
            assert info[5] > 0, name
    assert seen == {(1, 1, 1), (3, 1, 1), (3, 2, 1), (3, 2, 2), (3, 1, 2)}


def test_host_decode_matches_golden(host, golden_dir):
    g = np.load(os.path.join(golden_dir, "jpeg.npz"))
    assert str(g["pillow"]).startswith("12.") and str(g["libjpeg_turbo"]).startswith("3.")
    files = np.split(g["files"], g["file_ends"][:-1])
    pix = np.split(g["pixels"], g["pixel_ends"][:-1])
    assert len(files) >= 20
    for data, p, shape in zip(files, pix, g["shapes"]):
        for sub_bits in (KERNEL_SUB_BITS, TINY_SUB_BITS):
            st, out, _ = host_decode(host, data.tobytes(), sub_bits)
            assert st == 0 and np.array_equal(out, p.reshape(shape))


def test_declines_with_reason(host):
    for name, data, reason in JC.declined():
        info = np.zeros(6, np.int32)
        rc = host.h_parse(data, len(data), info.ctypes.data)
        assert rc > 0 and reason in host.h_reason(rc).decode(), (name, rc)
        assert _lib.load().ssp_jpeg_parse(data, len(data), info.ctypes.data) == rc
        assert reason in _lib.load().ssp_jpeg_decline_reason(rc).decode()


def test_read_jpeg_size(cases):
    for name, data in cases[::7]:
        assert read_jpeg_size(data) == JC.pillow_rgb(data).shape[1::-1], name
    assert read_jpeg_size(b"\x89PNG\r\n\x1a\n") is None and read_jpeg_size(b"\xff\xd8") is None


@pytest.fixture(scope="module")
def asan_driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("jpegasan") / "jpeg_asan")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                           "-DJPEG_HOST_MAIN", "-o", exe, SRC])
    return exe


def _run_malformed(asan_driver, tmp_path, blobs, sub_bits):
    paths = []
    for i, b in enumerate(blobs):
        p = str(tmp_path / ("f%05d.jpg" % i))
        with open(p, "wb") as f:
            f.write(b)
        paths.append(p)
    lst = str(tmp_path / "list.txt")
    with open(lst, "w") as f:
        f.write("\n".join(paths) + "\n")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([asan_driver, lst, str(sub_bits)], env=env, capture_output=True, text=True)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-3000:]
    flagged = 0
    for p, b in zip(paths, blobs):
        raw = open(p + ".out", "rb").read()
        st = int(np.frombuffer(raw[:4], np.int32)[0])
        if st != 0:
            flagged += 1
            continue
        try:
            want = JC.pillow_rgb(b)
        except Exception as e:                  # Pillow raises where the GPU path claimed a clean decode
            raise AssertionError("decoded a file Pillow rejects (%s): %s" % (e, p))
        assert np.array_equal(np.frombuffer(raw[4:], np.uint8).reshape(want.shape), want), p
    return flagged


def test_malformed_cut_every_97th_byte_under_sanitizers(asan_driver, tmp_path):
    base = JC.encode(JC.content("scene", 64, 48, 2), "420", 90, "rst_blocks3")
    blobs = [base[:n] for n in range(0, len(base), 97)]
    blobs += [base[:n] + b"\xff\xd9" for n in range(0, len(base) - 2, 97)]      # cut inside the scan, EOI appended
    flagged = _run_malformed(asan_driver, tmp_path, blobs, KERNEL_SUB_BITS)
    assert flagged == len(blobs)


@pytest.mark.parametrize("sub_bits", [KERNEL_SUB_BITS, TINY_SUB_BITS])
def test_malformed_bit_flips_under_sanitizers(asan_driver, tmp_path, sub_bits):
    rng = np.random.default_rng(7)
    blobs = []
    for sampling, option in (("420", "plain"), ("444", "rst_blocks1"), ("gray", "plain"), ("422", "rst_rows1")):
        base = bytearray(JC.encode(JC.content("scene", 48, 40, 5), sampling, 85, option))
        sos = base.index(b"\xff\xda")
        start = sos + 2 + (base[sos + 2] << 8 | base[sos + 3])
        for _ in range(60):
            b = bytearray(base)
            for _ in range(int(rng.integers(1, 4))):
                i = int(rng.integers(start, len(b) - 2))
                b[i] ^= 1 << int(rng.integers(0, 8))
            blobs.append(bytes(b))
    flagged = _run_malformed(asan_driver, tmp_path, blobs, sub_bits)
    assert flagged > 0                           # corrupt streams are caught, not only decoded alike


# ------------------------------------------------------------------------------------------------ the C ABI
def test_jpeg_abi_rejects_bad_arguments(cases):
    lib = _lib.load()
    info = np.zeros(6, np.int32)
    assert lib.ssp_jpeg_parse(None, 10, info.ctypes.data) < 0 and lib.ssp_jpeg_parse(b"\xff\xd8", 2, None) < 0
    assert lib.ssp_jpeg_parse(b"\xff\xd8", -1, info.ctypes.data) < 0
    assert lib.ssp_jpeg_parse(b"GIF89a", 6, info.ctypes.data) > 0

    Item = _lib.STRUCTS["ssp_jpeg_item"]
    good = cases[0][1]
    prog = JC.declined()[0][1]
    items = (Item * 2)(Item(C.cast(C.c_char_p(good), C.c_void_p), len(good), 1), Item(C.cast(C.c_char_p(good), C.c_void_p), len(good), 1))
    assert lib.ssp_jpeg_stage_bytes(items, 2) > 0 and lib.ssp_jpeg_work_bytes(items, 2) > 0
    assert lib.ssp_jpeg_stage_bytes(None, 2) < 0 and lib.ssp_jpeg_work_bytes(items, -1) < 0
    bad = (Item * 1)(Item(C.cast(C.c_char_p(prog), C.c_void_p), len(prog), 1))
    assert lib.ssp_jpeg_stage_bytes(bad, 1) < 0
    stage = np.zeros(int(lib.ssp_jpeg_stage_bytes(items, 2)), np.uint8)
    dims = (C.c_longlong * 4)()
    with pytest.raises(_lib.SspError, match="declines"):
        _lib.call("ssp_jpeg_batch_plan", bad, 1, stage.ctypes.data, stage.size, dims)
    with pytest.raises(_lib.SspError, match="staging buffer"):
        _lib.call("ssp_jpeg_batch_plan", items, 2, stage.ctypes.data, stage.size - 1, dims)
    with pytest.raises(_lib.SspError, match="null output"):
        nul = (Item * 1)(Item(C.cast(C.c_char_p(good), C.c_void_p), len(good), None))
        _lib.call("ssp_jpeg_batch_plan", nul, 1, stage.ctypes.data, stage.size, dims)
    assert _lib.call("ssp_jpeg_batch_plan", items, 2, stage.ctypes.data, stage.size, dims) == 0
    assert 0 < dims[3] <= stage.size
    d = C.c_void_p(1)
    with pytest.raises(_lib.SspError, match="work buffer"):
        _lib.call("ssp_jpeg_batch_run", d, 2, dims, d, dims[2] - 1, d, None)
    with pytest.raises(_lib.SspError, match="bad argument"):
        _lib.call("ssp_jpeg_batch_run", None, 2, dims, d, dims[2], d, None)
    with pytest.raises(_lib.SspError, match="bad argument"):
        _lib.call("ssp_jpeg_batch_run", d, -1, dims, d, dims[2], d, None)
    assert _lib.call("ssp_jpeg_batch_run", d, 0, dims, d, 0, d, None) == 0        # n = 0: no device access
