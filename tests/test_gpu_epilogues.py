"""The BatchNorm routing epilogues, the fused inference epilogue and the head GEMMs at the network's own geometries, against an
exact host emulation of their arithmetic and against fp64.

test_gpu_kernels.py covers each kernel on one destination at channel offset 0.  The network also writes two destinations at once
(layer 16: max-pooled into block 17 and directly into the route of block 25), places maps inside the 1280-channel concat plane
(block 26 reorganised at channel 0, block 24 at channel 256), reads fp16 gradient planes wider than the layer and runs the
multi-object head (1024 -> 160 channels).  Here every such path is checked on its own:

* ssp_bn_apply and ssp_conv_gemm_bnact bit for bit against a numpy emulation of fmaf + LeakyReLU + the saturating fp16 hi/lo
  split, with exact ties planted in the 2x2 pooling windows and every element outside the written region prefilled with a
  sentinel bit pattern that must survive;
* the fused epilogue byte for byte against ssp_conv_gemm(EPI_F32) + ssp_bn_apply (the same MMAs, the same epilogue arithmetic);
* the two-source BN backward against fp64 autograd, including the engine's quarter-resolution reduction of a pooled layer;
* the head's forward, data- and weight-gradient GEMMs and its bias gradient against fp64."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from singleshotpose_b200 import _lib
from singleshotpose_b200._lib import call, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"
DIRECT, POOL, REORG, F16 = _lib.ROUTE_DIRECT, _lib.ROUTE_POOL, _lib.ROUTE_REORG, _lib.ROUTE_F16
SENT16 = 0x7E5A              # an fp16 NaN no kernel writes: marks the 16-bit elements a kernel must leave alone
SENT32 = 0x7FC0DEAD          # the same for fp32 planes
EPS = 1e-4
# input size -> (layer-16 map, head grid): 416^2, 352x480, 608^2, 320^2
GEOMS = {"416": ((26, 26), (13, 13)), "352x480": ((22, 30), (11, 15)), "608": ((38, 38), (19, 19)), "320": ((20, 20), (10, 10))}


# ------------------------------------------------------------------------------------------------ layout helpers
def rows_of(N, H, W):
    return _lib.flat_alloc_rows(N, H, W)


def flat_index(N, H, W):
    """padded-flat row of every (n, h, w), in that order"""
    n, h, w = np.meshgrid(np.arange(N), np.arange(H), np.arange(W), indexing="ij")
    return (n * (H + 1) * (W + 1) + (h + 1) * (W + 1) + (w + 1)).reshape(-1)


def sentinel16(rows, ld):
    return torch.full((rows, ld), SENT16, dtype=torch.int16, device=DEV)


def sentinel32(rows, ld):
    return torch.full((rows, ld), SENT32, dtype=torch.int32, device=DEV)


def bits16(t):
    return t.cpu().numpy().view(np.uint16)


def flat_f32(y, ld=None):
    """NHWC fp32 numpy -> padded-flat fp32 device plane (zero pads)"""
    N, H, W, C = y.shape
    out = torch.zeros(rows_of(N, H, W), ld or C, device=DEV)
    out[torch.from_numpy(flat_index(N, H, W)).to(DEV), :C] = torch.from_numpy(np.ascontiguousarray(y.reshape(-1, C))).to(DEV)
    return out


def pack_nchw(x, ld=None, c0=0, split=True):
    """NCHW fp32 torch -> padded-flat fp16 planes through ssp_pack_nchw (hi/lo when split, else one rounded plane)"""
    N, C, H, W = x.shape
    rows = rows_of(N, H, W)
    hi = torch.zeros(rows, ld or C, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi) if split else None
    xd = x.to(DEV).contiguous()
    call("ssp_pack_nchw", ptr(xd), ptr(hi), ptr(lo), N, C, H, W, ld or C, c0, _lib.FMT_F16, 1.0, stream_ptr())
    return hi, lo, rows


def pack_weights(w, dgrad=False):
    """OIHW fp32 torch -> forward planes hi / lo [co][taps*ci] and, with dgrad, the tap-flipped transposed plane [ci][taps*co]"""
    co, ci, kh, kw = w.shape
    taps = kh * kw
    master = w.permute(0, 2, 3, 1).contiguous().to(DEV)
    ldf, ldd = (taps * ci + 7) // 8 * 8, (taps * co + 7) // 8 * 8
    hi = torch.zeros(co, ldf, dtype=torch.float16, device=DEV); lo = torch.zeros_like(hi)
    d = torch.zeros(ci, ldd, dtype=torch.float16, device=DEV) if dgrad else None
    call("ssp_pack_weights", ptr(master), co, taps, ci, ptr(hi), ptr(lo), ldf, ptr(d), ldd if dgrad else 0, _lib.FMT_F16, stream_ptr())
    return hi, lo, d


# ------------------------------------------------------------------------------------------------ exact host emulation
F32 = np.float32


def fmaf(a, b, c):
    """fp32 fused multiply-add, correctly rounded: the fp64 product of two fp32 values is exact, the fp64 sum keeps its rounding
    error (two-sum); rounding that sum to fp32 is correct except where it sits exactly halfway between two fp32 values while the
    exact sum does not -- then the error's sign picks the side"""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - p
    e = (p - (s - bp)) + (c - bp)
    r = s.astype(F32)
    d = s - r.astype(np.float64)
    nb = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))
    halfway = (d != 0) & (2 * d == nb.astype(np.float64) - r.astype(np.float64))
    return np.where(halfway & (e != 0) & ((e > 0) == (d > 0)), nb, r).astype(F32)


def leaky(z, slope):
    z = np.asarray(z, F32)
    return np.where(z > 0, z, z * F32(slope)).astype(F32)


def split(z, saturate=True):
    """fp16 hi / lo bit patterns of the device's split_f16 (saturate=False: the split before saturation was added)"""
    z = np.asarray(z, F32)
    lim = F32(65504)
    with np.errstate(over="ignore", invalid="ignore"):         # the unsaturated split overflows to +-inf and NaN by design
        hi = (np.clip(z, -lim, lim) if saturate else z).astype(np.float16)
        r = (z - hi.astype(F32)).astype(F32)
        lo = (np.clip(r, -lim, lim) if saturate else r).astype(np.float16)
    return hi.view(np.uint16), lo.view(np.uint16)


def windows(a):
    """(N, H, W, C) -> (N, H/2, W/2, 4, C), the 2x2 window of every pooled cell in (h, w) scan order"""
    N, H, W, C = a.shape
    return a.reshape(N, H // 2, 2, W // 2, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, H // 2, W // 2, 4, C)


def reorg(a):
    """Reorg(2) in marvis order (darknet.py:31-34): channel ((h % 2) * 2 + w % 2) * C + c of the half-resolution map"""
    N, H, W, C = a.shape
    return windows(a).reshape(N, H // 2, W // 2, 4 * C)


def first_max(z):
    """arg-max of every window, the first maximum in scan order winning (+0 and -0 tie)"""
    return np.argmax(windows(z), axis=3)


def emulate_apply(y, sc, sh, slope, dests):
    """expected bit patterns of ssp_bn_apply / ssp_conv_gemm_bnact: {dest index: (hi plane, lo plane)} with sentinels outside the
    written region, and the expected arg-max plane values"""
    N, H, W, C = y.shape
    z = leaky(fmaf(y, sc, sh), slope)
    best = first_max(z) if any(r == POOL for r, _, _ in dests) else None
    out = []
    for route, ld, c0 in dests:
        if route == DIRECT:
            g, v = (N, H, W), z
        elif route == POOL:
            g, v = (N, H // 2, W // 2), np.take_along_axis(windows(z), best[:, :, :, None, :], axis=3)[:, :, :, 0, :]
        else:
            g, v = (N, H // 2, W // 2), reorg(z)
        planes = []
        for part in split(v.reshape(-1, v.shape[-1])):
            p = np.full((rows_of(*g), ld), SENT16, np.uint16)
            p[flat_index(*g), c0:c0 + v.shape[-1]] = part
            planes.append(p)
        out.append(planes)
    ysel = None if best is None else np.take_along_axis(windows(y), best[:, :, :, None, :], axis=3)[:, :, :, 0, :]
    return out, ysel


# ------------------------------------------------------------------------------------------------ test data
def bn_affine(rng, C):
    """per-channel scale / shift of a folded BatchNorm: a third of the scales negative, some shifts exactly +0 or -0"""
    sc = (rng.uniform(0.2, 2.0, C) * np.where(np.arange(C) % 3 == 1, -1, 1)).astype(F32)
    sh = (rng.standard_normal(C) * 0.5).astype(F32)
    sh[np.arange(C) % 8 == 3] = 0.0
    sh[np.arange(C) % 8 == 5] = -0.0
    return sc, sh


def conv_output(rng, N, H, W, C, sign, zero_channels=()):
    """random conv output with exact ties planted in the 2x2 windows (H, W even).  sign[c] = the sign of channel c's BN scale,
    which decides where the activated maximum of a window lies: a tenth of the windows are four equal values (equal positives
    or, under the leaky slope, equal negatives), a fifth get a copy of their maximum at another position.  In zero_channels a
    tenth of the windows hold -0 and +0 above two values that activate below zero."""
    y = (rng.standard_normal((N, H, W, C)) * 1.7 + 0.3).astype(F32)
    if H % 2 or W % 2:
        return y
    w = windows(y).copy()                                           # (N, h, w, 4, C)
    pick = rng.random(w.shape[:3] + (C,))
    eq = pick < 0.1
    for q in range(1, 4):
        w[:, :, :, q, :][eq] = w[:, :, :, 0, :][eq]
    cp = (pick >= 0.1) & (pick < 0.3)
    src = np.argmax(w * sign.astype(F32), axis=3)                   # position of the activated maximum (monotone in y * sign)
    dst = (src + rng.integers(1, 4, src.shape)) % 4
    n, hh, ww, c = np.nonzero(cp)
    w[n, hh, ww, dst[cp], c] = w[n, hh, ww, src[cp], c]
    for c in zero_channels:
        m = rng.random(w.shape[:3]) < 0.1
        first = rng.random(w.shape[:3]) < 0.5
        # two zeros of opposite sign, in either order, then two values whose activation is negative
        w[m, 0, c] = np.where(first[m], -0.0, 0.0)
        w[m, 1, c] = np.where(first[m], 0.0, -0.0)
        w[m, 2, c] = -sign[c] * (1.0 + rng.random(m.sum()))
        w[m, 3, c] = -sign[c] * (1.0 + rng.random(m.sum()))
    N_, h, ww_, _, _ = w.shape
    return np.ascontiguousarray(w.reshape(N_, h, ww_, 2, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, H, W, C))


def count_ties_at_max(z):
    """windows whose activated maximum is reached more than once"""
    zw = windows(z)
    return int(((zw == zw.max(axis=3, keepdims=True)).sum(axis=3) > 1).sum())


# ------------------------------------------------------------------------------------------------ ssp_bn_finalize(train=0)
@pytest.mark.parametrize("C", [64, 160, 1000, 1024])
def test_bn_finalize_eval_matches_fp64(C):
    rng = np.random.default_rng(C)
    gamma = torch.from_numpy((rng.standard_normal(C) * 1.5).astype(F32)).to(DEV)
    beta = torch.from_numpy(rng.standard_normal(C).astype(F32)).to(DEV)
    rm = torch.from_numpy((rng.standard_normal(C) * 3).astype(F32)).to(DEV)
    rv = torch.from_numpy(np.exp(rng.uniform(-12, 4, C)).astype(F32)).to(DEV)     # down to 6e-6: eps matters
    rm0, rv0 = rm.clone(), rv.clone()
    mean, invstd, scale, shift = (torch.full((C,), float("nan"), device=DEV) for _ in range(4))
    call("ssp_bn_finalize", None, None, 1.0, ptr(gamma), ptr(beta), ptr(rm), ptr(rv), 0.1, EPS, 0,
         ptr(mean), ptr(invstd), ptr(scale), ptr(shift), C, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(rm.view(torch.int32), rm0.view(torch.int32)) and torch.equal(rv.view(torch.int32), rv0.view(torch.int32))
    g, b, m, v = (t.cpu().double() for t in (gamma, beta, rm0, rv0))
    inv64 = 1.0 / torch.sqrt(v + float(F32(EPS)))
    assert torch.equal(mean.cpu().double(), m)
    assert ((invstd.cpu().double() - inv64).abs() / inv64).max() < 1e-6
    sc64 = g * inv64
    assert ((scale.cpu().double() - sc64).abs() / sc64.abs()).max() < 1e-6
    sh64 = b - m * sc64
    assert ((shift.cpu().double() - sh64).abs() / (b.abs() + (m * sc64).abs())).max() < 1e-6


# ------------------------------------------------------------------------------------------------ ssp_bn_apply
# (name, N, H, W, C, y_ld, destinations [(route, ld, c0)], arg-max plane)
APPLY_CASES = [
    ("direct C64", 1, 26, 26, 64, 64, [(DIRECT, 64, 0)], False),
    ("direct C256 offset", 3, 22, 30, 256, 260, [(DIRECT, 264, 4)], False),
    ("direct C1024", 3, 10, 10, 1024, 1024, [(DIRECT, 1024, 0)], False),
    ("pool C512", 3, 26, 26, 512, 512, [(POOL, 512, 0)], True),
    ("pool C256 608", 1, 38, 38, 256, 256, [(POOL, 264, 8)], False),
    ("reorg C64", 3, 26, 26, 64, 64, [(REORG, 256, 0)], False),
    ("layer16 pool+direct", 3, 26, 26, 512, 512, [(POOL, 512, 0), (DIRECT, 512, 0)], True),
    ("layer16 direct+pool 352x480", 1, 22, 30, 512, 512, [(DIRECT, 516, 4), (POOL, 520, 8)], True),
    ("layer16 pool+direct 608", 3, 38, 38, 512, 512, [(POOL, 512, 0), (DIRECT, 512, 0)], True),
    ("layer16 direct+pool 320", 1, 20, 20, 512, 512, [(DIRECT, 512, 0), (POOL, 512, 0)], True),
    ("block26 reorg into concat", 3, 26, 26, 64, 64, [(REORG, 1280, 0)], False),
    ("block26 reorg into concat 352x480", 1, 22, 30, 64, 64, [(REORG, 1280, 0)], False),
    ("block24 direct into concat", 3, 13, 13, 1024, 1024, [(DIRECT, 1280, 256)], False),
    ("block24 direct into concat 608", 1, 19, 19, 1024, 1024, [(DIRECT, 1280, 256)], False),
]


@pytest.mark.parametrize("case", APPLY_CASES, ids=[c[0] for c in APPLY_CASES])
def test_bn_apply_bit_exact(case):
    _name, N, H, W, C, y_ld, dests, with_ypool = case
    rng = np.random.default_rng(zlib.crc32(case[0].encode()))
    sc, sh = bn_affine(rng, C)
    y = conv_output(rng, N, H, W, C, np.sign(sc), zero_channels=np.nonzero(sh == 0)[0][:8])
    want, ysel = emulate_apply(y, sc, sh, 0.1, dests)
    if any(r == POOL for r, _, _ in dests):
        assert count_ties_at_max(leaky(fmaf(y, sc, sh), 0.1)) > N * (H // 2) * (W // 2) * C // 10     # the tie rule is exercised
    yf = flat_f32(y, y_ld)
    scd, shd = torch.from_numpy(sc).to(DEV), torch.from_numpy(sh).to(DEV)
    planes, args = [], []
    for route, ld, c0 in dests:
        geo = (N, H, W) if route == DIRECT else (N, H // 2, W // 2)
        hi, lo = sentinel16(rows_of(*geo), ld), sentinel16(rows_of(*geo), ld)
        planes.append((hi, lo))
        args += [ptr(hi), ptr(lo), ld, c0, route]
    args += [None, None, 0, 0, 0] * (2 - len(dests))
    yp_ld = C + 4
    ypool = sentinel32(rows_of(N, H // 2, W // 2), yp_ld) if with_ypool else None
    call("ssp_bn_apply", ptr(yf), y_ld, ptr(scd), ptr(shd), N, C, H, W, 0.1, *args, ptr(ypool), yp_ld if with_ypool else 0, stream_ptr())
    torch.cuda.synchronize()
    for (hi, lo), (whi, wlo) in zip(planes, want):
        assert np.array_equal(bits16(hi), whi) and np.array_equal(bits16(lo), wlo)
    if with_ypool:
        wy = np.full((rows_of(N, H // 2, W // 2), yp_ld), SENT32, np.uint32)
        wy[flat_index(N, H // 2, W // 2), :C] = ysel.reshape(-1, C).view(np.uint32)
        assert np.array_equal(ypool.cpu().numpy().view(np.uint32), wy)


# ------------------------------------------------------------------------------------------------ ssp_conv_gemm_bnact
# (name, N, H, W, cin, cout, k, split operands, d_ld, d_c0)
BNACT_CASES = [
    ("block24 into concat", 3, 13, 13, 1024, 1024, 3, True, 1280, 256),
    ("block24 into concat single-term 608", 1, 19, 19, 1024, 1024, 3, False, 1280, 256),
    ("block28 cin1280", 1, 13, 13, 1280, 1024, 3, True, 1024, 0),
    ("block28 cin1280 single-term 352x480", 3, 11, 15, 1280, 1024, 3, False, 1032, 8),
    ("1x1 64 (N tile 64)", 3, 26, 26, 512, 64, 1, True, 64, 0),
    ("1x1 64 single-term 320", 1, 20, 20, 512, 64, 1, False, 72, 8),
    ("1x1 128", 1, 22, 30, 256, 128, 1, True, 136, 8),
    ("3x3 256", 3, 11, 15, 512, 256, 3, True, 256, 0),
    ("3x3 256 single-term", 1, 26, 26, 256, 256, 3, False, 264, 8),
]


@pytest.mark.parametrize("case", BNACT_CASES, ids=[c[0] for c in BNACT_CASES])
def test_conv_gemm_bnact(case):
    _name, N, H, W, cin, cout, k, nt3, d_ld, d_c0 = case
    taps = k * k
    g = torch.Generator().manual_seed(zlib.crc32(case[0].encode()))
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * taps) ** 0.5
    gamma = (torch.rand(cout, generator=g) + 0.5) * torch.where(torch.arange(cout) % 3 == 1, -1.0, 1.0)
    beta, rm = torch.randn(cout, generator=g) * 0.5, torch.randn(cout, generator=g) * 0.3
    rv = torch.rand(cout, generator=g) + 0.5
    xh, xl, rows = pack_nchw(x, split=nt3)
    wh, wl, _ = pack_weights(w)
    if not nt3:
        wl = None
    bn = [t.to(DEV) for t in (gamma, beta, rm, rv)]
    scale, shift, mean, invstd = (torch.zeros(cout, device=DEV) for _ in range(4))
    call("ssp_bn_finalize", None, None, 1.0, *map(ptr, bn), 0.1, EPS, 0, ptr(mean), ptr(invstd), ptr(scale), ptr(shift), cout, stream_ptr())
    a = [ptr(xh), ptr(xl), rows, cin, cin, ptr(wh), ptr(wl), cout, wh.shape[1]]
    impl = _lib.IMPL_TC2 if cout >= 128 else _lib.IMPL_TC
    fh, fl = sentinel16(rows, d_ld), sentinel16(rows, d_ld)
    call("ssp_conv_gemm_bnact", impl, *a, N, H, W, taps, cout, ptr(scale), ptr(shift), 0.1, ptr(fh), ptr(fl), d_ld, d_c0, stream_ptr())
    # the unfused chain: the same kernel's fp32 output, then ssp_bn_apply on the same scale / shift
    y = torch.zeros(rows, cout, device=DEV)
    call("ssp_conv_gemm", _lib.IMPL_TC, *a, _lib.FMT_F16, _lib.FMT_F16, N, H, W, taps, cout, ptr(y), cout, rows, _lib.EPI_F32, None, None, None,
         stream_ptr())
    uh, ul = sentinel16(rows, d_ld), sentinel16(rows, d_ld)
    call("ssp_bn_apply", ptr(y), cout, ptr(scale), ptr(shift), N, cout, H, W, 0.1, ptr(uh), ptr(ul), d_ld, d_c0, DIRECT,
         None, None, 0, 0, 0, None, 0, stream_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(bits16(fh), bits16(uh)) and np.array_equal(bits16(fl), bits16(ul))
    # the host emulation of the epilogue on the kernel's own accumulators (sentinels outside the valid rows and [d_c0, d_c0 + cout))
    idx = flat_index(N, H, W)
    yv = y.cpu().numpy()[idx].reshape(N, H, W, cout)
    (whi, wlo), = emulate_apply(yv, scale.cpu().numpy(), shift.cpu().numpy(), 0.1, [(DIRECT, d_ld, d_c0)])[0]
    assert np.array_equal(bits16(fh), whi) and np.array_equal(bits16(fl), wlo)
    # against fp64: conv -> BN(running statistics) -> leaky, the error of the conv scaled by each channel's |scale|
    xr, wr = (x, w) if nt3 else (x.half().float(), w.half().float())
    conv = F.conv2d(xr.double().to(DEV), wr.double().to(DEV), padding=(k - 1) // 2).cpu()
    sc64 = gamma.double() / torch.sqrt(rv.double() + float(F32(EPS)))
    z64 = F.leaky_relu(conv * sc64[None, :, None, None] + (beta.double() - rm.double() * sc64)[None, :, None, None], 0.1)
    got = (fh.view(torch.float16).float() + fl.view(torch.float16).float()).cpu()[torch.from_numpy(idx)][:, d_c0:d_c0 + cout]
    got = got.reshape(N, H, W, cout).permute(0, 3, 1, 2).double()
    err = ((got - z64).abs() / sc64.abs()[None, :, None, None]).max() / conv.abs().max()
    assert err < 2e-5 + 5e-9 * cin * taps, float(err)


# ------------------------------------------------------------------------------------------------ two-source BN backward
BWD_COMBOS = [(DIRECT, 0), (POOL, 0), (REORG, 0), (POOL, DIRECT), (DIRECT, POOL), (DIRECT, DIRECT), (DIRECT, REORG), (REORG, DIRECT)]
BWD_GEOMS = [("416", 3, 64), ("352x480", 1, 512), ("608", 1, 64), ("320", 3, 256)]


def _torch_windows(a):
    N, H, W, C = a.shape
    return a.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H // 2, W // 2, 4, C)


@pytest.mark.parametrize("geo", BWD_GEOMS, ids=[g[0] for g in BWD_GEOMS])
@pytest.mark.parametrize("combo", BWD_COMBOS, ids=["%d-%d" % c for c in BWD_COMBOS])
def test_bn_backward_two_sources(combo, geo):
    (H, W), _ = GEOMS[geo[0]]
    N, C = geo[1], geo[2]
    rng = np.random.default_rng(17 * combo[0] + 5 * combo[1] + H + C)
    gamma = (rng.uniform(0.5, 1.5, C) * np.where(np.arange(C) % 3 == 1, -1, 1)).astype(F32)
    beta = (rng.standard_normal(C) * 0.5).astype(F32)
    y = conv_output(rng, N, H, W, C, np.sign(gamma))
    # batch statistics in fp64 (the conv epilogue's sums in the network), folded on the device
    y64 = y.astype(np.float64)
    ssum = torch.from_numpy(y64.sum(axis=(0, 1, 2))).to(DEV); ssq = torch.from_numpy((y64 ** 2).sum(axis=(0, 1, 2))).to(DEV)
    gm, bt = torch.from_numpy(gamma).to(DEV), torch.from_numpy(beta).to(DEV)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    mean, invstd, scale, shift = (torch.zeros(C, device=DEV) for _ in range(4))
    call("ssp_bn_finalize", ptr(ssum), ptr(ssq), float(N * H * W), ptr(gm), ptr(bt), ptr(rm), ptr(rv), 0.1, EPS, 1,
         ptr(mean), ptr(invstd), ptr(scale), ptr(shift), C, stream_ptr())
    sc, sh = scale.cpu().numpy(), shift.cpu().numpy()
    pre = fmaf(y, sc, sh)                                  # the kernels' pre-activation: leaky' and the pooled arg-max follow it
    pooled = POOL in combo
    best = first_max(leaky(pre, 0.1)) if pooled else None
    if pooled:
        assert count_ties_at_max(leaky(pre, 0.1)) > N * (H // 2) * (W // 2) * C // 10
    # upstream gradients: fp16 planes wider than the layer at a channel offset, random everywhere (pads and other channels too)
    srcs, args, grads = [], [], []
    for s, route in enumerate(combo):
        if not route:
            args += [None, 0, 0, 0]
            continue
        geo_g = (N, H, W) if route == DIRECT else (N, H // 2, W // 2)
        width = 4 * C if route == REORG else C
        c0 = 256 if s == 0 else 8
        ld = c0 + width + 8
        plane = torch.randn(rows_of(*geo_g), ld, generator=torch.Generator(device=DEV).manual_seed(s), device=DEV).half()
        srcs.append(plane)
        args += [ptr(plane), ld, c0, route | F16]
        grads.append((route, plane.float().cpu().numpy()[flat_index(*geo_g), c0:c0 + width].reshape(*geo_g, width)))
    yf = flat_f32(y)
    head = [ptr(yf), C, ptr(scale), ptr(shift), ptr(mean), ptr(invstd), ptr(gm), N, C, H, W, 0.1]
    s1 = torch.zeros(C, dtype=torch.float64, device=DEV); s2 = torch.zeros_like(s1)
    call("ssp_bn_bwd_reduce", *head, *args, ptr(s1), ptr(s2), stream_ptr())
    if pooled:
        # the engine's decomposition: the pooled source reduced at a quarter of the resolution from the arg-max plane of the
        # forward, every other source at full resolution on its own
        hp = sentinel16(rows_of(N, H // 2, W // 2), C); lp = sentinel16(rows_of(N, H // 2, W // 2), C)
        ypool = sentinel32(rows_of(N, H // 2, W // 2), C)
        call("ssp_bn_apply", ptr(yf), C, ptr(scale), ptr(shift), N, C, H, W, 0.1, ptr(hp), ptr(lp), C, 0, POOL, None, None, 0, 0, 0,
             ptr(ypool), C, stream_ptr())
        ysel = np.take_along_axis(windows(y), best[:, :, :, None, :], axis=3)[:, :, :, 0, :]
        torch.cuda.synchronize()
        assert np.array_equal(ypool.cpu().numpy()[flat_index(N, H // 2, W // 2)].view(np.uint32), ysel.reshape(-1, C).view(np.uint32))
        t1 = torch.zeros_like(s1); t2 = torch.zeros_like(s2)
        for s, route in enumerate(combo):
            if not route:
                continue
            ptr_, ld, c0, _ = args[4 * s:4 * s + 4]
            if route == POOL:
                call("ssp_bn_bwd_reduce", ptr(ypool), C, *head[2:7], N, C, H // 2, W // 2, 0.1, ptr_, ld, c0, DIRECT | F16, None, 0, 0, 0,
                     ptr(t1), ptr(t2), stream_ptr())
            else:
                call("ssp_bn_bwd_reduce", *head, ptr_, ld, c0, route | F16, None, 0, 0, 0, ptr(t1), ptr(t2), stream_ptr())
        torch.cuda.synchronize()
        for t, s in ((t1, s1), (t2, s2)):
            assert torch.allclose(t, s, rtol=1e-6, atol=1e-6 * float(s.abs().max()))
    dy_ld = C + 4
    dy = sentinel16(rows_of(N, H, W), dy_ld)
    call("ssp_bn_bwd_apply", *head, *args, ptr(s1), ptr(s2), ptr(dy), dy_ld, _lib.FMT_F16, 1.0, stream_ptr())
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    call("ssp_bn_bwd_finalize", ptr(s1), ptr(s2), ptr(dg), ptr(db), C, 0, 1.0, stream_ptr())
    torch.cuda.synchronize()
    # fp64 autograd of BN(train) + leaky + the consumers, with leaky' and the pooled arg-max taken from the fp32 pre-activation
    yt = torch.from_numpy(y64).requires_grad_(True)
    gt = torch.from_numpy(gamma.astype(np.float64)).requires_grad_(True)
    btt = torch.from_numpy(beta.astype(np.float64)).requires_grad_(True)
    mu, var = yt.mean(dim=(0, 1, 2)), yt.var(dim=(0, 1, 2), unbiased=False)
    zp = (yt - mu) / torch.sqrt(var + EPS) * gt + btt
    act = torch.where(torch.from_numpy(pre > 0), zp, zp * 0.1)
    loss = 0
    for route, gv in grads:
        gv = torch.from_numpy(gv.astype(np.float64))
        if route == DIRECT:
            loss = loss + (act * gv).sum()
        elif route == POOL:
            sel = torch.gather(_torch_windows(act), 3, torch.from_numpy(best)[:, :, :, None, :]).squeeze(3)
            loss = loss + (sel * gv).sum()
        else:
            loss = loss + (_torch_windows(act).reshape(gv.shape) * gv).sum()
    loss.backward()
    assert torch.allclose(dg.cpu().double(), gt.grad, rtol=1e-4, atol=1e-4 * float(gt.grad.abs().max()))
    assert torch.allclose(db.cpu().double(), btt.grad, rtol=1e-4, atol=1e-4 * float(btt.grad.abs().max()))
    dyb = bits16(dy)
    idx = flat_index(N, H, W)
    got = dyb[idx][:, :C].view(np.float16).astype(np.float64).reshape(N, H, W, C)
    want = yt.grad.numpy()
    assert np.abs(got - want).max() < 2e-3 * np.abs(want).max()                        # fp16 storage of dY
    outside = np.ones(dyb.shape, bool); outside[idx, :C] = False
    assert (dyb[outside] == SENT16).all()


# ------------------------------------------------------------------------------------------------ head GEMMs
HEADS = [("416", 3), ("352x480", 1), ("608", 3)]


@pytest.mark.parametrize("geo", HEADS, ids=[h[0] for h in HEADS])
def test_head_forward_1024_to_160(geo):
    """the multi-object head: 1x1 1024 -> 160 with bias on SSP_IMPL_TC2 (one 128-channel and one 32-channel N tile)"""
    _, (H, W) = GEOMS[geo[0]]
    N, cin, cout, ld = geo[1], 1024, 160, 168
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
    b = torch.randn(cout, generator=g)
    xh, xl, rows = pack_nchw(x)
    wh, wl, _ = pack_weights(w)
    bd = b.to(DEV)
    out = sentinel32(rows, ld)
    call("ssp_conv_gemm", _lib.IMPL_TC2, ptr(xh), ptr(xl), rows, cin, cin, ptr(wh), ptr(wl), cout, wh.shape[1], _lib.FMT_F16, _lib.FMT_F16,
         N, H, W, 1, cout, ptr(out), ld, rows, _lib.EPI_BIAS, ptr(bd), None, None, stream_ptr())
    torch.cuda.synchronize()
    o = out.cpu()
    assert (o[:, cout:] == SENT32).all()
    got = o.view(torch.float32)[torch.from_numpy(flat_index(N, H, W))][:, :cout].reshape(N, H, W, cout).permute(0, 3, 1, 2).double()
    ref = F.conv2d(x.double(), w.double(), b.double())
    assert ((got - ref).abs().max() / ref.abs().max()) < 2e-5 + 5e-9 * cin


@pytest.mark.parametrize("geo", HEADS, ids=[h[0] for h in HEADS])
@pytest.mark.parametrize("cy,ld_y", [(20, 24), (160, 160)])
def test_head_data_gradient_into_1024(geo, cy, ld_y):
    """dX of the head (K = 20 single-object, 160 multi-object) into a 1024-channel fp16 plane on SSP_IMPL_TC2"""
    _, (H, W) = GEOMS[geo[0]]
    N, cx, ld16 = geo[1], 1024, 1032
    g = torch.Generator().manual_seed(cy + H)
    dy = torch.randn(N, cy, H, W, generator=g)
    w = torch.randn(cy, cx, 1, 1, generator=g) / cy ** 0.5
    dyh, _, rows = pack_nchw(dy, ld=ld_y, split=False)
    _, _, wd = pack_weights(w, dgrad=True)
    d16, d32 = sentinel16(rows, ld16), torch.zeros(rows, cx, device=DEV)
    for out, ld, epi in ((d16, ld16, _lib.EPI_F16), (d32, cx, _lib.EPI_F32)):
        call("ssp_conv_gemm", _lib.IMPL_TC2, ptr(dyh), None, rows, ld_y, cy, ptr(wd), None, cx, wd.shape[1], _lib.FMT_F16, _lib.FMT_F16,
             N, H, W, 1, cx, ptr(out), ld, rows, epi, None, None, None, stream_ptr())
    torch.cuda.synchronize()
    idx = flat_index(N, H, W)
    b16 = bits16(d16)
    assert (b16[:, cx:] == SENT16).all()
    assert np.array_equal(b16[idx][:, :cx], d32.cpu().numpy()[idx].astype(np.float16).view(np.uint16))
    got = torch.from_numpy(b16[idx][:, :cx].view(np.float16).astype(np.float64)).reshape(N, H, W, cx).permute(0, 3, 1, 2)
    ref = F.conv_transpose2d(dy.half().double(), w.half().double())
    assert (got - ref).abs().max() / ref.abs().max() < 1e-3


@pytest.mark.parametrize("geo", HEADS, ids=[h[0] for h in HEADS])
def test_head_weight_gradient_160x1024(geo):
    _, (H, W) = GEOMS[geo[0]]
    N, cy, cx = geo[1] + 1, 160, 1024
    g = torch.Generator().manual_seed(7 * H)
    x = torch.randn(N, cx, H, W, generator=g)
    dy = torch.randn(N, cy, H, W, generator=g)
    xh, _, rows = pack_nchw(x, split=False)
    dyh, _, _ = pack_nchw(dy, split=False)
    outs = []
    for _ in range(2):
        dw = torch.zeros(cy, cx, device=DEV)
        call("ssp_wgrad_gemm", _lib.IMPL_TC2, ptr(dyh), rows, cy, cy, _lib.FMT_F16, ptr(xh), rows, cx, cx, _lib.FMT_F16,
             N, H, W, 1, ptr(dw), cx, cx, 1.0, stream_ptr())
        outs.append(dw)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    ref = torch.nn.grad.conv2d_weight(x.half().double(), (cy, cx, 1, 1), dy.half().double())[:, :, 0, 0]
    assert (outs[0].cpu().double() - ref).abs().max() / ref.abs().max() < 1e-4


@pytest.mark.parametrize("N,C,HW", [(64, 20, 19 * 19), (64, 160, 19 * 19), (3, 160, 13 * 13), (1, 20, 11 * 15)])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_bias_grad_nchw(N, C, HW, accumulate):
    g = torch.Generator().manual_seed(N + C + accumulate)
    x = torch.randn(N, C, HW, generator=g) * 300.0
    db0 = torch.randn(C, generator=g)
    xd, db = x.to(DEV), db0.to(DEV)
    call("ssp_bias_grad_nchw", ptr(xd), ptr(db), N, C, HW, accumulate, 1.0 / 256, stream_ptr())
    torch.cuda.synchronize()
    v = x.double().sum(dim=(0, 2)) / 256
    ref = v + (db0.double() if accumulate else 0.0)
    tol = 1e-6 * (v.abs() + (db0.double().abs() if accumulate else 0.0))
    assert ((db.cpu().double() - ref).abs() <= tol).all()


# ------------------------------------------------------------------------------------------------ fp16 range edges
EDGES = np.array([65503, -65503, 65504, -65504, 65519, -65519, 65520, -65520, 70000, -70000, 131008, -131008, 1e6, -1e6,
                  1e-6, 6e-8, -0.0, 0.5], F32)


def _check_split_planes(hi, lo, z):
    """device planes (uint16) of the values z: finite, the saturating split, and the unsaturated split below 65520"""
    whi, wlo = split(z)
    assert np.array_equal(hi, whi) and np.array_equal(lo, wlo)
    assert np.isfinite(hi.view(np.float16)).all() and np.isfinite(lo.view(np.float16)).all()
    small = np.abs(z) < 65520
    ohi, olo = split(z, saturate=False)
    assert np.array_equal(hi[small], ohi[small]) and np.array_equal(lo[small], olo[small])


def test_fp16_range_edges_pack():
    C = 24
    x = np.resize(EDGES, (1, C, 2, 2)).astype(F32)
    x[0, :, 1, 1] *= F32(-0.75)
    hi, lo, _ = pack_nchw(torch.from_numpy(x))
    idx = flat_index(1, 2, 2)
    z = x.transpose(0, 2, 3, 1).reshape(-1, C)
    _check_split_planes(bits16(hi)[idx], bits16(lo)[idx], z)
    # NaN stays NaN, infinities saturate
    xs = torch.tensor([float("nan"), float("inf"), -float("inf"), 1.0]).view(1, 4, 1, 1)
    hi, lo, _ = pack_nchw(xs)
    r = int(flat_index(1, 1, 1)[0])
    h, l_ = hi.float().cpu()[r], lo.float().cpu()[r]
    assert torch.isnan(h[0]) and h[1] == 65504 and l_[1] == 65504 and h[2] == -65504 and l_[2] == -65504 and h[3] == 1 and l_[3] == 0


@pytest.mark.parametrize("slope", [0.1, 1.0])
def test_fp16_range_edges_bn_apply(slope):
    C = 32
    y = np.resize(EDGES, (1, 4, 4, C)).astype(F32)
    y[0, 2:] = y[0, 2:] / F32(3.0)
    sc = np.resize(np.array([1.0, 2.0, -1.0, 0.5], F32), C)
    sh = np.resize(np.array([0.0, -0.0, 3.0, -1.0], F32), C)
    want, _ = emulate_apply(y, sc, sh, slope, [(DIRECT, C, 0)])
    hi, lo = sentinel16(rows_of(1, 4, 4), C), sentinel16(rows_of(1, 4, 4), C)
    yf = flat_f32(y)
    scd, shd = torch.from_numpy(sc).to(DEV), torch.from_numpy(sh).to(DEV)
    call("ssp_bn_apply", ptr(yf), C, ptr(scd), ptr(shd), 1, C, 4, 4, slope, ptr(hi), ptr(lo), C, 0, DIRECT, None, None, 0, 0, 0, None, 0,
         stream_ptr())
    torch.cuda.synchronize()
    idx = flat_index(1, 4, 4)
    assert np.array_equal(bits16(hi), want[0][0]) and np.array_equal(bits16(lo), want[0][1])
    _check_split_planes(bits16(hi)[idx], bits16(lo)[idx], leaky(fmaf(y, sc, sh), slope).reshape(-1, C))


@pytest.mark.parametrize("nt3", [True, False])
def test_fp16_range_edges_conv_gemm_bnact(nt3):
    """conv = 1 exactly (one-hot input and weights), BN scale = the edge value: the fused epilogue's z is the value itself"""
    N, H, W, cin, cout = 1, 5, 6, 64, 32
    x = torch.zeros(N, cin, H, W); x[:, 0] = 1.0
    w = torch.zeros(cout, cin, 1, 1); w[:, 0] = 1.0
    vals = np.resize(EDGES, cout).astype(F32)
    scale = torch.from_numpy(vals).to(DEV)
    shift = torch.from_numpy(np.where(vals == 0, F32(-0.0), F32(0.0)).astype(F32)).to(DEV)        # fmaf(1, -0, -0) = -0
    xh, xl, rows = pack_nchw(x, split=nt3)
    wh, wl, _ = pack_weights(w)
    hi, lo = sentinel16(rows, cout), sentinel16(rows, cout)
    call("ssp_conv_gemm_bnact", _lib.IMPL_TC, ptr(xh), ptr(xl), rows, cin, cin, ptr(wh), ptr(wl) if nt3 else None, cout, wh.shape[1],
         N, H, W, 1, cout, ptr(scale), ptr(shift), 0.1, ptr(hi), ptr(lo), cout, 0, stream_ptr())
    torch.cuda.synchronize()
    y = np.ones((N, H, W, cout), F32)
    want, _ = emulate_apply(y, scale.cpu().numpy(), shift.cpu().numpy(), 0.1, [(DIRECT, cout, 0)])
    assert np.array_equal(bits16(hi), want[0][0]) and np.array_equal(bits16(lo), want[0][1])
    idx = flat_index(N, H, W)
    _check_split_planes(bits16(hi)[idx], bits16(lo)[idx], leaky(fmaf(y, scale.cpu().numpy(), shift.cpu().numpy()), 0.1).reshape(-1, cout))


# ------------------------------------------------------------------------------------------------ NaN and saturation, single-term fp16
# The backward's fp16 planes are stored by one conversion each (no hi/lo): the data-gradient epilogue SSP_EPI_F16 of the per-tap and
# the operand-swapped kernels, ssp_pack_nchw without a lo plane (the loss gradient), the dY store of ssp_bn_bwd_apply and the W_d
# planes of ssp_pack_weights and ssp_sgd_pack_step.  Each must give fp16(clamp(x, +-65504)) bit for bit and keep NaN a NaN.
NAN_EDGES = np.array([np.nan, np.inf, -np.inf, 65519, -65519, 65520, -65520, 1e6, -1e6, 65504, -65504, 65503, -0.0, 1.5, 6e-8,
                      -131008], F32)


def _check_f16_sat(got_bits, x):
    """device fp16 bits against numpy fp16(clip(x, +-65504)): NaN must come back as a NaN, everything else bit for bit"""
    x = np.asarray(x, F32)
    want = np.clip(x, F32(-65504), F32(65504)).astype(np.float16).view(np.uint16)
    got = np.asarray(got_bits, np.uint16)
    nan = np.isnan(x)
    assert np.isnan(got[nan].view(np.float16)).all(), "NaN did not survive the fp16 conversion: %s" % got[nan].view(np.float16)
    assert np.array_equal(got[~nan], want[~nan]), (x[~nan][got[~nan] != want[~nan]], got[~nan][got[~nan] != want[~nan]].view(np.float16))


def _fp16_parts(v, k):
    """k fp16 values whose exact sum is v (v a NaN / an infinity: that value, then zeros); the partial sums are integers or
    short dyadic values well inside fp32, so a tensor-core fp32 accumulation of them is exact in any order"""
    parts = np.zeros(k, np.float64)
    if not np.isfinite(v):
        parts[0] = v
        return parts
    r = float(v)
    for i in range(k):
        parts[i] = float(np.float16(np.clip(r, -65504, 65504)))
        r -= parts[i]
    assert r == 0.0, v
    return parts


@pytest.mark.parametrize("impl", [_lib.IMPL_TC2, _lib.IMPL_BANDT])
@pytest.mark.parametrize("tail_rows", [False, True])
def test_fp16_nan_and_saturation_data_gradient_epilogue(impl, tail_rows):
    """SSP_EPI_F16: dX[m][c] = sum_k dY[m][k] * W_d[c][k] with dY = 1 and W_d[c] the fp16 parts of an edge value.  48 channels: the
    per-tap kernel's packed 32-channel store and its channel tail; tail_rows: an output row count that ends inside the operand-swapped
    kernel's last 32-row chunk (its per-row tail store)"""
    N, H, W, K, cout = 2, 5, 7, 64, 48
    vals = np.resize(NAN_EDGES[(NAN_EDGES != 0) & (NAN_EDGES != F32(6e-8))], cout).astype(F32)   # -0 is not a sum of products, 6e-8 not one of fp16 values
    wd = torch.from_numpy(np.stack([_fp16_parts(v, K) for v in vals])).half().to(DEV)
    dy, _, rows = pack_nchw(torch.ones(N, K, H, W), split=False)
    out_rows = N * (H + 1) * (W + 1) + 5 if tail_rows else rows
    ld = (cout + 7) // 8 * 8
    dx = sentinel16(rows, ld)
    call("ssp_conv_gemm", impl, ptr(dy), None, rows, K, K, ptr(wd), None, cout, K, _lib.FMT_F16, _lib.FMT_F16,
         N, H, W, 1, cout, ptr(dx), ld, out_rows, _lib.EPI_F16, None, None, None, stream_ptr())
    torch.cuda.synchronize()
    idx = flat_index(N, H, W)
    got = bits16(dx)[idx, :cout]
    _check_f16_sat(got, np.broadcast_to(vals, got.shape))


def test_fp16_nan_and_saturation_pack_single_term():
    """ssp_pack_nchw with lo = NULL (the engine packs the loss gradient this way), loss scale 1 and 256"""
    C = NAN_EDGES.size
    x = np.ascontiguousarray(np.stack([NAN_EDGES, NAN_EDGES[::-1]]).T.reshape(1, C, 2, 1).astype(F32))
    for scale in (1.0, 256.0):
        hi = sentinel16(rows_of(1, 2, 1), C)
        xd = torch.from_numpy(x).to(DEV)
        call("ssp_pack_nchw", ptr(xd), ptr(hi), None, 1, C, 2, 1, C, 0, _lib.FMT_F16, scale, stream_ptr())
        torch.cuda.synchronize()
        got = bits16(hi)[flat_index(1, 2, 1)]
        _check_f16_sat(got, x.transpose(0, 2, 3, 1).reshape(-1, C) * F32(scale))


def test_fp16_nan_and_saturation_bn_backward_dy():
    """ssp_bn_bwd_apply's dY store: y = 1, scale 1, shift 0 (z > 0: leaky' = 1), mean 0, invstd 1, gamma 1 and zero sums, so
    dY = 1 * ((g + 0) - 0 - 1 * 0) = g + 0 (the second, absent source adds +0: -0 becomes +0)"""
    N, H, W, C = 1, 2, 3, NAN_EDGES.size
    g = np.resize(NAN_EDGES, (N, H, W, C)).astype(F32)
    g[0, 1] = g[0, 1, :, ::-1]
    yf, gf = flat_f32(np.ones((N, H, W, C), F32)), flat_f32(g)
    one, zero = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
    s1 = torch.zeros(C, dtype=torch.float64, device=DEV); s2 = torch.zeros_like(s1)
    dy = sentinel16(rows_of(N, H, W), C)
    call("ssp_bn_bwd_apply", ptr(yf), C, ptr(one), ptr(zero), ptr(zero), ptr(one), ptr(one), N, C, H, W, 0.1,
         ptr(gf), C, 0, DIRECT, None, 0, 0, _lib.ROUTE_NONE, ptr(s1), ptr(s2), ptr(dy), C, _lib.FMT_F16, 1.0, stream_ptr())
    torch.cuda.synchronize()
    got = bits16(dy)[flat_index(N, H, W)]
    _check_f16_sat(got, g.reshape(-1, C) + F32(0))


def test_fp16_nan_and_saturation_weight_planes():
    """the W_d plane [cin][taps*cout] of ssp_pack_weights and of the fused SGD + re-pack pass (vector path: cin % 4 == 0; scalar
    path: cin = 3), with a zero step (lr = momentum = weight decay = 0): p stays p except where 0 * p is a NaN (p = +-inf)"""
    for cout, taps, cin in [(16, 1, 64), (16, 9, 3)]:
        n = cout * taps * cin
        w = np.random.default_rng(cin).permutation(np.resize(NAN_EDGES, n)).reshape(cout, taps, cin).astype(F32)
        ld_f, ld_d = (taps * cin + 7) // 8 * 8, (taps * cout + 7) // 8 * 8
        d_want = lambda m: m.transpose(2, 1, 0)[:, ::-1, :].reshape(cin, taps * cout)       # k = (taps-1-tap)*cout + co
        master = torch.from_numpy(w).to(DEV)
        fh = torch.zeros(cout, ld_f, dtype=torch.float16, device=DEV); fl = torch.zeros_like(fh)
        d = sentinel16(cin, ld_d)
        call("ssp_pack_weights", ptr(master), cout, taps, cin, ptr(fh), ptr(fl), ld_f, ptr(d), ld_d, _lib.FMT_F16, stream_ptr())
        torch.cuda.synchronize()
        _check_f16_sat(bits16(d)[:, :taps * cout], d_want(w))
        # the same plane from ssp_sgd_pack_step
        tab = np.zeros(1, dtype=np.dtype(_lib.STRUCTS["ssp_sgd_segment"]))
        e = tab[0]
        d2 = sentinel16(cin, ld_d)
        e["off"], e["n"], e["cout"], e["taps"], e["cin"], e["ld_f"], e["ld_d"], e["d_fmt"] = 0, n, cout, taps, cin, ld_f, ld_d, _lib.FMT_F16
        e["f_hi"], e["f_lo"], e["d"], e["block0"] = fh.data_ptr(), fl.data_ptr(), d2.data_ptr(), 0
        nb = int(_lib.load().ssp_sgd_segment_blocks(cout, taps, cin, n))
        table = torch.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(DEV)
        p = master.clone().reshape(-1); gz = torch.zeros_like(p); v = torch.zeros_like(p)
        call("ssp_sgd_pack_step", ptr(table), 1, 0, nb, ptr(p), ptr(gz), ptr(v), 0.0, 0.0, 0.0, 1.0, stream_ptr())
        torch.cuda.synchronize()
        pw = p.cpu().numpy().reshape(cout, taps, cin)
        assert np.isnan(pw[np.isinf(w)]).all() and np.array_equal(pw[np.isfinite(w)].view(np.uint32), w[np.isfinite(w)].view(np.uint32))
        _check_f16_sat(bits16(d2)[:, :taps * cout], d_want(pw))


def test_nan_in_loss_gradient_reaches_head_weight_gradient(cfg_path):
    """end to end: one NaN element in the gradient of the logits must give NaN in the head's weight gradient (as autograd would)
    for the output channel it belongs to, and leave the other channels finite -- not a finite gradient of arbitrary sign"""
    from singleshotpose_b200 import Darknet, synth
    torch.manual_seed(0)
    m = Darknet(cfg_path).cuda().train()
    out = m(synth.images(2, 128, 128, seed=3).cuda())
    g = torch.zeros_like(out)
    g[1, 0, 2, 3] = float("nan")
    out.backward(g)
    head = m._engine.conv_modules()[-1][0]
    dw = head.weight.grad                                           # (20, 1024, 1, 1)
    assert torch.isnan(dw[0]).all(), "a NaN logit gradient gave a finite weight gradient: %s" % dw[0].flatten()[:4].tolist()
    assert torch.isfinite(dw[1:]).all()
