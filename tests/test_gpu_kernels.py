"""GPU parity of the individual kernels, called through the C ABI (ctypes), against plain torch fp32 references
of the same op computed on the CPU, and tensor-core kernels against their CUDA-core twins."""
import os

import pytest
import torch
import torch.nn.functional as F

from singleshotpose_b200 import _lib
from singleshotpose_b200._lib import call, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"


def flat_from_nchw(x, ld=None, c0=0, fmt=None, split=True):
    """NCHW fp32 (cuda) -> padded-flat planes via the pack kernel."""
    N, C, H, W = x.shape
    ld = ld or C
    rows = _lib.flat_alloc_rows(N, H, W)
    dt = torch.float16 if fmt in (None, _lib.FMT_F16) else torch.bfloat16
    hi = torch.zeros(rows, ld, dtype=dt, device=DEV)
    lo = torch.zeros(rows, ld, dtype=dt, device=DEV) if split else None
    call("ssp_pack_nchw", ptr(x.contiguous()), ptr(hi), ptr(lo), N, C, H, W, ld, c0, _lib.FMT_F16 if fmt is None else fmt, 1.0, stream_ptr())
    return hi, lo, rows


def nchw_from_flat(y, N, C, H, W, c0=0):
    out = torch.empty(N, C, H, W, dtype=torch.float32, device=DEV)
    call("ssp_unpack_nchw", ptr(y), ptr(out), N, C, H, W, y.shape[1], c0, stream_ptr())
    return out


def torch_flat_index(N, H, W):
    n, h, w = torch.meshgrid(torch.arange(N), torch.arange(H), torch.arange(W), indexing="ij")
    return (n * (H + 1) * (W + 1) + (h + 1) * (W + 1) + (w + 1)).reshape(-1)


def test_pack_layout_matches_definition():
    N, C, H, W = 2, 8, 5, 7
    x = torch.randn(N, C, H, W, device=DEV)
    hi, lo, rows = flat_from_nchw(x)
    v = (hi.float() + lo.float()).cpu()
    idx = torch_flat_index(N, H, W)
    ref = x.permute(0, 2, 3, 1).reshape(-1, C).cpu()
    assert (v[idx] - ref).abs().max() < 1e-6 * ref.abs().max() + 1e-7           # hi+lo carries ~22 bits
    mask = torch.ones(rows, dtype=torch.bool); mask[idx] = False
    assert v[mask].abs().max() == 0                                             # pads untouched (zero)
    back = nchw_from_flat(v.to(DEV).contiguous(), N, C, H, W)
    assert torch.equal(back.cpu(), v[idx].reshape(N, H, W, C).permute(0, 3, 1, 2))


def _pack_w(w, split=True, fmt=_lib.FMT_F16, dgrad=False):
    """w: OIHW fp32 cuda -> forward operand planes [co][taps*ci] (+ dgrad plane [ci][taps*co])."""
    co, ci, kh, kw = w.shape
    taps = kh * kw
    master = w.permute(0, 2, 3, 1).contiguous()                # [co][kh][kw][ci]
    ldf = (taps * ci + 7) // 8 * 8
    hi = torch.zeros(co, ldf, dtype=torch.float16, device=DEV)
    lo = torch.zeros(co, ldf, dtype=torch.float16, device=DEV)
    dt = torch.float16 if fmt == _lib.FMT_F16 else torch.bfloat16
    ldd = (taps * co + 7) // 8 * 8
    d = torch.zeros(ci, ldd, dtype=dt, device=DEV) if dgrad else None
    call("ssp_pack_weights", ptr(master), co, taps, ci, ptr(hi), ptr(lo), ldf, ptr(d), ldd, fmt, stream_ptr())
    return hi, (lo if split else None), d


CONV_CASES = [
    # N, H, W, cin, cout, k, bias
    (2, 12, 12, 64, 64, 3, False),
    (2, 40, 24, 32, 64, 3, False),           # block-2 shape class: band loads + resident weights
    (1, 13, 13, 128, 256, 3, False),
    (3, 5, 7, 64, 32, 3, False),
    (2, 26, 26, 256, 128, 1, False),
    (2, 13, 13, 1024, 20, 1, True),
    (1, 13, 13, 1280, 512, 3, False),
    (2, 13, 13, 1024, 160, 1, True),         # multi-object head: 160 channels, two N tiles of the per-tap kernel
]


def _operands(x, w, terms):
    """x (NCHW), w (OIHW) fp32 on the CPU -> padded-flat planes, weight planes and the fp64 reference operands of a forward with
    `terms` products: 3 = split fp16 (x_hi + x_lo, w_hi + w_lo; the reference takes the unrounded values), 1 = single term (no lo
    planes; the reference takes the fp16-rounded values, whose products are exact in the fp32 accumulator)"""
    xh, xl, rows = flat_from_nchw(x.to(DEV), split=terms == 3)
    wh, wl, _ = _pack_w(w.to(DEV), split=terms == 3)
    if terms == 1:
        x, w = x.half(), w.half()
    return xh, xl, rows, wh, wl, x.double(), w.double()


@pytest.mark.parametrize("case", [c + (3,) for c in CONV_CASES] + [c + (1,) for c in CONV_CASES])      # last field: operand terms
@pytest.mark.parametrize("impl", [_lib.IMPL_SIMT, _lib.IMPL_TC, _lib.IMPL_TC2, _lib.IMPL_BAND, _lib.IMPL_BANDT])
def test_conv_gemm_matches_torch(case, impl):
    N, H, W, cin, cout, k, use_bias, terms = case
    g = torch.Generator().manual_seed(hash(case[:7]) % 1000)
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) if use_bias else None
    xh, xl, rows, wh, wl, x64, w64 = _operands(x, w, terms)
    ref = F.conv2d(x64, w64, None if b is None else b.double(), padding=(k - 1) // 2).float()
    ldo = (cout + 3) // 4 * 4
    y = torch.zeros(rows, ldo, device=DEV)
    ssum = torch.zeros(cout, dtype=torch.float64, device=DEV); ssq = torch.zeros_like(ssum)
    epi = _lib.EPI_BIAS if use_bias else _lib.EPI_STATS
    bias = b.to(DEV) if use_bias else None
    call("ssp_conv_gemm", impl, ptr(xh), ptr(xl), rows, cin, cin, ptr(wh), ptr(wl), cout, wh.shape[1], 0, 0,
         N, H, W, k * k, cout, ptr(y), ldo, rows, epi, ptr(bias), ptr(ssum), ptr(ssq), stream_ptr())
    torch.cuda.synchronize()
    out = nchw_from_flat(y, N, cout, H, W).cpu()
    scale = ref.abs().max()
    # the tensor core's fp32 accumulation is ~10x less exact than FFMA and grows with K (measured: 5e-6 @ K=1152,
    # 3.6e-5 @ K=11520; independent of operand scale, i.e. not the fp16 lo parts) -- tolerance scales with K
    tol = 2e-5 + 5e-9 * cin * k * k
    assert (out - ref).abs().max() / scale < tol, (out - ref).abs().max() / scale
    if not use_bias:
        s_ref = ref.double().sum(dim=(0, 2, 3)); q_ref = (ref.double() ** 2).sum(dim=(0, 2, 3))
        assert (ssum.cpu() - s_ref).abs().max() < 1e-4 * q_ref.max().sqrt() * (N * H * W) ** 0.5
        assert ((ssq.cpu() - q_ref).abs() / q_ref).max() < 1e-4


def test_conv_gemm_single_term_bf16_dgrad_layout():
    """dX = conv_transpose(dY, W): the forward kernel with the tap-flipped / transposed weight plane."""
    N, H, W, cin, cout = 2, 13, 13, 128, 64
    g = torch.Generator().manual_seed(5)
    dy = torch.randn(N, cout, H, W, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
    dyq = dy.bfloat16().float(); wq = w.bfloat16().float()
    ref = F.conv_transpose2d(dyq.double(), wq.double(), padding=1).float()
    for impl in (_lib.IMPL_SIMT, _lib.IMPL_TC, _lib.IMPL_TC2, _lib.IMPL_BAND, _lib.IMPL_BANDT):
        dyh, _, rows = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_BF16, split=False)
        _, _, wd = _pack_w(w.to(DEV), fmt=_lib.FMT_BF16, dgrad=True)
        dx = torch.zeros(rows, cin, device=DEV)
        call("ssp_conv_gemm", impl, ptr(dyh), None, rows, cout, cout, ptr(wd), None, cin, wd.shape[1], 1, 1,
             N, H, W, 9, cin, ptr(dx), cin, rows, _lib.EPI_F32, None, None, None, stream_ptr())
        torch.cuda.synchronize()
        out = nchw_from_flat(dx, N, cin, H, W).cpu()
        assert (out - ref).abs().max() / ref.abs().max() < 1e-4, impl


WGRAD_CASES = [(2, 12, 12, 64, 64, 3), (1, 13, 13, 256, 128, 3), (2, 26, 26, 128, 64, 1), (2, 13, 13, 1024, 20, 1), (3, 5, 7, 64, 256, 3),
               (2, 20, 12, 32, 64, 3),      # cin 32: N tile 64 with a zero-filled upper half (block 2)
               (2, 13, 13, 128, 256, 3),    # cin 128: one N tile, two co tiles
               (1, 30, 22, 64, 128, 3)]     # cin 64 (blocks 3 / 5)


@pytest.mark.parametrize("case", WGRAD_CASES)
@pytest.mark.parametrize("impl", [_lib.IMPL_SIMT, _lib.IMPL_TC])
@pytest.mark.parametrize("dyfmt", [_lib.FMT_BF16, _lib.FMT_F16])      # both operands share the format (mixing is illegal)
def test_wgrad_gemm_matches_torch(case, impl, dyfmt):
    N, H, W, cin, cout, k = case
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, cin, H, W, generator=g)
    dy = torch.randn(N, cout, H, W, generator=g)
    xq = (x.bfloat16() if dyfmt == _lib.FMT_BF16 else x.half()).float()
    dyq = (dy.bfloat16() if dyfmt == _lib.FMT_BF16 else dy.half()).float()
    ref = torch.nn.grad.conv2d_weight(xq.double(), (cout, cin, k, k), dyq.double(), padding=(k - 1) // 2).float()
    xh, _, rows = flat_from_nchw(x.to(DEV), fmt=dyfmt, split=False)
    ld_dy = (cout + 7) // 8 * 8
    dyh, _, _ = flat_from_nchw(dy.to(DEV), ld=ld_dy, fmt=dyfmt, split=False)
    dw = torch.zeros(cout, k * k, cin, device=DEV)
    call("ssp_wgrad_gemm", impl, ptr(dyh), rows, ld_dy, cout, dyfmt, ptr(xh), rows, cin, cin, dyfmt,
         N, H, W, k * k, ptr(dw), cin, cin, 1.0, stream_ptr())
    torch.cuda.synchronize()
    out = dw.view(cout, k, k, cin).permute(0, 3, 1, 2).cpu()
    assert (out - ref).abs().max() / ref.abs().max() < 1e-4


# fp16 storage bound of the single-term backward GEMMs against the UNQUANTISED fp64 result: each operand is rounded once to fp16
# (relative 2^-12 rms, 2^-11 worst), so every product carries ~2^-11.5 rms relative error and the errors of a K-term sum of
# random-sign terms add in quadrature: ||d||_2 / ||ref||_2 ~ 3.5e-4 independent of K.  Asserted with a 3x margin in L2 and, since
# the largest element of a random-sign sum stands ~4 sigma above the rms error, 8e-3 in max-norm (relative to the largest element).
FP16_BWD_L2, FP16_BWD_MAX = 1.1e-3, 8e-3


@pytest.mark.parametrize("case", [(2, 13, 13, 256, 128, 3), (2, 26, 26, 128, 64, 1), (1, 13, 13, 1024, 512, 3)])
def test_wgrad_vs_unquantised_fp64(case):
    """weight gradient from fp16-stored dY and X against the fp64 gradient of the UNROUNDED operands (VERDICT r1 weak 6: the other
    wgrad tests round the reference's operands first and so cannot see the quantisation error)"""
    N, H, W, cin, cout, k = case
    g = torch.Generator().manual_seed(21)
    x = torch.randn(N, cin, H, W, generator=g)
    dy = torch.randn(N, cout, H, W, generator=g)
    ref = torch.nn.grad.conv2d_weight(x.double(), (cout, cin, k, k), dy.double(), padding=(k - 1) // 2)
    xh, _, rows = flat_from_nchw(x.to(DEV), fmt=_lib.FMT_F16, split=False)
    dyh, _, _ = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_F16, split=False)
    dw = torch.zeros(cout, k * k, cin, device=DEV)
    call("ssp_wgrad_gemm", _lib.IMPL_TC, ptr(dyh), rows, cout, cout, _lib.FMT_F16, ptr(xh), rows, cin, cin, _lib.FMT_F16,
         N, H, W, k * k, ptr(dw), cin, cin, 1.0, stream_ptr())
    torch.cuda.synchronize()
    out = dw.view(cout, k, k, cin).permute(0, 3, 1, 2).cpu().double()
    l2, mx = float((out - ref).norm() / ref.norm()), float((out - ref).abs().max() / ref.abs().max())
    assert l2 < FP16_BWD_L2 and mx < FP16_BWD_MAX, (l2, mx)
    assert l2 > 5e-5              # the test does see quantisation (an fp32-exact path would sit at ~1e-7)


@pytest.mark.parametrize("case", [(2, 13, 13, 256, 128, 3), (2, 26, 26, 128, 64, 1), (1, 13, 13, 512, 1024, 3)])
def test_dgrad_vs_unquantised_fp64(case):
    """data gradient from fp16-stored dY and fp16 tap-flipped weights against the fp64 conv_transpose of the UNROUNDED operands"""
    N, H, W, cin, cout, k = case
    g = torch.Generator().manual_seed(22)
    dy = torch.randn(N, cout, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    ref = F.conv_transpose2d(dy.double(), w.double(), padding=(k - 1) // 2)
    dyh, _, rows = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_F16, split=False)
    _, _, wd = _pack_w(w.to(DEV), fmt=_lib.FMT_F16, dgrad=True)
    impl = _lib.IMPL_TC2 if cin >= 128 else _lib.IMPL_TC
    dx = torch.zeros(rows, cin, device=DEV)
    call("ssp_conv_gemm", impl, ptr(dyh), None, rows, cout, cout, ptr(wd), None, cin, wd.shape[1], 0, 0,
         N, H, W, k * k, cin, ptr(dx), cin, rows, _lib.EPI_F32, None, None, None, stream_ptr())
    torch.cuda.synchronize()
    out = nchw_from_flat(dx, N, cin, H, W).cpu().double()
    l2, mx = float((out - ref).norm() / ref.norm()), float((out - ref).abs().max() / ref.abs().max())
    assert l2 < FP16_BWD_L2 and mx < FP16_BWD_MAX, (l2, mx)
    assert l2 > 5e-5


# long-K shapes whose K range the weight-gradient kernel splits over a thread-block cluster (csrc/wgrad_tc.cu: the split doubles while
# tiles x split < 132 SMs and every split keeps >= 32 k-blocks of 64 pixel rows); the comment gives the split on a 132-SM H100
WGRAD_SPLIT_CASES = [(24, 13, 13, 512, 256, 3),    # 72 tiles -> split 2
                     (64, 13, 13, 128, 128, 3),    # 9 tiles, 196 k-blocks -> split 4
                     (64, 26, 26, 64, 64, 1),      # 1 tile, 729 k-blocks -> split 8
                     (64, 26, 26, 32, 64, 3),      # cin 32 (N tile 64, zero-filled upper half), cout 64 (one M half) -> split 8
                     (64, 13, 13, 256, 256, 3)]    # 36 tiles -> split 4, two 128-channel co tiles


@pytest.mark.parametrize("case", WGRAD_SPLIT_CASES)
def test_wgrad_cluster_split_matches_torch(case):
    """weight gradient whose K range is split over the CTAs of a cluster and reduced through distributed shared memory: equal to
    torch's fp64 gradient of the same fp16 operands, the same bits on a second launch (fixed reduction order, no atomics), and the
    same bits through SSP_IMPL_TC2 (which selects this kernel on sm_90a)"""
    N, H, W, cin, cout, k = case
    g = torch.Generator().manual_seed(11)
    x = torch.randn(N, cin, H, W, generator=g)
    dy = torch.randn(N, cout, H, W, generator=g)
    xh, _, rows = flat_from_nchw(x.to(DEV), fmt=_lib.FMT_F16, split=False)
    dyh, _, _ = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_F16, split=False)
    outs = []
    for impl in (_lib.IMPL_TC, _lib.IMPL_TC, _lib.IMPL_TC2):
        dw = torch.zeros(cout, k * k, cin, device=DEV)
        call("ssp_wgrad_gemm", impl, ptr(dyh), rows, cout, cout, _lib.FMT_F16, ptr(xh), rows, cin, cin, _lib.FMT_F16,
             N, H, W, k * k, ptr(dw), cin, cin, 1.0, stream_ptr())
        torch.cuda.synchronize()
        outs.append(dw)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    ref = torch.nn.grad.conv2d_weight(x.half().double(), (cout, cin, k, k), dy.half().double(), padding=(k - 1) // 2).float()
    out = outs[0].view(cout, k, k, cin).permute(0, 3, 1, 2).cpu()
    assert (out - ref).abs().max() / ref.abs().max() < 1e-4


def _bn_ref(y, gamma, beta, route):
    """torch reference of BN(train)+leaky(+pool/reorg) and its autograd."""
    z = F.batch_norm(y, None, None, gamma, beta, training=True, eps=1e-4)
    z = F.leaky_relu(z, 0.1)
    if route == _lib.ROUTE_POOL:
        return F.max_pool2d(z, 2, 2)
    if route == _lib.ROUTE_REORG:
        B, C, H, W = z.shape
        t = z.view(B, C, H // 2, 2, W // 2, 2).transpose(3, 4).contiguous()
        t = t.view(B, C, (H // 2) * (W // 2), 4).transpose(2, 3).contiguous()
        t = t.view(B, C, 4, H // 2, W // 2).transpose(1, 2).contiguous()
        return t.view(B, 4 * C, H // 2, W // 2)
    return z


@pytest.mark.parametrize("gf16", [False, True])               # upstream gradient plane in fp32, or in fp16 as a GEMM with SSP_EPI_F16 writes it
@pytest.mark.parametrize("route", [_lib.ROUTE_DIRECT, _lib.ROUTE_POOL, _lib.ROUTE_REORG])
@pytest.mark.parametrize("C", [32, 256])
def test_bn_apply_and_backward(route, C, gf16):
    N, H, W = 3, 8, 6
    g = torch.Generator().manual_seed(11)
    y = (torch.randn(N, C, H, W, generator=g) * 1.7 + 0.3).requires_grad_(True)
    gamma = (torch.rand(C, generator=g) + 0.5).requires_grad_(True)
    gamma.data[::3] *= -1                                       # negative gammas: pooling must act on activated values
    beta = torch.randn(C, generator=g).requires_grad_(True)
    out_ref = _bn_ref(y, gamma, beta, route)
    gup = torch.randn(out_ref.shape, generator=g)
    if gf16:
        gup = gup.half().float()                               # the reference sees the values the fp16 plane holds
    out_ref.backward(gup)
    # ---- device: statistics come from the conv epilogue in production; here computed by torch in fp64 ----
    yd = y.detach().to(DEV)
    rows = _lib.flat_alloc_rows(N, H, W)
    yf = torch.zeros(rows, C, device=DEV)
    idx = torch_flat_index(N, H, W).to(DEV)
    yf[idx] = yd.permute(0, 2, 3, 1).reshape(-1, C)
    ssum = yd.double().sum(dim=(0, 2, 3)).contiguous(); ssq = (yd.double() ** 2).sum(dim=(0, 2, 3)).contiguous()
    gm, bt = gamma.detach().to(DEV), beta.detach().to(DEV)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    mean, invstd, scale, shift = (torch.zeros(C, device=DEV) for _ in range(4))
    call("ssp_bn_finalize", ptr(ssum), ptr(ssq), float(N * H * W), ptr(gm), ptr(bt), ptr(rm), ptr(rv), 0.1, 1e-4, 1,
         ptr(mean), ptr(invstd), ptr(scale), ptr(shift), C, stream_ptr())
    bn_t = torch.nn.BatchNorm2d(C, eps=1e-4); bn_t.train(); bn_t(y.detach())
    assert torch.allclose(rm.cpu(), bn_t.running_mean, rtol=1e-5, atol=1e-6)
    assert torch.allclose(rv.cpu(), bn_t.running_var, rtol=1e-5, atol=1e-6)
    assert float(ssum.abs().max()) == 0.0                      # accumulators cleared for the next step
    oN, oC, oH, oW = out_ref.shape
    orows = _lib.flat_alloc_rows(oN, oH, oW)
    ohi = torch.zeros(orows, oC, dtype=torch.float16, device=DEV); olo = torch.zeros_like(ohi)
    ypool = torch.zeros(orows, C, device=DEV) if route == _lib.ROUTE_POOL else None
    call("ssp_bn_apply", ptr(yf), C, ptr(scale), ptr(shift), N, C, H, W, 0.1, ptr(ohi), ptr(olo), oC, 0, route,
         None, None, 0, 0, 0, ptr(ypool), C, stream_ptr())
    got = torch.empty(oN, oC, oH, oW, device=DEV)
    call("ssp_unpack16_nchw", ptr(ohi), ptr(olo), ptr(got), oN, oC, oH, oW, oC, 0, 0, stream_ptr())
    assert (got.cpu() - out_ref.detach()).abs().max() < 2e-5 * out_ref.detach().abs().max()
    # ---- backward ----
    gf = torch.zeros(orows, oC, dtype=torch.float16 if gf16 else torch.float32, device=DEV)
    gf[torch_flat_index(oN, oH, oW).to(DEV)] = gup.to(DEV).permute(0, 2, 3, 1).reshape(-1, oC).to(gf.dtype)
    gflag = _lib.ROUTE_F16 if gf16 else 0
    s1 = torch.zeros(C, dtype=torch.float64, device=DEV); s2 = torch.zeros_like(s1)
    common = [ptr(yf), C, ptr(scale), ptr(shift), ptr(mean), ptr(invstd), ptr(gm), N, C, H, W, 0.1,
              ptr(gf), oC, 0, route | gflag, None, 0, 0, 0, ptr(s1), ptr(s2)]
    call("ssp_bn_bwd_reduce", *common, stream_ptr())
    if ypool is not None:
        # quarter-resolution first pass from the arg-max plane: the same S1 / S2 as the full-resolution reduction
        t1 = torch.zeros_like(s1); t2 = torch.zeros_like(s2)
        call("ssp_bn_bwd_reduce", ptr(ypool), C, ptr(scale), ptr(shift), ptr(mean), ptr(invstd), ptr(gm), N, C, H // 2, W // 2, 0.1,
             ptr(gf), oC, 0, _lib.ROUTE_DIRECT | gflag, None, 0, 0, 0, ptr(t1), ptr(t2), stream_ptr())
        torch.cuda.synchronize()
        assert torch.allclose(t1, s1, rtol=1e-6, atol=1e-6 * float(s1.abs().max()))
        assert torch.allclose(t2, s2, rtol=1e-6, atol=1e-6 * float(s2.abs().max()))
    dy = torch.zeros(rows, C, dtype=torch.float16, device=DEV)
    call("ssp_bn_bwd_apply", *common, ptr(dy), C, _lib.FMT_F16, 1.0, stream_ptr())
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    call("ssp_bn_bwd_finalize", ptr(s1), ptr(s2), ptr(dg), ptr(db), C, 0, 1.0, stream_ptr())
    torch.cuda.synchronize()
    assert torch.allclose(dg.cpu(), gamma.grad, rtol=1e-4, atol=1e-4 * gamma.grad.abs().max())
    assert torch.allclose(db.cpu(), beta.grad, rtol=1e-4, atol=1e-4 * beta.grad.abs().max())
    dyn = torch.empty(N, C, H, W, device=DEV)
    call("ssp_unpack16_nchw", ptr(dy), None, ptr(dyn), N, C, H, W, C, 0, 0, stream_ptr())
    assert (dyn.cpu() - y.grad).abs().max() < 2e-3 * y.grad.abs().max()        # fp16 storage of dY


def test_sgd_flat_matches_torch_sgd():
    n = 100003
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g); p_t = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([p_t], lr=0.01, momentum=0.9, dampening=0, weight_decay=0.032)
    p = p0.clone().to(DEV); v = torch.zeros(n, device=DEV)
    for _ in range(3):
        gr = torch.randn(n, generator=g)
        p_t.grad = gr.clone(); opt.step()
        call("ssp_sgd_step_flat", ptr(p), ptr(gr.to(DEV)), ptr(v), n, 0.01, 0.9, 0.032, 1.0, stream_ptr())
    assert torch.allclose(p.cpu(), p_t.detach(), rtol=1e-5, atol=1e-6)


def _seg_table(entries):
    """entries: dicts of ssp_sgd_segment fields -> (device table, total blocks)"""
    import numpy as np
    tab = np.zeros(len(entries), dtype=np.dtype(_lib.STRUCTS["ssp_sgd_segment"]))
    b0 = 0
    for e, d in zip(tab, entries):
        for k, v in d.items():
            e[k] = v
        e["block0"] = b0
        b0 += int(_lib.load().ssp_sgd_segment_blocks(int(e["cout"]), int(e["taps"]), int(e["cin"]), int(e["n"])))
    return torch.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(DEV), b0


def test_sgd_pack_step_matches_separate_kernels():
    """the fused optimiser + re-pack pass (csrc/sgd_pack.cu) writes exactly the bytes of ssp_sgd_step_flat followed by
    ssp_pack_weights: parameters, momentum, forward hi/lo planes and the transposed data-gradient plane; launched bucket by
    bucket (block sub-ranges) it gives the same result as in one launch"""
    shapes = [(32, 1, 27), (64, 9, 32), (130, 9, 70), (0, 0, 0, 70), (0, 0, 0, 5000), (20, 1, 1024), (256, 9, 128)]   # 4-tuples: plain tensors
    gen = torch.Generator(device=DEV).manual_seed(11)
    sizes = [(s[0] * s[1] * s[2]) if len(s) == 3 else s[3] for s in shapes]
    total = sum(sizes)
    p0 = torch.randn(total, device=DEV, generator=gen); g = torch.randn(total, device=DEV, generator=gen); v0 = torch.randn(total, device=DEV, generator=gen)
    hyper = (0.01, 0.9, 0.032, 0.5)
    # separate kernels
    p_ref, v_ref = p0.clone(), v0.clone()
    call("ssp_sgd_step_flat", ptr(p_ref), ptr(g), ptr(v_ref), total, *hyper, stream_ptr())
    planes_ref, planes, entries, off = [], [], [], 0
    for s, n in zip(shapes, sizes):
        if len(s) == 4:
            entries.append(dict(off=off, n=n)); planes_ref.append(None); planes.append(None)
        else:
            cout, taps, cin = s
            ld_f, ld_d = (taps * cin + 7) // 8 * 8, (taps * cout + 7) // 8 * 8
            mk = lambda: (torch.zeros(cout, ld_f, dtype=torch.float16, device=DEV), torch.zeros(cout, ld_f, dtype=torch.float16, device=DEV),
                          torch.zeros(cin, ld_d, dtype=torch.float16, device=DEV) if taps * cin != 27 else None)
            a, b = mk(), mk()
            call("ssp_pack_weights", ptr(p_ref[off:off + n]), cout, taps, cin, ptr(a[0]), ptr(a[1]), ld_f, ptr(a[2]), ld_d if a[2] is not None else 0, _lib.FMT_F16, stream_ptr())
            planes_ref.append(a); planes.append(b)
            entries.append(dict(off=off, n=n, cout=cout, taps=taps, cin=cin, ld_f=ld_f, ld_d=ld_d if b[2] is not None else 0, d_fmt=_lib.FMT_F16,
                                f_hi=b[0].data_ptr(), f_lo=b[1].data_ptr(), d=b[2].data_ptr() if b[2] is not None else 0))
        off += n
    table, nblocks = _seg_table(entries)
    for cuts in ([0, nblocks], None):
        if cuts is None:                 # bucket by bucket, last segments first (the data-parallel order)
            b0s = [int(x) for x in table.cpu().view(torch.int32).view(len(entries), 18)[:, 16]] + [nblocks]
            cuts = [b0s[0], b0s[3], b0s[5], nblocks]
        p, v = p0.clone(), v0.clone()
        for pl in planes:
            if pl is not None:
                for t in pl:
                    if t is not None:
                        t.zero_()
        for lo, hi in reversed(list(zip(cuts[:-1], cuts[1:]))):
            call("ssp_sgd_pack_step", ptr(table), len(entries), lo, hi, ptr(p), ptr(g), ptr(v), *hyper, stream_ptr())
        torch.cuda.synchronize()
        assert torch.equal(p, p_ref) and torch.equal(v, v_ref)
        for a, b in zip(planes_ref, planes):
            if a is not None:
                for x, y in zip(a, b):
                    if x is not None:
                        assert torch.equal(x.view(torch.int16), y.view(torch.int16))


def test_library_reports_errors():
    with pytest.raises(_lib.SspError):
        call("ssp_pnp_batched", None, 1, None, None, 9, 1, 20, None, None, None, stream_ptr())


@pytest.mark.parametrize("shape", [(2, 32, 64), (1, 48, 80), (3, 16, 32), (2, 34, 70)])
def test_l0_fused_blocks_match_torch(shape):
    """blocks 0-1 as one unit (csrc/l0_fused.cu: conv 3->32 + BatchNorm(batch statistics) + LeakyReLU + MaxPool 2x2, darknet.py:154-167)
    and their backward, against torch fp64 autograd of the same modules: Gram-matrix statistics, the pooled operand planes + arg-max
    codes, dW / dgamma / dbeta from the pooled gradient.  Shapes cover partial tiles in both directions."""
    N, H, W = shape
    g = torch.Generator().manual_seed(23)
    x = torch.rand(N, 3, H, W, generator=g)
    w = (torch.randn(32, 3, 3, 3, generator=g) * 0.3)
    gamma = torch.rand(32, generator=g) + 0.5
    beta = torch.randn(32, generator=g) * 0.2
    gpool = (torch.randn(N, 32, H // 2, W // 2, generator=g) * 256.0).half().float() / 256.0      # exactly representable in the loss-scaled fp16 plane
    # ---- reference: fp64 autograd
    wd = w.double().requires_grad_(True); gd = gamma.double().requires_grad_(True); bd = beta.double().requires_grad_(True)
    y = F.conv2d(x.double(), wd, padding=1)
    mean = y.mean(dim=(0, 2, 3)); var = y.var(dim=(0, 2, 3), unbiased=False)
    eps = 1e-4
    z = (y - mean[None, :, None, None]) / torch.sqrt(var + eps)[None, :, None, None] * gd[None, :, None, None] + bd[None, :, None, None]
    a = F.leaky_relu(z, 0.1)
    pooled, am = F.max_pool2d(a, 2, 2, return_indices=True)
    cnt = float(N * H * W)
    # ---- device
    xd = x.to(DEV)
    wm = w.permute(0, 2, 3, 1).contiguous().to(DEV)                      # master layout [co][kh][kw][ci]
    gram = torch.zeros(_lib.CONSTANTS["SSP_L0_GRAM_DOUBLES"], dtype=torch.float64, device=DEV)             # matrix + scratch
    ssum = torch.zeros(32, dtype=torch.float64, device=DEV); ssq = torch.zeros_like(ssum)
    s = stream_ptr()
    call("ssp_l0_gram", ptr(xd), N, H, W, ptr(gram), s)
    call("ssp_l0_stats", ptr(gram), ptr(wm), ptr(ssum), ptr(ssq), s)
    torch.cuda.synchronize()
    # Gram matrix against the im2col'ed patches (k = (kh*3+kw)*3 + c)
    P = F.unfold(x.double(), 3, padding=1).view(N, 3, 9, H * W).permute(0, 3, 2, 1).reshape(-1, 27)      # [px][tap][c]
    Q = torch.cat([P, torch.ones(P.shape[0], 1, dtype=torch.float64)], dim=1)
    Gref = Q.t() @ Q
    G = gram.cpu()[:784].view(28, 28)
    iu = torch.triu_indices(28, 28)
    assert ((G[iu[0], iu[1]] - Gref[iu[0], iu[1]]).abs() / Gref[iu[0], iu[1]].abs().clamp_min(1.0)).max() < 2e-6
    assert (ssum.cpu() - y.detach().sum(dim=(0, 2, 3))).abs().max() < 1e-5 * cnt
    q_ref = (y.detach() ** 2).sum(dim=(0, 2, 3))
    assert ((ssq.cpu() - q_ref).abs() / q_ref).max() < 2e-6
    rm = torch.zeros(32, device=DEV); rv = torch.ones(32, device=DEV)
    mean_d = torch.zeros(32, device=DEV); invstd_d = torch.zeros(32, device=DEV); scale_d = torch.zeros(32, device=DEV); shift_d = torch.zeros(32, device=DEV)
    gamma_d, beta_d = gamma.to(DEV), beta.to(DEV)                          # named: a temporary would be freed (and its memory reused) before the launch
    call("ssp_bn_finalize", ptr(ssum), ptr(ssq), cnt, ptr(gamma_d), ptr(beta_d), ptr(rm), ptr(rv), 0.1, eps, 1,
         ptr(mean_d), ptr(invstd_d), ptr(scale_d), ptr(shift_d), 32, s)
    assert (mean_d.cpu().double() - mean.detach()).abs().max() < 1e-6
    assert ((invstd_d.cpu().double() - 1.0 / torch.sqrt(var.detach() + eps)).abs() * torch.sqrt(var.detach() + eps)).max() < 1e-5
    prow = _lib.flat_alloc_rows(N, H // 2, W // 2)
    ld, c0 = 40, 4                                                       # destination wider than the layer: concat placement
    hi = torch.zeros(prow, ld, dtype=torch.float16, device=DEV); lo = torch.zeros_like(hi)
    code = torch.full((prow, 32), 255, dtype=torch.uint8, device=DEV)
    call("ssp_l0_fused_fwd", ptr(xd), ptr(wm), ptr(scale_d), ptr(shift_d), 0.1, N, H, W, ptr(hi), ptr(lo), ld, c0, ptr(code), s)
    torch.cuda.synchronize()
    idx = torch_flat_index(N, H // 2, W // 2)
    got = (hi.float() + lo.float()).cpu()[idx][:, c0:c0 + 32].reshape(N, H // 2, W // 2, 32).permute(0, 3, 1, 2)
    assert (got.double() - pooled.detach()).abs().max() / pooled.detach().abs().max() < 2e-5
    v = (hi.float() + lo.float()).cpu()
    mask = torch.ones(prow, dtype=torch.bool); mask[idx] = False
    assert float(v[mask].abs().max()) == 0.0 and float(v[:, :c0].abs().max()) == 0.0 and float(v[:, c0 + 32:].abs().max()) == 0.0
    # arg-max codes: position inside the window and the sign of the pre-activation there.  fp32-vs-fp64 rounding may pick the other
    # element of an (almost exact) tie: the selected VALUE must be the maximum, the position may differ on a vanishing fraction
    cd = code.cpu()[idx].reshape(N, H // 2, W // 2, 32).permute(0, 3, 1, 2).long()
    hh = torch.arange(H // 2).view(1, 1, -1, 1) * 2 + ((cd >> 1) & 1); ww = torch.arange(W // 2).view(1, 1, 1, -1) * 2 + (cd & 1)
    pos = hh * W + ww
    a_sel = a.detach().flatten(2).gather(2, pos.flatten(2)).view_as(pos)
    assert (a_sel - pooled.detach()).abs().max() < 1e-5 * pooled.detach().abs().max()
    assert float((pos != am).float().mean()) < 1e-3
    zsel = z.detach().flatten(2).gather(2, pos.flatten(2)).view_as(pos)
    sure = zsel.abs() > 1e-5
    assert torch.equal(((cd & 4) != 0)[sure], (zsel > 0)[sure])
    # reference backward routed through the device's arg-max positions (a valid subgradient; identical unless there was a tie)
    (a.flatten(2).gather(2, pos.flatten(2)).view_as(pos) * gpool.double()).sum().backward()
    assert int(code.cpu()[mask].min()) == 255                             # pad cells untouched
    # ---- backward from the pooled gradient (loss scale 256 carried like the engine does)
    gflat = torch.zeros(prow, ld, dtype=torch.float16, device=DEV)       # the engine's default: data gradients live in fp16 planes
    gflat[idx.to(DEV), c0:c0 + 32] = (gpool * 256.0).permute(0, 2, 3, 1).reshape(-1, 32).to(DEV).half()
    t1 = torch.zeros(28 * 32, dtype=torch.float64, device=DEV)
    dW = torch.zeros(32, 27, device=DEV); dga = torch.zeros(32, device=DEV); dbe = torch.zeros(32, device=DEV)
    call("ssp_l0_bwd", ptr(xd), ptr(gflat), 1, ld, c0, ptr(code), 0.1, N, H, W, ptr(t1), s)
    call("ssp_l0_bwd_finalize", ptr(t1), ptr(gram), ptr(wm), ptr(gamma_d), ptr(mean_d), ptr(invstd_d), cnt, 1.0 / 256.0,
         ptr(dW), ptr(dga), ptr(dbe), s)
    torch.cuda.synchronize()
    dW_ref = wd.grad.permute(0, 2, 3, 1).reshape(32, 27)
    assert (dW.cpu().double() - dW_ref).abs().max() / dW_ref.abs().max() < 1e-4
    assert (dga.cpu().double() - gd.grad).abs().max() / gd.grad.abs().max() < 1e-4
    assert (dbe.cpu().double() - bd.grad).abs().max() / bd.grad.abs().max() < 1e-4


BANDT_FWD = [
    # N, H, W, cin, cout, k, operand terms   (forward with BN statistics; split fp16, cout <= 64: W_hi / W_lo stacked on the M side;
    # single term, cout <= 128: channels 64-127 in the upper half (UP) of the M side)
    (2, 40, 24, 32, 64, 3, 3),     # block-2 class: 128-pixel tiles (nine resident 16 KB tiles leave room for two 136-row bands only)
    (4, 104, 104, 32, 64, 3, 3),   # 345 tiles: several tiles per CTA, every ring phase in use
    (2, 26, 26, 128, 64, 1, 3),    # 1x1, two K chunks
    (3, 5, 7, 64, 32, 3, 3),       # cout 32: half of each stacked plane is zero fill
    (1, 13, 13, 64, 24, 3, 3),     # cout not a multiple of 32
    (2, 40, 24, 32, 64, 3, 1),     # block 2 of the fast forward: the overlapping-row variant, single term
    (4, 104, 104, 64, 128, 3, 1),  # blocks 4 / 6 of the fast forward: UP 3x3, nine resident tiles, many tiles per CTA, every ring phase
    (2, 26, 26, 256, 128, 1, 1),   # block 9: UP 1x1, four K chunks
    (1, 13, 13, 64, 100, 3, 1),    # cout > 64 and not a multiple of 8: the weight tile's row count rounds up to 104
    (2, 26, 26, 512, 64, 1, 1),    # block 26: eight K chunks
    (2, 13, 13, 128, 64, 1, 1),    # block 5 class
]
BANDT_DGRAD = [
    # N, H, W, channels of dY (K per tap), channels of dX (<= 128), k      (single-term fp16)
    (2, 40, 24, 64, 32, 3),        # block-2 data gradient: 32 of the 128 accumulator rows carry output
    (4, 104, 104, 64, 32, 3),
    (2, 26, 26, 128, 64, 3),       # block-3/5 data gradient
    (2, 13, 13, 64, 128, 3),
    (2, 26, 26, 64, 128, 1),
]


@pytest.mark.parametrize("case", BANDT_FWD)
def test_conv_bandt_forward_runs_and_matches_torch(case):
    """operand-swapped kernel (csrc/conv_bandt.cu): the kernel itself must have run (launch counter), outputs / BN statistics
    against the fp64 torch convolution at the tolerance of the other tensor-core kernels.  The statistics are checked per 64-channel
    half of the M side: channels 64-127 come from the upper half of the accumulator, and only the valid pixel rows of each tile
    (its ballot mask) may contribute."""
    N, H, W, cin, cout, k, terms = case
    g = torch.Generator().manual_seed(31 + cin + cout + H)
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    xh, xl, rows, wh, wl, x64, w64 = _operands(x, w, terms)
    ref = F.conv2d(x64, w64, None, padding=(k - 1) // 2).float()
    ldo = (cout + 3) // 4 * 4
    y = torch.full((rows, ldo), float("nan"), device=DEV)
    ssum = torch.zeros(cout, dtype=torch.float64, device=DEV); ssq = torch.zeros_like(ssum)
    before = _lib.load().ssp_conv_bandt_launches()
    call("ssp_conv_gemm", _lib.IMPL_BANDT, ptr(xh), ptr(xl), rows, cin, cin, ptr(wh), ptr(wl), cout, wh.shape[1], 0, 0,
         N, H, W, k * k, cout, ptr(y), ldo, rows, _lib.EPI_STATS, None, ptr(ssum), ptr(ssq), stream_ptr())
    torch.cuda.synchronize()
    assert _lib.load().ssp_conv_bandt_launches() == before + 1
    out = nchw_from_flat(y, N, cout, H, W).cpu()
    tol = 2e-5 + 5e-9 * cin * k * k
    assert (out - ref).abs().max() / ref.abs().max() < tol
    s_ref = ref.double().sum(dim=(0, 2, 3)); q_ref = (ref.double() ** 2).sum(dim=(0, 2, 3))
    for c0 in range(0, cout, 64):
        c = slice(c0, min(cout, c0 + 64))
        assert (ssum.cpu()[c] - s_ref[c]).abs().max() < 1e-4 * q_ref[c].max().sqrt() * (N * H * W) ** 0.5, c0
        assert ((ssq.cpu()[c] - q_ref[c]).abs() / q_ref[c]).max() < 1e-4, c0


@pytest.mark.parametrize("out16", [False, True])              # fp32 plane, or the fp16 plane of SSP_EPI_F16
@pytest.mark.parametrize("case", BANDT_DGRAD)
def test_conv_bandt_dgrad_runs_and_matches_torch(case, out16):
    N, H, W, cy, cx, k = case
    g = torch.Generator().manual_seed(7 + cy + cx + H)
    dy = torch.randn(N, cy, H, W, generator=g)
    w = torch.randn(cy, cx, k, k, generator=g) / (cy * k * k) ** 0.5         # forward weight OIHW: cy = cout, cx = cin
    dyq = dy.half().float(); wq = w.half().float()
    ref = F.conv_transpose2d(dyq.double(), wq.double(), padding=(k - 1) // 2).float()
    dyh, _, rows = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_F16, split=False)
    _, _, wd = _pack_w(w.to(DEV), fmt=_lib.FMT_F16, dgrad=True)
    dx = torch.full((rows, cx), float("nan"), dtype=torch.float16 if out16 else torch.float32, device=DEV)
    before = _lib.load().ssp_conv_bandt_launches()
    call("ssp_conv_gemm", _lib.IMPL_BANDT, ptr(dyh), None, rows, cy, cy, ptr(wd), None, cx, wd.shape[1], 0, 0,
         N, H, W, k * k, cx, ptr(dx), cx, rows, _lib.EPI_F16 if out16 else _lib.EPI_F32, None, None, None, stream_ptr())
    torch.cuda.synchronize()
    assert _lib.load().ssp_conv_bandt_launches() == before + 1
    out = nchw_from_flat(torch.nan_to_num(dx.float()).contiguous(), N, cx, H, W).cpu()
    assert (out - ref).abs().max() / ref.abs().max() < (1e-3 if out16 else 1e-4)      # fp16 storage: 2^-11 relative per element


@pytest.mark.parametrize("case", [(2, 13, 13, 256, 512, 3), (2, 26, 26, 128, 256, 1), (1, 13, 13, 96, 40, 3)])
def test_conv_tc2_dgrad_fp16_plane(case):
    """SSP_EPI_F16 through SSP_IMPL_TC2 (the per-tap kernel, csrc/conv_tc.cu): the data gradient stored as fp16 equals the fp32 plane
    rounded once"""
    N, H, W, cy, cx, k = case
    g = torch.Generator().manual_seed(3 + cy)
    dy = torch.randn(N, cy, H, W, generator=g)
    w = torch.randn(cy, cx, k, k, generator=g) / (cy * k * k) ** 0.5
    dyh, _, rows = flat_from_nchw(dy.to(DEV), fmt=_lib.FMT_F16, split=False)
    _, _, wd = _pack_w(w.to(DEV), fmt=_lib.FMT_F16, dgrad=True)
    ld16 = (cx + 7) // 8 * 8
    d32 = torch.zeros(rows, (cx + 3) // 4 * 4, device=DEV); d16 = torch.zeros(rows, ld16, dtype=torch.float16, device=DEV)
    for out, ld, epi in ((d32, d32.shape[1], _lib.EPI_F32), (d16, ld16, _lib.EPI_F16)):
        call("ssp_conv_gemm", _lib.IMPL_TC2, ptr(dyh), None, rows, cy, cy, ptr(wd), None, cx, wd.shape[1], 0, 0,
             N, H, W, k * k, cx, ptr(out), ld, rows, epi, None, None, None, stream_ptr())
    torch.cuda.synchronize()
    idx = torch_flat_index(N, H, W).to(DEV)
    a = d32[idx][:, :cx]; b = d16[idx][:, :cx]
    assert torch.equal(a.half(), b)
    assert float(d16[:, cx:].abs().max()) == 0.0 if ld16 > cx else True
