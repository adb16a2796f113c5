"""Every GEMM of a real training step against fp64, at the input sizes of the multi-scale schedule.

Training draws a new square input for every batch (dataset.py: 7 to 26 cells, 224 to 832 pixels).  Here one step runs through the
public API (Darknet.train(), RegionLoss, forward, backward) at each of those geometries, and then every launch is checked against a
plain fp64 computation of the exact operand values the kernel read, taken from the engine's own retained state: the operand planes
x_hi / x_lo, the conv outputs y, the gradient planes dy / dx, the packed weights w_hi / w_lo / w_d and the flat gradient buffer.
No CPU network is involved, so the chaos of a random-init network plays no part and the bounds are those of one GEMM:

* forward: y = conv(x_hi + x_lo, w_hi + w_lo) (+ the head's bias), and the batch mean / invstd derived from its statistics; with
  SSP_PRECISION=fast y = conv(x_hi, w_hi), on the kernel configurations that only that mode selects;
* data gradient: dx = fp16(conv_transpose(dy, W_d)), loss-scaled and saturating;
* weight gradient: dW = conv2d_weight(x_hi, dy) / grad_scale, in the master layout [co][kh][kw][ci];
* blocks 0-1 (l0_fused.cu) at the real image size: Gram matrix, mean / invstd, pooled planes, dW0 / dgamma / dbeta;
* the invariants the engine relies on: zero pad rows and zero columns beyond the layer's channels, and no silent fall-back from
  the operand-swapped kernel (SSP_IMPL_BANDT)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from singleshotpose_b200 import Darknet, RegionLoss, _lib, synth
from singleshotpose_b200.predict import PosePredictor

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (N, H, W): batch 3 up to 608 (partial tiles at every layer), batch 1 at 832, the 352x480 training shape, and the real training batch
# (64) at 224 and 416, where the weight gradient's cluster split (a function of N*H*W) differs from the small batches
GEOMS = [(3, 224, 224), (3, 320, 320), (3, 416, 416), (3, 544, 544), (3, 608, 608), (1, 832, 832), (3, 352, 480),
         (64, 224, 224), (64, 416, 416)]

# the single-term forward (SSP_PRECISION=fast) at the sizes where its kernel configurations differ most: partial tiles (batch 3),
# the largest input, the non-square training shape, and blocks 4 / 6 at batch 64, 416^2 (thousands of 128-pixel tiles)
FAST_GEOMS = [(3, 416, 416), (3, 608, 608), (1, 832, 832), (3, 352, 480), (64, 416, 416)]
CASES = [("exact", g) for g in GEOMS] + [("fast", g) for g in FAST_GEOMS]
CASE_IDS = ["%dx%dx%d" % g for g in GEOMS] + ["fast-%dx%dx%d" % g for g in FAST_GEOMS]

# operand-swapped launches of one training step, the same at every geometry (eligibility depends on channel counts only).  Split
# operands (cout <= 64): the forwards of blocks 2, 5 and 26 and the data gradients of blocks 2, 4, 5 and 6.  Single term
# (cout <= 128): also the forwards of blocks 4, 6 (64 -> 128, 3x3) and 9 (256 -> 128, 1x1).  The engine routes three more launches
# to SSP_IMPL_BANDT that the kernel declines by design (conv_bandt.cu): the head's bias epilogue and the data gradients of blocks 8
# and 10 (256 -> 128 channels, 3x3: 36 resident 16-KB weight tiles do not fit next to two activation bands).
_BANDT_EXACT = {("fwd", 2), ("fwd", 5), ("fwd", 26), ("dgrad", 2), ("dgrad", 4), ("dgrad", 5), ("dgrad", 6)}
BANDT_STEP = {"exact": _BANDT_EXACT, "fast": _BANDT_EXACT | {("fwd", 4), ("fwd", 6), ("fwd", 9)}}
BANDT_DECLINED = {("fwd", 30), ("dgrad", 8), ("dgrad", 10)}


def _model(cfg_path, precision):
    """a random-init network whose engine runs `precision` (Engine reads SSP_PRECISION in its constructor only)"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("SSP_PRECISION", precision)
        torch.manual_seed(0)
        m = Darknet(cfg_path).cuda().train()
    assert m._engine.fast == (precision == "fast")
    return m


@pytest.fixture(scope="module")
def model(cfg_path, request):
    return _model(cfg_path, request.param)


def _idx(N, H, W):
    n, h, w = torch.meshgrid(torch.arange(N), torch.arange(H), torch.arange(W), indexing="ij")
    return (n * (H + 1) * (W + 1) + (h + 1) * (W + 1) + (w + 1)).reshape(-1).to(DEV)


def _nchw(plane, idx, N, h, w, C, sel=None):
    """padded-flat plane -> NCHW fp64 of its first C channels (or the channels `sel`)"""
    v = plane[idx, :C] if sel is None else plane[idx][:, sel]
    return v.double().view(N, h, w, -1).permute(0, 3, 1, 2)


def _channels(C, subset):
    """every channel, or (batch 64) a subset holding both ends of every 64- and 128-channel tile and the last channel"""
    if not subset:
        return torch.arange(C, device=DEV)
    return torch.tensor(sorted({c for c in range(C) if c % 64 in (0, 1, 62, 63)} | {C - 1}), device=DEV)


def _fp16_ulp(v):
    """spacing of the fp16 values around v (fp64 tensor of fp16 values): 2^(e-10), subnormal spacing 2^-24 below 2^-14"""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _step(model, N, H, W, seed):
    eng = model._engine
    lib = _lib.load()
    x = synth.images(N, H, W, seed=seed).cuda()
    tgt = synth.targets(N, seed=seed + 1)
    crit = RegionLoss(); crit.verbose = False
    torch.cuda.synchronize()
    n0 = int(lib.ssp_conv_bandt_launches())
    out = model(x)
    loss = crit(out, tgt, 20)
    loss.backward()
    torch.cuda.synchronize()
    return x, eng, eng.buffers(N, H, W, True), int(lib.ssp_conv_bandt_launches()) - n0


def _check_l0(eng, B, x, N, H, W, L):
    """blocks 0-1 against fp64 autograd of conv + batch-statistics BN + leaky + max-pool, with the tolerances of
    test_gpu_kernels.py::test_l0_fused_blocks_match_torch"""
    conv, bn = eng.conv_modules()[0]
    off, n, _ = eng._slices[id(conv.weight)]
    w = eng.flat_params[off:off + n].view(32, 3, 3, 3).permute(0, 3, 1, 2).double()          # master [co][kh][kw][ci] -> OIHW
    gamma, beta = bn.weight.detach().double(), bn.bias.detach().double()
    x64 = x.double()
    P = F.unfold(x64, 3, padding=1).view(N, 3, 9, H * W).permute(0, 3, 2, 1).reshape(-1, 27)  # [px][tap][c]
    Q = torch.cat([P, torch.ones(P.shape[0], 1, dtype=torch.float64, device=DEV)], dim=1)
    Gref = Q.t() @ Q
    del P, Q
    G = B.l0_gram[:784].view(28, 28)
    iu = torch.triu_indices(28, 28, device=DEV)
    gerr = ((G[iu[0], iu[1]] - Gref[iu[0], iu[1]]).abs() / Gref[iu[0], iu[1]].abs().clamp_min(1.0)).max()
    assert gerr < 2e-6, gerr
    wd = w.clone().requires_grad_(True); gd = gamma.clone().requires_grad_(True); bd = beta.clone().requires_grad_(True)
    y = F.conv2d(x64, wd, padding=1)
    mean = y.mean(dim=(0, 2, 3)); var = y.var(dim=(0, 2, 3), unbiased=False)
    st = B.stat[0]
    assert (st["mean"].double() - mean.detach()).abs().max() < 1e-6
    assert ((st["invstd"].double() - 1.0 / torch.sqrt(var.detach() + bn.eps)).abs() * torch.sqrt(var.detach() + bn.eps)).max() < 1e-5
    z = (y - mean[None, :, None, None]) / torch.sqrt(var + bn.eps)[None, :, None, None] * gd[None, :, None, None] + bd[None, :, None, None]
    a = F.leaky_relu(z, 0.1)
    pooled, am = F.max_pool2d(a, 2, 2, return_indices=True)
    h2, w2 = H // 2, W // 2
    ci, c0, _k = L.dests[0]
    pidx = _idx(N, h2, w2)
    got = (B.x_hi[ci][pidx, c0:c0 + 32].double() + B.x_lo[ci][pidx, c0:c0 + 32].double()).view(N, h2, w2, 32).permute(0, 3, 1, 2)
    perr = (got - pooled.detach()).abs().max() / pooled.detach().abs().max()
    assert perr < 2e-5, perr
    # arg-max codes: an (almost exact) tie may resolve to the other element; the selected value must be the maximum
    cd = B.l0_code[pidx].view(N, h2, w2, 32).permute(0, 3, 1, 2).long()
    hh = torch.arange(h2, device=DEV).view(1, 1, -1, 1) * 2 + ((cd >> 1) & 1)
    ww = torch.arange(w2, device=DEV).view(1, 1, 1, -1) * 2 + (cd & 1)
    pos = (hh * W + ww).flatten(2)
    a_sel = a.flatten(2).gather(2, pos).view_as(cd)
    assert (a_sel.detach() - pooled.detach()).abs().max() < 1e-5 * pooled.detach().abs().max()
    z_sel = z.flatten(2).gather(2, pos).view_as(cd)
    sure = z_sel.detach().abs() > 1e-5
    assert torch.equal(((cd & 4) != 0)[sure], (z_sel.detach() > 0)[sure])
    assert float((pos.view_as(am) != am).double().mean()) < 1e-3
    del am, pooled
    # backward from the pooled gradient the device read (dx of layer 1, loss-scaled fp16), routed through the device's positions and
    # its leaky slopes (bit 2 of the code): at a real image size some pre-activations lie within fp32 rounding of zero, where fp64
    # may take the other slope -- a valid subgradient either way, but a 0.9 g difference per such cell
    gpool = B.dx[ci][pidx, c0:c0 + 32].double().view(N, h2, w2, 32).permute(0, 3, 1, 2) / eng.grad_scale
    slope = torch.where((cd & 4) != 0, 1.0, 0.1).double()
    (z_sel * slope * gpool).sum().backward()
    dW = eng.flat_grads[off:off + n].view(32, 27).double()
    dW_ref = wd.grad.permute(0, 2, 3, 1).reshape(32, 27)
    assert (dW - dW_ref).abs().max() / dW_ref.abs().max() < 1e-4
    dga, dbe = eng.grad_view(bn.weight).double(), eng.grad_view(bn.bias).double()
    assert (dga - gd.grad).abs().max() / gd.grad.abs().max() < 1e-4
    assert (dbe - bd.grad).abs().max() / bd.grad.abs().max() < 1e-4


def _conv_ref(eng, B, L, N, h, w, idx, sel, bias, terms):
    """fp64 convolution of the operand values a forward with `terms` products reads: x_hi + x_lo and w_hi + w_lo (3), or x_hi and
    w_hi (1)"""
    i, k = L.index, L.size
    K = L.taps * L.cin
    A = _nchw(B.x_hi[i], idx, N, h, w, L.cin)
    Wf = eng.w_hi[i][:, :K].double()
    if terms == 3:
        A = A + _nchw(B.x_lo[i], idx, N, h, w, L.cin)
        Wf = Wf + eng.w_lo[i][:, :K].double()
    Wf = Wf.view(L.cout, k, k, L.cin).permute(0, 3, 1, 2)
    return F.conv2d(A, Wf[sel], bias, padding=(k - 1) // 2)


def _check_forward(eng, B, L, N, h, w, idx, sel, conv, bn):
    """returns, in fast mode, whether the three-term reference lies outside this layer's bound too (i.e. whether a kernel that read
    the lo planes would fail here)"""
    i = L.index
    K = L.taps * L.cin
    bias = conv.bias.detach().double()[sel] if not L.bn else None
    ref = _conv_ref(eng, B, L, N, h, w, idx, sel, bias, 1 if eng.fast else 3)
    got = _nchw(B.y[i], idx, N, h, w, L.cout, sel)
    scale = ref.abs().max()
    err = (got - ref).abs().max() / scale
    # the suite's tensor-core bound (test_gpu_kernels.py::test_conv_gemm_matches_torch): fp32 accumulation error grows with K
    tol = 2e-5 + 5e-9 * K
    assert err < tol, (L.block_ind, float(err))
    del got
    sees_lo = bool((_conv_ref(eng, B, L, N, h, w, idx, sel, bias, 3) - ref).abs().max() / scale > tol) if eng.fast else None
    if not L.bn:
        return sees_lo
    # batch statistics: the epilogue's fp64 sums are consumed (and zeroed) by ssp_bn_finalize, which leaves mean = sum / cnt and
    # invstd = 1 / sqrt(sum_sq / cnt - mean^2 + eps) in fp32.  With the sum bounds of test_conv_gemm_matches_torch,
    # |d sum| < 1e-4 sqrt(max sum_sq) sqrt(cnt) and |d sum_sq| < 1e-4 sum_sq, the mean is off by at most 1e-4 sqrt(max sum_sq / cnt)
    # (+ its fp32 rounding), the variance by 1e-4 sum_sq / cnt + 2 |mean| d mean, and invstd relatively by half of that over
    # (var + eps) (+ fp32 rounding)
    cnt = N * h * w
    s_ref = ref.sum(dim=(0, 2, 3)); q_ref = (ref ** 2).sum(dim=(0, 2, 3))
    m_ref = s_ref / cnt
    var_ref = q_ref / cnt - m_ref ** 2
    st = B.stat[i]
    dm = 1e-4 * (q_ref.max() / cnt).sqrt() + 2.0 ** -23 * m_ref.abs()
    assert ((st["mean"].double()[sel] - m_ref).abs() <= dm).all(), L.block_ind
    dvar = 1e-4 * q_ref / cnt + 2 * m_ref.abs() * dm
    rel = (st["invstd"].double()[sel] * torch.sqrt(var_ref + bn.eps) - 1).abs()
    assert (rel <= 0.5 * dvar / (var_ref + bn.eps) + 2.0 ** -21).all(), L.block_ind
    return sees_lo


def _check_dgrad(eng, B, L, N, h, w, idx, sel, master):
    i, k = L.index, L.size
    # W_d [cin][taps*cout], k = (taps-1-tap)*cout + co: the tap-flipped, transposed fp16 copy of the master weights
    Wq = eng.w_d[i][:, :L.taps * L.cout].double().view(L.cin, L.taps, L.cout).flip(1).permute(2, 0, 1).reshape(L.cout, L.cin, k, k)
    assert torch.equal(Wq, master.half().double()), L.block_ind
    dy = _nchw(B.dy[i], idx, N, h, w, L.cout)
    ref = F.conv_transpose2d(dy, Wq[:, sel], padding=(k - 1) // 2)
    ref16 = ref.clamp(-65504, 65504).half().double()
    got = _nchw(B.dx[i], idx, N, h, w, L.cin, sel)
    # one fp16 rounding of an fp32 sum: within one fp16 ulp of the rounded reference, plus the tensor-core accumulation error
    bound = _fp16_ulp(ref16) + 1e-4 * ref.abs().max()
    bad = (got - ref16).abs() > bound
    assert not bad.any(), (L.block_ind, int(bad.sum()), float(((got - ref16).abs() - bound).max()))


def _check_wgrad(eng, B, L, N, h, w, idx, sel, conv):
    i, k = L.index, L.size
    off, n, _ = eng._slices[id(conv.weight)]
    x = _nchw(B.x_hi[i], idx, N, h, w, L.cin)
    dy = _nchw(B.dy[i], idx, N, h, w, L.cout, sel)
    ref = torch.nn.grad.conv2d_weight(x, (len(sel), L.cin, k, k), dy, padding=(k - 1) // 2) / eng.grad_scale
    got = eng.flat_grads[off:off + n].view(L.cout, k, k, L.cin)[sel].permute(0, 3, 1, 2).double()
    err = (got - ref).abs().max() / ref.abs().max()
    # the reduction runs over the N*h*w pixels (2.8 million for block 2 at batch 64, 416^2): the suite's tensor-core bound
    # (test_conv_gemm_matches_torch: fp32 accumulation error grows with the reduction length) with that length, at least 1e-4
    assert err < max(1e-4, 2e-5 + 5e-9 * N * h * w), (L.block_ind, float(err))


def _check_invariants(B, L, idx):
    i = L.index
    pad = torch.ones(B.rows[i], dtype=torch.bool, device=DEV)
    pad[idx] = False
    for name, t in (("x_hi", B.x_hi[i]), ("x_lo", B.x_lo[i]), ("dy", B.dy[i])):
        assert not (t[pad] != 0).any(), (L.block_ind, name, "pad row written")
    assert not (B.dy[i][:, L.cout:] != 0).any(), (L.block_ind, "dy beyond cout")
    assert not (B.dx[i][:, L.cin:] != 0).any(), (L.block_ind, "dx beyond cin")


@pytest.mark.parametrize("model, geo", CASES, ids=CASE_IDS, indirect=["model"])
def test_train_step_gemms_match_fp64(model, geo):
    N, H, W = geo
    x, eng, B, bandt = _step(model, N, H, W, seed=H + W + N)
    precision = "fast" if eng.fast else "exact"
    subset = N >= 64
    mods = eng.conv_modules()
    sees_lo = []
    for L in eng.layers:
        conv, bn = mods[L.index]
        h, w = eng.spatial(L, H, W)
        if L.first:
            _check_l0(eng, B, x, N, H, W, L)
            continue
        idx = _idx(N, h, w)
        off, n, _ = eng._slices[id(conv.weight)]
        master = eng.flat_params[off:off + n].view(L.cout, L.size, L.size, L.cin).permute(0, 3, 1, 2).double()
        K = L.taps * L.cin
        assert torch.equal(eng.w_hi[L.index][:, :K].double().view(L.cout, L.size, L.size, L.cin).permute(0, 3, 1, 2),
                           master.half().double()), L.block_ind
        if _check_forward(eng, B, L, N, h, w, idx, _channels(L.cout, subset), conv, bn):
            sees_lo.append(L.block_ind)
        _check_dgrad(eng, B, L, N, h, w, idx, _channels(L.cin, subset), master)
        _check_wgrad(eng, B, L, N, h, w, idx, _channels(L.cout, subset), conv)
        _check_invariants(B, L, idx)
    if eng.fast:
        print("\n%dx%dx%d fast: the three-term reference is outside the bound at %d of %d GEMM layers: blocks %s"
              % (N, H, W, len(sees_lo), len(eng.layers) - 1, sees_lo))
        assert sees_lo                 # the single-term bound is tight enough to tell the two modes apart
    routed = {("fwd", L.block_ind) for L in eng.layers if not L.first and eng._conv_impl(L) == _lib.IMPL_BANDT}
    routed |= {("dgrad", L.block_ind) for L in eng.layers if not L.first and L.cin <= 128}
    assert bandt == len(BANDT_STEP[precision]), "%d operand-swapped launches, %d expected: a silent fall-back" % (bandt, len(BANDT_STEP[precision]))
    assert routed == BANDT_STEP[precision] | BANDT_DECLINED


# ---------------------------------------------------------------------------------------------------- fast-mode inference
def _route(z, kind):
    """the placement ssp_bn_apply / the fused epilogues give a layer's activated output: 2x2 max-pool, darknet's reorg, or as is"""
    if kind == _lib.ROUTE_POOL:
        return F.max_pool2d(z, 2, 2)
    if kind == _lib.ROUTE_REORG:
        B, C, H, W = z.shape
        t = z.reshape(B, C, H // 2, 2, W // 2, 2).transpose(3, 4).contiguous()
        t = t.view(B, C, (H // 2) * (W // 2), 4).transpose(2, 3).contiguous()
        t = t.view(B, C, 4, H // 2, W // 2).transpose(1, 2).contiguous()
        return t.view(B, 4 * C, H // 2, W // 2)
    return z


def _check_inference(eng, B, N, H, W):
    """every layer of an inference forward (fused epilogue, split-K or conv + bn_apply) from the planes the engine kept: the
    destination planes hi + lo against leaky(scale conv(x, w) + shift) in fp64, routed (direct, pool, reorg, concat offset),
    with the folded scale / shift the kernels read; y against conv(x, w) where the layer wrote it (and the head's bias).  x, w are
    the operand values the forward reads: x_hi, w_hi in fast mode, x_hi + x_lo, w_hi + w_lo in exact mode"""
    mods = eng.conv_modules()
    for L in eng.layers:
        conv, bn = mods[L.index]
        i, k = L.index, L.size
        h, w = eng.spatial(L, H, W)
        K = L.taps * L.cin
        if L.first:                               # blocks 0-1 read the image and the fp32 master weights
            off, n, _ = eng._slices[id(conv.weight)]
            A, Wf = B.x_image.double(), eng.flat_params[off:off + n].view(32, 3, 3, 3).permute(0, 3, 1, 2).double()
        else:
            idx = _idx(N, h, w)
            A = _nchw(B.x_hi[i], idx, N, h, w, L.cin)
            Wf = eng.w_hi[i][:, :K].double()
            if not eng.fast:
                A = A + _nchw(B.x_lo[i], idx, N, h, w, L.cin)
                Wf = Wf + eng.w_lo[i][:, :K].double()
            Wf = Wf.view(L.cout, k, k, L.cin).permute(0, 3, 1, 2)
        ref = F.conv2d(A, Wf, None if L.bn else conv.bias.detach().double(), padding=(k - 1) // 2)
        del A
        tol = 2e-5 + 5e-9 * K                     # the suite's tensor-core bound
        if not L.first and not B.splits[i] and not (L.bn and eng._fuse_eval_layer(L)):
            err = (_nchw(B.y[i], idx, N, h, w, L.cout) - ref).abs().max() / ref.abs().max()
            assert err < tol, (L.block_ind, "y", float(err))
        if not L.bn:
            continue
        sc, sh = B.stat[i]["scale"].double().view(1, -1, 1, 1), B.stat[i]["shift"].double().view(1, -1, 1, 1)
        y = ref * sc + sh
        z = torch.where(y > 0, y, L.slope * y)
        size = (ref.abs() * sc.abs()).max() + sh.abs().max()       # the largest term before the activation
        del y
        for (ci, c0, kind) in L.dests:
            want = _route(z, kind)
            _n, C, ho, wo = want.shape
            pidx, sel = _idx(N, ho, wo), torch.arange(c0, c0 + C, device=DEV)
            got = _nchw(B.x_hi[ci], pidx, N, ho, wo, C, sel) + _nchw(B.x_lo[ci], pidx, N, ho, wo, C, sel)
            err = (got - want).abs().max() / size
            assert err < tol, (L.block_ind, kind, float(err))


@pytest.fixture(scope="module")
def fast_eval_model(cfg_path):
    """the fast network in eval mode, its running statistics those of one training batch (momentum 1)"""
    m = _model(cfg_path, "fast")
    bns = [x for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.momentum = 1.0
    with torch.no_grad():
        m(synth.images(2, 416, 416, seed=5).cuda())
    for bn in bns:
        bn.momentum = 0.1
    return m.eval()


@pytest.mark.parametrize("geo", [(1, 416, 416), (3, 608, 608)], ids=["1x416x416", "3x608x608"])
def test_fast_eval_forward_layers_match_fp64(fast_eval_model, geo):
    N, H, W = geo
    m = fast_eval_model
    eng = m._engine
    with torch.no_grad():
        m(synth.images(N, H, W, seed=N + H).cuda())
    torch.cuda.synchronize()
    _check_inference(eng, eng.buffers(N, H, W, False), N, H, W)


@pytest.mark.parametrize("size", [416, 672])
def test_fast_predictor_layers_match_fp64(fast_eval_model, size):
    """the pose predictor's split-K forward (its private Buffers) in fast mode, per layer, and its logits against the model's
    unsplit fast forward of the same input"""
    m = fast_eval_model
    eng = m._engine
    pred = PosePredictor(m, synth.box_points(with_center=False).T.astype(np.float64), synth.intrinsics(), shape=(size, size), batch=1)
    n0 = eng.split_launches
    pred(np.random.default_rng(size).integers(0, 256, size=(1, 480, 640, 3), dtype=np.uint8))
    torch.cuda.synchronize()
    assert eng.split_launches > n0 and any(pred._bufs.splits)
    _check_inference(eng, pred._bufs, 1, size, size)
    logits = pred.logits.clone()
    with torch.no_grad():
        o_model = m(pred.input)
    rel = float((logits - o_model).abs().max() / o_model.abs().max())
    # split-K adds each split layer's fp32 partial sums in another order.  In fast mode the next layer reads only the fp16 hi part
    # of an activation, so such a last-bit difference moves a value that lies near an fp16 rounding boundary by a whole fp16 step
    # (2^-11 relative); the stack amplifies that to 2.8e-3 (416^2) and 2.3e-3 (672^2) relative on an H100 80GB HBM3 (700 W), ten
    # times the split operands' 1.4e-4 .. 2.1e-4 (test_gpu_predict.py::test_predictor_logits_match_oracle_and_model)
    assert rel < 1e-2, rel
