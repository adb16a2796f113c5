"""The multi-object network (yolo-pose-multi.cfg, BASELINE.json configs[3]) pinned like the single-object one.

The two networks share the backbone; the multi-object head is 1024 -> 160 channels with a bias (5 anchors x 32), so its forward,
data gradient and weight gradient run on the per-tap tensor-core kernels with one full 128-channel and one partial 32-channel
tile, and at the training batch (32) the weight gradient's K range is split over a thread-block cluster.  Here:

* every GEMM of a real training step against fp64 (the checks and bounds of test_gpu_train_geometry.py), at batch 32 over the
  whole multi-scale schedule (dataset_multi.py: 320 to 608 pixels), with the head's plumbing pinned bit for bit: the logits are
  its y plane, its dY plane is the loss-scaled fp16 loss gradient, and its bias gradient is the fp64 sum of that gradient;
* the loss and its gradient against the oracle on the device's own logits;
* the whole batch-32 step against the CPU oracle (slow);
* the weight gradients against a cuDNN noise floor measured in the test;
* the fused SGD step's operand planes against a re-pack of the same master weights;
* the pose predictor's split-K inference forward, layer by layer."""
import copy
import gc

import numpy as np
import pytest
import torch

from oracle import region_loss_multi_ref as RM
from oracle.darknet_ref import RefDarknet
from singleshotpose_b200 import FlatSGD, _lib, synth
from singleshotpose_b200.darknet_multi import Darknet
from singleshotpose_b200.predict_multi import MultiPosePredictor
from singleshotpose_b200.region_loss_multi import RegionLoss
from test_gpu_network import _grad_errors, _rel
from test_gpu_region_edges import MARGIN_CONF, MARGIN_OBJ, MARGIN_TCONF, margins, oracle as region_oracle
from test_gpu_train_geometry import (BANDT_STEP, DEV, _channels, _check_dgrad, _check_forward, _check_inference, _check_invariants,
                                     _check_l0, _check_wgrad, _idx)

pytestmark = pytest.mark.gpu
A = synth.MULTI_ANCHORS

# (N, H, W) and the cluster split of the head's weight gradient (160 x 1024: tiles = 2 co x 8 ci, _wgrad_split) the case is there
# for.  Batch 32 over the whole schedule: 320 (61 k-blocks) runs it unsplit, 352-448 split 2, 480-608 (128-200 k-blocks) split 4;
# batch 3 at 320 and 608 gives partial tiles at every layer, batch 1 the smallest step
GEOMS = [((32, s, s), 1 if s == 320 else 2 if s <= 448 else 4) for s in range(320, 609, 32)] + [
    ((3, 320, 320), 1), ((3, 608, 608), 1), ((1, 416, 416), 1)]
# the single-term forward (SSP_PRECISION=fast): batch 32 with the split-2 and split-4 head, and batch 3 at the largest size
FAST_GEOMS = [((32, 416, 416), 2), ((32, 608, 608), 4), ((3, 608, 608), 1)]
CASES = [("exact",) + g for g in GEOMS] + [("fast",) + g for g in FAST_GEOMS]
CASE_IDS = ["%s-%dx%dx%d-wgrad-split%d" % ((p,) + g + (s,)) for p, g, s in CASES]
# the operand-swapped kernel (SSP_IMPL_BANDT) also gets the data gradients of blocks 8 and 10, which it declines by design
# (conv_bandt.cu); unlike the single-object network's 20-channel head, the 160-channel head's forward is not routed there
BANDT_DECLINED = {("dgrad", 8), ("dgrad", 10)}


def _model(cfg, precision):
    """a random-init multi-object network whose engine runs `precision` (Engine reads SSP_PRECISION in its constructor only)"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("SSP_PRECISION", precision)
        torch.manual_seed(0)
        m = Darknet(cfg).cuda().train()
    assert m._engine.fast == (precision == "fast")
    assert m.num_anchors == 5 and m.num_classes == 13 and m.anchors == A
    return m


@pytest.fixture(scope="module")
def model(cfg_multi_path, request):
    return _model(cfg_multi_path, request.param)


def _wgrad_split(L, N, h, w, num_sms):
    """wgrad_tc.cu's K split (cluster size) of a layer's weight gradient: N tile 64 (cin <= 64) or 128, tiles = co tiles of 128 x
    ci tiles x taps, k-blocks of 64 padded-flat rows; doubled up to 8 while the tiles do not cover the SMs and every split keeps at
    least 32 k-blocks"""
    bn = 64 if L.cin <= 64 else 128
    tiles = -(-L.cout // 128) * -(-L.cin // bn) * L.taps
    kblocks = -(-N * (h + 1) * (w + 1) // 64)
    s = 1
    while s < 8 and tiles * s < num_sms and kblocks // (2 * s) >= 32:
        s *= 2
    return s


def test_sweep_covers_head_weight_gradient_splits(cfg_multi_path):
    """every case runs the head's weight gradient at the split it states, and the sweep covers split 1, 2 and 4"""
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    eng = Darknet(cfg_multi_path)._engine
    head = eng.layers[-1]
    assert (head.cin, head.cout, head.taps, head.bn) == (1024, 160, 1, False)
    for _p, (N, H, W), split in CASES:
        assert _wgrad_split(head, N, *eng.spatial(head, H, W), num_sms) == split, (N, H, W)
    assert {s for *_x, s in CASES} == {1, 2, 4}


def _step(model, N, H, W, seed):
    """one training step through the public API; returns the input, the logits (their gradient retained), the targets, the loss,
    the step's buffers and the number of operand-swapped launches"""
    eng = model._engine
    # a training step's buffers take up to 8 GiB at batch 32, 608^2, and the engine caches those of four shapes: keep only this
    # case's, and hand back what earlier tests left (a torn-down network is a model <-> engine cycle, freed by the collector only)
    eng._buffers.clear()
    gc.collect()
    torch.cuda.empty_cache()
    lib = _lib.load()
    x = synth.images(N, H, W, seed=seed).cuda()
    tgt = synth.targets_multi(N, seed=seed + 1)
    crit = RegionLoss(anchors=model.anchors); crit.verbose = False
    torch.cuda.synchronize()
    n0 = int(lib.ssp_conv_bandt_launches())
    out = model(x)
    out.retain_grad()
    loss = crit(out, tgt, 20)
    loss.backward()
    torch.cuda.synchronize()
    return x, out, tgt, crit, loss, eng.buffers(N, H, W, True), int(lib.ssp_conv_bandt_launches()) - n0


def _check_head(eng, B, L, conv, out, N, H, W):
    """the head's plumbing: logits = y plane, dY = fp16(g grad_scale), bias gradient = sum of g"""
    h, w = eng.spatial(L, H, W)
    idx = _idx(N, h, w)
    assert out.shape == (N, L.cout, h, w) == (N, 5 * 32, H // 32, W // 32)
    # ssp_unpack_nchw copies the y plane: the same bits
    assert torch.equal(out.detach(), B.y[L.index][idx, :L.cout].view(N, h, w, L.cout).permute(0, 3, 1, 2))
    # ssp_pack_nchw: the fp32 product g * grad_scale (a power of two: exact) rounded once to fp16, saturating at +-65504, NaN kept
    g = out.grad
    want = (g * eng.grad_scale).clamp(-65504, 65504).half()
    dy = B.dy[L.index]
    assert dy.shape[1] >= L.cout
    got = dy[idx, :L.cout].view(N, h, w, L.cout).permute(0, 3, 1, 2).contiguous()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan])
    # (_check_invariants: pad rows and the columns from cout to the plane's ld are zero)
    # ssp_bias_grad_nchw: the n = N h w values of a channel are summed in fp64 (exact fp32 inputs, in any order: error <= n 2^-53
    # sum |g|, and as much for the reference sum here) and rounded once to fp32 (2^-24 relative).  An fp32 accumulation would be off
    # by up to n 2^-24 sum |g| -- at batch 32, 608^2 (n = 11552) 7e-4 of sum |g|; the bound below is 2^28 times tighter in that term
    ref = g.double().sum(dim=(0, 2, 3))
    n = N * h * w
    bound = 2.0 ** -24 * ref.abs() + 2 * n * 2.0 ** -53 * g.double().abs().sum(dim=(0, 2, 3))
    db = eng.grad_view(conv.bias).double()
    assert ((db - ref).abs() <= bound).all(), float(((db - ref).abs() - bound).max())


def _check_loss(out, tgt, crit, loss):
    """the loss and its gradient against the oracle run on the device's own logits (test_gpu_multi.py's golden-test bounds), leaving
    out the cells inside a decision margin of test_gpu_region_edges.py, where the fp32 oracle may decide the other way"""
    o = out.detach().cpu()
    B, _, H, W = o.shape
    nA = 5
    rows_conf, rows_tconf, obj_near, _rec = margins(o, tgt, True)
    near = obj_near.clone()
    for r in rows_conf | rows_tconf:
        near[r // (nA * H * W), (r // (H * W)) % nA, (r // W) % H, r % W] = True
    l_ref, info, g_ref = region_oracle(o, tgt, 20, True)
    cells = near.numel()
    print("\n%dx%dx%d loss: %d of %d cells inside the decision margins (conf %d within %g of 0.6, tconf %d within %g of 0.5, "
          "objectness %d within %g of 0.25)" % (B, H * 32, W * 32, int(near.sum()), cells, len(rows_conf), MARGIN_CONF, len(rows_tconf),
                                                MARGIN_TCONF, int(obj_near.sum()), MARGIN_OBJ))
    assert int(near.sum()) <= 1e-3 * cells
    assert crit.stats()["nGT"] == info["nGT"]
    assert float(loss.detach()) == pytest.approx(float(l_ref.detach()), rel=1e-4)
    keep = ~near.view(B, nA, 1, H, W).expand(B, nA, 32, H, W).reshape(B, nA * 32, H, W)
    err = (out.grad.cpu() - g_ref).abs()[keep].max()
    assert err <= 1e-4 * g_ref.abs().max(), float(err / g_ref.abs().max())


@pytest.mark.parametrize("model, geo, split", CASES, ids=CASE_IDS, indirect=["model"])
def test_multi_train_step_gemms_match_fp64(model, geo, split):
    N, H, W = geo
    x, out, tgt, crit, loss, B, bandt = _step(model, N, H, W, seed=H + W + N)
    eng = model._engine
    precision = "fast" if eng.fast else "exact"
    subset = N >= 32
    mods = eng.conv_modules()
    head = eng.layers[-1]
    assert eng._conv_impl(head) == _lib.IMPL_TC2
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
        sel = _channels(L.cout, subset)
        if L is head:                     # the whole partial 32-channel tile of the head
            sel = torch.unique(torch.cat([sel, torch.arange(128, L.cout, device=DEV)]))
        if _check_forward(eng, B, L, N, h, w, idx, sel, conv, bn):
            sees_lo.append(L.block_ind)
        _check_dgrad(eng, B, L, N, h, w, idx, _channels(L.cin, subset), master)
        _check_wgrad(eng, B, L, N, h, w, idx, sel, conv)
        _check_invariants(B, L, idx)
    _check_head(eng, B, head, mods[head.index][0], out, N, H, W)
    _check_loss(out, tgt, crit, loss)
    if eng.fast:
        print("\n%dx%dx%d fast: the three-term reference is outside the bound at %d of %d GEMM layers: blocks %s"
              % (N, H, W, len(sees_lo), len(eng.layers) - 1, sees_lo))
        assert sees_lo                 # the single-term bound is tight enough to tell the two modes apart
    routed = {("fwd", L.block_ind) for L in eng.layers if not L.first and eng._conv_impl(L) == _lib.IMPL_BANDT}
    routed |= {("dgrad", L.block_ind) for L in eng.layers if not L.first and L.cin <= 128}
    assert bandt == len(BANDT_STEP[precision]), "%d operand-swapped launches, %d expected: a silent fall-back" % (bandt, len(BANDT_STEP[precision]))
    assert routed == BANDT_STEP[precision] | BANDT_DECLINED


# ---------------------------------------------------------------------------------------------------- the whole step, the oracle
@pytest.mark.slow
def test_batch32_multi_train_step_matches_oracle(cfg_multi_path):
    """BASELINE configs[3] -- yolo-pose-multi.cfg, batch 32, 416x416, train-mode BN, RegionLoss(epoch 20) -- against the CPU oracle:
    logits at 1e-3 overall and 2e-3 per image, the loss at 1e-3"""
    torch.manual_seed(0)
    ref = RefDarknet(cfg_multi_path).train()
    torch.manual_seed(0)
    dut = Darknet(cfg_multi_path).cuda().train()
    x, tgt = synth.images(32, seed=100), synth.targets_multi(32, seed=200)
    with torch.no_grad():
        o_ref = ref(x)
    l_ref, _info = RM.region_loss_multi_ref(o_ref, tgt, 20, A)
    crit = RegionLoss(anchors=dut.anchors); crit.verbose = False
    o = dut(x.cuda())
    loss = crit(o, tgt, 20)
    assert o.shape == (32, 160, 13, 13)
    assert _rel(o.detach().cpu(), o_ref) < 1e-3
    per_img = (o.detach().cpu() - o_ref).flatten(1).abs().max(dim=1).values / o_ref.flatten(1).abs().max(dim=1).values
    assert float(per_img.max()) < 2e-3, per_img.max()                       # no single image hides behind the batch maximum
    assert float(loss.detach()) == pytest.approx(float(l_ref), rel=1e-3)


# ---------------------------------------------------------------------------------------------------- weight gradients
def test_multi_gradient_error_against_live_cudnn_noise_floor(cfg_multi_path, capsys):
    """test_gpu_network.py::test_gradient_error_against_live_cudnn_noise_floor on the multi-object network: the oracle network runs
    on the CPU and through cuDNN (fp32, TF32 off) on this GPU; per weight-gradient tensor ours must stay within 1.5x of the cuDNN
    error, or under the noise ceiling (2.5e-2 L2, 2.5e-1 max-norm), and the median ratio over the conv weights under 1.5.  The
    table is printed."""
    torch.manual_seed(0)
    ref = RefDarknet(cfg_multi_path).train()
    torch.manual_seed(0)
    dut = Darknet(cfg_multi_path).cuda().train()
    cud = copy.deepcopy(ref).cuda().train()
    x, tgt = synth.images(2, seed=0), synth.targets_multi(2, seed=1)
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        o_ref = ref(x); RM.region_loss_multi_ref(o_ref, tgt, 20, A)[0].backward()
        o_cud = cud(x.cuda()); RM.region_loss_multi_ref(o_cud.cpu(), tgt, 20, A)[0].backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    crit = RegionLoss(anchors=dut.anchors); crit.verbose = False
    o = dut(x.cuda()); crit(o, tgt, 20).backward()
    e_cud = _grad_errors(list(cud.named_parameters()), list(ref.named_parameters()))
    e_our = _grad_errors(list(dut.named_parameters()), list(ref.named_parameters()))
    lines = ["logits rel: cudnn-vs-cpu %.3e  ours-vs-cpu %.3e" % (_rel(o_cud.detach().cpu(), o_ref.detach()), _rel(o.detach().cpu(), o_ref.detach())),
             "%-28s %10s %10s | %10s %10s" % ("param", "cudnn l2", "cudnn max", "ours l2", "ours max")]
    bad = []
    for (n, cl2, cmx), (_, ol2, omx) in zip(e_cud, e_our):
        lines.append("%-28s %10.2e %10.2e | %10.2e %10.2e" % (n, cl2, cmx, ol2, omx))
        if ol2 > max(1.5 * cl2, 2.5e-2) or omx > max(1.5 * cmx, 2.5e-1):
            bad.append(n)
    ratio = float(np.median([o[1] / max(c[1], 1e-12) for c, o in zip(e_cud, e_our) if ".conv" in c[0] and c[0].endswith("weight")]))
    lines.append("median over conv weights of ours_l2 / cudnn_l2 = %.2f" % ratio)
    with capsys.disabled():
        print("\n" + "\n".join(lines))
    assert not bad, bad
    assert ratio < 1.5, ratio


# ---------------------------------------------------------------------------------------------------- the optimiser
def test_multi_sgd_step_planes_equal_repack_and_torch_optimizer(cfg_multi_path):
    """FlatSGD's fused update rewrites every layer's operand planes (w_hi / w_lo [cout][taps*cin], w_d [cin][taps*cout], the head's
    160 x 1024 and 1024 x 160 among them) with the bits a re-pack of the updated master weights gives, and updates the parameters as
    torch.optim.SGD does"""
    torch.manual_seed(1)
    a = Darknet(cfg_multi_path).cuda()
    b = copy.deepcopy(a)
    x, tgt = synth.images(2, seed=3).cuda(), synth.targets_multi(2, seed=4)
    crit = RegionLoss(anchors=a.anchors); crit.verbose = False
    opt_a = FlatSGD(a, lr=1e-3, momentum=0.9, weight_decay=0.032)
    opt_b = torch.optim.SGD(b.parameters(), lr=1e-3, momentum=0.9, dampening=0, weight_decay=0.032)
    eng = a._engine
    gemm = [L for L in eng.layers if not L.first]
    for it in range(2):
        a.train()
        opt_a.zero_grad()
        crit(a(x), tgt, 20).backward()
        for pa, pb in zip(a.parameters(), b.parameters()):          # same gradients for both optimisers
            pb.grad = pa.grad.detach().clone()
        assert (eng.w_hi[-1].shape, eng.w_d[-1].shape) == ((160, 1024), (1024, 160))
        opt_a.step()
        opt_b.step()
        planes = [(eng.w_hi[L.index], eng.w_lo[L.index], eng.w_d[L.index]) for L in gemm]
        fused = [[t.clone() for t in p] for p in planes]
        # poison the real columns, so that a plane the re-pack did not write cannot pass
        for L, (hi, lo, d) in zip(gemm, planes):
            for t, k in ((hi, L.taps * L.cin), (lo, L.taps * L.cin), (d, L.taps * L.cout)):
                t[:, :k] = float("nan")
        eng.invalidate_packed_weights()
        a.eval()
        with torch.no_grad():
            a(x)                                                     # the next forward re-packs from the master weights
        for L, p, q in zip(gemm, planes, fused):
            for name, t, u in zip(("w_hi", "w_lo", "w_d"), p, q):
                assert torch.equal(t.view(torch.int16), u.view(torch.int16)), (it, L.block_ind, name)
        for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
            assert _rel(p.detach().cpu(), q.detach().cpu()) < 1e-5, (it, n)


# ---------------------------------------------------------------------------------------------------- predictor inference
@pytest.fixture(scope="module")
def eval_model(cfg_multi_path, request):
    """the network in eval mode, its running statistics those of one training batch (momentum 1), as
    test_gpu_train_geometry.py's fast_eval_model sets them"""
    m = _model(cfg_multi_path, request.param)
    bns = [x for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.momentum = 1.0
    with torch.no_grad():
        m(synth.images(2, 416, 416, seed=5).cuda())
    for bn in bns:
        bn.momentum = 0.1
    return m.eval()


@pytest.mark.parametrize("eval_model", ["exact", "fast"], indirect=True)
@pytest.mark.parametrize("size", [416, 608])
def test_multi_predictor_layers_match_fp64(eval_model, size):
    """MultiPosePredictor's split-K forward (its private Buffers), per layer, with the 160-channel head and its bias epilogue; and
    its logits against the model's unsplit forward of the same input"""
    m = eval_model
    eng = m._engine
    pred = MultiPosePredictor(m, {0: synth.box_points(with_center=False).T.astype(np.float64)}, synth.intrinsics(), shape=(size, size), batch=1)
    n0 = eng.split_launches
    pred(np.random.default_rng(size).integers(0, 256, size=(1, 480, 640, 3), dtype=np.uint8))
    torch.cuda.synchronize()
    assert eng.split_launches > n0 and any(pred._bufs.splits)
    assert not pred._bufs.splits[-1] and eng._conv_impl(eng.layers[-1]) == _lib.IMPL_TC2
    _check_inference(eng, pred._bufs, 1, size, size)
    logits = pred.logits.clone()
    with torch.no_grad():
        o_model = m(pred.input)
    rel = float((logits - o_model).abs().max() / o_model.abs().max())
    # split-K adds the split layers' fp32 partial sums in another order: in exact mode that stays at the last bits
    # (test_gpu_predict_multi.py: 5e-4); in fast mode the next layer reads the fp16 hi part only, and a value near an fp16 rounding
    # boundary moves by a whole fp16 step (test_gpu_train_geometry.py::test_fast_predictor_layers_match_fp64: 1e-2)
    assert rel < (1e-2 if eng.fast else 5e-4), rel
