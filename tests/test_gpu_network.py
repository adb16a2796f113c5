"""GPU parity of the whole hot path through the reference-facing API (Darknet / RegionLoss) against the oracle
network on the CPU and the reference-generated golden logits.  Tolerances are the north star's: 1e-3 relative
(inf-norm over the logits) for the forward pass and the loss.  Weight gradients are checked in relative L2 at 5e-2:
the random-init network is chaotic (leaky-slope / arg-max flips), PyTorch+cuDNN fp32 on the same GPU already differs
from PyTorch-CPU by 1.5e-2 L2 and up to 2e-1 in max-norm."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle.darknet_ref import RefDarknet
from oracle import region_loss_ref as RL
from singleshotpose_b200 import Darknet, RegionLoss, FlatSGD, synth
from singleshotpose_b200._lib import call, ptr, stream_ptr

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def _populate_eval(model):
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for bn in bns:
        bn.reset_running_stats(); bn.momentum = None
    model.train()
    with torch.no_grad():
        for s in (0, 10, 11):
            model(synth.images(2, seed=s))
    for bn in bns:
        bn.momentum = 0.1


@pytest.fixture(scope="module")
def pair(cfg_path):
    torch.manual_seed(0)
    ref = RefDarknet(cfg_path)
    torch.manual_seed(0)
    dut = Darknet(cfg_path)
    for a, b in zip(ref.state_dict().values(), dut.state_dict().values()):
        assert torch.equal(a, b)                                   # identical seeded initialisation
    return ref, dut.cuda()


def test_train_forward_backward_matches_oracle_and_golden(pair, golden_dir):
    ref, dut = pair
    g = np.load(os.path.join(golden_dir, "net_b2.npz"))
    x, tgt = synth.images(2, seed=0), synth.targets(2, seed=1)
    ref.train(); dut.train()
    out_ref = ref(x)
    out = dut(x.cuda())
    assert _rel(out.detach().cpu(), out_ref.detach()) < 1e-3
    assert _rel(out.detach().cpu(), torch.from_numpy(g["train_logits"])) < 1e-3          # reference's own output
    # running statistics after one train forward (momentum 0.1, unbiased variance)
    np.testing.assert_allclose(dut.models[0][1].running_mean.cpu().numpy(), g["running_mean0"], rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(dut.models[29][1].running_var.cpu().numpy(), g["running_var29"], rtol=1e-3, atol=1e-5)
    # loss + backward
    l_ref, _ = RL.region_loss_ref(out_ref, tgt, 20)
    l_ref.backward()
    crit = RegionLoss(); crit.verbose = False
    loss = crit(out, tgt, 20)
    loss.backward()
    assert float(loss) == pytest.approx(float(l_ref), rel=1e-3)
    assert float(loss) == pytest.approx(float(g["loss"]), rel=1e-3)
    worst = 0.0
    for (n, p), (_, q) in zip(dut.named_parameters(), ref.named_parameters()):
        assert p.grad is not None and p.grad.shape == q.grad.shape, n
        worst = max(worst, float((p.grad.cpu() - q.grad).norm() / q.grad.norm()))
    assert worst < 5e-2, worst
    gn = np.array([p.grad.double().norm().item() for p in dut.parameters()])
    np.testing.assert_allclose(gn, g["grad_norms"], rtol=5e-2)                             # reference's own gradient norms
    fw = torch.from_numpy(g["first_w_grad"])
    assert float((dut.models[0][0].weight.grad.cpu() - fw).norm() / fw.norm()) < 5e-2


def test_eval_forward_matches_oracle_and_golden(pair, golden_dir):
    ref, dut = pair
    g = np.load(os.path.join(golden_dir, "net_b2.npz"))
    ref2 = copy.deepcopy(ref)
    _populate_eval(ref2)
    dut.load_state_dict(ref2.state_dict())
    ref2.eval(); dut.eval()
    x = synth.images(2, seed=0)
    with torch.no_grad():
        o_ref = ref2(x)
        o = dut(x.cuda())
    assert _rel(o.cpu(), o_ref) < 1e-3
    assert _rel(o.cpu(), torch.from_numpy(g["eval_logits"])) < 1e-3
    # batch of one, like valid.py
    with torch.no_grad():
        o1 = dut(x[:1].cuda())
    assert _rel(o1.cpu(), o_ref[:1]) < 1e-3


def test_eval_fused_epilogue_matches_unfused(cfg_path):
    """inference folds BN(running stats)+LeakyReLU into the GEMM epilogue (ssp_conv_gemm_bnact); the unfused three-kernel chain
    (conv -> bn_finalize -> bn_apply) computes the same fmaf/leaky/split per element, so logits agree to rounding."""
    torch.manual_seed(5)
    m = Darknet(cfg_path).cuda().train()
    with torch.no_grad():
        for s in (0, 10, 11):                                 # non-trivial running statistics
            m(synth.images(2, seed=s).cuda())
    m.eval()
    eng = m._engine
    for n, hw in ((1, (416, 416)), (3, (352, 480))):
        x = synth.images(n, hw[0], hw[1], seed=7).cuda()
        with torch.no_grad():
            eng.fuse_eval = True
            l0 = eng.launches; o_f = m(x); n_f = eng.launches - l0
            eng.fuse_eval = False
            l0 = eng.launches; o_u = m(x); n_u = eng.launches - l0
            eng.fuse_eval = True
        assert n_f < n_u                                      # the fused path really ran (one launch fewer per fused layer)
        assert torch.isfinite(o_f).all() and _rel(o_f, o_u) < 2e-5


def test_fast_precision_trains_and_evaluates(cfg_path, monkeypatch, capsys):
    """SSP_PRECISION=fast: the forward GEMMs run one fp16 pass instead of three (blocks 0-1 stay the exact fused unit; the next
    layer reads only its hi plane).  No 1e-3 parity -- DESIGN section 2 emulates a single fp16 pass at 3.3e-2 -- but a training
    forward + backward + FlatSGD step and an eval forward must stay finite and within 1e-1 of the CPU oracle."""
    monkeypatch.setenv("SSP_PRECISION", "fast")
    torch.manual_seed(0)
    ref = RefDarknet(cfg_path).train()
    torch.manual_seed(0)
    dut = Darknet(cfg_path).cuda().train()
    assert dut._engine.fast
    x, tgt = synth.images(2, seed=0), synth.targets(2, seed=1)
    crit = RegionLoss(); crit.verbose = False
    opt = FlatSGD(dut, lr=1e-4, momentum=0.9, weight_decay=0.0005)
    with torch.no_grad():
        o_ref = ref(x)
    opt.zero_grad()
    o = dut(x.cuda())
    crit(o, tgt, 20).backward()
    assert all(torch.isfinite(p.grad).all() for p in dut.parameters())
    opt.step()
    assert all(torch.isfinite(p).all() for p in dut.parameters())
    e_train = _rel(o.detach().cpu(), o_ref)
    ref.load_state_dict({k: v.cpu() for k, v in dut.state_dict().items()})     # the stepped weights and the running statistics
    ref.eval(); dut.eval()
    with torch.no_grad():
        o_ref = ref(x)
        o = dut(x.cuda())
    assert torch.isfinite(o).all()
    e_eval = _rel(o.cpu(), o_ref)
    with capsys.disabled():
        print("\nSSP_PRECISION=fast logits rel err vs oracle: train %.2e, eval %.2e" % (e_train, e_eval))
    assert e_train < 1e-1 and e_eval < 1e-1, (e_train, e_eval)


@pytest.mark.parametrize("hw", [(352, 480), (224, 224), (672, 672)])
def test_other_resolutions_match_reference_golden(cfg_path, golden_dir, hw):
    """multi-resolution training shapes (dataset.py:66-90) and the 672^2 test shape: train-mode logits, batch 1, vs the reference"""
    g = np.load(os.path.join(golden_dir, "net_multires.npz"))
    torch.manual_seed(0)
    m = Darknet(cfg_path).cuda().train()
    x = synth.images(1, hw[0], hw[1], seed={(352, 480): 5, (224, 224): 6, (672, 672): 7}[hw])
    with torch.no_grad():
        o = m(x.cuda())
    want = torch.from_numpy(g["logits_%dx%d" % hw])
    assert o.shape == want.shape and _rel(o.cpu(), want) < 1e-3


def test_sgd_step_matches_torch_optimizer(cfg_path):
    """FlatSGD (one fused kernel) and torch.optim.SGD on the permuted parameter views give the same update."""
    torch.manual_seed(1)
    a = Darknet(cfg_path).cuda()
    b = copy.deepcopy(a)
    x, tgt = synth.images(2, seed=3).cuda(), synth.targets(2, seed=4)
    crit = RegionLoss(); crit.verbose = False
    opt_a = FlatSGD(a, lr=1e-3, momentum=0.9, weight_decay=0.032)
    opt_b = torch.optim.SGD(b.parameters(), lr=1e-3, momentum=0.9, dampening=0, weight_decay=0.032)
    for it in range(2):
        opt_a.zero_grad()
        crit(a(x), tgt, 20).backward()
        for pa, pb in zip(a.parameters(), b.parameters()):          # same gradients for both optimisers
            pb.grad = pa.grad.detach().clone()
        opt_a.step()
        opt_b.step()
        for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
            assert _rel(p.detach().cpu(), q.detach().cpu()) < 1e-5, (it, n)
    # and the unchanged train.py pattern (torch optimiser on our permuted parameter views) trains
    opt_b.zero_grad()
    l0 = crit(b(x), tgt, 20); l0.backward(); opt_b.step()
    assert torch.isfinite(l0)


def test_other_resolution_and_weights_roundtrip(cfg_path, tmp_path):
    torch.manual_seed(2)
    m = Darknet(cfg_path).cuda().eval()
    with torch.no_grad():
        o = m(synth.images(1, 352, 480, seed=5).cuda())            # multi-resolution training shapes (dataset.py:66-90)
    assert o.shape == (1, 20, 11, 15)
    with torch.no_grad():
        o672 = m(synth.images(1, m.test_height, m.test_width, seed=6).cuda())   # valid.py evaluates at test_width x test_height = 672
    assert o672.shape == (1, 20, 21, 21) and torch.isfinite(o672).all()
    dp = torch.nn.DataParallel(m, device_ids=[0])                           # train_multi.py:387 wraps the model like this
    with torch.no_grad():
        o_dp = dp(synth.images(1, 352, 480, seed=5).cuda())
    assert torch.equal(o_dp, o) and dp.module.num_keypoints == 9
    f = str(tmp_path / "m.weights")
    m.seen = 1234
    m.save_weights(f)
    m2 = Darknet(cfg_path)
    m2.load_weights(f)
    assert int(m2.seen) == 1234
    for (n, p), (_, q) in zip(m.state_dict().items(), m2.state_dict().items()):
        if "num_batches" not in n:
            assert torch.equal(p.cpu(), q), n


def test_cpu_tensor_is_rejected(cfg_path):
    from singleshotpose_b200._lib import SspError
    m = Darknet(cfg_path)
    with pytest.raises(SspError):
        m(synth.images(1))


def test_graphed_train_step_matches_eager(cfg_path):
    """The CUDA-graph replay of the whole step produces the same losses / weights as the eager launch path."""
    from singleshotpose_b200 import GraphedTrainStep
    torch.manual_seed(4)
    a = Darknet(cfg_path).cuda().train()
    b = copy.deepcopy(a)
    x, tgt = synth.images(2, seed=8), synth.targets(2, seed=9)
    crit = RegionLoss(); crit.verbose = False
    opt_a = FlatSGD(a, lr=1e-5, momentum=0.9, weight_decay=0.01)
    opt_b = FlatSGD(b, lr=1e-5, momentum=0.9, weight_decay=0.01)
    g = GraphedTrainStep(b, RegionLoss(), opt_b, (2, 3, 416, 416), (2, 1050), 20, torch.device("cuda"), warmup=0)
    g.criterion.verbose = False
    # warm-up allocations on the eager model only; the graphed model captures from the same initial weights
    g._warmup = 1
    state = copy.deepcopy(b.state_dict())
    g.x.copy_(x); g.t.copy_(tgt)
    g.capture()
    b.load_state_dict(state)                                   # undo the warm-up + capture-time updates (capture does not execute)
    opt_b._v.zero_()
    for it in range(3):
        opt_a.zero_grad()
        la = crit(a(x.cuda()), tgt, 20); la.backward(); opt_a.step()
        if it == 1:
            g.stage(x.pin_memory(), tgt.pin_memory()); lb = g.run_staged()      # prefetch path
        else:
            lb = g(x.pin_memory(), tgt.pin_memory())
        assert float(lb) == pytest.approx(float(la), rel=2e-3), it
        if it == 0:      # identical after the first step; later steps diverge chaotically from 1e-7 differences
            for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
                assert _rel(p.detach().cpu(), q.detach().cpu()) < 1e-5, n


def test_load_weights_after_forward_refreshes_operand_planes(cfg_path, tmp_path):
    """ADVICE r1 (high): load_weights() after a forward pass must not leave the packed fp16 conv operands stale -- forward,
    load_weights, forward equals a freshly built model that loaded the same file (darknet.py:251-297)."""
    torch.manual_seed(5)
    src = Darknet(cfg_path)
    f = str(tmp_path / "w.weights")
    src.save_weights(f)
    x = synth.images(1, seed=12).cuda()
    torch.manual_seed(6)
    m = Darknet(cfg_path).cuda().eval()
    with torch.no_grad():
        before = m(x).clone()
        m.load_weights(f)
        after = m(x).clone()
    fresh = Darknet(cfg_path)
    fresh.load_weights(f)
    fresh = fresh.cuda().eval()
    with torch.no_grad():
        want = fresh(x)
    assert torch.equal(after, want)
    assert not torch.equal(before, after)


def _plain_sgd_step(opt):
    """the unfused update FlatSGD.step() is checked against: ssp_sgd_step_flat over the engine's flat buffers and the optimizer's
    momentum buffer, then a re-pack of the operand planes at the next forward"""
    eng = opt.model._engine
    if opt._v is None:
        opt._v = torch.zeros_like(eng.flat_params)
    g = opt.param_groups[0]
    call("ssp_sgd_step_flat", ptr(eng.flat_params), ptr(eng.flat_grads), ptr(opt._v), eng.flat_params.numel(),
         float(g["lr"]), float(g["momentum"]), float(g["weight_decay"]), 1.0, stream_ptr())
    eng.invalidate_packed_weights()


def test_fused_sgd_repack_and_bucketed_step_match_plain(cfg_path, monkeypatch):
    """FlatSGD's fused update + operand-plane rewrite (csrc/sgd_pack.cu), also issued bucket by bucket in reverse layer order
    (the data-parallel overlap path, world size 1 here), gives the weights AND the next forward of the unfused path
    (ssp_sgd_step_flat, re-pack at the next forward)."""
    torch.manual_seed(7)
    base = Darknet(cfg_path).cuda().train()
    x, tgt = synth.images(2, seed=13).cuda(), synth.targets(2, seed=14)
    crit = RegionLoss(); crit.verbose = False
    outs = []
    for mode in ("plain", "plain", "fused", "bucketed"):      # the second plain run measures the run-to-run noise of step 2
        m = copy.deepcopy(base)
        opt = FlatSGD(m, lr=1e-4, momentum=0.9, weight_decay=0.032)
        logits = []
        for it in range(2):
            opt.zero_grad()
            o = m(x)
            logits.append(o.detach().clone())
            crit(o, tgt, 20).backward()
            if mode == "bucketed" and it == 0:
                opt.overlap_all_reduce(4)
                assert len(opt._buckets) == 4 and opt._buckets[-1][1][0] == 0 and opt._buckets[0][1][1] == m._engine.flat_params.numel()
                assert all(a[1][0] == b[1][1] for a, b in zip(opt._buckets[:-1], opt._buckets[1:]))     # contiguous, last layers first
            opt.all_reduce_grads()
            if mode == "plain":
                _plain_sgd_step(opt)
            else:
                opt.step()
            if it == 0:
                first = [p.detach().clone() for p in m.parameters()]
        outs.append((logits, first, [p.detach().clone() for p in m.parameters()]))
    # Step 2 re-amplifies any weight difference left after step 1 (chaotic net).  Parameters that start at zero (BN beta, biases) are
    # pure sums of gradients after two steps, so their relative difference IS the step-2 gradient noise: bounded like the
    # gradient-parity tests (5e-2; the plain path against ITSELF is printed).  Everything else moves by lr * grad << its own size: 2e-3.
    floor = max(_rel(p, q) for p, q in zip(outs[1][2], outs[0][2]))
    print("plain-vs-plain step-2 noise floor (max over tensors): %.2e" % floor)
    for logits, first, params in outs[2:]:
        assert torch.equal(logits[0], outs[0][0][0])
        for p, q in zip(first, outs[0][1]):
            assert _rel(p, q) < 1e-6                          # one step: the same update up to the atomics' summation order
        assert _rel(logits[1], outs[0][0][1]) < 1e-4          # second forward used the planes the optimiser wrote
        for p, q, p0 in zip(params, outs[0][2], base.parameters()):
            zero_init = float(p0.detach().abs().max()) == 0.0
            assert _rel(p, q) < (5e-2 if zero_init else 2e-3)


def _grad_errors(model_params, ref_params):
    """per weight-gradient tensor: (||d||_2 / ||ref||_2, ||d||_inf / ||ref||_inf)"""
    out = []
    for (n, p), (_, q) in zip(model_params, ref_params):
        d = p.grad.detach().cpu().double() - q.grad.detach().cpu().double()
        out.append((n, float(d.norm() / q.grad.double().norm()), float(d.abs().max() / q.grad.double().abs().max())))
    return out


def test_gradient_error_against_live_cudnn_noise_floor(cfg_path, capsys):
    """Parameter gradients of the fp16 single-term backward, judged against a noise floor measured IN THE TEST (VERDICT r1 weak 6): the same oracle network (torch.nn, fp32, TF32 off) runs once on the
    CPU (the reference path) and once through PyTorch/cuDNN on this GPU.  The random-init network is chaotic (LeakyReLU-slope and
    max-pool arg-max flips turn 1e-4 forward differences into percent-level gradient differences), so cuDNN-fp32 itself differs
    from the CPU by ~1.5e-2 L2 per tensor (up to 2e-2 on single BN tensors); ours must stay within 1.5x of that, tensor by tensor, or
    under the noise ceiling where cuDNN happens to sit below it (2.5e-2 L2: 23 layers of 3.5e-4 quantisation noise re-amplified by the BN backward's mean
    subtraction; 2.5e-1 max-norm: single flipped activations).  The table is printed with pytest -s."""
    torch.manual_seed(0)
    ref = RefDarknet(cfg_path).train()
    torch.manual_seed(0)
    dut = Darknet(cfg_path).cuda().train()
    cud = copy.deepcopy(ref).cuda().train()
    x, tgt = synth.images(2, seed=0), synth.targets(2, seed=1)
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        o_ref = ref(x); RL.region_loss_ref(o_ref, tgt, 20)[0].backward()
        o_cud = cud(x.cuda()); RL.region_loss_ref(o_cud.cpu(), tgt, 20)[0].backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    crit = RegionLoss(); crit.verbose = False
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


@pytest.mark.slow
def test_batch64_train_step_matches_oracle(cfg_path):
    """BASELINE configs[1] itself -- batch 64, 416x416, train-mode BN, RegionLoss(epoch 20) -- against the CPU oracle: logits and loss
    at the north star's 1e-3 (the oracle step takes ~10-20 s of host time), every image checked, not a sample"""
    torch.manual_seed(0)
    ref = RefDarknet(cfg_path).train()
    torch.manual_seed(0)
    dut = Darknet(cfg_path).cuda().train()
    x, tgt = synth.images(64, seed=100), synth.targets(64, seed=200)
    with torch.no_grad():
        o_ref = ref(x)
    l_ref, parts = RL.region_loss_ref(o_ref, tgt, 20)
    crit = RegionLoss(); crit.verbose = False
    o = dut(x.cuda())
    loss = crit(o, tgt, 20)
    assert o.shape == (64, 20, 13, 13)
    assert _rel(o.detach().cpu(), o_ref) < 1e-3
    per_img = (o.detach().cpu() - o_ref).flatten(1).abs().max(dim=1).values / o_ref.flatten(1).abs().max(dim=1).values
    assert float(per_img.max()) < 2e-3, per_img.max()                       # no single image hides behind the batch maximum
    assert float(loss) == pytest.approx(float(l_ref), rel=1e-3)
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in dut.parameters())
