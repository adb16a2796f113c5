"""Both loss heads (region.cu, region_multi.cu) at every grid of the multi-scale schedule, with targets planted on the edges where a
kernel's decisions go wrong: centroids exactly on a cell boundary and one fp32 ulp below it, the last row and column, saturated
logits, the epoch where the confidence term switches on, and for the multi-object head 50 ground truths in one image, two ground
truths on one cell and anchor (the last one's targets win, both count), two on one cell with different anchors, a box that overlaps
no anchor (python's best_n = -1, i.e. the last anchor) and large class logits.

Discrete outputs (nGT, nCorrect, nProposals, and which cells receive a coordinate gradient) must equal the fp32 oracle's exactly:
`make_case` nudges every logit whose corner confidence lies within 1e-4 of thresh, whose tconf lies within 1e-4 of 0.5 or whose
objectness lies within 1e-6 of 0.25, so an fp32 expf difference cannot flip a decision.  Continuous outputs (the loss parts and the
gradient) are compared with the oracle's formula evaluated in float64 on the fp32 oracle's masks and targets."""
import numpy as np
import pytest
import torch

from oracle import region_loss_multi_ref as RM
from oracle import region_loss_ref as RL
from singleshotpose_b200 import RegionLoss, synth
from singleshotpose_b200.region_loss_multi import RegionLoss as RegionLossMulti

pytestmark = pytest.mark.gpu
K, NL = 9, 21
THRESH, MARGIN_CONF, MARGIN_TCONF, MARGIN_OBJ = 0.6, 1e-4, 1e-4, 1e-6
A = synth.MULTI_ANCHORS
NA, NC_MULTI = 5, 13
SINGLE_GRIDS, MULTI_GRIDS = list(range(7, 27)), list(range(10, 20))


# ------------------------------------------------------------------------------------------------ planted targets
def _gt(rng, x0, y0, w=0.2, h=0.2, cls=0):
    row = np.zeros(NL, np.float32)
    row[0], row[1], row[2] = cls, x0, y0
    row[3:19] = np.clip(np.repeat([x0, y0], 8) + rng.uniform(-0.15, 0.15, 16), 0.01, 0.99)
    row[19], row[20] = w, h
    return row


def _edge_xy(rng, H, W, kind):
    """a centroid (fp32) of the given kind: on a boundary k / W, one ulp below it, in the last row and column, or anywhere"""
    kx, ky = int(rng.integers(1, W)), int(rng.integers(1, H))
    if kind == "boundary":
        return np.float32(kx / W), np.float32(ky / H)
    if kind == "below":
        return np.nextafter(np.float32(kx / W), np.float32(0)), np.nextafter(np.float32(ky / H), np.float32(0))
    if kind == "last":
        return np.float32((W - 1 + rng.uniform(0.05, 0.95)) / W), np.float32((H - 1 + rng.uniform(0.05, 0.95)) / H)
    return np.float32(rng.uniform(0.05, 0.95)), np.float32(rng.uniform(0.05, 0.95))


KINDS = ["boundary", "below", "last", "free"]


def _plant_prediction(out, row, b, a, H, W, nch):
    """logits at the ground truth's own cell (anchor a) that decode close to its keypoints: tconf > 0.5 occurs"""
    gi, gj = int(np.float32(row[1]) * np.float32(W)), int(np.float32(row[2]) * np.float32(H))
    for k in range(K):
        vx = float(np.float32(row[1 + 2 * k]) * np.float32(W)) - gi
        vy = float(np.float32(row[2 + 2 * k]) * np.float32(H)) - gj
        if k == 0:
            vx, vy = [float(np.log(min(max(v, 1e-3), 1 - 1e-3) / (1 - min(max(v, 1e-3), 1 - 1e-3)))) for v in (vx, vy)]
        out[b, a * nch + 2 * k, gj, gi] = vx + 0.01
        out[b, a * nch + 2 * k + 1, gj, gi] = vy - 0.01


def _record(multi):
    """a build_targets hook recording every corner confidence the oracle computed: per image the confidences of all its
    predictions (the conf_mask threshold) and per ground truth its tconf with the row of pred_corners it was read from"""
    mod = RM if multi else RL
    rec = dict(confs=[], tconf=[])

    def hook(pred_corners, *args):
        orig_s, orig_m = mod.corner_confidences_ref, mod.corner_confidence_ref
        base = pred_corners.storage_offset()

        def confs(gt, pr):
            c = orig_s(gt, pr)
            rec["confs"].append(((pr.storage_offset() - base) // (2 * K), c.clone()))
            return c

        def conf1(gt, pr):
            c = orig_m(gt, pr)
            rec["tconf"].append(((pr.storage_offset() - base) // (2 * K), float(c)))
            return c
        mod.corner_confidences_ref, mod.corner_confidence_ref = confs, conf1
        try:
            return (RM.build_targets_multi_ref if multi else RL.build_targets_ref)(pred_corners, *args)
        finally:
            mod.corner_confidences_ref, mod.corner_confidence_ref = orig_s, orig_m
    return hook, rec


def oracle(out, tgt, epoch, multi, dtype=torch.float32, build_targets=None):
    o = out.to(dtype).clone().requires_grad_(True)
    kw = dict(build_targets=build_targets) if build_targets else {}
    if multi:
        loss, info = RM.region_loss_multi_ref(o, tgt, epoch, A, **kw)
    else:
        loss, info = RL.region_loss_ref(o, tgt, epoch, **kw)
    loss.backward()
    return loss, info, o.grad


def margins(out, tgt, multi):
    """(near-threshold prediction rows, near-0.5 tconf rows, near-0.25 objectness mask) under the fp32 oracle"""
    hook, rec = _record(multi)
    oracle(out, tgt, 20, multi, build_targets=hook)
    B, _, H, W = out.shape
    nA = NA if multi else 1
    rows_conf = set()
    for r0, c in rec["confs"]:
        near = torch.nonzero((c - THRESH).abs() < MARGIN_CONF).flatten().tolist()
        rows_conf |= {r0 + int(i) for i in near}
    rows_tconf = {r % (B * nA * H * W) for r, c in rec["tconf"] if abs(c - 0.5) < MARGIN_TCONF}
    nch = out.shape[1] // nA
    obj = torch.sigmoid(out.view(B, nA, nch, H, W)[:, :, 2 * K])
    return rows_conf, rows_tconf, (obj - 0.25).abs() < MARGIN_OBJ, rec


def make_case(B, H, W, multi, seed):
    """logits and targets with the edges planted, nudged off every decision threshold of the fp32 oracle"""
    rng = np.random.default_rng(seed)
    nA, nC = (NA, NC_MULTI) if multi else (1, 1)
    nch = 2 * K + 1 + nC
    out = torch.from_numpy(rng.standard_normal((B, nA * nch, H, W)).astype(np.float32))
    tgt = np.zeros((B, 50 * NL), np.float32)
    for b in range(B):
        rows = []
        x0, y0 = _edge_xy(rng, H, W, KINDS[b % 4])
        if not multi:
            rows.append(_gt(rng, x0, y0))
        elif b == 0:
            # 50 ground truths; rows 0-1 share a cell and a box size (one anchor), rows 2-3 share a cell with different anchors, row 4
            # has gw = 0 (overlaps no anchor: the last one)
            rows += [_gt(rng, x0, y0, 0.1, 0.2, 3), _gt(rng, x0, y0, 0.1, 0.2, 7)]
            x1, y1 = _edge_xy(rng, H, W, "free")
            rows += [_gt(rng, x1, y1, 0.05, 0.07, 1), _gt(rng, x1, y1, 0.4, 0.5, 2)]
            rows.append(_gt(rng, *_edge_xy(rng, H, W, "below"), 0.0, 0.3, 5))
            while len(rows) < 50:
                rows.append(_gt(rng, *_edge_xy(rng, H, W, KINDS[len(rows) % 4]), *rng.uniform(0.02, 0.5, 2), int(rng.integers(0, nC))))
        else:
            rows += [_gt(rng, x0, y0, *rng.uniform(0.02, 0.5, 2), int(rng.integers(0, nC))) for _ in range(1 + b % 3)]
        for t, r in enumerate(rows):
            tgt[b, t * NL:(t + 1) * NL] = r
    for b in range(B):
        if b % 3 == 1:
            out[b] = torch.from_numpy(np.where(rng.random((nA * nch, H, W)) < 0.5, -40.0, 40.0).astype(np.float32))     # saturated
        if multi:
            if b % 3 != 1:
                out.view(B, nA, nch, H, W)[b, :, 2 * K + 1:] *= 15.0       # large class logits for the cross-entropy
            # the tconf of image b + 1 is read from image b's last anchor (b = B - 1 wraps to image 0)
            nb = (b + 1) % B
            nxt = tgt[nb, :NL]
            if nxt[1] != 0 and b % 2 == 0:
                _plant_prediction(out, nxt, b, nA - 1, H, W, nch)
        elif b % 2 == 0:
            _plant_prediction(out, tgt[b, :NL], b, 0, H, W, nch)
    tgt = torch.from_numpy(tgt)
    for it in range(50):
        rows_conf, rows_tconf, obj_near, _ = margins(out, tgt, multi)
        if not rows_conf and not rows_tconf and not obj_near.any():
            return out, tgt
        v = out.view(B, nA, nch, H, W)
        for r in rows_conf | rows_tconf:
            b, a, j, i = r // (nA * H * W), (r // (H * W)) % nA, (r // W) % H, r % W
            v[b, a, :2 * K, j, i] += torch.from_numpy(rng.choice([-0.02, 0.02], 2 * K).astype(np.float32))
        v[:, :, 2 * K][obj_near] += 0.01
    raise AssertionError("could not move the logits off the decision thresholds")


# ------------------------------------------------------------------------------------------------ the GPU comparison
def _compare(out, tgt, epoch, multi):
    B, _, H, W = out.shape
    bt = RM.build_targets_multi_ref if multi else RL.build_targets_ref
    kept = {}

    def keep(*args):
        kept["r"] = bt(*args)
        return kept["r"]
    _, info32, _ = oracle(out, tgt, epoch, multi, build_targets=keep)
    # the float64 evaluation of the formula on the fp32 oracle's masks and targets
    loss64, info64, grad64 = oracle(out, tgt, epoch, multi, torch.float64, lambda *args: kept["r"])
    crit = RegionLossMulti(anchors=A) if multi else RegionLoss()
    crit.verbose = False
    od = out.cuda().requires_grad_(True)
    loss = crit(od, tgt, epoch)
    loss.backward()
    st = crit.stats()
    # discrete: exactly the fp32 oracle's
    assert (st["nGT"], st["nCorrect"], st["nProposals"]) == (info32["nGT"], info32["nCorrect"], info32["nProposals"])
    nA = NA if multi else 1
    nch = out.shape[1] // nA
    g = od.grad.cpu().double().view(B, nA, nch, H, W)
    coord = (g[:, :, :2 * K] != 0).any(dim=2)
    assert torch.equal(coord, info32["coord_mask"] > 0)
    # continuous: float64 formula on the fp32 masks and targets, within 1e-5 of the largest value.  The coordinate terms add one
    # more error: the kernel forms x - tx in fp32 from operands up to M = max|logit| + max(H, W) (a linear keypoint logit against
    # gx - gi, which runs up to the grid size), so each difference carries up to 2 ulp(M) <= 4 eps M of absolute error however small
    # it is (a planted prediction sits 0.01 from its target): 4 eps M per gradient element, and for loss_x / loss_y, sums of d^2 / 2
    # over n <= K nGT terms, 4 eps M sum|d| <= 4 eps M sqrt(2 n loss)
    eps = 2.0 ** -24
    M = float(out.abs().max()) + max(H, W)
    n = K * st["nGT"]
    parts = ["loss_x", "loss_y", "loss_conf"] + (["loss_cls"] if multi else [])
    tol = {}
    for p in parts:
        ref = float(info64[p])
        tol[p] = 1e-5 * abs(ref) + (4 * eps * M * (2 * n * abs(ref)) ** 0.5 if p in ("loss_x", "loss_y") else 0.0) + 1e-12
        assert abs(st[p] - ref) <= tol[p], (p, st[p], ref)
    gr = grad64.view(B, nA, nch, H, W)
    assert (g - gr).abs().max() <= 1e-5 * gr.abs().max() + 4 * eps * M, float((g - gr).abs().max() / gr.abs().max())
    # the returned loss: the parts the epoch includes, rounded to fp32 once
    used = [p for p in parts if p != "loss_conf" or epoch > 15]
    assert abs(float(loss) - float(loss64)) <= sum(tol[p] for p in used) + eps * abs(float(loss64))


@pytest.mark.parametrize("grid", SINGLE_GRIDS)
@pytest.mark.parametrize("B", [1, 5, 64])
def test_region_loss_edges(grid, B):
    out, tgt = make_case(B, grid, grid, False, seed=1000 * grid + B)
    for epoch in (15, 16):                  # pretrain_num_epochs: the confidence loss and its gradient off, then on
        _compare(out, tgt, epoch, False)


@pytest.mark.parametrize("grid", MULTI_GRIDS)
@pytest.mark.parametrize("B", [1, 4, 64])
def test_region_loss_multi_edges(grid, B):
    out, tgt = make_case(B, grid, grid, True, seed=2000 * grid + B)
    for epoch in (15, 16):
        _compare(out, tgt, epoch, True)
