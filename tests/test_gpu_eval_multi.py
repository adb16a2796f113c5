"""GPU tests of the multi-object evaluation tail (utils_multi.evaluate_multi_poses_batched, ssp_eval_multi_select) against the
reference's valid_multi.valid() through tests/golden/eval_multi.npz and against oracle/eval_multi_ref.py."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import eval_multi_ref as EM
from singleshotpose_b200 import synth
from singleshotpose_b200.utils_multi import evaluate_multi_poses_batched, get_multi_region_boxes, projection_accuracy, get_3D_corners

pytestmark = pytest.mark.gpu
K, NC, NA, NL = 9, 13, 5, 21
A = synth.MULTI_ANCHORS


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "eval_multi.npz"))


def _mesh(n=500, seed=0):
    rng = np.random.default_rng(seed)
    half = np.array([0.038, 0.039, 0.046])
    V = np.concatenate([synth.box_points(with_center=False).astype(np.float64), rng.uniform(-1, 1, (n - 8, 3)) * half])
    V = np.c_[V, np.ones(n)].T
    return V, get_3D_corners(V)


def _evaluate(out, tgt, V, corners, thresh=0.05):
    return evaluate_multi_poses_batched(out, tgt, thresh, NC, K, NA, V, corners, synth.intrinsics())


def _angle_deg(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


def test_eval_multi_matches_reference_golden(golden):
    r = _evaluate(torch.from_numpy(golden["outputs"]).cuda(), torch.from_numpy(golden["targets"]), golden["vertices"], golden["corners3D"],
                  float(golden["conf_thresh"]))
    G = len(golden["pos"])
    assert r["box"].shape[0] == G
    assert r["image"].cpu().tolist() == list(golden["image"])
    flags = (r["fallback"].int() + 2 * r["carried"].int()).cpu().numpy()
    np.testing.assert_array_equal(flags, golden["flags"])
    pr = r["box"][:, :2 * K].cpu().numpy().reshape(G, K, 2) * np.array([640, 480], np.float32)
    np.testing.assert_allclose(pr, golden["pnp_points2d"][1::2], rtol=1e-5)
    for name, sl in (("gt", slice(0, None, 2)), ("pr", slice(1, None, 2))):
        R, t = r["R_" + name].cpu().numpy(), r["t_" + name].cpu().numpy()
        Rg, tg = golden["pnp_R"][sl], golden["pnp_t"][sl][..., 0]
        for g in range(G):
            assert _angle_deg(R[g], Rg[g]) < 1e-2, (name, g)
            assert np.abs(t[g] - tg[g]).max() * 1e3 < 1e-2, (name, g)
    np.testing.assert_allclose(r["pixel_err"].cpu().numpy(), golden["pixel_err"], rtol=1e-3)
    assert projection_accuracy(r["pixel_err"]) == list(golden["accuracy"])


def _random_case(B, seed, H=13, W=13, max_gts=3, num_classes=4):
    gen = torch.Generator().manual_seed(seed)
    out = torch.randn(B, (2 * K + 1 + NC) * NA, H, W, generator=gen)
    out[:, [18 + 32 * a for a in range(NA)]] += 1.0                     # many boxes above 0.05
    tgt = synth.targets_multi(B, seed=seed + 1, num_classes=num_classes, max_gts=max_gts)
    return out, tgt


def test_batch_equals_per_image_calls():
    out, tgt = _random_case(16, 40)
    tgt[3] = 0                                                          # an image without ground truths
    V, corners = _mesh()
    r = _evaluate(out.cuda(), tgt, V, corners)
    G, gi = r["box"].shape[0], 0
    for b in range(16):
        one = _evaluate(out[b:b + 1].cuda(), tgt[b:b + 1], V, corners)
        n = one["box"].shape[0]
        for key in ("box", "fallback", "carried", "R_gt", "t_gt", "R_pr", "t_pr", "pixel_err", "cls", "gt_index"):
            assert torch.equal(r[key][gi:gi + n], one[key]), (b, key)
        gi += n
    assert gi == G


@pytest.mark.parametrize("H", [13, 26])
def test_selection_matches_oracle_random(H):
    B = 8 if H == 13 else 2
    out, tgt = _random_case(B, 50 + H, H, H)
    V, corners = _mesh()
    r = _evaluate(out.cuda(), tgt, V, corners)
    box, flags = r["box"].cpu().numpy(), (r["fallback"].int() + 2 * r["carried"].int()).cpu().numpy()
    gi, listed = 0, 0
    for b in range(B):
        res, boxes = EM.evaluate_image_multi_ref(out[b:b + 1], tgt[b].numpy(), 0.05, NC, K, A, NA, None, None, None, with_pose=False)
        listed += len(boxes)
        for x in res:
            assert flags[gi] == x["fallback"] + 2 * x["carried"], (b, gi)
            np.testing.assert_allclose(box[gi], x["box"], rtol=1e-5, atol=1e-7)
            gi += 1
    assert gi == box.shape[0] and listed > 20 * B


def test_chosen_box_is_an_element_of_get_multi_region_boxes():
    """B = 1: the box the select kernel picks is bit-equal to one of the decode kernel's boxes (one shared device function)"""
    V, corners = _mesh()
    for seed in range(4):
        out, tgt = _random_case(1, 70 + seed)
        if seed == 3:
            out[:, [18 + 32 * a for a in range(NA)]] -= 9.0                # nothing listed: the fallback box
        r = _evaluate(out.cuda(), tgt, V, corners)
        boxes = get_multi_region_boxes(out.cuda(), 0.05, NC, K, A, NA, int(tgt[0][0]), only_objectness=0)[0]
        dec = torch.tensor([[float(v) for v in bx] for bx in boxes], dtype=torch.float32)
        for g in range(r["box"].shape[0]):
            assert (dec == r["box"][g].cpu()).all(1).any(), (seed, g)
        if seed == 3:
            assert bool(r["fallback"][0])


def test_full_label_and_empty_batch():
    """a label with all 50 rows filled is evaluated in full; a batch without ground truths returns empty tensors"""
    out, tgt = _random_case(2, 90)
    tgt[1] = tgt[0, :NL].repeat(50)
    V, corners = _mesh()
    r = _evaluate(out.cuda(), tgt, V, corners)
    assert r["box"].shape[0] == int((tgt[0].view(-1, NL)[:, 1] != 0).int().cumprod(0).sum()) + 50
    assert torch.isfinite(r["box"]).all()
    e = _evaluate(out.cuda(), torch.zeros(2, 50 * NL), V, corners)
    assert all(v.shape[0] == 0 for v in e.values())


def test_end_to_end_dataset_network_eval(tmp_path, cfg_multi_path):
    """test-mode listDataset -> GpuMultiCollate -> Darknet (multi cfg, eval) -> evaluate_multi_poses_batched, against the oracle loop
    on the same network output"""
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.dataset_multi import listDataset, GpuMultiCollate
    root = str(tmp_path)
    synth.write_linemod_multi_like(root, n=3)
    paths = [os.path.join(root, "LINEMOD", o, "JPEGImages", "%06d.png" % i) for o in ("ape", "can", "duck") for i in range(3)]
    with open(os.path.join(root, "test.txt"), "w") as f:
        f.write("\n".join(paths) + "\n")
    random.seed(0)
    ds = listDataset(os.path.join(root, "test.txt"), shape=(416, 416), shuffle=False, objclass="ape", train=False)
    data, target = GpuMultiCollate("cuda")([ds[i] for i in range(len(ds))])
    torch.manual_seed(0)
    net = Darknet(cfg_multi_path).cuda().eval()
    with torch.no_grad():
        out = net(data)
    V, corners = _mesh()
    r = evaluate_multi_poses_batched(out, target.cuda(), 0.05, NC, K, NA, V, corners, synth.intrinsics())
    oc = out.detach().cpu()
    gi = 0
    box, flags = r["box"].cpu().numpy(), (r["fallback"].int() + 2 * r["carried"].int()).cpu().numpy()
    for b in range(len(ds)):
        res, _ = EM.evaluate_image_multi_ref(oc[b:b + 1], target[b].numpy(), 0.05, NC, K, A, NA, None, None, None, with_pose=False)
        for x in res:
            assert flags[gi] == x["fallback"] + 2 * x["carried"], (b, gi)
            np.testing.assert_allclose(box[gi], x["box"], rtol=1e-5, atol=1e-7)
            gi += 1
    assert gi == box.shape[0] > 0
