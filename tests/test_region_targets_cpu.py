"""The planted loss-head targets of test_gpu_region_edges.py hit the edges they are meant to, according to the CPU oracle: the
boundary centroids, the last row and column, the collisions of the multi-object image, the anchor-less box, and a margin around
every decision threshold.  Runs without a GPU, so the generator can be rehearsed anywhere."""
import numpy as np
import pytest
import torch

from oracle import region_loss_multi_ref as RM
from test_gpu_region_edges import A, K, NA, NL, margins, make_case, oracle


def _cell(row, H, W):
    return int(np.float32(row[1]) * np.float32(W)), int(np.float32(row[2]) * np.float32(H))


def _best_anchor(row, H, W):
    gw, gh = np.float32(row[19]) * np.float32(W), np.float32(row[20]) * np.float32(H)
    best_iou, best_n = 0.0, -1
    for n in range(NA):
        iou = RM.bbox_iou_ref([0, 0, A[2 * n], A[2 * n + 1]], [0, 0, float(gw), float(gh)])
        if iou > best_iou:
            best_iou, best_n = iou, n
    return best_n


@pytest.mark.parametrize("grid,B", [(7, 5), (13, 1), (26, 5), (17, 64)])
def test_single_object_targets_hit_the_edges(grid, B):
    out, tgt = make_case(B, grid, grid, False, seed=1000 * grid + B)
    t = tgt.numpy()
    for b in range(B):
        x0, y0 = t[b, 1], t[b, 2]
        gi, gj = _cell(t[b], grid, grid)
        kind = b % 4
        if kind == 0:          # exactly k / W in fp32
            assert any(x0 == np.float32(k / grid) for k in range(1, grid)) and any(y0 == np.float32(k / grid) for k in range(1, grid))
        elif kind == 1:        # one ulp below k / W
            assert any(np.nextafter(x0, np.float32(1)) == np.float32(k / grid) for k in range(1, grid))
        elif kind == 2:
            assert gi == grid - 1 and gj == grid - 1
    rows_conf, rows_tconf, obj_near, _ = margins(out, tgt, False)
    assert not rows_conf and not rows_tconf and not obj_near.any()
    _, info, _ = oracle(out, tgt, 16, False)
    assert info["nGT"] == B and info["nCorrect"] >= (B + 1) // 2          # every even image has a planted prediction
    if B > 1:
        assert float(out[1].abs().min()) == 40.0                          # a saturated image


@pytest.mark.parametrize("grid,B", [(10, 1), (13, 4), (19, 4)])
def test_multi_object_targets_hit_the_edges(grid, B):
    out, tgt = make_case(B, grid, grid, True, seed=2000 * grid + B)
    t = tgt.numpy()
    rows = t[0].reshape(50, NL)
    assert (rows[:, 1] != 0).all()                                        # 50 ground truths in image 0
    c0, c1 = _cell(rows[0], grid, grid), _cell(rows[1], grid, grid)
    n0, n1 = _best_anchor(rows[0], grid, grid), _best_anchor(rows[1], grid, grid)
    assert c0 == c1 and n0 == n1 >= 0                                     # one cell, one anchor
    assert _cell(rows[2], grid, grid) == _cell(rows[3], grid, grid) and _best_anchor(rows[2], grid, grid) != _best_anchor(rows[3], grid, grid)
    assert rows[4, 19] == 0 and _best_anchor(rows[4], grid, grid) == -1    # no anchor overlaps: python's [-1]
    rows_conf, rows_tconf, obj_near, _ = margins(out, tgt, True)
    assert not rows_conf and not rows_tconf and not obj_near.any()
    hook_out = {}

    def keep(*args):
        hook_out["r"] = RM.build_targets_multi_ref(*args)
        return hook_out["r"]
    _, info, _ = oracle(out, tgt, 16, True, build_targets=keep)
    nGT, nCorrect, coord_mask, conf_mask, cls_mask, txs, tys, tconf, tcls = hook_out["r"]
    assert nGT == int((t.reshape(B, 50, NL)[:, :, 1] != 0).sum()) and nCorrect >= 1
    gi, gj = c0
    assert float(tcls[0, n0, gj, gi]) == rows[1, 0] != rows[0, 0]          # the last ground truth on a slot wins
    assert float(txs[1][0, n0, gj, gi]) == pytest.approx(float(np.float32(rows[1, 3]) * np.float32(grid)) - gi)
    gi4, gj4 = _cell(rows[4], grid, grid)
    assert float(coord_mask[0, NA - 1, gj4, gi4]) == 1
    assert float(out.view(B, NA, 2 * K + 14, grid, grid)[0, :, 2 * K + 1:].abs().max()) > 30    # large class logits
