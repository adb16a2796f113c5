"""Cost of lens distortion in the pose solve and projection (csrc/pnp_dist.cu) against the zero-distortion kernels.  All device times
from CUDA events after warm-up, median over the repetitions.  Prints the card's name and power limit first, then one JSON line per
measurement:

  * `solve`: one ssp_pnp_dist launch against one ssp_pnp_batched launch, per launch, for n = 1, 13, 256 and 10^4 problems of the 9
    box points under the barrel calibration (k1, k2, p1, p2, k3) = (-0.3, 0.12, 1e-3, -5e-4, -0.02), the box 0.6-1.0 m away towards
    a frame corner, one keypoint moved by 40-150 px (oracle/pnp_dist_ref.corner_problems); both solve the same keypoints;
  * `consensus`: ssp_pnp_consensus_dist against ssp_pnp_consensus on the same problems (60 subset hypotheses);
  * `predictor`: PosePredictor and MultiPosePredictor (all 13 classes) with dist_coeffs against without, captured, host frames
    (640 x 480 uint8) -> device results, at B = 1 and 8; the difference is what the distortion costs per call.
    python tools/bench_pnp_dist.py [--reps 50]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_pnp_consensus import NC, _gpu_name, _time                        # noqa: E402
from oracle.pnp_dist_ref import corner_problems, dist8                      # noqa: E402
from singleshotpose_b200 import synth                                       # noqa: E402
from singleshotpose_b200._lib import call, ptr, stream_ptr                  # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402
from singleshotpose_b200.utils import consensus_subsets, consensus_work_bytes   # noqa: E402

BARREL = (-0.3, 0.12, 1e-3, -5e-4, -0.02)


def bench_solve(reps):
    dev = "cuda"
    K = synth.intrinsics()
    P3 = synth.box_points(with_center=True)
    tab = consensus_subsets(P3)
    dd = torch.from_numpy(dist8(BARREL)).to(dev)
    for n in (1, 13, 256, 10000):
        uv, _out, _r, _t = corner_problems(n, n, K, BARREL, P3)
        P3d, uvd, Kd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (P3, uv, K.astype(np.float32)))
        R = torch.empty(n, 9, dtype=torch.float64, device=dev)
        t = torch.empty(n, 3, dtype=torch.float64, device=dev)
        p = torch.empty(n, 6, dtype=torch.float64, device=dev)
        inl = torch.empty(n, dtype=torch.int32, device=dev)
        hyp = torch.empty(n, dtype=torch.int32, device=dev)
        wb = consensus_work_bytes(9, len(tab), n)
        work = torch.empty(wb // 8, dtype=torch.float64, device=dev)

        def plain():
            call("ssp_pnp_batched", ptr(P3d), 1, ptr(uvd), ptr(Kd), 9, n, 20, ptr(R), ptr(t), None, stream_ptr())

        def dist():
            call("ssp_pnp_dist", ptr(P3d), 1, ptr(uvd), ptr(Kd), ptr(dd), 9, n, 1, None, None, None, 20, ptr(R), ptr(t), None, None, stream_ptr())

        def cons():
            call("ssp_pnp_consensus", ptr(P3d), 1, ptr(uvd), ptr(Kd), 9, n, 1, None, tab.ctypes.data, len(tab), 8.0, 20, ptr(R), ptr(t), ptr(p),
                 ptr(inl), ptr(hyp), ptr(work), wb, stream_ptr())

        def cons_dist():
            call("ssp_pnp_consensus_dist", ptr(P3d), 1, ptr(uvd), ptr(Kd), ptr(dd), 9, n, 1, None, tab.ctypes.data, len(tab), 8.0, 20, ptr(R),
                 ptr(t), ptr(p), ptr(inl), ptr(hyp), ptr(work), wb, stream_ptr())
        res = {f: [] for f in (plain, dist, cons, cons_dist)}
        for _ in range(3):                                                  # alternate the pairs in one process
            for f in res:
                res[f].append(_time(f, max(reps // 3, 5)))
        tp, td, tc, tcd = (float(np.median(res[f])) for f in (plain, dist, cons, cons_dist))
        print(json.dumps(dict(bench="solve", n=n, plain_us=round(tp, 1), dist_us=round(td, 1), ratio=round(td / tp, 2))), flush=True)
        print(json.dumps(dict(bench="consensus", n=n, hypotheses=len(tab) + 1, plain_us=round(tc, 1), dist_us=round(tcd, 1),
                              ratio=round(tcd / tc, 2))), flush=True)


def bench_predictors(reps):
    from singleshotpose_b200 import Darknet
    from singleshotpose_b200.darknet_multi import Darknet as DarknetMulti
    from singleshotpose_b200.predict import PosePredictor
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    import tempfile
    tmp = tempfile.mkdtemp()
    torch.manual_seed(0)
    single = Darknet(write_cfg(os.path.join(tmp, "yolo-pose.cfg"))).cuda().eval()
    multi = DarknetMulti(write_cfg(os.path.join(tmp, "yolo-pose-multi.cfg"), multi=True)).cuda().eval()
    corners = synth.box_points(with_center=False).T.astype(np.float64)
    KM = synth.intrinsics()
    for B in (1, 8):
        frames = np.random.default_rng(B).integers(0, 256, size=(B, 480, 640, 3), dtype=np.uint8)
        for name, make in (("PosePredictor", lambda d: PosePredictor(single, corners, KM, batch=B, dist_coeffs=d)),
                           ("MultiPosePredictor", lambda d: MultiPosePredictor(multi, {c: corners for c in range(NC)}, KM, batch=B,
                                                                               conf_thresh=0.02, dist_coeffs=d))):
            preds = {"none": make(None), "barrel": make(BARREL)}
            for pr in preds.values():
                pr(frames)
            res = {k: [] for k in preds}
            for _ in range(3):                                              # alternate the two in one process
                for k, pr in preds.items():
                    res[k].append(_time(lambda: pr(frames), max(reps // 3, 5)))
            tn, tb = float(np.median(res["none"])), float(np.median(res["barrel"]))
            print(json.dumps(dict(bench="predictor", predictor=name, B=B, problems=B * (NC if name == "MultiPosePredictor" else 1),
                                  no_dist_us=round(tn, 1), dist_us=round(tb, 1), extra_us=round(tb - tn, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pnp_dist needs a CUDA device")
    print(json.dumps(dict(gpu=_gpu_name())), flush=True)
    bench_solve(a.reps)
    bench_predictors(a.reps)


if __name__ == "__main__":
    main()
