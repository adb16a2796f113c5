"""Cost of the consensus PnP (utils.pnp_consensus_batched, ssp_pnp_consensus) against the plain solve (ssp_pnp_batched).  All device
times from CUDA events after warm-up, median over the repetitions.

  * `solve`: one ssp_pnp_consensus launch pair against one ssp_pnp_batched launch, per launch, for n = 1, 13, 256 and 10^4 problems
    at 9 points (60 subset hypotheses) and 8 points (28).  The problems have sigma = 1 px noise and 0-3 keypoints moved by
    40-150 px, so the refinement runs in most of them;
  * `predictor`: PosePredictor and MultiPosePredictor (all 13 classes) with pnp="consensus" against pnp="plain", captured, host
    frames (640 x 480 uint8) -> device results, at B = 1 and 8; the difference is what the consensus solve costs per call.
Then the card's name and power limit.  One JSON line per measurement.
    python tools/bench_pnp_consensus.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from singleshotpose_b200 import synth                                       # noqa: E402
from singleshotpose_b200._lib import call, ptr, stream_ptr                  # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402
from singleshotpose_b200.utils import consensus_subsets, consensus_work_bytes   # noqa: E402

NC = 13


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _time(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def _problems(n, npts, seed=0):
    pr = synth.pnp_problems(n, sigma=1.0, seed=seed, with_center=npts == 9)
    rng = np.random.default_rng(seed)
    uv = pr["uv"].astype(np.float64)
    for i in range(n):
        k = int(rng.integers(0, 4))
        bad = rng.choice(npts, k, replace=False)
        ang, rad = rng.uniform(0, 2 * np.pi, k), rng.uniform(40, 150, k)
        uv[i, bad] += np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
    return pr["P3"], uv.astype(np.float32), pr["K"]


def bench_solve(reps):
    dev = "cuda"
    for npts in (9, 8):
        for n in (1, 13, 256, 10000):
            P3, uv, K = _problems(n, npts)
            tab = consensus_subsets(P3)
            P3d, uvd, Kd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (P3, uv, K.astype(np.float32)))
            R = torch.empty(n, 9, dtype=torch.float64, device=dev)
            t = torch.empty(n, 3, dtype=torch.float64, device=dev)
            p = torch.empty(n, 6, dtype=torch.float64, device=dev)
            inl = torch.empty(n, dtype=torch.int32, device=dev)
            hyp = torch.empty(n, dtype=torch.int32, device=dev)
            wb = consensus_work_bytes(npts, len(tab), n)
            work = torch.empty(wb // 8, dtype=torch.float64, device=dev)

            def plain():
                call("ssp_pnp_batched", ptr(P3d), 1, ptr(uvd), ptr(Kd), npts, n, 20, ptr(R), ptr(t), None, stream_ptr())

            def consensus():
                call("ssp_pnp_consensus", ptr(P3d), 1, ptr(uvd), ptr(Kd), npts, n, 1, None, tab.ctypes.data, len(tab), 8.0, 20, ptr(R),
                     ptr(t), ptr(p), ptr(inl), ptr(hyp), ptr(work), wb, stream_ptr())
            tp, tc = _time(plain, reps), _time(consensus, reps)
            refined = float(((hyp > 0).sum()).item()) / n
            print(json.dumps(dict(bench="solve", points=npts, hypotheses=len(tab) + 1, n=n, plain_us=round(tp, 1), consensus_us=round(tc, 1),
                                  ratio=round(tc / tp, 2), share_not_hyp0=round(refined, 3))), flush=True)


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
        for name, make in (("PosePredictor", lambda pnp: PosePredictor(single, corners, KM, batch=B, pnp=pnp)),
                           ("MultiPosePredictor", lambda pnp: MultiPosePredictor(multi, {c: corners for c in range(NC)}, KM, batch=B,
                                                                                 conf_thresh=0.02, pnp=pnp))):
            preds = {pnp: make(pnp) for pnp in ("plain", "consensus")}
            for pr in preds.values():
                pr(frames)
            res = {pnp: [] for pnp in preds}
            for _ in range(3):                                              # alternate the two in one process
                for pnp, pr in preds.items():
                    res[pnp].append(_time(lambda: pr(frames), max(reps // 3, 5)))
            tp, tc = float(np.median(res["plain"])), float(np.median(res["consensus"]))
            print(json.dumps(dict(bench="predictor", predictor=name, B=B, problems=B * (NC if name == "MultiPosePredictor" else 1),
                                  plain_us=round(tp, 1), consensus_us=round(tc, 1), extra_us=round(tc - tp, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pnp_consensus needs a CUDA device")
    bench_solve(a.reps)
    bench_predictors(a.reps)
    print(json.dumps(dict(gpu=_gpu_name())))


if __name__ == "__main__":
    main()
