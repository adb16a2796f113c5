"""Cost of the multi-view fusion (ssp_fuse_views, utils.fuse_views_batched, the predictors' rig=).  All device times from CUDA
events after warm-up, median over --reps.

  * `launch`: the ssp_fuse_views call alone (its stages: the per-row PnP, the hypotheses and the selection) at C = 2 and 4 pinhole
    cameras for 1, 13 and 64 x 13 captures, the CPU tests' rigs (cameras 0.6-1.0 m from the object, 45-135 degrees apart) and 2 px
    keypoint noise, so that every capture fuses all its views; device buffers allocated once; per call.  Beside it ssp_pnp_batched
    of the same rows alone (the per-row PnP the call contains), and the difference: the fusion's own cost;
  * `pose`: the captured PosePredictor at B = 2 (416^2) with a two-camera rig against the single-camera predictor at the same batch,
    host frames.  The network is the GPU tests' posed model (constant logits that decode a box's projection), and the rig's two
    cameras share K and the extrinsics, so both views agree and the hypotheses and the LM run over two views on every call; the
    two predictors alternated, and the pair timed twice (the second round is the spread);
every row carries the card's name and power limit.
    python tools/bench_multiview.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from singleshotpose_b200 import synth, utils                                # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402
from test_multiview_cpu import P9, observe, random_object, random_rig      # noqa: E402


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _events_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def bench_launch(reps, gpu):
    from singleshotpose_b200._lib import call, ptr, stream_ptr
    for C in (2, 4):
        rng = np.random.default_rng(C)
        rig = random_rig(rng, C)
        K32, K64, D, Rr, tr = utils.rig_tensors(rig, "cuda")
        P3 = torch.from_numpy(P9).cuda()
        for G in (1, 13, 64 * 13):
            uv = torch.from_numpy(np.concatenate([observe(rig, *random_object(rng), rng) for _ in range(G)])).cuda()
            B = G * C
            ok = torch.ones(B, dtype=torch.bool, device="cuda")
            f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device="cuda")
            R, t, corners = f64(B, 3, 3), f64(B, 3), torch.empty(B, 9, 2, dtype=torch.float32, device="cuda")
            Rw, tw, cov, err = f64(G, 3, 3), f64(G, 3), f64(G, 6, 6), f64(G, C)
            views = torch.empty(G, C, dtype=torch.bool, device="cuda")
            hyp, st = (torch.empty(G, dtype=torch.int32, device="cuda") for _ in range(2))
            cw = torch.empty(B, 9, 2, dtype=torch.float32, device="cuda")
            work = f64(max(utils.fuse_work_bytes(G, C, 1), 8) // 8)
            s = stream_ptr()

            def launch():
                call("ssp_fuse_views", ptr(P3), 1, ptr(uv), ptr(ok), 9, G, C, 1, ptr(K32), ptr(K64), ptr(D), ptr(Rr), ptr(tr), 40.0, 8.0, 2.0,
                     20, ptr(R), ptr(t), ptr(corners), ptr(Rw), ptr(tw), ptr(cov), ptr(views), ptr(err), ptr(hyp), ptr(st), ptr(cw),
                     ptr(work), work.numel() * 8, s)
            for _ in range(3):
                launch()
            def pnp():
                call("ssp_pnp_batched", ptr(P3), 1, ptr(uv), ptr(K32[0]), 9, B, 20, ptr(R), ptr(t), None, s)
            for _ in range(3):
                pnp()
            ms, ms_pnp = _events_ms(launch, reps), _events_ms(pnp, reps)
            launch()
            print(json.dumps(dict(kind="launch", cameras=C, captures=G, us=round(ms * 1e3, 1), pnp_rows_us=round(ms_pnp * 1e3, 1),
                                  fusion_us=round((ms - ms_pnp) * 1e3, 1), status0=int((st == 0).sum()),
                                  mean_views=float(views.float().sum(1).mean()), gpu=gpu)), flush=True)


def bench_predictor(reps, gpu):
    from singleshotpose_b200.predict import PosePredictor
    from test_gpu_refine_depth import CORNERS, _posed_model
    tmp = tempfile.mkdtemp()
    K = synth.intrinsics()
    m = _posed_model(write_cfg(os.path.join(tmp, "yolo-pose.cfg")))
    rig = utils.camera_rig([K, K], [np.eye(3), np.eye(3)], [np.zeros(3), np.zeros(3)])
    fr = np.random.default_rng(1).integers(0, 256, size=(2, 480, 640, 3)).astype(np.uint8)
    base = PosePredictor(m, CORNERS, K, shape=(416, 416), batch=2)
    fused = PosePredictor(m, CORNERS, None, shape=(416, 416), batch=2, rig=rig, conf_thresh=0.0)
    for _ in range(3):
        base(fr); r = fused(fr)
    torch.cuda.synchronize()
    fused_views = int(r["views"].sum())
    for i in range(2):
        b = _events_ms(lambda: base(fr), reps)
        f = _events_ms(lambda: fused(fr), reps)
        print(json.dumps(dict(kind="pose", B=2, cameras=2, fused_views=fused_views, round=i, single_ms=round(b, 4), rig_ms=round(f, 4),
                              rig_minus_single_us=round((f - b) * 1e3, 1), gpu=gpu)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    gpu = _gpu_name()
    bench_launch(a.reps, gpu)
    bench_predictor(a.reps, gpu)


if __name__ == "__main__":
    main()
