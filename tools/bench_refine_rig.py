"""Cost of the rig refinement (ssp_refine_depth_rig, the predictors' rig= with mesh=).  All device times from CUDA events after
warm-up, median over --reps, two rounds (the second is the spread).

  * `launch`: ssp_refine_depth_rig alone at C = 1, 2, 4, 8 and 16 cameras and G S = 1, 13 and 256 problems (one capture, its slots
    sharing the capture's depth), a 6002-vertex mesh (synth.closed_mesh), 640 x 480 depth frames rendered in every camera with
    a table plane (tests/test_refine_rig_cpu.py's scenes), 10 iterations, start poses moved up to 2 cm and 5 degrees; per launch;
  * `single`: at C = 1 (identity extrinsics), ssp_refine_depth on the same problems, alternated launch by launch with the rig
    launch;
  * `pose`: the captured PosePredictor(rig) of 2 cameras at B = 2 and 8 (416^2, random weights), with mesh= against without,
    host frames and host depth, alternated call by call;
then the card's name and power limit.
    python tools/bench_refine_rig.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from singleshotpose_b200 import synth, utils                                # noqa: E402
from singleshotpose_b200._lib import call, ptr, stream_ptr                  # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402
from test_refine_rig_cpu import BOX, make_rig, perturb_world, random_pose, rig_depth   # noqa: E402

SCALE = 0.001


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _alternate_ms(fns, reps):
    """median event time of each fn, the fns called in turn rep by rep"""
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts[i].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in ts]


def bench_launch(reps):
    V, F = synth.closed_mesh()
    model, offsets, diam = utils.refine_model_table({0: (V, F)}, 1, "cuda")
    table = torch.from_numpy(BOX).cuda()
    s = stream_ptr()
    for C in (1, 2, 4, 8, 16):
        rng = np.random.default_rng(C)
        rig = make_rig(rng, C) if C > 1 else utils.camera_rig([synth.intrinsics()], [np.eye(3)], [np.zeros(3)])
        R_true, t_true = random_pose(rng)
        if C == 1:                                                         # the identity rig: the world frame is the camera's
            t_true = t_true + np.array([0.0, 0.0, 0.8])
        D = torch.from_numpy(rig_depth(rig, R_true, t_true, table=C > 1).view(np.int16)).cuda()
        _K32, K64, Dd, Rr, tr = utils.rig_tensors(rig, "cuda")
        for n in (1, 13, 256):
            P = [perturb_world(R_true, t_true, rng) for _ in range(n)]
            R = torch.from_numpy(np.stack([p[0] for p in P])).cuda()
            t = torch.from_numpy(np.stack([p[1] for p in P])).cuda()
            cls = torch.zeros(n, dtype=torch.int32, device="cuda")
            Ro, to = torch.empty_like(R), torch.empty_like(t)
            pts, st = torch.empty(n, dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
            rmse = torch.empty(n, dtype=torch.float64, device="cuda")
            vp, vr = torch.empty(n, C, dtype=torch.int32, device="cuda"), torch.empty(n, C, dtype=torch.float64, device="cuda")
            crn = torch.empty(C, n, 9, 2, dtype=torch.float32, device="cuda")

            def rig_launch():
                call("ssp_refine_depth_rig", ptr(D), 640, 480, SCALE, C, ptr(K64), ptr(Dd), ptr(Rr), ptr(tr), ptr(model), ptr(offsets), ptr(diam),
                     ptr(table), 9, 1, ptr(cls), 1, n, None, None, ptr(R), ptr(t), 10, 0.5, 0.02, ptr(Ro), ptr(to), ptr(pts), ptr(rmse), ptr(st),
                     ptr(vp), ptr(vr), ptr(crn), s)
            Ro1, to1 = torch.empty_like(R), torch.empty_like(t)
            pts1, st1, rmse1 = torch.empty_like(pts), torch.empty_like(st), torch.empty_like(rmse)

            def single():
                call("ssp_refine_depth", ptr(D), 640, 480, SCALE, ptr(K64), None, ptr(model), ptr(offsets), ptr(diam), 1, ptr(cls), 1, n, None,
                     ptr(R), ptr(t), 10, 0.5, 0.02, ptr(Ro1), ptr(to1), ptr(pts1), ptr(rmse1), ptr(st1), s)
            fns = [rig_launch, single] if C == 1 else [rig_launch]
            for _ in range(3):
                for fn in fns:
                    fn()
            for rnd in range(2):
                ms = _alternate_ms(fns, reps)
                row = dict(kind="launch", C=C, n=n, vertices=len(V), iters=10, round=rnd, us=round(ms[0] * 1e3, 1), status0=int((st == 0).sum()),
                           mean_points=float(pts.double().mean()))
                if C == 1:
                    row.update(single_us=round(ms[1] * 1e3, 1), single_status0=int((st1 == 0).sum()))
                print(json.dumps(row), flush=True)


def bench_predictor(reps):
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.predict import PosePredictor
    tmp = tempfile.mkdtemp()
    V, F = synth.closed_mesh()
    corners = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    torch.manual_seed(0)
    m = Darknet(write_cfg(os.path.join(tmp, "yolo-pose.cfg"))).cuda().eval()
    rng = np.random.default_rng(1)
    rig = make_rig(rng, 2)
    depth2 = rig_depth(rig, *random_pose(rng), table=True)
    for B in (2, 8):
        fr = rng.integers(0, 256, size=(B, 480, 640, 3)).astype(np.uint8)
        depth = np.concatenate([depth2] * (B // 2))
        base = PosePredictor(m, corners, None, shape=(416, 416), batch=B, rig=rig, conf_thresh=0.0)
        ref = PosePredictor(m, corners, None, shape=(416, 416), batch=B, rig=rig, conf_thresh=0.0, mesh=(V, F))
        fns = [lambda: base(fr), lambda: ref(fr, depth=depth)]
        for _ in range(3):
            for fn in fns:
                fn()
        for rnd in range(2):
            b, r = _alternate_ms(fns, reps)
            print(json.dumps(dict(kind="pose", C=2, B=B, round=rnd, plain_ms=round(b, 4), refined_ms=round(r, 4),
                                  refine_minus_plain_us=round((r - b) * 1e3, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=_gpu_name())), flush=True)
    bench_launch(a.reps)
    bench_predictor(a.reps)
    print(json.dumps(dict(gpu=_gpu_name())))


if __name__ == "__main__":
    main()
