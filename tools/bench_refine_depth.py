"""Cost of the depth refinement (ssp_refine_depth, utils.refine_depth_batched, the predictors' mesh= / meshes=).  All device times
from CUDA events after warm-up, median over --reps.

  * `launch`: ssp_refine_depth alone at n = 1, 13 and 256 problems, a 6002-vertex mesh (synth.closed_mesh), 640 x 480 depth frames
    rendered at 4 object poses (oracle/refine_depth_ref.py's renderer, a table plane behind the object), 10 iterations, input poses
    perturbed as the CPU value test perturbs them (up to 3 cm along the ray, 5 mm across, 5 degrees); per launch;
  * `pose`: the captured PosePredictor at B = 1 (416^2, random weights) with mesh= against without, host frames and host depth;
  * `instances`: the captured InstancePosePredictor at B = 1 and 8 (416^2, 13 classes, each a 6002-vertex mesh, 32 slots, random
    weights at conf_thresh 0.02, so the slots are full), with meshes= against without;
the two predictors of a pair alternated, and each pair timed twice (the second round is the spread); then the card's name and
power limit.
    python tools/bench_refine_depth.py [--reps 50]
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

from oracle.pose_filter_ref import so3_exp                                  # noqa: E402
from oracle.refine_depth_ref import render_depth_ref                        # noqa: E402
from singleshotpose_b200 import synth, utils                                # noqa: E402
from singleshotpose_b200._lib import call, ptr, stream_ptr                  # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402

NC = 13
SCALE = 0.001


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


def _scene(V, F, K, R, t):
    Pc = np.concatenate([V @ R.T + t, [[-2, -2, t[2] + 0.06], [2, -2, t[2] + 0.06], [2, 2, t[2] + 0.06], [-2, 2, t[2] + 0.06]]])
    Fs = np.concatenate([F, np.array([[0, 1, 2], [0, 2, 3]]) + len(V)])
    return render_depth_ref(Pc, Fs, K, 640, 480, SCALE)


def _perturb(R, t, rng):
    ray = t / np.linalg.norm(t)
    side = np.cross(ray, rng.normal(size=3))
    side /= np.linalg.norm(side)
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    return so3_exp(ax * np.radians(rng.uniform(0, 5))) @ R, t + ray * rng.uniform(-0.03, 0.03) + side * rng.uniform(0, 0.005)


def bench_launch(reps):
    V, F = synth.closed_mesh()
    K = synth.intrinsics()
    Rs, ts = synth.object_poses(4, seed=3)
    frames = np.stack([_scene(V, F, K, Rs[i], ts[i]) for i in range(4)])
    model, offsets, diam = utils.refine_model_table({0: (V, F)}, 1, "cuda")
    Kd = torch.from_numpy(K).cuda()
    rng = np.random.default_rng(0)
    for n in (1, 13, 256):
        P = [_perturb(Rs[i % 4], ts[i % 4], rng) for i in range(n)]
        R = torch.from_numpy(np.stack([p[0] for p in P])).cuda()
        t = torch.from_numpy(np.stack([p[1] for p in P])).cuda()
        D = torch.from_numpy(frames[np.arange(n) % 4].view(np.int16)).cuda()
        cls = torch.zeros(n, dtype=torch.int32, device="cuda")
        Ro, to = torch.empty_like(R), torch.empty_like(t)
        pts, st = torch.empty(n, dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
        rmse = torch.empty(n, dtype=torch.float64, device="cuda")
        s = stream_ptr()

        def launch():
            call("ssp_refine_depth", ptr(D), 640, 480, SCALE, ptr(Kd), None, ptr(model), ptr(offsets), ptr(diam), 1, ptr(cls), n, 1, None, ptr(R),
                 ptr(t), 10, 0.5, 0.02, ptr(Ro), ptr(to), ptr(pts), ptr(rmse), ptr(st), s)
        for _ in range(3):
            launch()
        ms = _events_ms(launch, reps)
        row = dict(kind="launch", n=n, vertices=len(V), iters=10, us=round(ms * 1e3, 1), status0=int((st == 0).sum()),
                   mean_points=float(pts.double().mean()))
        print(json.dumps(row), flush=True)


def _pair(make, frames, depth, reps):
    base, ref = make(False), make(True)
    for _ in range(3):
        base(frames); ref(frames, depth=depth)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(2):
        b = _events_ms(lambda: base(frames), reps)
        r = _events_ms(lambda: ref(frames, depth=depth), reps)
        rounds.append((b, r))
    return rounds


def bench_predictors(reps):
    from singleshotpose_b200.darknet import Darknet as Single
    from singleshotpose_b200.darknet_multi import Darknet as Multi
    from singleshotpose_b200.predict import PosePredictor
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    tmp = tempfile.mkdtemp()
    K = synth.intrinsics()
    V, F = synth.closed_mesh()
    corners = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    depth1 = _scene(V, F, K, *[a[0] for a in synth.object_poses(1, seed=3)])
    torch.manual_seed(0)
    single = Single(write_cfg(os.path.join(tmp, "yolo-pose.cfg"))).cuda().eval()
    rng = np.random.default_rng(1)
    fr = rng.integers(0, 256, size=(1, 480, 640, 3)).astype(np.uint8)
    make = lambda m: PosePredictor(single, corners, K, shape=(416, 416), batch=1, **(dict(mesh=(V, F)) if m else {}))
    for i, (b, r) in enumerate(_pair(make, fr, depth1[None], reps)):
        print(json.dumps(dict(kind="pose", B=1, round=i, plain_ms=round(b, 4), refined_ms=round(r, 4), refine_minus_plain_us=round((r - b) * 1e3, 1))),
              flush=True)
    torch.manual_seed(0)
    multi = Multi(write_cfg(os.path.join(tmp, "yolo-pose-multi.cfg"), multi=True)).cuda().eval()
    meshes = {c: synth.closed_mesh(seed=c) for c in range(NC)}
    objects = {c: utils.get_3D_corners(np.c_[v, np.ones((len(v), 1))].T) for c, (v, _f) in meshes.items()}
    for B in (1, 8):
        fr = rng.integers(0, 256, size=(B, 480, 640, 3)).astype(np.uint8)
        depth = np.repeat(depth1[None], B, 0)
        make = lambda m: InstancePosePredictor(multi, objects, K, shape=(416, 416), batch=B, conf_thresh=0.02, max_instances=32,
                                               **(dict(meshes=meshes) if m else {}))
        for i, (b, r) in enumerate(_pair(make, fr, depth, reps)):
            print(json.dumps(dict(kind="instances", B=B, slots=32, round=i, plain_ms=round(b, 4), refined_ms=round(r, 4),
                                  refine_minus_plain_us=round((r - b) * 1e3, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    bench_launch(a.reps)
    bench_predictors(a.reps)
    print(json.dumps(dict(gpu=_gpu_name())))


if __name__ == "__main__":
    main()
