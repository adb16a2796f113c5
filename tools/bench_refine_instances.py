"""Cost of refining a rig's world instances with depth-pixel ownership (ssp_refine_instances_rig, InstancePosePredictor's rig= with
meshes=).  All device times from CUDA events after warm-up, median over --reps, two rounds (the second is the spread).

  * `launch`: ssp_refine_instances_rig alone at G = 1 capture, C = 1, 2, 4, 8 and 16 cameras and M = 1, 8, 32 and 256 world slots,
    a 6002-vertex mesh with its 12000 faces (synth.closed_mesh), 640 x 480 depth frames of a pile of 6 instances on a table
    (tests/test_refine_instances_cpu.py's scenes; slot w starts near instance w % 6, moved up to 1 cm and 3 degrees), 10
    iterations; alternated call by call with ssp_refine_depth_rig over the same slots, so the cost of ownership (the draws and the
    per-iteration launches) is the difference;
  * `instances`: the captured InstancePosePredictor(rig) of C = 2 and 4 cameras at B = 2C (416^2, random weights, conf_thresh 0 so
    every one of the 32 slots per frame is a detection), with meshes= against without, host frames and host depth, alternated call
    by call;
then the card's name and power limit.
    python tools/bench_refine_instances.py [--reps 30]
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
from test_refine_instances_cpu import pile_depth, pile_poses               # noqa: E402
from test_refine_rig_cpu import make_rig, perturb_world                     # noqa: E402

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
    meshes = utils.check_instance_meshes({0: (V, F)}, 1)
    model, offsets, diam = utils.refine_model_table(meshes, 1, "cuda")
    faces, foff, max_faces = utils.refine_face_table(meshes, 1, "cuda")
    table = torch.from_numpy(utils.mesh_box_table(meshes, 1)).cuda()
    s = stream_ptr()
    for C in (1, 2, 4, 8, 16):
        rng = np.random.default_rng(C)
        rig = make_rig(rng, C)
        truth = pile_poses(rng, 6)
        D = torch.from_numpy(pile_depth(rig, truth, noise=True).view(np.int16)).cuda()
        _K32, K64, Dd, Rr, tr = utils.rig_tensors(rig, "cuda")
        for M in (1, 8, 32, 256):
            P = [perturb_world(*truth[w % 6], rng, move=0.01, angle_deg=3.0) for w in range(M)]
            R = torch.from_numpy(np.stack([p[0] for p in P])).cuda()
            t = torch.from_numpy(np.stack([p[1] for p in P])).cuda()
            cls = torch.zeros(M, dtype=torch.int32, device="cuda")
            f64 = lambda *sh: torch.empty(*sh, dtype=torch.float64, device="cuda")
            i32 = lambda *sh: torch.empty(*sh, dtype=torch.int32, device="cuda")
            o = (f64(M, 3, 3), f64(M, 3), i32(M), f64(M), i32(M), i32(M, C), f64(M, C), i32(M, C),
                 torch.empty(C, M, 9, 2, dtype=torch.float32, device="cuda"), torch.empty(C, 480, 640, dtype=torch.int16, device="cuda"))
            work = torch.empty(utils.refine_instances_work_bytes(1, C, M, 640, 480) // 8, dtype=torch.float64, device="cuda")
            o1 = (f64(M, 3, 3), f64(M, 3), i32(M), f64(M), i32(M), i32(M, C), f64(M, C), torch.empty(C, M, 9, 2, dtype=torch.float32, device="cuda"))

            def owned():
                call("ssp_refine_instances_rig", ptr(D), 640, 480, SCALE, C, ptr(K64), ptr(Dd), ptr(Rr), ptr(tr), ptr(model), ptr(offsets),
                     ptr(diam), ptr(faces), ptr(foff), max_faces, ptr(table), 9, 1, ptr(cls), 1, M, None, None, ptr(R), ptr(t), 10, 0.5, 0.02,
                     *(ptr(x) for x in o), ptr(work), work.numel() * 8, s)

            def per_slot():
                call("ssp_refine_depth_rig", ptr(D), 640, 480, SCALE, C, ptr(K64), ptr(Dd), ptr(Rr), ptr(tr), ptr(model), ptr(offsets), ptr(diam),
                     ptr(table), 9, 1, ptr(cls), 1, M, None, None, ptr(R), ptr(t), 10, 0.5, 0.02, *(ptr(x) for x in o1), s)
            fns = [owned, per_slot]
            for _ in range(3):
                for fn in fns:
                    fn()
            for rnd in range(2):
                ms = _alternate_ms(fns, reps)
                print(json.dumps(dict(kind="launch", C=C, M=M, vertices=len(V), faces=len(F), iters=10, round=rnd, owned_us=round(ms[0] * 1e3, 1),
                                      per_slot_us=round(ms[1] * 1e3, 1), status0=int((o[4] == 0).sum()), per_slot_status0=int((o1[4] == 0).sum()),
                                      hidden=int(o[7].sum()))), flush=True)


def bench_predictor(reps):
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    tmp = tempfile.mkdtemp()
    V, F = synth.closed_mesh()
    corners = utils.get_3D_corners(np.c_[V, np.ones((len(V), 1))].T)
    torch.manual_seed(0)
    m = Darknet(write_cfg(os.path.join(tmp, "yolo-pose.cfg"))).cuda().eval()
    for C in (2, 4):
        rng = np.random.default_rng(C)
        rig = make_rig(rng, C)
        B = 2 * C
        fr = rng.integers(0, 256, size=(B, 480, 640, 3)).astype(np.uint8)
        depth = np.concatenate([pile_depth(rig, pile_poses(rng, 6), noise=True)] * 2)
        kw = dict(shape=(416, 416), batch=B, rig=rig, conf_thresh=0.0, max_instances=32)
        base = InstancePosePredictor(m, {0: corners}, None, **kw)
        ref = InstancePosePredictor(m, {0: corners}, None, meshes={0: (V, F)}, **kw)
        fns = [lambda: base(fr), lambda: ref(fr, depth=depth)]
        for _ in range(3):
            for fn in fns:
                fn()
        for rnd in range(2):
            b, r = _alternate_ms(fns, reps)
            print(json.dumps(dict(kind="instances", C=C, B=B, round=rnd, world_count=ref._last.fi["world_count"].tolist(), plain_ms=round(b, 4),
                                  refined_ms=round(r, 4), refine_minus_plain_us=round((r - b) * 1e3, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=_gpu_name())), flush=True)
    bench_launch(a.reps)
    bench_predictor(a.reps)
    print(json.dumps(dict(gpu=_gpu_name())))


if __name__ == "__main__":
    main()
