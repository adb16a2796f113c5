"""Throughput of the multi-object evaluation tail (singleshotpose_b200/utils_multi.py evaluate_multi_poses_batched): N synthetic
13x13 network outputs of the multi-object head (many boxes above the threshold) with 1-3 ground truths each, a mesh of about 6k
vertices, evaluated in batches of B.  Prints one JSON line:
  images/s and objects/s of the GPU tail, timed by wall clock around the calls of all batches and a final synchronise,
  device time per batch (CUDA events around each call),
  the reference loop (oracle/eval_multi_ref.py: the box list, the selection, cv2.solvePnP through the oracle's points and the
  numpy projection, one thread) on a bounded sample of the same images, and the card name and power limit.
    python tools/bench_eval_multi.py [--images 1024] [--batch 64] [--reps 3] [--ref-images 16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

K, NC, NA = 9, 13, 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-images", type=int, default=16)
    ap.add_argument("--vertices", type=int, default=6000)
    a = ap.parse_args()
    import torch
    from singleshotpose_b200 import synth
    from singleshotpose_b200.utils_multi import evaluate_multi_poses_batched, get_3D_corners
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_multi needs a CUDA device")
    gen = torch.Generator().manual_seed(0)
    out = torch.randn(a.images, (2 * K + 1 + NC) * NA, 13, 13, generator=gen)
    out[:, [18 + 32 * i for i in range(NA)]] += 1.0
    tgt = synth.targets_multi(a.images, seed=1, num_classes=NC, max_gts=3)
    rng = np.random.default_rng(2)
    half = np.array([0.038, 0.039, 0.046])
    V = np.concatenate([synth.box_points(with_center=False).astype(np.float64), rng.uniform(-1, 1, (a.vertices - 8, 3)) * half])
    V = np.c_[V, np.ones(len(V))].T
    corners = get_3D_corners(V)
    Kc = synth.intrinsics()
    out_d, tgt_d = out.cuda(), tgt.cuda()
    batches = [(out_d[i:i + a.batch], tgt_d[i:i + a.batch]) for i in range(0, a.images, a.batch)]
    run = lambda o, t: evaluate_multi_poses_batched(o, t, 0.05, NC, K, NA, V, corners, Kc)
    for o, t in batches[:2]:                                                # warm-up
        run(o, t)
    torch.cuda.synchronize()
    n_obj = sum(int(run(o, t)["pixel_err"].shape[0]) for o, t in batches)
    walls, dev = [], []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev = []
        for o, t in batches:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(o, t)
            e1.record()
            ev.append((e0, e1))
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
        dev.append(float(np.mean([e0.elapsed_time(e1) for e0, e1 in ev])))
    wall = min(walls)
    res = {"images": a.images, "batch": a.batch, "objects": n_obj, "vertices": a.vertices,
           "gpu_images_per_s": a.images / wall, "gpu_objects_per_s": n_obj / wall, "gpu_wall_s": walls,
           "device_ms_per_batch": dev}
    if a.ref_images:
        from oracle import eval_multi_ref as EM
        import cv2
        cv2.setNumThreads(1)
        torch.set_num_threads(1)
        P3 = np.array(np.transpose(np.concatenate((np.zeros((3, 1)), corners[:3]), axis=1)), dtype="float32")
        Kf = np.array(Kc, dtype="float32")
        t0 = time.perf_counter()
        n_ref = 0
        for b in range(a.ref_images):
            res_b, _ = EM.evaluate_image_multi_ref(out[b:b + 1], tgt[b].numpy(), 0.05, NC, K, synth.MULTI_ANCHORS, NA, None, None, None,
                                                   with_pose=False)
            for x in res_b:                                                  # the reference's pnp (cv2) and projection per object
                poses = []
                for uv in (x["uv_gt"], x["uv_pr"]):
                    _, rv, tv = cv2.solvePnP(P3, np.ascontiguousarray(uv.reshape(-1, 1, 2)), Kf, np.zeros((8, 1), "float32"),
                                             flags=cv2.SOLVEPNP_ITERATIVE)
                    poses.append((cv2.Rodrigues(rv)[0], tv))
                EM.pixel_error(V, poses[0][0], poses[0][1], poses[1][0], poses[1][1], Kc)
                n_ref += 1
        dt = time.perf_counter() - t0
        res.update(ref_images=a.ref_images, ref_objects=n_ref, ref_1thread_images_per_s=a.ref_images / dt,
                   ref_1thread_objects_per_s=n_ref / dt)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        res["gpu"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        res["gpu"] = torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
