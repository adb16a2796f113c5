"""Cost of tracking the world instances of a rig (ssp_world_track_associate, ssp_world_track_commit).

  * Each launch on preallocated device buffers (no uploads, no allocation) with full slots: every one of the M world slots of a
    capture holds an instance and every one of the T track slots is alive (max_misses large, so none dies), for G = 1 and 13
    captures, T = 64 and 256, M = 8 and 32, without motion and with the constant-velocity filter (every filter started).
  * What tracking adds to the captured predictor: WorldTrackingPosePredictor and InstancePosePredictor(rig=...) at the same
    batch, alternated call by call, on a posed network (tests/test_gpu_refine_depth.py) whose detections fill the slots and fuse
    into world instances in every capture, so every world slot is tracked.

CUDA events, median of --runs timed calls per case, repeated --rounds times; prints the card's name and power limit, then one line
per case and round.

    python tools/bench_world_track.py [--runs 50 --rounds 2]"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))


def _median_us(fns, runs):
    """median µs of each fn in fns, the fns alternated call by call"""
    for _ in range(3):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(runs):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts[i].append(a.elapsed_time(b) * 1e3)
    return [float(np.median(t)) for t in ts]


def _launchers(G, C, T, M, motion):
    """(associate, commit): closures launching the two kernels on preallocated buffers with full slots"""
    from singleshotpose_b200._lib import call, ptr, stream_ptr
    dev = "cuda"
    rng = np.random.default_rng(G * 1000 + T + M)
    f64 = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32, device=dev)
    world_count = torch.full((G,), M, dtype=torch.int32, device=dev)
    world_cls = torch.as_tensor(np.tile(np.arange(M) % 2, (G, 1)), dtype=torch.int32, device=dev)
    t_world = torch.as_tensor(rng.uniform(-0.3, 0.3, (G, M, 3)), device=dev)
    R_world = torch.eye(3, dtype=torch.float64, device=dev).repeat(G, M, 1, 1)
    world_cov = (1e-6 * torch.eye(6, dtype=torch.float64, device=dev)).repeat(G, M, 1, 1)
    fuse_status = i32(G, M)
    world_index = torch.as_tensor(np.tile(np.arange(M), (G * C, 1)), dtype=torch.int32, device=dev)
    size = torch.tensor([0.175, 0.172], dtype=torch.float64, device=dev)
    tracks = i32(G, T, 5)
    tracks[..., 0] = 1
    tracks[..., 1] = torch.arange(T, dtype=torch.int32, device=dev)
    tracks[..., 2] = torch.arange(T, dtype=torch.int32, device=dev) % 2
    poses = f64(G, T, 12)
    poses[..., 9:] = t_world[:, torch.arange(T, device=dev) % M] + 0.01
    next_id = torch.full((G,), T, dtype=torch.int32, device=dev)
    wslot, wid, matched, track_id = i32(G, M), i32(G, M), i32(G, M), i32(G * C, M)
    filt = dt = None
    outs = [None] * 5
    if motion:
        filt = f64(G, T, 163)
        filt[..., :9] = torch.eye(3, dtype=torch.float64, device=dev).reshape(9)
        filt[..., 9:12] = poses[..., 9:]
        filt[..., 18:162] = (1e-4 * torch.eye(12, dtype=torch.float64, device=dev)).reshape(144)
        filt[..., 162] = 1.0
        dt = torch.full((G,), 1 / 30.0, dtype=torch.float64, device=dev)
        outs = [f64(G, M, 9), f64(G, M, 3), f64(G, M, 36), f64(G, M, 6), i32(G, M)]
    big = 1 << 30

    def associate():
        call("ssp_world_track_associate", G, C, T, M, ptr(world_count), ptr(world_cls), ptr(t_world), ptr(world_index), ptr(size), 2, 0.5, big,
             ptr(tracks), ptr(poses), ptr(filt), ptr(dt), 2.0, 1.0, ptr(next_id), ptr(wslot), ptr(wid), ptr(matched), ptr(track_id), stream_ptr())

    def commit():
        call("ssp_world_track_commit", G, T, M, ptr(world_count), ptr(R_world), ptr(t_world), ptr(world_cov), ptr(fuse_status), ptr(wslot),
             ptr(matched), ptr(tracks), ptr(poses), ptr(filt), 1.0, 0.5, 22.46, *map(ptr, outs), stream_ptr())
    associate()
    torch.cuda.synchronize()
    assert int(matched.sum()) == G * M, "every world slot should find its track"
    return associate, commit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    from singleshotpose_b200.cfgs import write_cfg
    from singleshotpose_b200.predict_instances import InstancePosePredictor, WorldTrackingPosePredictor
    from test_gpu_multiview import _rig2
    from test_gpu_refine_depth import CORNERS, _posed_model
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s; nvidia-smi name, power limit: %s" % (torch.cuda.get_device_name(), q.stdout.strip() or q.stderr.strip()))
    m = _posed_model(write_cfg(os.path.join(tempfile.mkdtemp(), "yolo-pose.cfg")))
    objects = {0: CORNERS}
    C = 4
    for rnd in range(args.rounds):
        for motion in (None, "constant_velocity"):
            for G in (1, 13):
                for T in (64, 256):
                    for M in (8, 32):
                        a, c = _launchers(G, C, T, M, motion)
                        ua, uc = _median_us([a, c], args.runs)
                        print("round %d  motion=%-17s G=%2d T=%3d M=%2d: associate %6.1f us, commit %6.1f us"
                              % (rnd, motion, G, T, M, ua, uc))
        rig = _rig2(False)
        for G in (1, 4):
            fr = np.random.default_rng(8).integers(0, 256, size=(2 * G, 480, 640, 3), dtype=np.uint8)
            for motion in (None, "constant_velocity"):
                kw = dict(shape=(416, 416), batch=2 * G, conf_thresh=0.5, max_instances=32, rig=rig)
                plain = InstancePosePredictor(m, objects, None, **kw)
                tracked = WorldTrackingPosePredictor(m, objects, motion=motion, max_tracks=64, **kw)
                a, b = _median_us([lambda: tracked(fr), lambda: plain(fr)], args.runs)
                r = tracked(fr)
                n, k = int(r["world_count"].sum()), int((r["world_track_id"] >= 0).sum())
                print("round %d  captured predictor C=2 G=%d M=32 motion=%-17s %d world instances, %d tracked: %.1f us tracked, %.1f us "
                      "untracked (%+.1f us)" % (rnd, G, motion, n, k, a, b, a - b))


if __name__ == "__main__":
    main()
