"""Cost of the instance fusion across a rig (ssp_fuse_instances).

  * One ssp_fuse_instances launch sequence on preallocated device buffers (no uploads, no allocation): at C = 2 and 4 cameras,
    M = 8 and 32 slots and 1 / 13 captures, on seeded scenes (2 classes, 1-5 instances each, missed and spurious detections:
    sparse slots) and on the worst case, the detections of a random multi-object network at conf_thresh 0.02 (every slot full)
    repeated over the captures.  Each case also times the same call with every count zero, which is the per-row stage over every
    slot (empty ones included) plus an empty fusion.
  * What a rig adds to the captured InstancePosePredictor: the predictor with the rig and the one-camera predictor at the same
    batch, alternated call by call.

CUDA events, median of --runs timed calls per case, repeated --rounds times; prints one line per case and round.

    python tools/bench_fuse_instances.py [--runs 30 --rounds 2]"""
import argparse
import os
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


def _launcher(table, uv, cls, count, rig):
    """a closure that launches ssp_fuse_instances on preallocated buffers"""
    from singleshotpose_b200._lib import call, ptr, stream_ptr
    from singleshotpose_b200.utils import fuse_instances_outputs, fuse_instances_work_bytes, rig_tensors
    B, M, npts = uv.shape[:3]
    C = len(rig.K)
    dev = uv.device
    K32, K64, D, Rr, tr = rig_tensors(rig, dev)
    o = fuse_instances_outputs(B, C, M, npts, dev)
    work = torch.empty(max(fuse_instances_work_bytes(B // C, C, M), 8) // 8, dtype=torch.float64, device=dev)
    outs = [ptr(v) for v in o.values()]
    return lambda cnt=count: call("ssp_fuse_instances", ptr(table), table.shape[0], ptr(uv), ptr(cls), ptr(cnt), npts, B // C, C, M, ptr(K32),
                                  ptr(K64), ptr(D), ptr(Rr), ptr(tr), 40.0, 8.0, 2.0, 20, *outs, ptr(work), work.numel() * 8, stream_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    from singleshotpose_b200 import utils
    from singleshotpose_b200.cfgs import write_cfg
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import InstancePosePredictor
    from test_fuse_instances_cpu import TABLE, scene, scene_rig
    print("device: %s" % torch.cuda.get_device_name())
    cfg = write_cfg(os.path.join(tempfile.mkdtemp(), "yolo-pose-multi.cfg"), multi=True)
    torch.manual_seed(0)
    m = Darknet(cfg).cuda().eval()
    objects = {c: utils.get_3D_corners(np.c_[np.random.default_rng(c).normal(0, 0.04, (50, 3)), np.ones((50, 1))].T) for c in (0, 3, 7)}
    table_full = torch.zeros(m.num_classes, 9, 3, device="cuda")
    for c, corners in objects.items():
        table_full[c, 1:] = torch.as_tensor(corners[:3].T)
    table_scene = torch.as_tensor(TABLE).cuda()
    for rnd in range(args.rounds):
        for n_cams in (2, 4):
            rig = scene_rig(np.random.default_rng(n_cams), n_cams)
            fr = np.random.default_rng(8).integers(0, 256, size=(n_cams, 480, 640, 3), dtype=np.uint8)
            for M in (8, 32):
                with_rig = InstancePosePredictor(m, objects, None, batch=n_cams, conf_thresh=0.02, max_instances=M, rig=rig)
                plain = InstancePosePredictor(m, objects, rig.K[0], batch=n_cams, conf_thresh=0.02, max_instances=M)
                r = with_rig(fr)
                full = [r["keypoints_px"].clone(), r["cls"].clone(), r["count"].clone()]
                for G in (1, 13):
                    rng = np.random.default_rng(n_cams * 100 + M + G)
                    caps = [scene(rng, rig, M=M) for _ in range(G)]
                    sc = [torch.as_tensor(np.concatenate([c[i] for c in caps])).cuda().contiguous() for i in range(3)]
                    fu = [x.repeat((G,) + (1,) * (x.dim() - 1)).contiguous() for x in full]
                    for name, table, (uv, cl, cn) in (("seeded scenes", table_scene, sc), ("full slots", table_full, fu)):
                        launch = _launcher(table, uv, cl, cn, rig)
                        zero = torch.zeros_like(cn)
                        us, us0 = _median_us([launch, lambda: launch(zero)], args.runs)
                        print("round %d  %-13s C=%d M=%2d captures=%2d detections=%4d: %7.1f us per launch (all counts zero: %6.1f us)"
                              % (rnd, name, n_cams, M, G, int(cn.sum()), us, us0))
                a, b = _median_us([lambda: with_rig(fr), lambda: plain(fr)], args.runs)
                print("round %d  captured InstancePosePredictor C=%d M=%2d, full slots: %.1f us with the rig, %.1f us without (%+.1f us)"
                      % (rnd, n_cams, M, a, b, a - b))


if __name__ == "__main__":
    main()
