"""Cost of every-instance detection (singleshotpose_b200/predict_instances.py).  All device times from CUDA events after warm-up.

  * `detect`: ssp_detect_instances alone (all 13 classes of yolo-pose-multi.cfg, nms_thresh 0.4, max_instances 32) on the
    logits the predictor's own forward produced for the timed frames, per launch and per frame;
  * `instances` against `multi`: InstancePosePredictor and MultiPosePredictor (both captured, the same model, frames and
    conf_thresh) end to end, host frames (640 x 480 uint8) -> device results, median device time per call;
  * the oracle's numpy NMS loop (oracle/detect_ref.py nms_ref) on one CPU thread over the same candidates, per frame;
at B = 1 and 8 for network inputs 416^2 and 672^2, with the candidate count of the frames, then the card's name and power limit.
    python tools/bench_detect.py [--reps 50] [--conf 0.02]
A randomly initialised network is used: its det_conf * cls_max_conf is near 1/13 * 1/2, so --conf 0.02 lists most entries and the
detect kernel sorts and suppresses thousands of candidates per frame, more than a trained network lists.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import detect_ref as DR                                         # noqa: E402
from singleshotpose_b200 import synth                                       # noqa: E402
from singleshotpose_b200._lib import call, ptr, stream_ptr                  # noqa: E402
from singleshotpose_b200.cfgs import write_cfg                              # noqa: E402
from singleshotpose_b200.darknet_multi import Darknet                       # noqa: E402
from singleshotpose_b200.predict_instances import InstancePosePredictor     # noqa: E402
from singleshotpose_b200.predict_multi import MultiPosePredictor            # noqa: E402
from singleshotpose_b200.utils_multi import multi_region_dense              # noqa: E402

NC, NA, K9 = 13, 5, 9


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--conf", type=float, default=0.02)
    a = ap.parse_args()
    torch.set_num_threads(1)
    import tempfile
    cfg = write_cfg(os.path.join(tempfile.mkdtemp(), "yolo-pose-multi.cfg"), multi=True)
    torch.manual_seed(0)
    model = Darknet(cfg).cuda().eval()
    objects = {c: synth.box_points((0.038 + 0.002 * c, 0.039, 0.046), with_center=False).T.astype(np.float64) for c in range(NC)}
    K = synth.intrinsics()
    cls = np.arange(NC, dtype=np.int32)
    rows = []
    for size in (416, 672):
        for B in (1, 8):
            frames = np.random.default_rng(size + B).integers(0, 256, size=(B, 480, 640, 3), dtype=np.uint8)
            ip = InstancePosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf)
            mp = MultiPosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf)
            for _ in range(3):
                ip(frames); mp(frames)
            torch.cuda.synchronize()
            logits = ip.logits.clone()
            h, w = logits.shape[2:]
            M = 32
            bufs = [torch.empty(B, M, 2 * K9 + 3, device="cuda"), torch.empty(B, M, dtype=torch.int32, device="cuda"),
                    torch.empty(B, M, K9, 2, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"),
                    torch.empty(B, dtype=torch.int32, device="cuda")]

            def detect():
                call("ssp_detect_instances", ptr(logits), B, K9, NC, NA, h, w, C.c_void_p(cls.ctypes.data), NC, a.conf, 0.4, M, 640.0, 480.0,
                     *[ptr(t) for t in bufs], stream_ptr())

            def detect_many(n=20):
                for _ in range(n):
                    detect()
            detect_many()
            t_det = _events_ms(detect_many, a.reps) / 20
            t_ip = t_mp = None
            ips, mps = [], []
            for _ in range(3):                                       # alternate the two predictors
                ips.append(_events_ms(lambda: ip(frames), a.reps))
                mps.append(_events_ms(lambda: mp(frames), a.reps))
            t_ip, t_mp = float(np.median(ips)), float(np.median(mps))
            dense = multi_region_dense(logits, NC, K9, NA, -1, only_objectness=0)["boxes"].cpu().numpy()
            cands, t_cpu = [], 0.0
            for b in range(B):
                d = dense[b]
                px = d[:, :2 * K9].reshape(-1, K9, 2) * np.float32([640, 480])
                sel = np.nonzero(d[:, 18] * d[:, 19] > np.float32(a.conf))[0]
                cands.append(len(sel))
                t0 = time.perf_counter()
                DR.nms_ref(d[sel, 18], d[sel, 20].astype(np.int64), px[sel], 0.4, M)
                t_cpu += time.perf_counter() - t0
            row = dict(shape=size, B=B, grid=[h, w], candidates_per_frame=float(np.mean(cands)), kept=bufs[4].cpu().tolist(),
                       detect_us=round(t_det * 1e3, 2), detect_us_per_frame=round(t_det * 1e3 / B, 2),
                       instances_ms=round(t_ip, 4), multi_ms=round(t_mp, 4), instances_minus_multi_us=round((t_ip - t_mp) * 1e3, 1),
                       cpu_nms_ms_per_frame=round(t_cpu * 1e3 / B, 2))
            print(json.dumps(row), flush=True)
            rows.append(row)
    print(json.dumps(dict(gpu=_gpu_name(), torch_threads=torch.get_num_threads(), rows=len(rows))))


if __name__ == "__main__":
    main()
