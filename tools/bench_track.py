"""Cost of tracking across frames (predict_instances.TrackingPosePredictor).  All device times from CUDA events after warm-up.

  * `track`: ssp_track_associate + ssp_track_commit alone, on the detections of the timed frames (the track state is put back after
    the timing), per frame pair of launches;
  * `pnp_warm` against `pnp_cold`: ssp_pnp_batched_guess with the slots' warm starts against ssp_pnp_batched_counted over the same
    slots, and the mean accepted LM iterations and linear solves per solved slot of each (work counters; warm starts skip the DLT);
  * `tracking` against `instances`: TrackingPosePredictor and InstancePosePredictor (both captured, the same model, frames and
    conf_thresh) end to end, host frames (640 x 480 uint8) -> device results, median device time per call;
at B = 1 and 8 for network inputs 416^2 and 672^2 with all 13 classes requested, then the card's name and power limit.
    python tools/bench_track.py [--reps 50] [--conf 0.02]
The frames are a slowly changing scene (one random frame plus a little noise per call), so most instances match a track.  A
randomly initialised network is used: with --conf 0.02 it lists far more instances than a trained one, so max_instances (32) slots
are full in every frame.
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
from singleshotpose_b200.darknet_multi import Darknet                       # noqa: E402
from singleshotpose_b200.predict_instances import InstancePosePredictor, TrackingPosePredictor   # noqa: E402

NC, K9 = 13, 9


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
    import tempfile
    cfg = write_cfg(os.path.join(tempfile.mkdtemp(), "yolo-pose-multi.cfg"), multi=True)
    torch.manual_seed(0)
    model = Darknet(cfg).cuda().eval()
    objects = {c: synth.box_points((0.038 + 0.002 * c, 0.039, 0.046), with_center=False).T.astype(np.float64) for c in range(NC)}
    K = synth.intrinsics()
    rows = []
    for size in (416, 672):
        for B in (1, 8):
            rng = np.random.default_rng(size + B)
            f0 = rng.integers(0, 256, size=(B, 480, 640, 3)).astype(np.int16)
            seq = [np.clip(f0 + rng.integers(-4, 5, size=f0.shape), 0, 255).astype(np.uint8) for _ in range(8)]
            tp = TrackingPosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf)
            ip = InstancePosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf)
            for fr in seq:
                tp(fr); ip(fr)
            torch.cuda.synchronize()
            c, tr, M, T = tp._last, tp._tracker, tp.max_instances, tp.max_tracks
            saved = tr.snapshot()

            def track():
                s = stream_ptr()
                call("ssp_track_associate", B, T, M, ptr(c.count), ptr(c.cls), ptr(c.kp), tr.match_iou, tr.max_misses, ptr(tr.state_tracks),
                     ptr(tr.state_rects), ptr(tr.state_poses), ptr(tr.state_next_id), ptr(c.slot), ptr(c.track_id), ptr(c.guess),
                     ptr(c.use_guess), s)
                call("ssp_track_commit", B, T, M, ptr(c.count), ptr(c.kp), ptr(c.slot), ptr(c.params), ptr(tr.state_tracks),
                     ptr(tr.state_rects), ptr(tr.state_poses), s)
            tr.restore(saved)
            track()                                                    # the last frame's association: its warm starts
            guess, use = c.guess.clone(), c.use_guess.clone()
            t_track = _events_ms(lambda: [track() for _ in range(20)], a.reps) / 20
            tr.restore(saved)
            R = torch.empty(B, M, 3, 3, dtype=torch.float64, device="cuda"); t = torch.empty(B, M, 3, dtype=torch.float64, device="cuda")
            params = torch.empty(B, M, 6, dtype=torch.float64, device="cuda")
            work_w = torch.zeros(B, M, 3, dtype=torch.int32, device="cuda"); work_c = torch.zeros_like(work_w)
            zero = torch.zeros_like(use)

            def warm(work=None):
                call("ssp_pnp_batched_guess", ptr(c.P3), ptr(c.kp), ptr(tp._K32), K9, B, M, ptr(c.count), ptr(guess), ptr(use), 20, ptr(R),
                     ptr(t), ptr(params), ptr(work) if work is not None else None, stream_ptr())

            def cold():
                call("ssp_pnp_batched_counted", ptr(c.P3), ptr(c.kp), ptr(tp._K32), K9, B, M, ptr(c.count), 20, ptr(R), ptr(t), stream_ptr())
            warm(work_w)
            call("ssp_pnp_batched_guess", ptr(c.P3), ptr(c.kp), ptr(tp._K32), K9, B, M, ptr(c.count), ptr(guess), ptr(zero), 20, ptr(R),
                 ptr(t), ptr(params), ptr(work_c), stream_ptr())      # use_guess 0: the counted solve, with its work counters
            solved = (torch.arange(M, device="cuda")[None] < c.count[:, None])
            nw, ns = int((solved & (use != 0)).sum()), int(solved.sum())
            t_warm = _events_ms(warm, a.reps)
            t_cold = _events_ms(cold, a.reps)
            tps, ips = [], []
            for _ in range(3):                                        # alternate the two predictors
                tps.append(_events_ms(lambda: tp(seq[0]), a.reps))
                ips.append(_events_ms(lambda: ip(seq[0]), a.reps))
            t_tp, t_ip = float(np.median(tps)), float(np.median(ips))
            sv = solved.cpu().numpy()
            ww, wc = work_w.cpu().numpy()[sv], work_c.cpu().numpy()[sv]
            row = dict(shape=size, B=B, solved_slots=ns, warm_slots=nw, track_us=round(t_track * 1e3, 2),
                       pnp_warm_us=round(t_warm * 1e3, 1), pnp_cold_us=round(t_cold * 1e3, 1),
                       lm_iters_warm=round(float(ww[:, 1].mean()), 2) if len(ww) else None,
                       lm_iters_cold=round(float(wc[:, 1].mean()), 2) if len(wc) else None,
                       lm_solves_warm=round(float(ww[:, 2].mean()), 2) if len(ww) else None,
                       lm_solves_cold=round(float(wc[:, 2].mean()), 2) if len(wc) else None,
                       tracking_ms=round(t_tp, 4), instances_ms=round(t_ip, 4), tracking_minus_instances_us=round((t_tp - t_ip) * 1e3, 1))
            print(json.dumps(row), flush=True)
            rows.append(row)
    print(json.dumps(dict(gpu=_gpu_name(), rows=len(rows))))


if __name__ == "__main__":
    main()
