"""Cost of the constant-velocity pose filter of tracked instances (TrackingPosePredictor(motion="constant_velocity")).  All device
times from CUDA events after warm-up.

  * `predict`, `cov`, `update`: ssp_track_predict, ssp_pose_covariance and ssp_track_filter_update alone, each on the state and the
    detection slots of the last timed frame (the tracker state is put back before each timing), per launch.  The random network's
    PnP solutions collapse onto the camera centre, so their covariances are unusable and `update` times the restart of every
    matched filter;
  * `update_matched`: ssp_track_filter_update with every slot matched to a started filter and a usable covariance (a synthetic pose
    0.8 m in front of the camera, measured where the filter already is): the Kalman update with its gate and Joseph form, per launch;
  * `filtered` against `tracking`: TrackingPosePredictor with and without the filter (both captured, the same model, frames and
    conf_thresh) end to end, host frames (640 x 480 uint8) -> device results, median device time per call, the two alternated;
at B = 1 and 8 for the network input 416^2 with all 13 classes requested, then the card's name and power limit.
    python tools/bench_pose_filter.py [--reps 50] [--conf 0.02]
The frames are a slowly changing scene (one random frame plus a little noise per call).  A randomly initialised network is used:
with --conf 0.02 it lists far more instances than a trained one, so max_instances (32) slots are full in every frame and every
slot has a track.
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
from singleshotpose_b200.predict_instances import TrackingPosePredictor     # noqa: E402

NC, K9 = 13, 9


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _events_ms(fn, reps, restore=None):
    ts = []
    for _ in range(reps):
        if restore:
            restore()
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
    size = 416
    for B in (1, 8):
        rng = np.random.default_rng(size + B)
        f0 = rng.integers(0, 256, size=(B, 480, 640, 3)).astype(np.int16)
        seq = [np.clip(f0 + rng.integers(-4, 5, size=f0.shape), 0, 255).astype(np.uint8) for _ in range(8)]
        fp = TrackingPosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf, motion="constant_velocity")
        tp = TrackingPosePredictor(model, objects, K, shape=(size, size), batch=B, conf_thresh=a.conf)
        for fr in seq:
            fp(fr); tp(fr)
        torch.cuda.synchronize()
        c, tr, M, T = fp._last, fp._tracker, fp.max_instances, fp.max_tracks
        saved = tr.snapshot()
        s = stream_ptr()
        dist = None

        def predict():
            call("ssp_track_predict", B, T, ptr(tr.state_tracks), ptr(tr.state_rects), ptr(tr.state_poses), ptr(tr.state_filter), ptr(tr._dt),
                 ptr(tr._P3_table), tr.num_classes, ptr(tr._K64), dist, tr.accel_sigma[0], tr.accel_sigma[1], ptr(c.pred_poses),
                 ptr(c.pred_rects), s)

        def cov():
            call("ssp_pose_covariance", ptr(c.P3), 0, ptr(tr._K32), dist, K9, B, M, ptr(c.count), ptr(c.R), ptr(c.t), tr.keypoint_sigma,
                 ptr(c.cov_m), ptr(c.cov_status), s)

        def update():
            call("ssp_track_filter_update", B, T, M, ptr(c.count), ptr(c.slot), ptr(c.use_guess), ptr(c.R), ptr(c.t), ptr(c.cov_m),
                 ptr(c.cov_status), ptr(tr.state_filter), tr.init_velocity_sigma[0], tr.init_velocity_sigma[1], tr.gate, ptr(c.R_filt),
                 ptr(c.t_filt), ptr(c.pose_cov), ptr(c.velocity), ptr(c.reinit_i), s)
        restore = lambda: tr.restore(saved)
        t_pred = _events_ms(predict, a.reps, restore)
        t_cov = _events_ms(cov, a.reps)
        t_upd = _events_ms(update, a.reps, restore)
        tr.restore(saved)
        n = c.count.cpu().numpy()
        tid, warm, reinit = c.track_id.cpu().numpy(), c.use_guess.cpu().numpy() != 0, c.reinit.cpu().numpy()
        # the update path: every slot a synthetic pose with a usable covariance, started once (births), then measured again
        R0, t0, use0 = c.R.clone(), c.t.clone(), c.use_guess.clone()
        c.R.copy_(torch.eye(3, dtype=torch.float64, device="cuda")); c.t.copy_(torch.tensor([0.0, 0.0, 0.8], dtype=torch.float64, device="cuda"))
        cov()
        c.use_guess.zero_(); update()
        started = tr.snapshot()
        c.use_guess.copy_(((torch.arange(M, device="cuda")[None] < c.count[:, None]) & (c.slot >= 0)).int())
        t_upd_m = _events_ms(update, a.reps, lambda: tr.restore(started))
        n_upd = int(((c.reinit_i == 0) & (c.use_guess != 0)).sum())
        c.R.copy_(R0); c.t.copy_(t0); c.use_guess.copy_(use0); cov()
        tr.restore(saved)
        valid = np.arange(M)[None] < n[:, None]
        fps, tps = [], []
        for _ in range(3):                                        # alternate the two predictors
            fps.append(_events_ms(lambda: fp(seq[0]), a.reps))
            tps.append(_events_ms(lambda: tp(seq[0]), a.reps))
        t_fp, t_tp = float(np.median(fps)), float(np.median(tps))
        row = dict(shape=size, B=B, slots=int(valid.sum()), tracked=int((valid & (tid >= 0)).sum()),
                   matched=int((valid & warm).sum()), restarted=int((valid & warm & reinit).sum()), alive_tracks=int(tr.state_tracks[..., 0].sum()),
                   predict_us=round(t_pred * 1e3, 2), cov_us=round(t_cov * 1e3, 2), update_us=round(t_upd * 1e3, 2),
                   update_matched_us=round(t_upd_m * 1e3, 2), update_matched_slots=n_upd,
                   filtered_ms=round(t_fp, 4), tracking_ms=round(t_tp, 4), filtered_minus_tracking_us=round((t_fp - t_tp) * 1e3, 1))
        print(json.dumps(row), flush=True)
        rows.append(row)
    print(json.dumps(dict(gpu=_gpu_name(), rows=len(rows))))


if __name__ == "__main__":
    main()
