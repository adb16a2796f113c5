#!/usr/bin/env python
"""Golden of TrackingPosePredictor's outputs without a motion model, written by the tracker as it was before the pose filter existed
(the commit that added lens distortion, 9b67a94), so that the tracker with motion=None can be checked against it bit for bit.

  the multi-object cfg of cfgs.write_cfg(multi=True) with torch.manual_seed(0) weights; 4 requested classes; B = 2 streams of 6
  frames of a slowly changing scene (one random 640 x 480 frame plus a little noise per call); conf_thresh 0.02, max_instances 16,
  max_tracks 8, graph replay; every output of every frame, then the track state.
run() uses only what both versions have.  Needs an H100 (the same GPU the suite runs on); writes tests/golden/track_motion_none.npz.

    python tests/golden/make_golden_track_motion_none.py [out.npz]
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CLASSES = (0, 4, 7, 11)
KEYS = ("count", "kept", "cls", "R", "t", "conf", "cls_conf", "keypoints_px", "corners_px", "track_id", "warm")


def _corners(c):
    from singleshotpose_b200 import synth
    s = 1.0 + 0.1 * c
    return synth.box_points((0.038 * s, 0.039 * s, 0.046 * (2.0 - 0.05 * c)), with_center=False).T.astype(np.float64)


def run():
    """-> {name: array}: the outputs '<key>_<frame>' and the state 'state_<i>' of the scenario above"""
    import torch
    from singleshotpose_b200 import synth
    from singleshotpose_b200.cfgs import write_cfg
    from singleshotpose_b200.darknet_multi import Darknet
    from singleshotpose_b200.predict_instances import TrackingPosePredictor
    cfg = write_cfg(os.path.join(tempfile.mkdtemp(), "yolo-pose-multi.cfg"), multi=True)
    torch.manual_seed(0)
    model = Darknet(cfg).cuda().eval()
    tp = TrackingPosePredictor(model, {c: _corners(c) for c in CLASSES}, synth.intrinsics(), batch=2, conf_thresh=0.02, max_instances=16,
                               max_tracks=8)
    rng = np.random.default_rng(3)
    f0 = rng.integers(0, 256, size=(2, 480, 640, 3)).astype(np.int16)
    out = {}
    for f in range(6):
        frame = np.clip(f0 + rng.integers(-6, 7, size=f0.shape), 0, 255).astype(np.uint8)
        r = tp(frame, to_host=True)
        out.update(("%s_%d" % (k, f), r[k]) for k in KEYS)
    for i, t in enumerate(tp._tracker._state()[:4]):
        out["state_%d" % i] = t.cpu().numpy()
    return out


def main():
    sys.path.insert(0, ROOT)
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "track_motion_none.npz")
    out = run()
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %d warm slots" % (path, len(out), sum(int(v.sum()) for k, v in out.items() if k.startswith("warm_"))))


if __name__ == "__main__":
    main()
