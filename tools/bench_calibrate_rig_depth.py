"""Cost of the depth calibration of a rig (ssp_calibrate_rig_depth, utils.calibrate_rig_depth_batched).  Device times from CUDA
events after a warm-up, median over --reps; then one torch.profiler run per size for the time of each kernel.

  * C = 2, 4 and 8 cameras, G = 60 and 600 captures of one slot, a 6002-vertex mesh (synth.closed_mesh), 640 x 480 depth frames
    rendered in every camera with a table plane (tests/test_refine_rig_cpu.py's scenes; 6 distinct captures repeated, since the
    cost does not depend on which capture a frame shows), 10 iterations, the true rig perturbed by 0.5 degrees and 5 mm per free
    camera and the world poses by 1 degree and 3 mm;
  * `call_ms`: one calibrate_rig_depth_batched call on device inputs, between two events (it includes the wrapper's host checks,
    the mesh table's upload and mesh_diameter, and the copy of the statuses back); `kernels_ms`: each kernel's summed device time
    over one call, from the profiler;
then the card's name and power limit, printed beside every line.
    python tools/bench_calibrate_rig_depth.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from singleshotpose_b200 import utils                                         # noqa: E402
from test_calibrate_rig_depth_cpu import start                                # noqa: E402
from test_refine_depth_cpu import F, V                                        # noqa: E402


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def problem(C, G):
    """-> a function that runs calibrate_rig_depth_batched once on device depth"""
    _true, rig0, depth6, R6, t6 = start(300 + C, C, 6)[:5]
    depth = torch.from_numpy(np.concatenate([depth6[(g % 6) * C:(g % 6) * C + C] for g in range(G)]).view(np.int16)).cuda().view(torch.uint16)
    calib = dict(R=rig0.R, t=rig0.t, cam_status=np.zeros(C, np.int32), R_world=np.stack([R6[g % 6] for g in range(G)]),
                 t_world=np.stack([t6[g % 6] for g in range(G)]), views=np.ones((G, C), bool), linked=np.ones(G, bool))
    calib = {k: torch.as_tensor(v).cuda() for k, v in calib.items()}
    return lambda: utils.calibrate_rig_depth_batched(depth, V, F, rig0.K, calib)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="write the JSON lines here too")
    a = ap.parse_args()
    gpu = _gpu_name()
    lines = []
    for C in (2, 4, 8):
        for G in (60, 600):
            run = problem(C, G)
            assert run()["status"] == 0
            torch.cuda.synchronize()
            ts = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and "cd_" in ev.key:
                    name = ev.key.split("cd_")[1].split("_kernel")[0]
                    kern[name] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3, 3)
            line = dict(C=C, G=G, vertices=len(V), frame="640x480", iters=10, call_ms=round(float(np.median(ts)), 3),
                        call_ms_min=round(float(np.min(ts)), 3), kernels_ms=kern, gpu=gpu)
            print(json.dumps(line), flush=True)
            lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
