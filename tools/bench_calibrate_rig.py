"""Device time of ssp_calibrate_rig per stage, from torch.profiler's kernel records, at C = 2 / 4 / 8 cameras and 60 / 600 / 6000
observations (2 px noise, 10 % missed and 10 % wrong views), the whole call from CUDA events, and the numpy oracle and scipy's
bundle adjustment on the CPU at the small size for scale.  Prints the card's name and power limit with the numbers.

    python tools/bench_calibrate_rig.py [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from singleshotpose_b200 import utils  # noqa: E402
from test_calibrate_rig_cpu import moving_object, record  # noqa: E402
from test_multiview_cpu import P9, random_rig  # noqa: E402

STAGES = (("per-view solve", ("fuse_rows",)), ("pair scoring", ("pair_list", "pair_score", "tree_kernel")),
          ("fusion", ("fuse_hyp", "fuse_obs", "round_kernel")), ("BA terms", ("obs_terms",)), ("BA reduce", ("block_kernel",)),
          ("BA factor", ("factor_kernel", "cov_kernel")), ("BA back-sub + accept", ("backsub", "accept")), ("finish", ("finish_kernel",)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def problem(n_cams, n_obs, seed=0):
    rng = np.random.default_rng(seed)
    rig = random_rig(rng, n_cams)
    uv, valid = record(rig, moving_object(rng, n_obs), rng, 2.0, 0.1, 0.1)
    return rig, uv, valid


def stage_times(rig, uv, valid):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        utils.calibrate_rig_batched(P9, uv, rig.K, valid=valid)
        torch.cuda.synchronize()
    us = {name: 0.0 for name, _ in STAGES}
    for e in prof.key_averages():
        for name, keys in STAGES:
            if any(k in e.key for k in keys):
                us[name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("device: %s" % card())
    for n_cams in (2, 4, 8):
        for n_obs in (60, 600, 6000):
            rig, uv, valid = problem(n_cams, n_obs)
            o = utils.calibrate_rig_batched(P9, uv, rig.K, valid=valid)          # warm-up
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            best = np.inf
            for _ in range(a.reps):
                ev[0].record()
                utils.calibrate_rig_batched(P9, uv, rig.K, valid=valid)
                ev[1].record()
                torch.cuda.synchronize()
                best = min(best, ev[0].elapsed_time(ev[1]))
            st = stage_times(rig, uv, valid)
            print("C=%d obs=%5d: whole call %.2f ms (rounds %d, LM steps %d); per stage (us): %s"
                  % (n_cams, n_obs, best, o["rounds"], o["iterations"], ", ".join("%s %.0f" % (k, v) for k, v in st.items())))
    # the CPU at the small size, for scale
    from oracle.calibrate_rig_ref import calibrate_ref
    rig, uv, valid = problem(2, 60)
    o = utils.calibrate_rig_batched(P9, uv, rig.K, valid=valid)
    G = len(uv) // 2
    sh = lambda x: np.asarray(x).reshape(G, 2, *np.shape(x)[1:])
    t0 = time.perf_counter()
    calibrate_ref(rig.K, None, np.repeat(P9[None, None], G, 0).repeat(2, 1), sh(uv), sh(valid), sh(o["R_rows"].cpu().numpy()),
                  sh(o["t_rows"].cpu().numpy()))
    t1 = time.perf_counter()
    from scipy.optimize import least_squares
    from test_calibrate_rig_cpu import _joint_residuals
    linked = np.flatnonzero(o["linked"].cpu().numpy())
    views = o["views"].cpu().numpy()
    sets = {int(g): views[g] for g in linked}
    poses = [(o["R_world"][g].cpu().numpy(), o["t_world"][g].cpu().numpy()) for g in linked]
    f = lambda x: _joint_residuals(rig.K, None, o["R"].cpu().numpy(), o["t"].cpu().numpy(), uv.reshape(G, 2, 9, 2), sets, poses, [1], x)
    t2 = time.perf_counter()
    least_squares(f, np.zeros(6 + 6 * len(linked)), method="lm")
    t3 = time.perf_counter()
    print("CPU at C=2 obs=60: numpy oracle %.0f ms, scipy least_squares bundle adjustment %.0f ms" % (1e3 * (t1 - t0), 1e3 * (t3 - t2)))


if __name__ == "__main__":
    main()
