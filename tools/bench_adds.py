"""Speed of the pose errors over the mesh (utils.adi_batched, utils.mesh_diameter, evaluate_poses_batched(adds=True)) on the GPU
and of the reference's CPU functions they replace.  Prints one JSON line:
  adi_batched at Nv vertices for n = 64 and n = 1024 pose pairs: device time (CUDA events around the call, mean over the
    timed repetitions), poses/s, pair evaluations/s (n * Nv^2) and achieved fp64 FLOP/s (8 flop per pair: 3 subtractions,
    one multiply, two FMAs) against the data sheet's 34 TFLOP/s FP64 (non-tensor) of an H100 SXM, which assumes 700 W;
  mesh_diameter at Nv vertices (CUDA events; the call waits for its result);
  evaluate_poses_batched at B = 64 with and without adds (CUDA events around the call);
  the CPU baselines, one thread: utils_host.adi (scipy cKDTree, as the reference's adi) per pose pair and calc_pts_diameter,
    with the CPU model;
  the card name and power limit, read in the same run.
    python tools/bench_adds.py [--vertices 6000] [--reps 20] [--cpu-poses 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FP64_PEAK = 34e12          # H100 SXM data sheet, FP64 without tensor cores
FLOP_PER_PAIR = 8


def _events_ms(fn, reps, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _poses(rng, n):
    from singleshotpose_b200 import synth
    R = synth._rodrigues(rng.normal(size=(n, 3)))
    t = np.stack([rng.uniform(-.1, .1, n), rng.uniform(-.07, .07, n), rng.uniform(.6, 1.1, n)], 1)
    dR = synth._rodrigues(rng.normal(size=(n, 3)) * 0.05)
    return np.concatenate([dR @ R, (t + rng.normal(0, .01, (n, 3)))[:, :, None]], 2), np.concatenate([R, t[:, :, None]], 2)


def _cpu_model():
    import platform
    try:
        with open("/proc/cpuinfo") as f:
            name = next(line.split(":", 1)[1].strip() for line in f if line.startswith("model name"))
    except (OSError, StopIteration):
        name = platform.processor()
    return "%s (%s, %d logical CPUs)" % (name, platform.machine(), os.cpu_count())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vertices", type=int, default=6000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-poses", type=int, default=8)
    a = ap.parse_args()
    import torch
    from singleshotpose_b200 import synth, utils, utils_host
    if not torch.cuda.is_available():
        raise SystemExit("bench_adds needs a CUDA device")
    torch.set_num_threads(1)
    rng = np.random.default_rng(0)
    nv = a.vertices
    X = np.round(rng.uniform(-1, 1, (nv, 3)) * np.array([0.038, 0.039, 0.046]), 6)
    Xd = torch.from_numpy(X).cuda()
    res = {"vertices": nv}
    for n in (64, 1024):
        E, G = _poses(rng, n)
        Ed, Gd = torch.from_numpy(E).cuda(), torch.from_numpy(G).cuda()
        ms = _events_ms(lambda: utils.adi_batched(Xd, Ed, Gd), a.reps if n == 64 else max(a.reps // 4, 3))
        pairs = float(n) * nv * nv
        res["adi_batched_n%d" % n] = {"device_ms": ms, "poses_per_s": n / ms * 1e3, "pairs_per_s": pairs / ms * 1e3,
                                      "fp64_tflops": pairs * FLOP_PER_PAIR / ms * 1e-9, "share_of_34tflops": pairs * FLOP_PER_PAIR / ms * 1e3 / FP64_PEAK}
    res["mesh_diameter_ms"] = _events_ms(lambda: utils.mesh_diameter(Xd), a.reps)
    # the single-object tail at B = 64 on a synthetic batch: the same PnP work with and without ADD-S
    B = 64
    pr = synth.pnp_problems(B, sigma=0.5, seed=1)
    out = (torch.randn(B, 20, 13, 13, generator=torch.Generator().manual_seed(2)) * 0.3).cuda()
    tgt = torch.zeros(B, 21)
    tgt[:, 1:19] = torch.from_numpy((pr["uv"] / np.array([640.0, 480.0], np.float32)).reshape(B, -1))
    verts = np.c_[X, np.ones(nv)].T
    Kc = synth.intrinsics()
    for adds in (False, True):
        res["evaluate_poses_batched_b64_adds_%s_ms" % adds] = _events_ms(
            lambda: utils.evaluate_poses_batched(out, tgt, verts, pr["P3"], Kc, adds=adds), a.reps)
    # CPU baselines, one thread
    E, G = _poses(rng, a.cpu_poses)
    Xh = np.c_[X, np.ones(nv)].T
    utils_host.adi((E[0] @ Xh).T, (G[0] @ Xh).T)                      # imports scipy.spatial outside the timed loop
    t0 = time.perf_counter()
    cpu = [utils_host.adi((E[p] @ Xh).T, (G[p] @ Xh).T) for p in range(a.cpu_poses)]
    res["cpu_adi_ms_per_pose"] = (time.perf_counter() - t0) / a.cpu_poses * 1e3
    gpu = utils.adi_batched(X, E, G).cpu().numpy()
    res["cpu_gpu_adi_max_rel_diff"] = float(np.max(np.abs(gpu - cpu) / np.abs(cpu)))
    t0 = time.perf_counter()
    d_cpu = utils_host.calc_pts_diameter(X)
    res["cpu_calc_pts_diameter_ms"] = (time.perf_counter() - t0) * 1e3
    res["diameter_bit_identical"] = utils.mesh_diameter(X) == d_cpu
    res["cpu"] = _cpu_model()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        res["gpu"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        res["gpu"] = torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
