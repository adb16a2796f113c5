"""Speed of making a training set from camera poses (utils.render_masks, python -m singleshotpose_b200.make_dataset) on the GPU,
and of a one-thread CPU rasteriser.  Prints one JSON line:
  render: ssp_render_masks for the synthetic closed mesh (synth.closed_mesh: 6002 vertices, 12000 faces) at 640 x 480, n = 1024
    poses, preallocated buffers: device time from CUDA events (mean over the timed repetitions) and masks/s, the device time of
    each kernel of one launch (torch.profiler, a separate pass); and utils.render_masks (allocation and the Python wrapper
    included);
  make_dataset: the command end to end on --images synthetic 640 x 480 JPEGs (host clock: pose checks, label rows, the masks
    rendered, copied to the host and written as PNG), images/s;
  cpu: cv2.fillConvexPoly over every triangle, one thread, with the same 1/256-px fixed-point vertices (shift = 8), for
    --cpu-poses poses: masks/s, and the share of pixels on which it agrees with the GPU mask (OpenCV's fill rule differs on
    edges, so this is not 1);
  the card name and power limit, read in the same run.
    python tools/bench_render.py [--poses 1024] [--reps 10] [--images 256] [--cpu-poses 16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _events_ms(fn, reps, warmup=2):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--cpu-poses", type=int, default=16)
    a = ap.parse_args()
    import cv2
    import torch
    from PIL import Image
    from singleshotpose_b200 import _lib, make_dataset, synth, utils
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a CUDA device")
    W, H, n = 640, 480, a.poses
    V, F = synth.closed_mesh()
    K = synth.intrinsics()
    R, t = synth.object_poses(n, seed=1)
    Rt = np.concatenate([R, t[:, :, None]], 2)
    res = {"vertices": len(V), "faces": len(F), "width": W, "height": H, "poses": n}
    # the kernel launches alone
    X = torch.from_numpy(np.ascontiguousarray(V.T, np.float32)).cuda()
    Fd = torch.from_numpy(F).cuda()
    Td, Kd = torch.from_numpy(Rt).cuda(), torch.from_numpy(K).cuda()
    wb = int(_lib.load().ssp_render_work_bytes(len(V), len(F), n, W, H))
    work = torch.empty(wb, dtype=torch.uint8, device="cuda")
    masks = torch.empty(n, H, W, dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    run = lambda: _lib.call("ssp_render_masks", _lib.ptr(X), 3, len(V), _lib.ptr(Fd), len(F), _lib.ptr(Td), _lib.ptr(Kd), n, W, H,
                            _lib.ptr(masks), _lib.ptr(status), _lib.ptr(work), wb, _lib.stream_ptr())
    ms = _events_ms(run, a.reps)
    cover = float((masks > 0).float().mean())
    res["render"] = {"device_ms": ms, "masks_per_s": n / ms * 1e3, "work_bytes": wb, "mean_covered_share": cover,
                     "status_nonzero": int((status != 0).sum())}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:        # one launch, for the share of each kernel
        run()
        torch.cuda.synchronize()
    res["render"]["kernel_us"] = {e.key: e.device_time_total for e in prof.key_averages() if e.device_time_total > 0}
    ms = _events_ms(lambda: utils.render_masks(V, F, Rt, K, W, H), a.reps)
    res["render_masks_call"] = {"ms": ms, "masks_per_s": n / ms * 1e3}
    # make_dataset end to end
    with tempfile.TemporaryDirectory() as d:
        jd = os.path.join(d, "obj", "JPEGImages")
        os.makedirs(jd)
        img = Image.fromarray(synth.photo_sample(0, W, H, 8, 8)[0])
        paths = []
        for i in range(a.images):
            p = os.path.join(jd, "%06d.jpg" % i)
            img.save(p, quality=95)
            paths.append(p)
        ply = os.path.join(d, "obj.ply")
        synth.write_ply(ply, V, F)
        np.savez(os.path.join(d, "poses.npz"), paths=np.array(paths), R=R[:a.images], t=t[:a.images])
        make_dataset.make_dataset(ply, os.path.join(d, "poses.npz"), K, "obj", os.path.join(d, "warm.data"), log=lambda s: None)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        make_dataset.make_dataset(ply, os.path.join(d, "poses.npz"), K, "obj", os.path.join(d, "obj.data"), log=lambda s: None)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        res["make_dataset"] = {"images": a.images, "s": s, "images_per_s": a.images / s}
    # one-thread CPU baseline
    cv2.setNumThreads(1)
    uv = utils.project_points_batched(V.T, Rt[:a.cpu_poses], K).cpu().numpy()
    ref = masks[:a.cpu_poses].cpu().numpy()
    agree = []
    t0 = time.perf_counter()
    for p in range(a.cpu_poses):
        m = np.zeros((H, W), np.uint8)
        pts = np.rint(uv[p].T * 256).astype(np.int32)
        for f in F:
            cv2.fillConvexPoly(m, pts[f], 255, lineType=cv2.LINE_8, shift=8)
        agree.append(float((m == ref[p]).mean()))
    s = time.perf_counter() - t0
    res["cpu_fillConvexPoly"] = {"poses": a.cpu_poses, "masks_per_s": a.cpu_poses / s, "pixel_agreement_with_gpu": float(np.mean(agree))}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        res["gpu"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        res["gpu"] = torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
