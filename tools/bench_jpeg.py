"""Measures the batched GPU JPEG decoder (singleshotpose_b200/jpeg.py) against Pillow on the same files.

Content: seeded synthetic photo-like images (smooth gradients, a disc, Gaussian noise of sigma 3), 4:2:0, at quality 75 and
95, in two sizes: 640x480 (LINEMOD) and 500x375 (a typical VOC background).  Reports, with the card name and power limit read
in the same run: the compressed sizes; GPU decode time per batch of 64 / 128 / 192 (CUDA events around the whole decoder call,
host parse and staging included), images/s and compressed MB/s, and the share of 1024-bit subsequences the entropy decode had
to walk serially; the per-kernel device time from torch.profiler in a separate pass; Pillow decode in one thread and in
os.cpu_count() processes; GpuCollate for 64 training samples with listDataset(gpu_decode=True / False).  Prints JSON lines.

    python tools/bench_jpeg.py [--iters 5]
"""
import argparse
import io
import json
import os
import platform
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def scene(w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    f = rng.uniform(15, 40, 4)
    img = np.stack([128 + 100 * np.sin(xx / f[0]) * np.cos(yy / f[1]), 255 * xx / (w - 1), 255 * yy / (h - 1)], -1)
    cx, cy, r = rng.uniform(0.2, 0.8) * w, rng.uniform(0.2, 0.8) * h, rng.uniform(0.1, 0.3) * min(w, h)
    img[(xx - cx) ** 2 + (yy - cy) ** 2 < r * r] = rng.uniform(0, 255, 3)
    img += rng.normal(0, 3, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def make_files(w, h, q, n):
    from PIL import Image
    out = []
    for i in range(n):
        b = io.BytesIO()
        Image.fromarray(scene(w, h, i)).save(b, "JPEG", quality=q)
        out.append(b.getvalue())
    return out


def collate_bench(iters):
    """GpuCollate of 64 training samples (640x480 JPEG images, PNG masks, 500x375 JPEG backgrounds) -> 416x416; the samples are
    built once beforehand: the worker-side work (file reads or Pillow decodes, draws, labels) is not in the time."""
    import random
    import tempfile
    import torch
    from PIL import Image
    from singleshotpose_b200 import dataset
    res = {}
    with tempfile.TemporaryDirectory() as root:
        base = os.path.join(root, "LINEMOD", "ape")
        for d in ("JPEGImages", "mask", "labels"):
            os.makedirs(os.path.join(base, d))
        lines, bgs = [], []
        for i in range(64):
            Image.fromarray(scene(640, 480, 1000 + i)).save(os.path.join(base, "JPEGImages", "%06d.jpg" % i), quality=95)
            m = np.zeros((480, 640, 3), np.uint8); m[120:360, 200:440] = 255
            Image.fromarray(m).save(os.path.join(base, "mask", "%04d.png" % i))
            open(os.path.join(base, "labels", "%06d.txt" % i), "w").write(" ".join(["0"] + ["0.5"] * 20) + "\n")
            lines.append(os.path.join(base, "JPEGImages", "%06d.jpg" % i))
            bg = os.path.join(root, "bg%d.jpg" % i)
            Image.fromarray(scene(500, 375, 2000 + i)).save(bg, quality=75)
            bgs.append(bg)
        lf = os.path.join(root, "train.txt")
        open(lf, "w").write("\n".join(lines) + "\n")
        for gd in (False, True):
            random.seed(0)
            ds = dataset.listDataset(lf, shape=(416, 416), shuffle=False, train=True, bg_file_names=bgs, batch_size=64, num_workers=1,
                                     gpu_decode=gd)
            samples = [ds[i] for i in range(64)]
            coll = dataset.GpuCollate("cuda")
            coll(samples)
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(iters):
                coll(samples)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t) / iters * 1e3
            res["gpu_decode_%s" % gd] = {"ms_per_batch": round(ms, 2), "samples_per_s": round(64 / ms * 1e3, 1)}
    return res


def _pillow(blobs):
    from PIL import Image
    for b in blobs:
        np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))
    return len(blobs)


def pillow_rate(blobs, procs):
    if procs == 1:
        t = time.perf_counter(); _pillow(blobs); return len(blobs) / (time.perf_counter() - t)
    chunks = [blobs[i::procs] for i in range(procs)]
    with ProcessPoolExecutor(procs) as ex:
        list(ex.map(_pillow, chunks))                     # warm the workers
        t = time.perf_counter()
        list(ex.map(_pillow, chunks))
        return len(blobs) / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from singleshotpose_b200.jpeg import GpuJpegDecoder
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cpu = platform.processor() or "unknown"
    try:
        with open("/proc/cpuinfo") as f:
            cpu = next((l.split(":", 1)[1].strip() for l in f if l.startswith("model name")), cpu)
    except OSError:
        pass
    res = {"gpu": smi, "cpu": cpu, "cpu_count": os.cpu_count(), "sets": []}
    dec = GpuJpegDecoder("cuda")
    for (w, h) in ((640, 480), (500, 375)):
        for q in (75, 95):
            files = make_files(w, h, q, 192)
            mean_kb = float(np.mean([len(b) for b in files])) / 1e3
            kb = np.array([len(b) for b in files]) / 1e3
            entry = {"size": "%dx%d" % (w, h), "quality": q, "mean_compressed_kB": round(mean_kb, 1),
                     "compressed_kB_min_median_max": [round(float(np.min(kb)), 1), round(float(np.median(kb)), 1), round(float(np.max(kb)), 1)],
                     "gpu": {}}
            for B in (64, 128, 192):
                batch = files[:B]
                outs = dec(batch)
                assert dec.fallbacks == 0, dec.fallback_reasons
                nsub = sum((len(b) * 8 + 1023) // 1024 for b in batch)          # about: header bytes and stuffing included
                serial = dec.serial_subsequences
                from PIL import Image
                assert np.array_equal(outs[0].cpu().numpy(), np.asarray(Image.open(io.BytesIO(batch[0])).convert("RGB")))
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    dec(batch)
                e1.record(); e1.synchronize()
                ms = e0.elapsed_time(e1) / args.iters
                entry["gpu"][str(B)] = {"ms_per_batch": round(ms, 2), "images_per_s": round(B / ms * 1e3, 1),
                                        "compressed_MB_per_s": round(B * mean_kb / 1e3 / ms * 1e3, 1), "h2d_bytes": dec.h2d_bytes,
                                        "serial_subsequences": serial, "subsequences_about": nsub}
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                dec(files[:64])
                torch.cuda.synchronize()
            entry["kernels_ms_batch64"] = {e.key: round(e.device_time_total / 1e3, 3) for e in prof.key_averages()
                                           if "kernel" in e.key or "Memcpy" in e.key}
            entry["pillow_1thread_images_per_s"] = round(pillow_rate(files[:64], 1), 1)
            entry["pillow_%dproc_images_per_s" % os.cpu_count()] = round(pillow_rate(files * 2, os.cpu_count()), 1)
            res["sets"].append(entry)
            print(json.dumps(entry), flush=True)
    res["collate_64_train_samples"] = collate_bench(args.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
