"""Throughput of the multi-object training-image pipeline (singleshotpose_b200/image_multi.py GpuMultiAugmenter): one batch of
B samples at SIZE^2 from a synthetic 640x480 LINEMOD tree (singleshotpose_b200.synth.write_linemod_multi_like), written to a
temporary directory.  Prints one JSON line:
  cold  - the first batch (object bank empty: every view is decoded and copied once),
  warm  - later batches (bank filled: attempts cost no decode and no copy),
  wall time per batch, and the summed span of the launched work of each round / phase on the stream (CUDA events around each
  H2D copy + launch sequence: device time, without the host's draws, decoding and waits between rounds),
  rounds per batch, attempts per sample (mean, max), decodes and host->device bytes per batch,
  a 1-thread PIL baseline of the same sample sequence (Pillow calls as the reference makes them) and whether its last sample
  matched the GPU bytes, and the card name and power limit.
    python tools/bench_augment_multi.py [--batch 64] [--size 416] [--batches 4] [--pil-samples 4] [--views 8]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pil_sample(path, bgpath, shape, rng, root, jitter=0.1):
    """image_multi.load_data_detection's pixel path with Pillow calls (1 thread); returns (uint8 image, attempts)"""
    from PIL import Image, ImageChops
    from singleshotpose_b200 import image_multi as IM
    from singleshotpose_b200.image import mask_luts
    pos, neg = mask_luts()
    rgb = lambda p: Image.open(p).convert("RGB")

    def sel(a, m, b):          # a * round(m/255) + b * round(1 - m/255): what the ImageMath expressions compute
        return np.clip(np.asarray(a).astype(np.int32) * pos[m] + np.asarray(b).astype(np.int32) * neg[m], 0, 255).astype(np.uint8)

    def crop_resize(im, p):
        return im.crop((p["pleft"], p["ptop"], p["pleft"] + p["cw"], p["ptop"] + p["ch"])).resize(shape)
    bg = rgb(bgpath)
    add = IM.get_add_objs(os.path.basename(os.path.dirname(os.path.dirname(path))))
    rng.shuffle(add)
    img, mask = rgb(path), rgb(IM.mask_path(path))
    p = IM.draw_main(img.size[0], img.size[1], shape, jitter, rng)
    img, mask = (ImageChops.offset(crop_resize(a, p), p["shift_x"], p["shift_y"]) for a in (img, mask))
    if p["flip"]:
        img, mask = img.transpose(Image.FLIP_LEFT_RIGHT), mask.transpose(Image.FLIP_LEFT_RIGHT)
    m0 = np.asarray(mask)
    main = sel(img, m0, np.zeros_like(m0))
    tm, ti, attempts = m0, main, 0
    for obj in add:
        while True:
            attempts += 1
            with open(os.path.join(root, "LINEMOD", obj, "train.txt")) as f:
                lines = f.readlines()
            vp = os.path.join(root, lines[rng.randint(0, len(lines) - 1)].rstrip())
            v, vm = rgb(vp), rgb(IM.mask_path(vp))
            v = Image.fromarray(sel(v, np.asarray(vm), np.zeros_like(np.asarray(vm))))
            c = IM.draw_crop(v.size[0], v.size[1], jitter, rng)
            v, vm = crop_resize(v, c), crop_resize(vm, c)
            if c["flip"]:
                v, vm = v.transpose(Image.FLIP_LEFT_RIGHT), vm.transpose(Image.FLIP_LEFT_RIGHT)
            m = np.asarray(vm)
            xx = m > 200
            s = int(xx.sum())
            if s and float(int((xx & (tm > 200)).sum())) / float(s) < 0.2:
                tm = np.clip(m.astype(np.int32) + tm.astype(np.int32) * neg[m], 0, 255).astype(np.uint8)
                ti = sel(v, m, ti)
                break
    ti = sel(main, m0, ti)
    return sel(ti, tm, bg.resize(shape)), attempts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--pil-samples", type=int, default=4)
    ap.add_argument("--views", type=int, default=8, help="views per object in the synthetic tree")
    ap.add_argument("--max-attempts", type=int, default=1000, help="per pasted object; the reference has no bound")
    a = ap.parse_args()
    import torch
    from singleshotpose_b200 import image_multi as IM, synth
    B, shape = a.batch, (a.size, a.size)
    with tempfile.TemporaryDirectory() as root:
        bgs = synth.write_linemod_multi_like(root, n=a.views, ow=640, oh=480, num_bg=4, spread=True)
        objs = [o for o in synth.LINEMOD_OBJECTS]
        samples = [(os.path.join(root, "LINEMOD", objs[i % 13], "JPEGImages", "%06d.png" % (i // 13 % a.views)), bgs[i % len(bgs)])
                   for i in range(B)]
        aug = IM.GpuMultiAugmenter("cuda", root=root, keep_u8=True, max_attempts=a.max_attempts, timing=True)
        runs = []
        for b in range(a.batches):
            seeds = [1000 * b + i for i in range(B)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            x, labels = aug(samples, shape, [random.Random(s) for s in seeds])
            torch.cuda.synchronize()
            att = [sum(v) for v in aug.attempts]
            span = sum(e0.elapsed_time(e1) for e0, e1 in aug.timing)
            runs.append(dict(wall_s=time.perf_counter() - t0, span_ms=span, rounds=aug.rounds, decodes=aug.decodes,
                             h2d=aug.h2d_bytes, att_mean=float(np.mean(att)), att_max=int(max(att)), seeds=seeds))
            print("batch %d: %.2f s, %d rounds" % (b, runs[-1]["wall_s"], aug.rounds), file=sys.stderr, flush=True)
        last_u8 = aug.u8[a.pil_samples - 1].cpu().numpy() if a.pil_samples else None
        warm = runs[1:] or runs
        res = {"batch": B, "size": a.size, "source": "640x480 synthetic LINEMOD tree, 13 objects x %d views, objects spread over the central 3/4 of the frame "
                                               "(synth spread=True: fewer rejections than the test tree)" % a.views,
               "cold_images_per_s": B / runs[0]["wall_s"], "warm_images_per_s": B / float(np.mean([r["wall_s"] for r in warm])),
               "cold_device_ms": runs[0]["span_ms"], "warm_device_ms": float(np.mean([r["span_ms"] for r in warm])),
               "rounds_per_batch": [r["rounds"] for r in runs], "attempts_per_sample_mean": [r["att_mean"] for r in runs],
               "attempts_per_sample_max": [r["att_max"] for r in runs], "decodes_per_batch": [r["decodes"] for r in runs],
               "h2d_bytes_per_batch": [r["h2d"] for r in runs]}
        if a.pil_samples:
            t0 = time.perf_counter()
            for i in range(a.pil_samples):
                out, _att = pil_sample(samples[i][0], samples[i][1], shape, random.Random(runs[-1]["seeds"][i]), root)
            dt = (time.perf_counter() - t0) / a.pil_samples
            res.update(pil_1thread_ms_per_sample=dt * 1e3, pil_1thread_images_per_s=1.0 / dt, pil_last_sample_byte_identical=bool(
                np.array_equal(out, last_u8)))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        res["gpu"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        res["gpu"] = torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
