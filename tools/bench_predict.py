"""Latency and throughput of PosePredictor (singleshotpose_b200/predict.py): camera frames (640 x 480 uint8, host memory) -> poses.

Reports, all device times from CUDA events after warm-up:
  * per configuration (B = 1 at 416^2 and at 672^2 = valid.py's test shape, B = 8 and 64 at 416^2), alternating in rounds:
      - `pred`        the captured predictor (split-K on where the rule picks it)
      - `pred_nosplit` the same with split-K forced off (Engine.split_override = 0)
      - `eager`       today's chain: load_validation_batch + bench.py's infer_step (model(x), region_boxes_batched, pnp_batched)
    end-to-end latency host frame -> host result (median wall time) and frames/s;
  * device time per stage (image, forward, head) of one eager predictor call;
  * the captured forward alone, split-K on / off: achieved weight-plane bandwidth and MMA rate against the data-sheet floors
    (hi/lo fp16 weight planes at 3.35 TB/s; 3 x algorithmic FLOPs at 989 TFLOP/s dense fp16), naming the floor that bounds it;
  * the reference chain on the CPU at B = 1 (oracle Darknet in eval mode, the restated decode, cv2.solvePnP), with the thread
    count and CPU model;
  * the card's name and power limit.
    python tools/bench_predict.py [--reps 50] [--rounds 3]

--multi measures MultiPosePredictor (singleshotpose_b200/predict_multi.py) instead, with the same method: yolo-pose-multi.cfg at
416^2, B = 1 and 8, all 13 classes requested; the captured predictor against graph=False; the device time per stage (image,
forward, head) of one eager call; the reference chain on the CPU at B = 1 (oracle Darknet in eval mode, get_multi_region_boxes_ref
and valid_multi.py's selection for each class, cv2.solvePnP, the projection); the card's name and power limit.
    python tools/bench_predict.py --multi [--reps 50] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from singleshotpose_b200 import Darknet, synth, utils        # noqa: E402
from singleshotpose_b200.cfgs import write_cfg               # noqa: E402
from singleshotpose_b200.engine import Buffers               # noqa: E402
from singleshotpose_b200.image import load_validation_batch  # noqa: E402
from singleshotpose_b200.predict import PosePredictor        # noqa: E402

HBM_BPS, MMA_FLOPS = 3.35e12, 989e12


def _gpu_name():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _cpu_model():
    """model name, or vendor / family / model numbers where the name is hidden (virtual machines)"""
    info = {}
    try:
        for line in open("/proc/cpuinfo"):
            k, _, v = line.partition(":")
            info.setdefault(k.strip(), v.strip())
    except OSError:
        return "unknown"
    name = info.get("model name", "unknown")
    if name == "unknown":
        name = "%s family %s model %s" % (info.get("vendor_id", "?"), info.get("cpu family", "?"), info.get("model", "?"))
    return name


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def _forward_graph_ms(eng, x, split, reps):
    """device time of the eval forward alone, captured in a CUDA graph with private buffers"""
    N, _, H, W = x.shape
    old = eng.split_override
    eng.split_override = None if split else 0
    B = Buffers(eng, N, H, W, False, split_k=True)
    eng.split_override = old
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eng.forward(x, False, False, split_k=True, buffers=B)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.forward(x, False, False, split_k=True, buffers=B)
    for _ in range(3):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, sum(1 for v in B.splits if v)


def _stage_split(pred, frames, n=10):
    """median device time per stage of eager predictor calls"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    st = {"image": [], "forward": [], "head": []}
    for _ in range(n):
        pred(frames, events=ev)
        ev[3].synchronize()
        st["image"].append(ev[0].elapsed_time(ev[1])); st["forward"].append(ev[1].elapsed_time(ev[2])); st["head"].append(ev[2].elapsed_time(ev[3]))
    return {k: float(np.median(v)) for k, v in st.items()}


def main_multi(args):
    import ctypes as C
    from singleshotpose_b200._lib import call, ptr, stream_ptr
    from singleshotpose_b200.darknet_multi import Darknet as DarknetMulti
    from singleshotpose_b200.predict_multi import MultiPosePredictor
    cfg = write_cfg(multi=True)
    torch.manual_seed(0)
    model = DarknetMulti(cfg).cuda().eval()
    K = synth.intrinsics()
    objects = {c: synth.box_points((0.03 + 0.002 * c, 0.039, 0.046), with_center=False).T for c in range(13)}
    res = {"gpu": _gpu_name(), "frame": [640, 480], "classes": 13, "configs": {}}
    for bsz in (1, 8):
        frames = np.random.default_rng(bsz).integers(0, 256, size=(bsz, 480, 640, 3), dtype=np.uint8)
        pred = MultiPosePredictor(model, objects, K, batch=bsz)
        eager = MultiPosePredictor(model, objects, K, batch=bsz, graph=False)
        arms = {"pred": lambda: pred(frames, to_host=True), "pred_nograph": lambda: eager(frames, to_host=True)}
        for f in arms.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        reps = args.reps if bsz == 1 else max(5, args.reps // 5)
        lat = {k: [] for k in arms}
        for _ in range(args.rounds):                         # alternate the arms
            for k, f in arms.items():
                lat[k].append(_median_ms(f, reps))
        c = {k: {"ms": float(np.median(v)), "frames_per_s": bsz / (float(np.median(v)) * 1e-3), "rounds_ms": v} for k, v in lat.items()}
        c["eager_stage_device_ms"] = _stage_split(pred, frames)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(10):
            e0.record(); pred(frames); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        c["replay_device_ms"] = float(np.median(ts))
        c["detected"] = int(pred(frames)["detected"].sum())
        # the select kernel alone (one CTA per frame, 13 classes) on the predictor's logits; the rest of the head is the PnP
        # launch (one thread per slot), the projection and three small copies
        lg, ch = pred.logits, pred._last
        sel = lambda: call("ssp_predict_multi_select", ptr(lg), bsz, 9, 13, 5, lg.shape[2], lg.shape[3], C.c_void_p(pred._cls_host.ctypes.data), 13,
                           pred.conf_thresh, 640.0, 480.0, ptr(ch.boxes), ptr(ch.flags), ptr(ch.kp), stream_ptr())
        sel()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(100):
            sel()
        e1.record(); e1.synchronize()
        c["select_kernel_us"] = e0.elapsed_time(e1) * 10.0
        res["configs"]["B%d_416" % bsz] = c
        del pred, eager
        print(json.dumps({"B%d_416" % bsz: c}), flush=True)
    # reference chain on the CPU, B = 1 at 416^2: every class as valid_multi.py evaluates a first ground truth of that class
    import cv2
    from oracle import eval_multi_ref as EM
    from oracle.darknet_ref import RefDarknet
    from oracle.decode_multi_ref import get_multi_region_boxes_ref
    from oracle.eval_ref import compute_projection
    torch.manual_seed(0)
    ref = RefDarknet(cfg).eval()
    xb = synth.images(1, seed=0)
    K32 = K.astype(np.float32)
    thr = float(model.blocks[0]["conf_thresh"])

    def ref_chain():
        with torch.no_grad():
            o = ref(xb)
        for c, corners in objects.items():
            boxes = get_multi_region_boxes_ref(o, thr, 13, 9, synth.MULTI_ANCHORS, 5, c, only_objectness=0)[0]
            truths = np.zeros((50, 21), np.float32)
            truths[0, 0], truths[0, 1:] = c, 0.5
            (j, _carried), = EM.select_ref(boxes, truths, 9)
            uv = np.array([[float(boxes[j][2 * k]) * 640, float(boxes[j][2 * k + 1]) * 480] for k in range(9)], dtype=np.float32)
            P = np.concatenate([np.zeros((3, 1)), corners[:3]], 1)
            _ok, rvec, t = cv2.solvePnP(np.ascontiguousarray(P.T, dtype=np.float32), uv, K32, None, flags=cv2.SOLVEPNP_ITERATIVE)
            R, _ = cv2.Rodrigues(rvec)
            compute_projection(np.concatenate([P, np.ones((1, 9))], 0), np.concatenate([R, t], 1), K)
    ref_chain()
    res["cpu_reference_B1_416"] = {"ms": _median_ms(ref_chain, 5), "threads": torch.get_num_threads(), "cpu": _cpu_model()}
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--multi", action="store_true", help="measure the multi-object predictor (13 classes) instead")
    args = ap.parse_args()
    if args.multi:
        return main_multi(args)
    dev = torch.device("cuda")
    cfg = write_cfg()
    torch.manual_seed(0)
    model = Darknet(cfg).cuda().eval()
    eng = model._engine
    corners, K = synth.box_points(with_center=False).T, synth.intrinsics()
    P3 = torch.from_numpy(synth.box_points()).to(dev)
    K32 = torch.from_numpy(synth.intrinsics(np.float32)).to(dev)
    scale = torch.tensor([640.0, 480.0], device=dev)

    def infer_step(xb):                                      # bench.py's eager inference chain
        with torch.no_grad():
            o = model(xb)
            boxes, _, _ = utils.region_boxes_batched(o, 1, 9)
            return utils.pnp_batched(P3, boxes[:, :18].reshape(-1, 9, 2) * scale, K32)

    res = {"gpu": _gpu_name(), "frame": [640, 480], "configs": {}}
    for bsz, size in ((1, 416), (1, 672), (8, 416), (64, 416)):
        frames = np.random.default_rng(bsz + size).integers(0, 256, size=(bsz, 480, 640, 3), dtype=np.uint8)
        pred = PosePredictor(model, corners, K, shape=(size, size), batch=bsz)
        eng.split_override = 0
        pred_off = PosePredictor(model, corners, K, shape=(size, size), batch=bsz)
        eng.split_override = None

        def eager():
            R, t = infer_step(load_validation_batch(list(frames), (size, size), dev))
            return R.cpu(), t.cpu()
        arms = {"pred": lambda: pred(frames, to_host=True), "pred_nosplit": lambda: pred_off(frames, to_host=True), "eager": eager}
        for f in arms.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        reps = args.reps if bsz == 1 else max(5, args.reps // 5)
        lat = {k: [] for k in arms}
        for _ in range(args.rounds):                         # alternate the arms
            for k, f in arms.items():
                lat[k].append(_median_ms(f, reps))
        c = {k: {"ms": float(np.median(v)), "frames_per_s": bsz / (float(np.median(v)) * 1e-3), "rounds_ms": v} for k, v in lat.items()}
        # device time per stage, eager predictor call
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        st = {"image": [], "forward": [], "head": []}
        for _ in range(10):
            pred(frames, events=ev)
            ev[3].synchronize()
            st["image"].append(ev[0].elapsed_time(ev[1])); st["forward"].append(ev[1].elapsed_time(ev[2])); st["head"].append(ev[2].elapsed_time(ev[3]))
        c["eager_stage_device_ms"] = {k: float(np.median(v)) for k, v in st.items()}
        # device time of one replay (H2D copy of the frames + the whole chain)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(10):
            e0.record(); pred(frames); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        c["replay_device_ms"] = float(np.median(ts))
        # the forward alone against the floors
        x = pred.input.clone()
        wbytes = sum(t.numel() * t.element_size() for t in eng.w_hi + eng.w_lo if t is not None)
        flops = 0.0
        for L in eng.layers:
            h, w = eng.spatial(L, size, size)
            flops += 2.0 * bsz * h * w * L.cout * L.cin * L.taps
        fw = {}
        for split in (True, False):
            ms, nsplit = _forward_graph_ms(eng, x, split, reps)
            t = ms * 1e-3
            fw["split" if split else "nosplit"] = {"ms": ms, "split_layers": nsplit, "weight_TBps": wbytes / t / 1e12,
                                                   "mma_TFLOPs": 3 * flops / t / 1e12}
        floors = {"weights_us": wbytes / HBM_BPS * 1e6, "mma_us": 3 * flops / MMA_FLOPS * 1e6}
        fw["floors"] = floors
        fw["bounding_floor"] = "weight traffic" if floors["weights_us"] >= floors["mma_us"] else "MMA work"
        fw["split_vs_floor"] = fw["split"]["ms"] * 1e3 / max(floors.values())
        c["forward_graph"] = fw
        res["configs"]["B%d_%d" % (bsz, size)] = c
        del pred, pred_off
        print(json.dumps({"B%d_%d" % (bsz, size): c}), flush=True)
    # reference chain on the CPU, B = 1 at 416^2
    import cv2
    from oracle.darknet_ref import RefDarknet
    from oracle.decode_ref import get_region_boxes_ref
    torch.manual_seed(0)
    ref = RefDarknet(cfg).eval()
    xb = synth.images(1, seed=0)
    P3n = synth.box_points().astype(np.float32)

    def ref_chain():
        with torch.no_grad():
            o = ref(xb)
        box = get_region_boxes_ref(o, 1, 9)
        uv = np.array([[float(box[2 * j]) * 640, float(box[2 * j + 1]) * 480] for j in range(9)], dtype=np.float32)
        cv2.solvePnP(P3n, uv, synth.intrinsics(np.float32), None, flags=cv2.SOLVEPNP_ITERATIVE)
    ref_chain()
    res["cpu_reference_B1_416"] = {"ms": _median_ms(ref_chain, 5), "threads": torch.get_num_threads(), "cpu": _cpu_model()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
