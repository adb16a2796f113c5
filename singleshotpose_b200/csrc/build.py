"""Build libssp_b200.so in-tree with nvcc for sm_90a (no other architectures, no JIT cache)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["abi.cu", "conv_tc.cu", "conv_band.cu", "conv_bandt.cu", "wgrad_tc.cu", "conv_simt.cu", "l0_fused.cu", "elementwise.cu", "sgd_pack.cu", "region.cu", "region_multi.cu", "pnp.cu", "pnp_consensus.cu", "pnp_dist.cu", "track.cu", "pose_filter.cu", "refine_depth.cu", "refine_rig.cu", "refine_instances.cu", "multiview_rows.cu", "multiview.cu", "multiview_instances.cu", "calibrate_rig.cu", "calibrate_rig_depth.cu", "world_track.cu", "augment.cu", "adds.cu", "jpeg.cu", "render.cu"]
# augment.cu restates Pillow's float/double pixel arithmetic bit for bit: no multiply-add contraction there
# pose_filter.cu: the fp64 filter arithmetic is rounded as the host harness (g++ -ffp-contract=off) rounds it
# refine_depth.cu, refine_rig.cu, refine_instances.cu: likewise, so the refinements' sums equal the harness's bit for bit
# multiview.cu, multiview_instances.cu: the fusion stages likewise (multiview_rows.cu keeps the contraction of pnp.cu, whose bits its
# PnP reproduces); world_track.cu: the pose filter of the world tracks likewise; calibrate_rig.cu,
# calibrate_rig_depth.cu: the rig calibrations likewise
EXTRA = {"augment.cu": ["-fmad=false"], "pose_filter.cu": ["-fmad=false"], "refine_depth.cu": ["-fmad=false"], "refine_rig.cu": ["-fmad=false"], "refine_instances.cu": ["-fmad=false"],
         "multiview.cu": ["-fmad=false"],
         "multiview_instances.cu": ["-fmad=false"], "world_track.cu": ["-fmad=false"],
         "calibrate_rig.cu": ["-fmad=false"], "calibrate_rig_depth.cu": ["-fmad=false"]}
LIB = os.path.join(HERE, "libssp_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cu", ".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "..", "include", "ssp_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC, *FLAGS, *EXTRA.get(src, []), "-c", os.path.join(HERE, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("== %s ==\n%s\n" % (src, out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB, *objs])   # static cudart (nvcc default)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
