"""Layout checks of the BN launchers and of the fused inference epilogue (include/ssp_b200.h): a misaligned vector address, a
leading dimension that is not a multiple of the vector width or a channel range that runs past the row is SSP_ERR_ARG before
any CUDA call, instead of a misaligned-address fault in the kernel.

The pointers are fabricated and never dereferenced.  The calls run in a child process with an empty CUDA_VISIBLE_DEVICES, so a
call that passes the argument stage cannot reach a device either: it fails with a CUDA / driver error, which is also what a
missing check looks like."""
import json
import os
import subprocess
import sys

import pytest

from singleshotpose_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG, ERR_CUDA, ERR_DRIVER = (_lib.CONSTANTS[k] for k in ("SSP_ERR_ARG", "SSP_ERR_CUDA", "SSP_ERR_DRIVER"))
DIRECT, POOL, REORG, F16 = _lib.ROUTE_DIRECT, _lib.ROUTE_POOL, _lib.ROUTE_REORG, _lib.ROUTE_F16

# runs [[symbol, args], ...] from stdin and prints [[return code, ssp_last_error()], ...]; _lib.py is loaded by path so that the
# child imports neither torch nor the package
_CHILD = r"""
import importlib.util, json, sys
spec = importlib.util.spec_from_file_location("ssp_lib", sys.argv[1])
m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
lib = m.load()
out = []
for name, args in json.load(sys.stdin):
    rc = getattr(lib, name)(*args)
    out.append([rc, lib.ssp_last_error().decode()])
print(json.dumps(out))
"""


def run_without_device(calls):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(REPO, "singleshotpose_b200", "_lib.py")], input=json.dumps(calls),
                       capture_output=True, text=True, env=env, cwd=REPO, timeout=120)
    assert p.returncode == 0, p.stderr
    return json.loads(p.stdout.strip().splitlines()[-1])


# fabricated device addresses: 4 KiB aligned bases, offsets added per case
Y, SC, SH, MU, IS, GM, D0H, D0L, D1H, D1L, YP, G0, G1, S1, S2, DY, AH, AL, BH, BL = (0x7F0000000000 + (i << 32) for i in range(20))
N, H, W = 3, 26, 26


def bn_apply(y=Y, y_ld=512, C=512, d0=(D0H, D0L, 512, 0, POOL), d1=(D1H, D1L, 512, 0, DIRECT), ypool=YP, ypool_ld=512):
    """layer 16 of yolo-pose: 512 channels at 26x26, max-pooled into block 17 and routed directly to block 25"""
    return ["ssp_bn_apply", [y, y_ld, SC, SH, N, C, H, W, 0.1, *d0, *d1, ypool, ypool_ld, None]]


def bn_apply_splitk(y=Y, splits=1, y_ld=512, C=512, d0=(D0H, D0L, 1280, 256, DIRECT)):
    slab = _lib.load().ssp_flat_alloc_rows(1, 13, 13) * y_ld
    return ["ssp_bn_apply_splitk", [y, splits, slab, y_ld, SC, SH, 1, C, 13, 13, 0.1, *d0, None, None, 0, 0, 0, None]]


def bn_bwd(name, y=Y, y_ld=512, C=512, g0=(G0, 512, 0, POOL | F16), g1=(G1, 512, 0, DIRECT | F16), dy=(DY, 512)):
    args = [y, y_ld, SC, SH, MU, IS, GM, N, C, H, W, 0.1, *g0, *g1, S1, S2]
    if name == "ssp_bn_bwd_apply":
        args += [*dy, _lib.FMT_F16, 1.0]
    return [name, args + [None]]


def bnact(d_hi=D0H, d_lo=D0L, d_ld=1280, d_c0=256, cout=1024, cin=1024, taps=9):
    """block 24 of yolo-pose: 3x3 1024 -> 1024 at 13x13 into the 1280-channel concat plane at channel 256"""
    rows = _lib.load().ssp_flat_alloc_rows(1, 13, 13)
    return ["ssp_conv_gemm_bnact", [_lib.IMPL_TC2, AH, AL, rows, cin, cin, BH, BL, cout, taps * cin, 1, 13, 13, taps, cout, SC, SH, 0.1,
                                    d_hi, d_lo, d_ld, d_c0, None]]


BAD = {
    # ssp_bn_apply: y, the arg-max plane, each destination
    "apply y misaligned": bn_apply(y=Y + 8),
    "apply y_ld % 4": bn_apply(y_ld=514),
    "apply y_ld < C": bn_apply(y_ld=508),
    "apply ypool misaligned": bn_apply(ypool=YP + 4),
    "apply d0 hi misaligned": bn_apply(d0=(D0H + 4, D0L, 512, 0, POOL)),
    "apply d0 lo misaligned": bn_apply(d0=(D0H, D0L + 2, 512, 0, POOL)),
    "apply d0 c0 % 4": bn_apply(d0=(D0H, D0L, 1280, 2, POOL)),
    "apply d0 ld % 4": bn_apply(d0=(D0H, D0L, 1282, 0, POOL)),
    "apply d0 ld < c0 + C": bn_apply(d0=(D0H, D0L, 1280, 772, POOL)),
    "apply d1 hi misaligned": bn_apply(d1=(D1H + 2, D1L, 512, 0, DIRECT)),
    "apply d1 c0 % 4": bn_apply(d1=(D1H, D1L, 1280, 258, DIRECT)),
    "apply d1 ld < c0 + C": bn_apply(d1=(D1H, D1L, 1280, 1024, DIRECT)),
    "apply reorg ld < c0 + 4C": bn_apply(C=64, y_ld=64, d0=(D0H, D0L, 1280, 1028, REORG), d1=(None, None, 0, 0, 0), ypool=None, ypool_ld=0),
    # ssp_bn_apply_splitk: the same rules with one slab (splits = 1 checked nothing about y before)
    "splitk y misaligned": bn_apply_splitk(y=Y + 4),
    "splitk y_ld % 4": bn_apply_splitk(y_ld=518),
    "splitk d0 c0 % 4": bn_apply_splitk(d0=(D0H, D0L, 1280, 254, DIRECT)),
    "splitk d0 ld < c0 + C": bn_apply_splitk(splits=2, d0=(D0H, D0L, 1280, 772, DIRECT)),
    "splitk d0 lo misaligned": bn_apply_splitk(d0=(D0H, D0L + 4, 1280, 256, DIRECT)),
}
for name in ("ssp_bn_bwd_reduce", "ssp_bn_bwd_apply"):
    k = name[7:]
    BAD.update({
        k + " y misaligned": bn_bwd(name, y=Y + 8),
        k + " y_ld % 4": bn_bwd(name, y_ld=510),
        k + " y_ld < C": bn_bwd(name, y_ld=500),
        k + " fp16 source misaligned": bn_bwd(name, g0=(G0 + 4, 512, 0, POOL | F16)),
        k + " fp32 source misaligned": bn_bwd(name, g1=(G1 + 8, 512, 0, DIRECT)),
        k + " source c0 % 4": bn_bwd(name, g1=(G1, 1280, 2, DIRECT | F16)),
        k + " source ld % 4": bn_bwd(name, g0=(G0, 514, 0, POOL | F16)),
        k + " source ld < c0 + C": bn_bwd(name, g0=(G0, 1024, 768, POOL | F16)),
        k + " reorg source ld < c0 + 4C": bn_bwd(name, C=64, y_ld=64, g0=(G0, 1280, 1028, REORG | F16), g1=(None, 0, 0, 0)),
    })
BAD.update({
    "bwd_apply dy misaligned": bn_bwd("ssp_bn_bwd_apply", dy=(DY + 2, 512)),
    "bwd_apply dy_ld % 4": bn_bwd("ssp_bn_bwd_apply", dy=(DY, 514)),
    "bwd_apply dy_ld < C": bn_bwd("ssp_bn_bwd_apply", dy=(DY, 256)),
    "bnact d_hi misaligned": bnact(d_hi=D0H + 8),
    "bnact d_lo misaligned": bnact(d_lo=D0L + 8),
    "bnact d_ld < d_c0 + cout": bnact(d_c0=264),
    "bnact 1x1 d_ld < d_c0 + cout": bnact(d_ld=1280, d_c0=1280 - 56, cout=64, cin=256, taps=1),
})

GOOD = {
    "apply layer 16 pool + direct": bn_apply(),
    "apply direct into the concat plane at 256": bn_apply(C=1024, y_ld=1024, d0=(D0H, D0L, 1280, 256, DIRECT), d1=(None, None, 0, 0, 0), ypool=None),
    "apply reorg into the concat plane at 0": bn_apply(C=64, y_ld=64, d0=(D0H, D0L, 1280, 0, REORG), d1=(None, None, 0, 0, 0), ypool=None),
    "apply single plane": bn_apply(d0=(D0H, None, 516, 4, POOL), d1=(None, None, 0, 0, 0)),
    "splitk one slab": bn_apply_splitk(),
    "splitk two slabs": bn_apply_splitk(splits=2),
    "bwd_reduce pool + direct": bn_bwd("ssp_bn_bwd_reduce"),
    "bwd_apply pool + direct": bn_bwd("ssp_bn_bwd_apply"),
    "bwd_apply fp32 sources at offsets": bn_bwd("ssp_bn_bwd_apply", g0=(G0 + 16, 1024, 512, POOL), g1=(G1, 1280, 764, DIRECT | F16), dy=(DY + 8, 516)),
    "bwd_apply reorg source": bn_bwd("ssp_bn_bwd_apply", C=64, y_ld=64, g0=(G0, 1280, 0, REORG | F16), g1=(G1, 64, 0, DIRECT | F16), dy=(DY, 64)),
    "bnact block 24": bnact(),
    "bnact 1x1 64 channels": bnact(d_ld=64, d_c0=0, cout=64, cin=256, taps=1),
}


@pytest.fixture(scope="module")
def results():
    names = list(BAD) + list(GOOD)
    got = run_without_device([BAD.get(n) or GOOD[n] for n in names])
    return dict(zip(names, got))


@pytest.mark.parametrize("case", list(BAD))
def test_bad_layout_is_an_argument_error(results, case):
    rc, msg = results[case]
    assert rc == ERR_ARG, (case, rc, msg)
    assert "aligned" in msg and ">=" in msg, msg               # the message states the rule


@pytest.mark.parametrize("case", list(GOOD))
def test_good_layout_passes_the_argument_stage(results, case):
    rc, msg = results[case]
    assert rc in (ERR_CUDA, ERR_DRIVER), (case, rc, msg)       # no device in the child: the first CUDA call fails
