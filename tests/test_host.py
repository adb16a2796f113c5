"""CPU-only tests: host logic (cfg parsing, execution plan, .weights format), the C-ABI surface and its binding, and the N>1
gradient all-reduce path with the gloo backend (world size 2).  No GPU, no compute calls into the library."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from singleshotpose_b200 import _lib, Darknet
from singleshotpose_b200.cfg import parse_cfg, layer_shapes, print_cfg
from singleshotpose_b200.cfgs import yolo_pose_cfg_text
from singleshotpose_b200.engine import build_plan

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cfg_parse_semantics(cfg_path, cfg_multi_path, capsys):
    b = parse_cfg(cfg_path)
    assert len(b) == 33 and b[0]["type"] == "net" and b[-1]["type"] == "region"
    assert b[1]["batch_normalize"] == "1" and b[-2]["batch_normalize"] == 0        # default for [convolutional]
    assert b[-1]["anchors"] == "" and b[-1]["classes"] == "1"
    shp = layer_shapes(b)
    assert [s[0] for s in shp].count("conv") == 23
    assert shp[29][1:3] == (1280, 1024) and shp[30][2] == 20 and shp[30][5:7] == (13, 13)
    bm = parse_cfg(cfg_multi_path)
    assert layer_shapes(bm)[30][2] == 160 and bm[-1]["num"] == "5"
    print_cfg(b)
    out = capsys.readouterr().out
    assert "   29 conv   1024  3 x 3 / 1    13 x  13 x1280   ->    13 x  13 x1024" in out
    assert "   28 route  27 24" in out


def test_execution_plan_with_fused_first_blocks(cfg_path):
    layers = build_plan(parse_cfg(cfg_path))
    assert len(layers) == 23
    l16 = [L for L in layers if L.block_ind == 16][0]
    assert sorted(k for (_, _, k) in l16.dests) == [_lib.ROUTE_DIRECT, _lib.ROUTE_POOL]     # maxpool 17 + route 25
    l29 = [L for L in layers if L.block_ind == 29][0]
    assert l29.cin == 1280
    assert [(layers[s].block_ind, k, c0, c) for (s, k, c0, c) in l29.leaves] == [(26, _lib.ROUTE_REORG, 0, 256), (24, _lib.ROUTE_DIRECT, 256, 1024)]
    assert layers[0].first and not any(L.first for L in layers[1:])                 # blocks 0-1: conv 3 -> 32 + BN + leaky, maxpool 2/2
    assert (layers[0].cin, layers[0].cout, layers[0].taps, layers[0].bn) == (3, 32, 9, True)
    assert layers[0].dests == [(1, 0, _lib.ROUTE_POOL)]
    assert not layers[-1].bn and layers[-1].cout == 20


def test_unsupported_blocks_raise(tmp_path):
    txt = yolo_pose_cfg_text().replace("[maxpool]\nsize=2\nstride=2", "[maxpool]\nsize=2\nstride=1", 1)
    p = tmp_path / "bad.cfg"
    p.write_text(txt)
    with pytest.raises(NotImplementedError):
        Darknet(str(p))


def test_first_conv_without_maxpool_raises(tmp_path):
    """blocks 0-1 run as one fused unit (conv 3 -> 32 + BN + leaky + max-pool 2/2): a first conv that feeds another conv is refused"""
    conv = "[convolutional]\nbatch_normalize=1\nfilters=32\nsize=1\nstride=1\npad=1\nactivation=leaky\n"
    txt = yolo_pose_cfg_text().replace("[maxpool]\nsize=2\nstride=2\n", conv, 1)
    assert txt != yolo_pose_cfg_text()
    p = tmp_path / "bad.cfg"
    p.write_text(txt)
    with pytest.raises(NotImplementedError, match="blocks 0-1"):
        Darknet(str(p))


def test_parameter_names_and_counts(cfg_path):
    torch.manual_seed(0)
    m = Darknet(cfg_path)
    names = [n for n, _ in m.named_parameters()]
    assert len(names) == 68 and names[0] == "models.0.conv1.weight" and names[1] == "models.0.bn1.weight"
    assert names[-2:] == ["models.30.conv23.weight", "models.30.conv23.bias"]
    assert sum(p.numel() for p in m.parameters()) == 50547764
    assert (m.width, m.height, m.test_width, m.num_keypoints, m.num_classes, m.num_anchors) == (416, 416, 672, 9, 1, 1)
    assert m.models[-1].noobject_scale == 0.1 and m.models[-1].object_scale == 5.0     # cfg values land on the unused head


def test_weights_file_format_roundtrip(cfg_path, tmp_path):
    torch.manual_seed(3)
    m = Darknet(cfg_path)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.normal_(); mod.running_var.uniform_(0.5, 2.0)
    m.seen = 4711
    f = str(tmp_path / "a.weights")
    m.save_weights(f)
    assert os.path.getsize(f) == 16 + 4 * 50568436                      # header + fp32 stream (SURVEY a7)
    raw = np.fromfile(f, dtype=np.float32, offset=16)
    bn0, conv0 = m.models[0][1], m.models[0][0]
    np.testing.assert_array_equal(raw[:32], bn0.bias.detach().numpy())            # order: bn.bias, bn.weight, mean, var, conv.weight
    np.testing.assert_array_equal(raw[64:96], bn0.running_mean.numpy())
    np.testing.assert_array_equal(raw[128:128 + 864], conv0.weight.detach().numpy().reshape(-1))   # OIHW order
    torch.manual_seed(4)
    m2 = Darknet(cfg_path)
    m2.load_weights(f)
    assert int(m2.seen) == 4711
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        if "num_batches" not in k:
            assert torch.equal(a, b), k
    torch.manual_seed(5)
    m3 = Darknet(cfg_path)
    last_before = m3.models[30][0].weight.detach().clone()
    m3.load_weights_until_last(f)
    assert torch.equal(m3.models[29][0].weight, m.models[29][0].weight)
    assert torch.equal(m3.models[30][0].weight, last_before)                       # last conv untouched (darknet.py:310)


def test_abi_exports_every_declared_symbol():
    hdr = open(os.path.join(REPO, "include", "ssp_b200.h")).read()
    declared = set(re.findall(r"\b(ssp_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.ssp_version() >= 100
    assert _lib.flat_alloc_rows(64, 416, 416) >= 64 * 417 * 417 + 417 + 2


# (restype, argtypes) of the entry points with the most mixed argument lists, written out by hand: what _lib must read from the header
_p, _i, _ll, _f, _d = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double
_PINNED = {
    "ssp_last_error": (C.c_char_p, []),
    "ssp_flat_alloc_rows": (_ll, [_i, _i, _i]),
    "ssp_jpeg_decline_reason": (C.c_char_p, [_i]),
    "ssp_conv_gemm": (_i, [_i, _p, _p, _ll, _i, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _i, _ll, _i, _p, _p, _p, _p]),
    "ssp_wgrad_gemm": (_i, [_i, _p, _ll, _i, _i, _i, _p, _ll, _i, _i, _i, _i, _i, _i, _i, _p, _i, _i, _f, _p]),
    "ssp_bn_finalize": (_i, [_p, _p, _d, _p, _p, _p, _p, _f, _f, _i, _p, _p, _p, _p, _i, _p]),
    "ssp_l0_bwd_finalize": (_i, [_p, _p, _p, _p, _p, _p, _d, _f, _p, _p, _p, _p]),
    "ssp_pnp_batched": (_i, [_p, _i, _p, _p, _i, _ll, _i, _p, _p, _p, _p]),
    "ssp_jpeg_batch_run": (_i, [_p, _i, _p, _p, _ll, _p, _p]),
    "ssp_render_masks": (_i, [_p, _i, _i, _p, _i, _p, _p, _ll, _i, _i, _p, _p, _p, _ll, _p]),
}


def test_abi_signatures_read_from_the_header():
    for name, (restype, argtypes) in _PINNED.items():
        assert (_lib.RETURNS[name], _lib.SIGNATURES[name]) == (restype, argtypes), name
    lib = _lib.load()
    assert all(getattr(lib, n).argtypes == a and getattr(lib, n).restype == _lib.RETURNS[n] for n, a in _lib.SIGNATURES.items())
    wide = {n for n, r in _lib.RETURNS.items() if r is not _i}          # every return that is not an int status
    assert wide == {"ssp_last_error", "ssp_jpeg_decline_reason", "ssp_flat_alloc_rows", "ssp_flat_row", "ssp_jpeg_stage_bytes",
                    "ssp_jpeg_work_bytes", "ssp_aug_resize_work_bytes", "ssp_aug_sample_work_bytes", "ssp_aug_batch_table_bytes",
                    "ssp_augm_work_bytes", "ssp_augm_table_bytes", "ssp_adds_work_bytes", "ssp_render_work_bytes"}


_STRUCT_NAMES = ["ssp_sgd_segment", "ssp_aug_item", "ssp_augm_item", "ssp_jpeg_info", "ssp_jpeg_item"]


@pytest.fixture(scope="module")
def compiled_header(tmp_path_factory):
    """what the C compiler makes of include/ssp_b200.h: sizeof and every offsetof of the structs, the value of every macro"""
    d = tmp_path_factory.mktemp("abi")
    layout = ["sizeof(%s)" % s + "".join(", offsetof(%s, %s)" % (s, f) for f, _ in _lib.STRUCTS[s]._fields_) for s in _STRUCT_NAMES]
    (d / "abi.c").write_text('#include <stddef.h>\n#include "ssp_b200.h"\nconst long long layout[] = {%s};\nconst long long constants[] = {%s};\n'
                             % (", ".join(layout), ", ".join(_lib.CONSTANTS)))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-I", os.path.join(REPO, "include"), "-o", str(d / "libabi.so"), str(d / "abi.c")])
    return C.CDLL(str(d / "libabi.so"))


def test_abi_struct_layouts_match_the_compiler(compiled_header):
    assert sorted(_lib.STRUCTS) == sorted(_STRUCT_NAMES)
    want = []
    for s in _STRUCT_NAMES:
        cls = _lib.STRUCTS[s]
        want += [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    assert list((C.c_longlong * len(want)).in_dll(compiled_header, "layout")) == want
    assert C.sizeof(_lib.STRUCTS["ssp_sgd_segment"]) == np.dtype(_lib.STRUCTS["ssp_sgd_segment"]).itemsize == 72
    hdr = open(os.path.join(REPO, "include", "ssp_b200.h")).read()
    for s in _STRUCT_NAMES:                      # no declarator lost: as many fields as names before a ';' or ',' in the struct's body
        body = re.search(r"typedef struct %s \{(.*?)\}" % s, re.sub(r"/\*.*?\*/", "", hdr, flags=re.S), re.S).group(1)
        assert [f for f, _ in _lib.STRUCTS[s]._fields_] == re.findall(r"(\w+)\s*[;,]", body), s


def test_abi_constants_match_the_compiler(compiled_header):
    hdr = open(os.path.join(REPO, "include", "ssp_b200.h")).read()
    assert set(_lib.CONSTANTS) == set(re.findall(r"^#define (SSP_\w+)[ \t]+\S", hdr, re.M))       # all but the include guard
    got = list((C.c_longlong * len(_lib.CONSTANTS)).in_dll(compiled_header, "constants"))
    assert got == list(_lib.CONSTANTS.values())
    assert (_lib.CONSTANTS["SSP_ERR_ARG"], _lib.CONSTANTS["SSP_L0_GRAM_DOUBLES"], _lib.CONSTANTS["SSP_JPEG_ST_OVERFLOW"]) == (-1, 2816, 8)
    assert (_lib.FMT_BF16, _lib.IMPL_BANDT, _lib.EPI_F16, _lib.ROUTE_REORG, _lib.ROUTE_F16) == (1, 4, 8, 3, 16)


@pytest.mark.parametrize("text, complaint", [
    ("int ssp_a(int n, size_t bytes);", "unknown type 'size_t'"),
    ("short ssp_a(void);", "unknown type 'short'"),
    ("int ssp_a(int, float x);", "no 'type name'"),
    ("typedef struct ssp_s { int a; long long b;\nint ssp_a(const ssp_s* s);", "neither a prototype nor a struct"),
    ("#define SSP_N (1 << 4)", "not an integer literal"),
])
def test_abi_parser_refuses_what_it_cannot_read(text, complaint):
    with pytest.raises(_lib.SspError, match=re.escape(complaint)):
        _lib.parse_header(text)


def test_abi_parser_reads_each_construct():
    sig, ret, const, structs = _lib.parse_header("#define SSP_N (-3)\ntypedef struct ssp_s { unsigned* p; int a, b; } ssp_s;\n"
                                                 "const char* ssp_a(const ssp_s* s, /* note */ double x);")
    assert (sig, ret, const) == ({"ssp_a": [_p, _d]}, {"ssp_a": C.c_char_p}, {"SSP_N": -3})
    assert structs["ssp_s"]._fields_ == [("p", _p), ("a", _i), ("b", _i)]


def test_no_cpu_fallback(cfg_path):
    from singleshotpose_b200 import RegionLoss
    with pytest.raises(_lib.SspError):
        Darknet(cfg_path)(torch.zeros(1, 3, 416, 416))
    with pytest.raises(_lib.SspError):
        RegionLoss()(torch.zeros(1, 20, 13, 13), torch.zeros(1, 1050), 0)


def test_product_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(REPO, "singleshotpose_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from singleshotpose_b200.optim import all_reduce_flat_, dp_hyperparams
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
r = dist.get_rank()
g = torch.arange(10, dtype=torch.float32) * (r + 1)          # rank-dependent "gradient of a sum-loss"
all_reduce_flat_(g)
assert torch.equal(g, torch.arange(10, dtype=torch.float32) * 3), g
lr, wd = dp_hyperparams(0.001 * 0.1, 0.0005, per_gpu_batch=64)
assert abs(lr - 1e-4 / 128) < 1e-12 and abs(wd - 0.0005 * 128) < 1e-9
dist.barrier(); dist.destroy_process_group()
print("ok", r)
'''


def test_gradient_allreduce_two_ranks_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = str(29500 + os.getpid() % 2000)
    ps = [subprocess.Popen([sys.executable, str(script), REPO, port, str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
          for r in range(2)]
    outs = [p.communicate(timeout=120)[0] for p in ps]
    assert all(p.returncode == 0 for p in ps), outs
    assert all("ok" in o for o in outs)


def test_bench_reference_arm_other_ranks_exit():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                       env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_optimizer_state_checkpoint_interchanges_with_torch_sgd(cfg_path):
    """FlatSGD.state_dict()/load_state_dict() speak torch.optim.SGD's format (SURVEY 8f.4): momentum buffers are stored flat in
    the kernel's OHWI layout but exchanged as OIHW tensors, so a checkpoint moves between FlatSGD and train.py:388's optimiser."""
    import torch
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.optim import FlatSGD
    torch.manual_seed(0)
    m = Darknet(cfg_path)
    m._engine.materialize(torch.device("cpu"))                       # flat buffers + views; no kernel involved
    params = list(m.parameters())
    ref = torch.optim.SGD(params, lr=1e-3, momentum=0.9, dampening=0, weight_decay=0.032)
    gen = torch.Generator().manual_seed(1)
    for p in params[:6] + params[-2:]:                               # optim.SGD keeps buffers only for parameters it stepped
        ref.state[p]["momentum_buffer"] = torch.randn(p.shape, generator=gen)
    sd = ref.state_dict()
    opt = FlatSGD(m, lr=5.0, momentum=0.0, weight_decay=0.0)
    opt.load_state_dict(sd)
    assert opt.param_groups[0] == dict(lr=1e-3, momentum=0.9, weight_decay=0.032)
    w0 = params[0]
    off, n, _ = m._engine._slices[id(w0)]
    want = sd["state"][0]["momentum_buffer"].permute(0, 2, 3, 1).reshape(-1)          # flat storage is [co][kh][kw][ci]
    assert torch.equal(opt._v[off:off + n], want)
    out = opt.state_dict()
    assert set(out["state"]) == set(range(len(params)))
    for i, p in enumerate(params):
        got = out["state"][i]["momentum_buffer"]
        exp = sd["state"][i]["momentum_buffer"] if i in sd["state"] else torch.zeros(p.shape)
        assert got.is_contiguous() and torch.equal(got, exp), i
    ref2 = torch.optim.SGD(params, lr=1.0)
    ref2.load_state_dict(out)                                        # and back into the stock optimiser
    assert ref2.param_groups[0]["momentum"] == 0.9 and torch.equal(ref2.state[params[3]]["momentum_buffer"], out["state"][3]["momentum_buffer"])
    with pytest.raises(ValueError):
        bad = {"state": {}, "param_groups": [dict(sd["param_groups"][0], nesterov=True)]}
        opt.load_state_dict(bad)


def test_checkpoint_weights_plus_optimizer_state(cfg_path, tmp_path):
    import torch
    from singleshotpose_b200.darknet import Darknet
    from singleshotpose_b200.optim import FlatSGD
    from singleshotpose_b200.checkpoint import save_checkpoint, load_checkpoint
    torch.manual_seed(3)
    a = Darknet(cfg_path); a._engine.materialize(torch.device("cpu"))
    oa = FlatSGD(a, lr=1e-4, momentum=0.9, weight_decay=0.032)
    oa._v = torch.randn(a._engine.flat_params.numel(), generator=torch.Generator().manual_seed(4))
    a.seen, a.iter = 6400, 100
    f = str(tmp_path / "ck.weights")
    save_checkpoint(a, oa, f)
    torch.manual_seed(9)
    b = Darknet(cfg_path); b._engine.materialize(torch.device("cpu"))
    ob = FlatSGD(b, lr=1.0)
    assert load_checkpoint(b, ob, f) is True
    assert (b.seen, b.iter) == (6400, 100) and ob.param_groups[0]["momentum"] == 0.9
    assert torch.equal(ob._v, oa._v)
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(p, q), n
    os.remove(f + ".optim.pt")
    with pytest.raises(FileNotFoundError):
        load_checkpoint(b, ob, f)
    assert load_checkpoint(b, ob, f, strict=False) is False
