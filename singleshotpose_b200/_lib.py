"""ctypes binding of libssp_b200.so (include/ssp_b200.h).  There is NO fallback: if the library is missing
or a call fails, an exception is raised -- the product path never routes through the CPU oracle."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SSP_LIB") or os.path.join(_HERE, "csrc", "libssp_b200.so")   # SSP_LIB: A/B experiments only

FMT_F16, FMT_BF16 = 0, 1
IMPL_TC, IMPL_SIMT, IMPL_TC2, IMPL_BAND, IMPL_BANDT = 0, 1, 2, 3, 4
EPI_F32, EPI_STATS, EPI_BIAS, EPI_F16 = 0, 1, 2, 8
ROUTE_NONE, ROUTE_DIRECT, ROUTE_POOL, ROUTE_REORG = 0, 1, 2, 3
ROUTE_F16 = 16          # OR-ed into a gradient route of ssp_bn_bwd_*: that plane holds fp16

_p, _i, _ll, _f, _d = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double

# name -> argtypes (restype int unless stated); must list every symbol of include/ssp_b200.h
SIGNATURES = {
    "ssp_version": [],
    "ssp_last_error": [],
    "ssp_flat_alloc_rows": [_i, _i, _i],
    "ssp_flat_row": [_i, _i, _i, _i, _i],
    "ssp_pack_nchw": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _f, _p],
    "ssp_unpack_nchw": [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    "ssp_unpack16_nchw": [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "ssp_conv_gemm": [_i, _p, _p, _ll, _i, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _i, _ll, _i, _p, _p, _p, _p],
    "ssp_conv_bandt_launches": [],
    "ssp_l0_gram": [_p, _i, _i, _i, _p, _p],
    "ssp_l0_stats": [_p, _p, _p, _p, _p],
    "ssp_l0_fused_fwd": [_p, _p, _p, _p, _f, _i, _i, _i, _p, _p, _i, _i, _p, _p],
    "ssp_l0_bwd": [_p, _p, _i, _i, _i, _p, _f, _i, _i, _i, _p, _p],
    "ssp_l0_bwd_finalize": [_p, _p, _p, _p, _p, _p, _d, _f, _p, _p, _p, _p],
    "ssp_conv_gemm_bnact": [_i, _p, _p, _ll, _i, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _f, _p, _p, _i, _i, _p],
    "ssp_conv_gemm_splitk": [_p, _p, _ll, _i, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p, _ll, _i, _p],
    "ssp_conv_splitk_count": [_i, _i, _i, _i, _i, _i, _i],
    "ssp_bn_apply_splitk": [_p, _i, _ll, _i, _p, _p, _i, _i, _i, _i, _f, _p, _p, _i, _i, _i, _p, _p, _i, _i, _i, _p],
    "ssp_wgrad_gemm": [_i, _p, _ll, _i, _i, _i, _p, _ll, _i, _i, _i, _i, _i, _i, _i, _p, _i, _i, _f, _p],
    "ssp_bn_finalize": [_p, _p, _d, _p, _p, _p, _p, _f, _f, _i, _p, _p, _p, _p, _i, _p],
    "ssp_bn_apply": [_p, _i, _p, _p, _i, _i, _i, _i, _f, _p, _p, _i, _i, _i, _p, _p, _i, _i, _i, _p, _i, _p],
    "ssp_bn_bwd_reduce": [_p, _i, _p, _p, _p, _p, _p, _i, _i, _i, _i, _f, _p, _i, _i, _i, _p, _i, _i, _i, _p, _p, _p],
    "ssp_bn_bwd_apply": [_p, _i, _p, _p, _p, _p, _p, _i, _i, _i, _i, _f, _p, _i, _i, _i, _p, _i, _i, _i, _p, _p, _p, _i, _i, _f, _p],
    "ssp_bn_bwd_finalize": [_p, _p, _p, _p, _i, _i, _f, _p],
    "ssp_bias_grad_nchw": [_p, _p, _i, _i, _i, _i, _f, _p],
    "ssp_pack_weights": [_p, _i, _i, _i, _p, _p, _i, _p, _i, _i, _p],
    "ssp_sgd_step_flat": [_p, _p, _p, _ll, _f, _f, _f, _f, _p],
    "ssp_sgd_segment_blocks": [_i, _i, _i, _ll],
    "ssp_sgd_pack_step": [_p, _i, _i, _i, _p, _p, _p, _f, _f, _f, _f, _p],
    "ssp_region_loss_fwd_bwd": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _f, _f, _f, _f, _i, _f, _p],
    "ssp_region_decode_argmax": [_p, _i, _i, _i, _i, _i, _i, _p, _p, _p, _p],
    "ssp_region_loss_multi_fwd_bwd": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p, _i, _f, _f, _f, _f, _f, _i, _f, _p],
    "ssp_region_decode_multi": [_p, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p],
    "ssp_eval_multi_select": [_p, _i, _i, _i, _i, _i, _i, _p, _i, _p, _f, _f, _f, _p, _p, _p, _p],
    "ssp_predict_multi_select": [_p, _i, _i, _i, _i, _i, _i, _p, _i, _f, _f, _f, _p, _p, _p, _p],
    "ssp_pnp_batched": [_p, _i, _p, _p, _i, _ll, _i, _p, _p, _p, _p],
    "ssp_pnp_batched_work": [_p, _i, _p, _p, _i, _ll, _i, _p, _p, _p, _p],
    "ssp_project_points": [_p, _i, _i, _p, _p, _ll, _p, _p],
    "ssp_adds_work_bytes": [_i, _ll],
    "ssp_adds_batched": [_p, _i, _p, _p, _ll, _p, _p, _p, _ll, _p],
    "ssp_mesh_diameter": [_p, _i, _p, _p],
    "ssp_render_work_bytes": [_i, _i, _ll, _i, _i],
    "ssp_render_masks": [_p, _i, _i, _p, _i, _p, _p, _ll, _i, _i, _p, _p, _p, _ll, _p],
    "ssp_aug_resize_work_bytes": [_i, _i, _i, _i, _i],
    "ssp_aug_resize_u8": [_p, _i, _i, _i, _i, _i, _i, _p, _i, _i, _i, _p, _ll, _p],
    "ssp_aug_rgb2hsv_u8": [_p, _p, _ll, _p],
    "ssp_aug_hsv2rgb_u8": [_p, _p, _ll, _p],
    "ssp_aug_to_tensor_u8": [_p, _ll, _p, _p],
    "ssp_aug_batch_table_bytes": [_i],
    "ssp_aug_batch_plan": [_p, _i, _i, _i, _i, _p, _ll, _p],
    "ssp_aug_batch_run": [_p, _i, _p, _p],
    "ssp_aug_sample_work_bytes": [_i, _i, _i, _i, _i, _i, _i, _i, _i],
    "ssp_augm_work_bytes": [_i, _i, _i, _i, _i],
    "ssp_augm_table_bytes": [_i],
    "ssp_augm_plan_begin": [_p, _i, _i, _i, _i, _p, _ll, _p],
    "ssp_augm_plan_attempt": [_p, _i, _i, _i, _i, _p, _ll, _p],
    "ssp_augm_plan_finish": [_p, _i, _i, _i, _i, _p, _ll, _p],
    "ssp_augm_run": [_p, _i, _p, _p],
    "ssp_jpeg_parse": [_p, _ll, _p],
    "ssp_jpeg_decline_reason": [_i],
    "ssp_jpeg_stage_bytes": [_p, _i],
    "ssp_jpeg_work_bytes": [_p, _i],
    "ssp_jpeg_batch_plan": [_p, _i, _p, _ll, _p],
    "ssp_jpeg_batch_run": [_p, _i, _p, _p, _ll, _p, _p],
}
_RESTYPE = {"ssp_last_error": C.c_char_p, "ssp_flat_alloc_rows": _ll, "ssp_flat_row": _ll,
            "ssp_jpeg_decline_reason": C.c_char_p, "ssp_jpeg_stage_bytes": _ll, "ssp_jpeg_work_bytes": _ll,
            "ssp_aug_resize_work_bytes": _ll, "ssp_aug_sample_work_bytes": _ll, "ssp_aug_batch_table_bytes": _ll,
            "ssp_augm_work_bytes": _ll, "ssp_augm_table_bytes": _ll, "ssp_adds_work_bytes": _ll, "ssp_render_work_bytes": _ll}

_lib = None


class SspError(RuntimeError):
    pass


def load():
    """Load the CUDA library (building is __graft_entry__.build()'s job).  Raises if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SspError("libssp_b200.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "-- singleshotpose_b200 has no CPU fallback" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(lib, name)            # AttributeError if the .so lacks a declared symbol
            fn.argtypes = args
            fn.restype = _RESTYPE.get(name, _i)
        _lib = lib
    return _lib


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise SspError("%s failed (%d): %s" % (name, rc, lib.ssp_last_error().decode()))
    return rc


def ptr(t):
    """device (or host) pointer of a torch tensor / None."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def flat_alloc_rows(N, H, W):
    return int(load().ssp_flat_alloc_rows(N, H, W))
