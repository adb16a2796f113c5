"""Execution plan of the yolo-pose conv stack on the sm_90a kernels (libssp_b200.so).

Turns the cfg block list into a per-conv-layer program:

  forward   conv GEMM (wgmma, split-fp16 3-term) -> fp32 Y (+ per-channel batch statistics in the epilogue)
            -> bn_finalize -> bn_apply (+LeakyReLU, fused 2x2 max-pool / reorg / concat placement) which
            writes the NEXT layers' operand planes directly (route / reorg / maxpool blocks never run as
            kernels of their own; reference darknet.py:82-130 walks them one by one).
  backward  bn_bwd_reduce / bn_bwd_apply (BN + leaky + pool/reorg/route routing in one pass) -> dY plane
            -> wgrad GEMM (dW, fp32 atomics into the flat gradient buffer) and dgrad GEMM (dX, fp32).

All parameters live in ONE flat fp32 buffer (conv weights stored [cout][kh][kw][cin]; the nn.Parameter the
user sees is a permuted view with the reference's OIHW shape), all gradients in a second flat buffer: one
NCCL all-reduce and one fused SGD kernel per step (train.py:388, SURVEY 8e).
"""
from __future__ import annotations

import os

import torch

from . import _lib
from ._lib import call, ptr, stream_ptr
from .cfg import layer_shapes


def _rup(x, m):
    return (x + m - 1) // m * m


class ConvLayer:
    """Static description of one [convolutional] block (stride 1, 1x1 or 3x3 'same')."""

    def __init__(self, block_ind, cin, cout, size, bn, slope, H, W):
        self.block_ind, self.cin, self.cout, self.size = block_ind, cin, cout, size
        self.bn, self.slope, self.H, self.W = bn, slope, H, W
        self.taps = size * size
        self.leaves = []      # inputs: (producer layer index or -1 for the image, route kind, channel offset, channels)
        self.dests = []       # outputs: (consumer layer index, channel offset, route kind)
        self.first = False


def build_plan(blocks):
    """blocks (cfg.parse_cfg) -> list[ConvLayer] in execution order."""
    shapes = layer_shapes(blocks)
    exprs = []          # per block: expression tree of its output
    layers = []
    cur = ("input", int(blocks[0].get("channels", 3)))
    for ind, (block, sh) in enumerate(zip(blocks[1:], shapes)):
        t = block["type"]
        kind, ic, oc, ih, iw, oh, ow, ex = sh
        if t == "convolutional":
            if ex["stride"] != 1 or ex["size"] not in (1, 3) or (ex["size"] == 3 and ex["pad"] != 1):
                raise NotImplementedError("conv block %d: only stride-1 1x1 / 3x3-same convolutions are on the hot path" % ind)
            act = block.get("activation", "linear")
            if act not in ("leaky", "linear"):
                raise NotImplementedError("activation %r" % act)
            L = ConvLayer(ind, ic, oc, ex["size"], int(block["batch_normalize"]) == 1, 0.1 if act == "leaky" else 1.0, ih, iw)
            L.index = len(layers)
            L.leaves = _flatten(cur)
            layers.append(L)
            cur = ("conv", L.index, oc)
        elif t == "maxpool":
            if ex["size"] != 2 or ex["stride"] != 2:
                raise NotImplementedError("maxpool block %d: only 2x2 stride 2" % ind)
            cur = ("pool", cur)
        elif t == "reorg":
            if ex["stride"] != 2:
                raise NotImplementedError("reorg stride != 2")
            cur = ("reorg", cur)
        elif t == "route":
            ls = ex["layers"]
            cur = exprs[ls[0]] if len(ls) == 1 else ("cat", [exprs[l] for l in ls])
        elif t == "region":
            pass
        else:
            raise NotImplementedError("block type %r is not on the hot path" % t)
        exprs.append(cur)
    if not layers or layers[-1].bn or layers[-1].slope != 1.0 or cur[0] != "conv":
        raise NotImplementedError("the network must end in a linear, bias-only convolution (region head)")
    for L in layers[1:]:
        for (src, kind, c0, c) in L.leaves:
            if src < 0:
                raise NotImplementedError("only the first layer may read the image")
            layers[src].dests.append((L.index, c0, kind))
    first = layers[0]
    if (first.leaves != [(-1, _lib.ROUTE_DIRECT, 0, first.cin)] or first.size != 3 or first.cin != 3 or first.cout != 32 or not first.bn
            or len(first.dests) != 1 or first.dests[0][2] != _lib.ROUTE_POOL):
        raise NotImplementedError("blocks 0-1 must be a 3x3 convolution 3 -> 32 of the image with batch_normalize, then a 2x2 / 2 max-pool "
                                  "(one fused unit, csrc/l0_fused.cu)")
    first.first = True
    for L in layers[:-1]:
        if not L.bn:
            raise NotImplementedError("hidden convolution without batch_normalize")
        if not 1 <= len(L.dests) <= 2:
            raise NotImplementedError("conv block %d feeds %d consumers (1 or 2 supported)" % (L.block_ind, len(L.dests)))
    return layers


def _flatten(expr, kind=_lib.ROUTE_DIRECT, c0=0):
    """expression -> [(producer, route kind, channel offset, channels)]"""
    tag = expr[0]
    if tag == "input":
        return [(-1, kind, c0, expr[1])]
    if tag == "conv":
        c = expr[2] * (4 if kind == _lib.ROUTE_REORG else 1)
        return [(expr[1], kind, c0, c)]
    if tag in ("pool", "reorg"):
        if kind != _lib.ROUTE_DIRECT:
            raise NotImplementedError("chained pool/reorg")
        return _flatten(expr[1], _lib.ROUTE_POOL if tag == "pool" else _lib.ROUTE_REORG, c0)
    if tag == "cat":
        out = []
        for e in expr[1]:
            part = _flatten(e, kind, c0)
            out += part
            c0 += sum(p[3] for p in part)
        return out
    raise NotImplementedError(tag)


class Buffers:
    """Device buffers for one input shape (N, H, W); zero-initialised so that pad rows stay zero."""

    def __init__(self, eng, N, H, W, train, split_k=False):
        dev = eng.device
        self.N, self.H, self.W = N, H, W
        self.generation = 0
        # inference split-K (Engine.forward(split_k=True)): per-layer split count (0 = the layer keeps its kernels) and ONE fp32
        # workspace of max(splits * slab) elements, slab = the layer's rows x ld, shared by the layers (they run one after another)
        self.split_k = bool(split_k)
        self.splits = [eng.split_count(L, N, H, W) if split_k else 0 for L in eng.layers]
        self.split_ld = [_rup(L.cout, 4) for L in eng.layers]
        self.split_slab = [_lib.flat_alloc_rows(N, *eng.spatial(L, H, W)) * ld for L, ld in zip(eng.layers, self.split_ld)]
        ws = max([s * slab for s, slab in zip(self.splits, self.split_slab)] or [0])
        self.split_ws = torch.empty(ws, dtype=torch.float32, device=dev) if ws else None
        f16 = torch.float16
        self.x_hi, self.x_lo, self.y, self.rows = [], [], [], []
        self.dy, self.dx, self.ypool = [], [], []
        # per-layer BN state (batch sums, mean / invstd, folded scale / shift, backward sums) lives with the activations it
        # describes: a forward of another shape or mode between a training forward and its backward cannot overwrite it
        self.stat = []
        for L in eng.layers:
            st = {k: torch.zeros(L.cout, dtype=torch.float64, device=dev) for k in ("ssum", "ssq", "s1", "s2")}
            st.update({k: torch.zeros(L.cout, dtype=torch.float32, device=dev) for k in ("mean", "invstd", "scale", "shift")})
            self.stat.append(st)
            # spatial size of this layer for the actual input resolution
            h, w = eng.spatial(L, H, W)
            rows = _lib.flat_alloc_rows(N, h, w)
            self.rows.append(rows)
            if L.first:
                # blocks 0-1 run as one unit (csrc/l0_fused.cu): no operand planes, no full-resolution conv output, no dY plane --
                # the 28x28 Gram matrix of the image patches, a 1-byte code per pooled cell and 28x32 backward sums instead
                self.x_hi.append(None); self.x_lo.append(None); self.y.append(None)
                self.l0_gram = torch.zeros(_lib.CONSTANTS["SSP_L0_GRAM_DOUBLES"], dtype=torch.float64, device=dev)      # the 28x28 matrix + ssp_l0_gram's scratch
                if train:
                    self.l0_code = torch.zeros(_lib.flat_alloc_rows(N, h // 2, w // 2), 32, dtype=torch.uint8, device=dev)
                    self.l0_t1 = torch.zeros(28 * 32, dtype=torch.float64, device=dev)
                    self.ypool.append(None); self.dy.append(None); self.dx.append(None)
                continue
            self.x_hi.append(torch.zeros(rows, L.cin, dtype=f16, device=dev))
            self.x_lo.append(torch.zeros(rows, L.cin, dtype=f16, device=dev))
            self.y.append(torch.zeros(rows, _rup(L.cout, 4), dtype=torch.float32, device=dev))
            if train:
                pooled = any(k == _lib.ROUTE_POOL for (_c, _o, k) in L.dests)
                # y at the arg-max of every 2x2 window (pooled geometry): the BN-backward reduction of a pooled layer reads this
                # plane + the pooled gradient (8 B per window) instead of the four full-resolution y values + the gradient (20 B)
                self.ypool.append(torch.zeros(_lib.flat_alloc_rows(N, h // 2, w // 2), _rup(L.cout, 4), dtype=torch.float32, device=dev) if pooled else None)
                self.dy.append(torch.zeros(rows, _rup(L.cout, 8), dtype=f16, device=dev))
                # data gradients dX in fp16 (loss-scaled, saturating): the BN backward reads every dX twice, the GEMM epilogue writes it
                # once -- 6 of the ~22 bytes per activation element of the backward pass
                self.dx.append(torch.zeros(rows, _rup(L.cin, 8), dtype=f16, device=dev))


class Engine:
    def __init__(self, model):
        self.model = model
        self.layers = build_plan(model.blocks)
        self.device = None
        self.flat_params = None
        self.flat_grads = None
        self._views = None
        self._buffers = {}
        self._weights_version = None
        self.fuse_eval = True        # inference: BN + leaky in the GEMM epilogue (False: conv, bn_finalize, bn_apply as in training)
        # backward operands: one 16-bit format for dY, W and X (wgmma takes both 16-bit operands in one format).  fp16 + a static
        # loss scale (saturating conversion) is 8x more precise than bf16, and the activation planes are fp16 anyway.
        self.grad_scale = float(os.environ.get("SSP_GRAD_SCALE", "256"))
        # SSP_PRECISION: "exact" (default: split-fp16 hi + lo forward, three products) or "fast" (single-term fp16 forward, no lo
        # planes), case-insensitive; anything else is refused, so that a misspelt value cannot silently select the default
        precision = os.environ.get("SSP_PRECISION", "exact").lower()
        if precision not in ("exact", "fast"):
            raise _lib.SspError("SSP_PRECISION=%r: expected 'exact' (the default) or 'fast'" % os.environ["SSP_PRECISION"])
        self.fast = precision == "fast"
        self.launches = 0
        # inference split-K (forward(split_k=True)): launches of ssp_conv_gemm_splitk so far; split_override (internal, for tests and
        # tools/bench_predict.py): None = ssp_conv_splitk_count's rule, 0 = split-K off, k >= 1 = k splits (at most the k-block
        # count) for every layer the rule would consider, k = 1 included
        self.split_launches = 0
        self.split_override = None
        self._num_sms = None
        self._side = None
        self.grad_ready_hook = None  # fn(first layer index, stream): every gradient of layers >= that index is complete in `stream` order
        self.profile = None          # set to [] to record (kind, layer block, algorithmic flops, start event, end event) per GEMM launch
        net = model.blocks[0]
        self.base_hw = (int(net["height"]), int(net["width"]))

    # ------------------------------------------------------------------ geometry
    def spatial(self, L, H, W):
        """spatial size of layer L when the network input is H x W (cfg sizes scale with the /2 pools)."""
        bh, bw = self.base_hw
        if (H * L.H) % bh or (W * L.W) % bw:
            raise ValueError("input %dx%d is not compatible with the cfg's pooling pyramid" % (H, W))
        return H * L.H // bh, W * L.W // bw

    # ------------------------------------------------------------------ parameters
    def conv_modules(self):
        out = []
        for L in self.layers:
            seq = self.model.models[L.block_ind]
            out.append((seq[0], seq[1] if L.bn else None))
        return out

    def materialize(self, device):
        """Move all parameters into one flat fp32 buffer on `device` (conv weights as [co][kh][kw][ci]) and make the
        nn.Parameters views of it; idempotent (checked through data_ptr)."""
        params = list(self.model.parameters())
        if self.flat_params is not None and self.flat_params.device == device and self._views is not None:
            if all(p.data_ptr() == v for p, v in zip(params, self._views)):
                return
        total = sum(p.numel() for p in params)
        flat = torch.empty(total, dtype=torch.float32, device=device)
        grads = torch.zeros(total, dtype=torch.float32, device=device)
        conv_w = {id(c.weight) for c, _ in self.conv_modules()}
        off = 0
        self._slices = {}
        views = []
        for p in params:
            n = p.numel()
            if id(p) in conv_w:
                co, ci, kh, kw = p.shape
                view = flat[off:off + n].view(co, kh, kw, ci).permute(0, 3, 1, 2)
                gview = grads[off:off + n].view(co, kh, kw, ci).permute(0, 3, 1, 2)
            else:
                view = flat[off:off + n].view(p.shape)
                gview = grads[off:off + n].view(p.shape)
            view.copy_(p.data.to(device=device, dtype=torch.float32))
            p.data = view
            p.grad = None
            self._slices[id(p)] = (off, n, gview)
            views.append(view.data_ptr())
            off += n
        for _, bn in self.conv_modules():
            if bn is not None:
                bn.running_mean.data = bn.running_mean.data.to(device=device, dtype=torch.float32).contiguous()
                bn.running_var.data = bn.running_var.data.to(device=device, dtype=torch.float32).contiguous()
        self.flat_params, self.flat_grads, self._views, self.device = flat, grads, views, device
        self._alloc_layer_state(device)
        self._buffers = {}
        self._weights_version = None
        self._seg_table = None

    def _alloc_layer_state(self, dev):
        """fp16 operand planes of the GEMM layers' weights: W_hi / W_lo [cout][taps*cin] (forward), W_d [cin][taps*cout] (data
        gradient).  Layer 0 has none: the fused unit of blocks 0-1 reads the fp32 master weights."""
        self.w_hi, self.w_lo, self.w_d = [], [], []
        f16 = torch.float16
        for L in self.layers:
            if L.first:
                self.w_hi.append(None); self.w_lo.append(None); self.w_d.append(None)
                continue
            kf = _rup(L.taps * L.cin, 8)
            self.w_hi.append(torch.zeros(L.cout, kf, dtype=f16, device=dev))
            self.w_lo.append(torch.zeros(L.cout, kf, dtype=f16, device=dev))
            self.w_d.append(torch.zeros(L.cin, _rup(L.taps * L.cout, 8), dtype=f16, device=dev))

    # ------------------------------------------------------------------ fused SGD + re-pack work list, gradient buckets
    def sgd_segments(self):
        """device table (ssp_sgd_segment, include/ssp_b200.h) for ssp_sgd_pack_step: one entry per parameter tensor in flat order.
        Returns (table tensor, [(block0, nblocks)] per parameter)."""
        if getattr(self, "_seg_table", None) is not None:
            return self._seg_table, self._seg_blocks
        import numpy as np
        lib = _lib.load()
        # the GEMM layers' weights also rewrite their operand planes; every other tensor (layer 0's weight included) is plain
        conv_of = {id(conv.weight): L for L, (conv, _) in zip(self.layers, self.conv_modules()) if not L.first}
        params = list(self.model.parameters())
        tab = np.zeros(len(params), dtype=np.dtype(_lib.STRUCTS["ssp_sgd_segment"]))
        blocks, b0 = [], 0
        for k, p in enumerate(params):
            off, n, _g = self._slices[id(p)]
            e = tab[k]
            e["off"], e["n"], e["block0"] = off, n, b0
            L = conv_of.get(id(p))
            if L is not None:
                i = L.index
                e["cout"], e["taps"], e["cin"] = L.cout, L.taps, L.cin
                e["d"], e["ld_d"], e["d_fmt"] = self.w_d[i].data_ptr(), self.w_d[i].shape[1], _lib.FMT_F16
                e["f_hi"], e["f_lo"], e["ld_f"] = self.w_hi[i].data_ptr(), self.w_lo[i].data_ptr(), self.w_hi[i].shape[1]
            nb = int(lib.ssp_sgd_segment_blocks(int(e["cout"]), int(e["taps"]), int(e["cin"]), n))
            blocks.append((b0, nb))
            b0 += nb
        self._seg_table = torch.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(self.device)
        self._seg_blocks = blocks
        return self._seg_table, blocks

    def grad_buckets(self, n_buckets=4):
        """contiguous runs of layers, LAST layers first (the order in which backward completes their gradients), each about
        1/n_buckets of the parameters: [(first layer index, (elem lo, elem hi), (block lo, block hi))].  SURVEY 8e: 'bucket in
        reverse layer order to overlap with backward'."""
        _tab, blocks = self.sgd_segments()
        params = list(self.model.parameters())
        index_of = {id(p): k for k, p in enumerate(params)}
        per_layer = []                     # (layer index, first param k, last param k)
        for L, (conv, bn) in zip(self.layers, self.conv_modules()):
            ks = [index_of[id(q)] for q in ([conv.weight] + ([bn.weight, bn.bias] if bn is not None else [conv.bias]))]
            per_layer.append((L.index, min(ks), max(ks)))
        total = self.flat_params.numel()
        target = 0.9 * total / max(1, n_buckets)
        out, acc, hi_k = [], 0, None
        for (li, k0, k1) in reversed(per_layer):
            hi_k = k1 if hi_k is None else hi_k
            acc += sum(self._slices[id(params[k])][1] for k in range(k0, k1 + 1))
            if acc >= target and len(out) < n_buckets - 1 and li > 0:
                out.append((li, k0, hi_k)); acc, hi_k = 0, None
        if hi_k is not None:
            out.append((0, 0, hi_k))
        res = []
        for (li, k0, k1) in out:
            e0 = self._slices[id(params[k0])][0]
            e1 = self._slices[id(params[k1])][0] + self._slices[id(params[k1])][1]
            res.append((li, (e0, e1), (blocks[k0][0], blocks[k1][0] + blocks[k1][1])))
        return res

    def grad_view(self, p):
        return self._slices[id(p)][2]

    def _params_version(self):
        return tuple(p._version for p in self.model.parameters())

    def invalidate_packed_weights(self):
        """the fp32 master weights changed behind the version counters (load_weights, a graph replay, an external optimiser
        writing through .data): the next forward re-packs W_hi / W_lo / W_d"""
        self._weights_version = None

    def pack_weights(self, force=False):
        ver = self._params_version()
        if not force and ver == self._weights_version:
            return
        s = stream_ptr()
        for L, (conv, _) in zip(self.layers, self.conv_modules()):
            if L.first:
                continue
            i = L.index
            off, n, _g = self._slices[id(conv.weight)]
            call("ssp_pack_weights", ptr(self.flat_params[off:off + n]), L.cout, L.taps, L.cin, ptr(self.w_hi[i]), ptr(self.w_lo[i]),
                 self.w_hi[i].shape[1], ptr(self.w_d[i]), self.w_d[i].shape[1], _lib.FMT_F16, s)
            self.launches += 1
        self._weights_version = ver

    def buffers(self, N, H, W, train, split_k=False):
        key = (N, H, W, bool(train), bool(split_k))
        b = self._buffers.get(key)
        if b is None:
            if len(self._buffers) >= 4:
                self._buffers.clear()
            b = Buffers(self, N, H, W, train, split_k)
            self._buffers[key] = b
        return b

    def _fuse_eval_layer(self, L):
        """inference layers whose BN + leaky run in the GEMM epilogue (ssp_conv_gemm_bnact)"""
        return (L.bn and self.fuse_eval and not L.first and len(L.dests) == 1 and L.dests[0][2] == _lib.ROUTE_DIRECT
                and L.cout % 32 == 0)

    def split_count(self, L, N, H, W):
        """split-K count of an inference forward of layer L on an N x 3 x H x W input: 0 = the layer keeps its kernels.  Only BN
        layers whose forward runs on the per-tap tensor-core kernel are split; the rule is ssp_conv_splitk_count's."""
        if not L.bn or L.first or self.split_override == 0:
            return 0
        if not (self._fuse_eval_layer(L) or self._conv_impl(L) in (_lib.IMPL_TC, _lib.IMPL_TC2)):
            return 0
        h, w = self.spatial(L, H, W)
        if self.split_override is not None:
            return min(int(self.split_override), L.taps * ((L.cin + 63) // 64))
        if self._num_sms is None:
            self._num_sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        s = int(_lib.load().ssp_conv_splitk_count(N, h, w, L.taps, L.cin, L.cout, self._num_sms))
        if s < 0:
            raise _lib.SspError("ssp_conv_splitk_count failed: %s" % _lib.load().ssp_last_error().decode())
        return s if s >= 2 else 0

    def _conv_impl(self, L):
        """forward kernel of a GEMM layer.  Few output channels: operands swapped (weights on the M side, 128 / 256 pixels as the MMA's
        N; csrc/conv_bandt.cu); the ABI falls back to the kernels below by itself when the layer's weights do not fit next to two
        activation bands.  From 128 output channels the per-tap kernel (SSP_IMPL_TC2 = SSP_IMPL_TC on sm_90a), else the
        activation-band kernel for 3x3 layers."""
        if L.cout <= (128 if self.fast else 64):
            return _lib.IMPL_BANDT
        if L.cout >= 128:
            return _lib.IMPL_TC2
        return _lib.IMPL_BAND if L.taps == 9 else _lib.IMPL_TC

    def _gemm(self, kind, L, N, h, w, name, *args, stream=None):
        """launch one GEMM-shaped kernel; optionally bracket it with CUDA events on the launching stream (bench roofline)."""
        self.launches += 1
        if self.profile is None:
            call(name, *args)
            return
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call(name, *args)
        e1.record(stream)
        self.profile.append((kind, L.block_ind, 2.0 * N * h * w * L.cout * L.cin * L.taps, e0, e1))

    def _bn_finalize(self, bn, st, C, s, count=None, train=False):
        """mean / invstd and the folded scale / shift of one BatchNorm into `st`: from the running statistics when count is None
        (inference), else from the batch sums over `count` values when `train` (which also updates the running statistics)"""
        if count is None:
            sums, count, momentum = (None, None), 1.0, 0.1
        else:
            sums, momentum = (ptr(st["ssum"]), ptr(st["ssq"])), bn.momentum if bn.momentum is not None else 0.1
        call("ssp_bn_finalize", *sums, float(count), ptr(bn.weight.data), ptr(bn.bias.data), ptr(bn.running_mean), ptr(bn.running_var),
             float(momentum), float(bn.eps), 1 if train else 0, ptr(st["mean"]), ptr(st["invstd"]), ptr(st["scale"]), ptr(st["shift"]), C, s)
        self.launches += 1

    @staticmethod
    def _dests(B, L):
        """the two destination slots (hi, lo, ld, channel offset, route) of ssp_bn_apply / ssp_bn_apply_splitk for layer L"""
        d = []
        for (ci, c0, kind) in L.dests:
            d += [ptr(B.x_hi[ci]), ptr(B.x_lo[ci]), B.x_hi[ci].shape[1], c0, kind]
        return d + [None, None, 0, 0, _lib.ROUTE_NONE] * (2 - len(L.dests))

    # ------------------------------------------------------------------ forward
    def forward(self, x, train_bn, keep_for_backward, split_k=False, buffers=None):
        """x: (N,3,H,W) fp32 CUDA -> logits (N,Cout,h,w) fp32.  train_bn: batch statistics + running-stat update.
        split_k (inference only): the layers with a split count (split_count, ssp_conv_splitk_count) run ssp_conv_gemm_splitk +
        ssp_bn_apply_splitk; their result is deterministic but differs in the last bits from the unsplit forward.
        buffers: a private Buffers of this input shape (built with split_k=True when split_k is set) instead of the engine's cache."""
        if not x.is_cuda:
            raise _lib.SspError("singleshotpose_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor")
        if split_k and (train_bn or keep_for_backward):
            raise _lib.SspError("split_k is an inference mode: no batch statistics, no backward")
        x = x.contiguous().float()
        N, C, H, W = x.shape
        self.materialize(x.device)
        self.pack_weights()
        if buffers is not None:
            if (buffers.N, buffers.H, buffers.W) != (N, H, W) or buffers.split_k != bool(split_k) or buffers.dy:
                raise _lib.SspError("buffers were built for input %s (split_k=%s), not %s (split_k=%s) in inference mode"
                                    % ((buffers.N, 3, buffers.H, buffers.W), buffers.split_k, (N, C, H, W), bool(split_k)))
            B = buffers
        else:
            B = self.buffers(N, H, W, keep_for_backward, split_k)
        B.generation += 1
        s = stream_ptr()
        mods = self.conv_modules()
        B.x_image = x                               # the layer-0 backward reads the image again (kept alive with the activations)
        for L in self.layers:
            i = L.index
            conv, bn = mods[i]
            h, w = self.spatial(L, H, W)
            st = B.stat[i]
            if L.first:
                # blocks 0-1 (conv + BN + leaky + 2x2 max-pool) as one unit from the raw image and the fp32 master weights
                off, n, _gv = self._slices[id(conv.weight)]
                w0 = ptr(self.flat_params[off:off + n])
                if train_bn or keep_for_backward:      # the Gram matrix of the image patches: batch statistics without a pass over y, and
                    call("ssp_l0_gram", ptr(x), N, H, W, ptr(B.l0_gram), s)      # the backward's correction terms (also for a frozen-BN forward)
                    self.launches += 3
                if train_bn:
                    call("ssp_l0_stats", ptr(B.l0_gram), w0, ptr(st["ssum"]), ptr(st["ssq"]), s)
                    self.launches += 1
                self._bn_finalize(bn, st, L.cout, s, N * h * w, train_bn)
                ci, c0, _k = L.dests[0]
                call("ssp_l0_fused_fwd", ptr(x), w0, ptr(st["scale"]), ptr(st["shift"]), L.slope, N, H, W, ptr(B.x_hi[ci]), ptr(B.x_lo[ci]),
                     B.x_hi[ci].shape[1], c0, ptr(B.l0_code) if keep_for_backward else None, s)
                self.launches += 1
                continue
            xin = B.x_hi[i]
            a_lo = None if self.fast else ptr(B.x_lo[i])
            b_lo = None if self.fast else ptr(self.w_lo[i])
            S = B.splits[i]
            if S:
                # split-K inference: S partial GEMMs over slices of K into the workspace, then BN(running stats) + leaky + routing
                # from their sum, in a fixed order (csrc/conv_tc.cu SPLIT, csrc/elementwise.cu bn_apply_kernel SPLIT)
                self._bn_finalize(bn, st, L.cout, s)
                ws, slab, ld = ptr(B.split_ws), B.split_slab[i], B.split_ld[i]
                self._gemm("fwd", L, N, h, w, "ssp_conv_gemm_splitk", ptr(xin), a_lo, B.rows[i], xin.shape[1], L.cin, ptr(self.w_hi[i]), b_lo,
                           L.cout, self.w_hi[i].shape[1], N, h, w, L.taps, L.cout, S, ws, slab, ld, s)
                call("ssp_bn_apply_splitk", ws, S, slab, ld, ptr(st["scale"]), ptr(st["shift"]), N, L.cout, h, w, L.slope, *self._dests(B, L), s)
                self.launches += 1
                self.split_launches += 1
                continue
            if not train_bn and not keep_for_backward and self._fuse_eval_layer(L):
                # inference: BN(running stats) + LeakyReLU folded into the GEMM epilogue, which writes the consumer's operand
                # planes directly -- no fp32 Y, no bn_apply pass (reference: conv, bn, leaky as three modules, darknet.py:154-164)
                self._bn_finalize(bn, st, L.cout, s)
                ci, c0, _k = L.dests[0]
                self._gemm("fwd", L, N, h, w, "ssp_conv_gemm_bnact", _lib.IMPL_TC2 if L.cout >= 128 else _lib.IMPL_TC, ptr(xin), a_lo,
                           B.rows[i], xin.shape[1], L.cin, ptr(self.w_hi[i]), b_lo, L.cout, self.w_hi[i].shape[1], N, h, w, L.taps, L.cout,
                           ptr(st["scale"]), ptr(st["shift"]), L.slope, ptr(B.x_hi[ci]), ptr(B.x_lo[ci]), B.x_hi[ci].shape[1], c0, s)
                continue
            if L.bn:
                epi, bias = (_lib.EPI_STATS if train_bn else _lib.EPI_F32), None
            else:
                epi, bias = _lib.EPI_BIAS, ptr(conv.bias.data)
            self._gemm("fwd", L, N, h, w, "ssp_conv_gemm", self._conv_impl(L), ptr(xin), a_lo, B.rows[i], xin.shape[1], L.cin,
                       ptr(self.w_hi[i]), b_lo, L.cout, self.w_hi[i].shape[1], _lib.FMT_F16, _lib.FMT_F16,
                       N, h, w, L.taps, L.cout, ptr(B.y[i]), B.y[i].shape[1], B.rows[i], epi, bias,
                       ptr(st["ssum"]), ptr(st["ssq"]), s)
            if not L.bn:
                continue
            self._bn_finalize(bn, st, L.cout, s, N * h * w, train_bn)
            yp = B.ypool[i] if keep_for_backward else None
            call("ssp_bn_apply", ptr(B.y[i]), B.y[i].shape[1], ptr(st["scale"]), ptr(st["shift"]), N, L.cout, h, w, L.slope, *self._dests(B, L),
                 ptr(yp), yp.shape[1] if yp is not None else 0, s)
            self.launches += 1
        last = self.layers[-1]
        h, w = self.spatial(last, H, W)
        out = torch.empty(N, last.cout, h, w, dtype=torch.float32, device=x.device)
        call("ssp_unpack_nchw", ptr(B.y[-1]), ptr(out), N, last.cout, h, w, B.y[-1].shape[1], 0, s)
        self.launches += 1
        return out, B, B.generation

    # ------------------------------------------------------------------ backward
    def backward(self, B, generation, grad_out):
        """grad_out: (N,Cout,h,w) fp32 -> fills self.flat_grads (dW for every conv, dgamma/dbeta, dbias)."""
        if B.generation != generation:
            raise RuntimeError("activations of this forward pass were overwritten by a later forward of the same shape")
        N, H, W = B.N, B.H, B.W
        s = stream_ptr()
        mods = self.conv_modules()
        self.flat_grads.zero_()
        g = grad_out.contiguous().float()
        # Weight-gradient GEMMs (tensor/L2 bound) run on a side stream so that they overlap the HBM-bound BN-backward
        # kernels of the next layer on the main stream; joined before returning.  Serial when per-launch profiling is on.
        overlap = self.profile is None
        main = torch.cuda.current_stream()
        if overlap:
            if self._side is None or self._side.device != main.device:
                self._side = torch.cuda.Stream(device=main.device)
            side = self._side
            side.wait_stream(main)
            ws, wstream = _lib.C.c_void_p(side.cuda_stream), side
        else:
            ws, wstream = s, None
        inv = 1.0 / self.grad_scale        # the whole backward chain carries the loss scale; undone where grads are written
        for L in reversed(self.layers):
            i = L.index
            conv, bn = mods[i]
            h, w = self.spatial(L, H, W)
            st = B.stat[i]
            if L.first:
                # dW0 / dgamma / dbeta from the pooled gradient, the arg-max codes and the image (csrc/l0_fused.cu); runs where the
                # weight gradients run, after the data gradient of layer 1 (the last kernel of the main stream)
                ci, c0, _k = L.dests[0]
                off, n, _gv = self._slices[id(conv.weight)]
                if overlap:
                    ev = torch.cuda.Event()
                    ev.record(main)
                    side.wait_event(ev)
                self._gemm("l0_bwd", L, N, h, w, "ssp_l0_bwd", ptr(B.x_image), ptr(B.dx[ci]), 1, B.dx[ci].shape[1], c0, ptr(B.l0_code), L.slope,
                           N, H, W, ptr(B.l0_t1), ws, stream=wstream)
                call("ssp_l0_bwd_finalize", ptr(B.l0_t1), ptr(B.l0_gram), ptr(self.flat_params[off:off + n]), ptr(bn.weight.data),
                     ptr(st["mean"]), ptr(st["invstd"]), float(N * h * w), inv, ptr(self.flat_grads[off:off + n]),
                     ptr(self.grad_view(bn.weight)), ptr(self.grad_view(bn.bias)), ws)
                self.launches += 1
                if self.grad_ready_hook is not None:
                    self.grad_ready_hook(i, side if overlap else main)
                continue
            dy = B.dy[i]
            if L.bn:
                srcs = []
                f16 = _lib.ROUTE_F16
                for (ci, c0, kind) in L.dests:
                    srcs += [ptr(B.dx[ci]), B.dx[ci].shape[1], c0, kind | f16]
                if len(L.dests) == 1:
                    srcs += [None, 0, 0, _lib.ROUTE_NONE]
                common = [ptr(B.y[i]), B.y[i].shape[1], ptr(st["scale"]), ptr(st["shift"]), ptr(st["mean"]), ptr(st["invstd"]),
                          ptr(bn.weight.data), N, L.cout, h, w, L.slope, *srcs, ptr(st["s1"]), ptr(st["s2"])]
                yp = B.ypool[i]
                if yp is not None:
                    # pooled consumer(s): only the arg-max position of a 2x2 window receives gradient, so S1 / S2 are sums over
                    # pooled cells -- reduce at a quarter of the resolution from the arg-max plane; S1 / S2 are linear in the
                    # upstream gradient, so any other consumer (layer 16 also feeds the reorg branch) adds its own pass
                    head = common[:7]
                    for (ci, c0, kind) in L.dests:
                        if kind == _lib.ROUTE_POOL:
                            call("ssp_bn_bwd_reduce", ptr(yp), yp.shape[1], *head[2:], N, L.cout, h // 2, w // 2, L.slope,
                                 ptr(B.dx[ci]), B.dx[ci].shape[1], c0, _lib.ROUTE_DIRECT | f16, None, 0, 0, _lib.ROUTE_NONE, ptr(st["s1"]), ptr(st["s2"]), s)
                        else:
                            call("ssp_bn_bwd_reduce", *head, N, L.cout, h, w, L.slope, ptr(B.dx[ci]), B.dx[ci].shape[1], c0, kind | f16,
                                 None, 0, 0, _lib.ROUTE_NONE, ptr(st["s1"]), ptr(st["s2"]), s)
                        self.launches += 1
                else:
                    call("ssp_bn_bwd_reduce", *common, s)
                    self.launches += 1
                call("ssp_bn_bwd_apply", *common, ptr(dy), dy.shape[1], _lib.FMT_F16, 1.0, s)
                call("ssp_bn_bwd_finalize", ptr(st["s1"]), ptr(st["s2"]), ptr(self.grad_view(bn.weight)), ptr(self.grad_view(bn.bias)),
                     L.cout, 0, inv, s)
                self.launches += 2
            else:
                call("ssp_pack_nchw", ptr(g), ptr(dy), None, N, L.cout, h, w, dy.shape[1], 0, _lib.FMT_F16, self.grad_scale, s)
                call("ssp_bias_grad_nchw", ptr(g), ptr(self.grad_view(conv.bias)), N, L.cout, h * w, 0, 1.0, s)
                self.launches += 2
            off, n, _gv = self._slices[id(conv.weight)]
            dw = self.flat_grads[off:off + n]
            xh = B.x_hi[i]
            if overlap:
                ev = torch.cuda.Event()
                ev.record(main)                      # dY of this layer is complete
            # data gradient first: it is on the critical path of the next layer.  The fp16 dX planes need a kernel with the fp16
            # epilogue: the operand-swapped one where the layer is narrow enough, else the per-tap kernel.
            wd = self.w_d[i]
            dimpl = _lib.IMPL_BANDT if L.cin <= 128 else _lib.IMPL_TC2
            self._gemm("dgrad", L, N, h, w, "ssp_conv_gemm", dimpl, ptr(dy), None, B.rows[i], dy.shape[1], L.cout,
                       ptr(wd), None, L.cin, wd.shape[1], _lib.FMT_F16, _lib.FMT_F16, N, h, w, L.taps, L.cin, ptr(B.dx[i]),
                       B.dx[i].shape[1], B.rows[i], _lib.EPI_F16, None, None, None, s)
            if overlap:
                side.wait_event(ev)
            self._gemm("wgrad", L, N, h, w, "ssp_wgrad_gemm", _lib.IMPL_TC2, ptr(dy), B.rows[i], dy.shape[1], L.cout, _lib.FMT_F16,
                       ptr(xh), B.rows[i], xh.shape[1], L.cin, _lib.FMT_F16, N, h, w, L.taps, ptr(dw), L.cin, L.cin, inv, ws, stream=wstream)
            if self.grad_ready_hook is not None:
                # the weight-gradient stream has waited for this layer's dY event, i.e. for every main-stream gradient write
                # (dgamma / dbeta / dbias) of the layers >= i as well
                self.grad_ready_hook(i, side if overlap else main)
        if overlap:
            main.wait_stream(side)
