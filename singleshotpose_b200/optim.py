"""Fused SGD over the engine's flat parameter / gradient buffers: optim.SGD(momentum, dampening=0, weight_decay)
of train.py:388 as ONE kernel (read p, g, v; write p, v), plus the optional NCCL gradient all-reduce for
one-process-per-GPU data parallelism (SURVEY 8e: sum over ranks, lr already divided by the global batch)."""
from __future__ import annotations

import torch

from ._lib import call, ptr, stream_ptr


def all_reduce_flat_(flat):
    """SUM all-reduce of the flat gradient buffer over the data-parallel group (NCCL on GPUs, gloo in the CPU tests).
    The loss is a SUM over images (region_loss.py:149-161), so gradients add across ranks."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    return flat


def dp_hyperparams(learning_rate, decay, per_gpu_batch):
    """train.py:388 divides lr and multiplies weight decay by the batch size: with data parallelism that is the GLOBAL batch."""
    import torch.distributed as dist
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    gb = per_gpu_batch * world
    return learning_rate / gb, decay * gb


class FlatSGD:
    """optim.SGD(model.parameters(), lr, momentum, dampening=0, weight_decay) of train.py:388 as one kernel over the engine's flat
    buffers, which also rewrites the conv operand planes from the updated weights (csrc/sgd_pack.cu).

    Data parallelism (SURVEY 8e): `overlap_all_reduce(n_buckets)` splits the flat gradient buffer into contiguous buckets in
    REVERSE layer order; backward hands each bucket to NCCL on a communication stream as soon as its last weight gradient has
    been launched, so the exchange of the big tail layers (L29 / L24 / L23 = 60 % of the bytes) runs under the rest of backward;
    `step()` then updates bucket after bucket as the all-reduces retire."""

    def __init__(self, model, lr, momentum=0.0, weight_decay=0.0):
        self.model = model
        self.param_groups = [dict(lr=lr, momentum=momentum, weight_decay=weight_decay)]   # adjust_learning_rate() writes lr here
        self._v = None
        self._buckets = None          # [(first layer, (elem lo, hi), (block lo, hi))] when overlap_all_reduce() is on
        self._comm = None
        self._done = {}               # bucket -> event recorded on the communication stream after its all-reduce
        self._group = None

    def zero_grad(self, set_to_none=True):
        for p in self.model.parameters():
            p.grad = None

    # ------------------------------------------------------------------ gradient exchange
    def overlap_all_reduce(self, n_buckets=4, group=None):
        """switch the gradient all-reduce from one call after backward to per-bucket calls issued DURING backward.  Needs
        materialised parameters (one forward pass, or model._engine.materialize(device))."""
        eng = self.model._engine
        if eng.flat_params is None:
            raise RuntimeError("overlap_all_reduce() needs materialised parameters: run one forward pass first")
        self._buckets = eng.grad_buckets(n_buckets)
        self._group = group
        self._first = {b[0]: k for k, b in enumerate(self._buckets)}
        eng.grad_ready_hook = self._bucket_ready
        return self

    def _bucket_ready(self, layer_index, stream):
        k = self._first.get(layer_index)
        if k is None:
            return
        import torch.distributed as dist
        if self._comm is None or self._comm.device != stream.device:
            self._comm = torch.cuda.Stream(device=stream.device)
        lo, hi = self._buckets[k][1]
        ev = torch.cuda.Event()
        ev.record(stream)
        self._comm.wait_event(ev)
        with torch.cuda.stream(self._comm):
            if dist.is_available() and dist.is_initialized() and dist.get_world_size(self._group) > 1:
                dist.all_reduce(self.model._engine.flat_grads[lo:hi], op=dist.ReduceOp.SUM, group=self._group)
            done = torch.cuda.Event()
            done.record(self._comm)
        self._done[k] = done

    def all_reduce_grads(self):
        if self._buckets is None:
            all_reduce_flat_(self.model._engine.flat_grads)
        # bucketed mode: the all-reduces were issued by backward; step() waits for them bucket by bucket

    def step(self, grad_scale=1.0):
        eng = self.model._engine
        if eng.flat_params is None:
            raise RuntimeError("FlatSGD.step() before the first forward pass")
        if self._v is None or self._v.data_ptr() == 0 or self._v.numel() != eng.flat_params.numel() or self._v.device != eng.flat_params.device:
            self._v = torch.zeros_like(eng.flat_params)
        g = self.param_groups[0]
        hyper = (float(g["lr"]), float(g["momentum"]), float(g["weight_decay"]), float(grad_scale))
        table, blocks = eng.sgd_segments()
        n_seg = len(blocks)
        if self._buckets is not None and self._done:
            cur = torch.cuda.current_stream()
            for k, (_li, _el, (b0, b1)) in enumerate(self._buckets):       # completion order: last layers first
                ev = self._done.get(k)
                if ev is not None:
                    cur.wait_event(ev)
                call("ssp_sgd_pack_step", ptr(table), n_seg, b0, b1, ptr(eng.flat_params), ptr(eng.flat_grads), ptr(self._v), *hyper, stream_ptr())
                eng.launches += 1
            self._done = {}
        else:
            call("ssp_sgd_pack_step", ptr(table), n_seg, 0, blocks[-1][0] + blocks[-1][1], ptr(eng.flat_params), ptr(eng.flat_grads),
                 ptr(self._v), *hyper, stream_ptr())
            eng.launches += 1
        eng._weights_version = eng._params_version()       # the operand planes were rewritten from the updated weights

    # ------------------------------------------------------------------ checkpointing (SURVEY 8f.4; absent in the reference,
    # which only saves model weights -- train.py:409).  The layout is torch.optim.SGD's own state_dict, so a checkpoint moves
    # freely between FlatSGD and the `optim.SGD(model.parameters(), ...)` of train.py:388.
    def _momentum_views(self):
        """per-parameter views of the flat momentum buffer, shaped like the parameters (conv weights: OIHW view of OHWI storage)"""
        eng = self.model._engine
        out = []
        for p in self.model.parameters():
            off, n, _g = eng._slices[id(p)]
            v = self._v[off:off + n]
            if p.dim() == 4:
                co, ci, kh, kw = p.shape
                out.append(v.view(co, kh, kw, ci).permute(0, 3, 1, 2))
            else:
                out.append(v.view(p.shape))
        return out

    def state_dict(self):
        g = self.param_groups[0]
        n = len(list(self.model.parameters()))
        group = dict(lr=g["lr"], momentum=g["momentum"], dampening=0, weight_decay=g["weight_decay"], nesterov=False,
                     maximize=False, foreach=None, differentiable=False, fused=None, params=list(range(n)))
        state = {}
        if self._v is not None:
            state = {i: {"momentum_buffer": v.detach().clone().contiguous()} for i, v in enumerate(self._momentum_views())}
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        eng = self.model._engine
        if eng.flat_params is None:
            raise RuntimeError("FlatSGD.load_state_dict() needs materialised parameters: move the model to its device and run one "
                               "forward pass (or call model._engine.materialize(device)) first")
        groups = sd["param_groups"]
        if len(groups) != 1:
            raise ValueError("FlatSGD has one parameter group (train.py:388 passes model.parameters()), got %d" % len(groups))
        g = groups[0]
        if g.get("dampening", 0) != 0 or g.get("nesterov", False):
            raise ValueError("FlatSGD implements optim.SGD(dampening=0, nesterov=False) only (train.py:388)")
        params = list(self.model.parameters())
        if len(g["params"]) != len(params):
            raise ValueError("checkpoint has %d parameters, the model %d" % (len(g["params"]), len(params)))
        self.param_groups[0].update(lr=g["lr"], momentum=g["momentum"], weight_decay=g["weight_decay"])
        state = sd.get("state", {})
        if not state:
            self._v = None
            return
        self._v = torch.zeros_like(eng.flat_params)
        for i, (p, view) in enumerate(zip(params, self._momentum_views())):
            ent = state.get(i, state.get(str(i)))
            if ent is None or ent.get("momentum_buffer") is None:
                continue                      # optim.SGD creates buffers lazily; a missing one is zero
            buf = ent["momentum_buffer"]
            if tuple(buf.shape) != tuple(p.shape):
                raise ValueError("momentum_buffer %d has shape %s, parameter %s" % (i, tuple(buf.shape), tuple(p.shape)))
            view.copy_(buf.to(device=view.device, dtype=torch.float32))
