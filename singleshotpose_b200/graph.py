"""CUDA-graph capture of one whole training step (forward + RegionLoss + backward + optional gradient all-reduce + SGD).

The step is ~200 short launches; replaying them as one graph removes the host launch path (ctypes + Python) from the
critical path, which matters as soon as the host waits for the loss every step (the reference's train.py prints it,
train.py:97 / region_loss.py:173).  Inputs are copied into static device buffers before each replay."""
from __future__ import annotations

import torch

from .optim import FlatSGD


class GraphedTrainStep:
    def __init__(self, model, criterion, optimizer, batch_shape, target_shape, epoch, device, all_reduce=False, warmup=3):
        self.model, self.criterion, self.optimizer, self.epoch = model, criterion, optimizer, epoch
        # any other optimizer (torch.optim.SGD on the parameter views) leaves the conv operand planes stale after its step
        self._sgd_repacks = isinstance(optimizer, FlatSGD)
        self.x = torch.zeros(batch_shape, dtype=torch.float32, device=device)
        self.t = torch.zeros(target_shape, dtype=torch.float32, device=device)
        self.all_reduce = all_reduce
        self.graph = None
        self.loss = None
        self._warmup = warmup
        self._captured = None

    def _hyper(self):
        """everything the captured launches carry BY VALUE: lr / momentum / weight decay (kernel scalars of ssp_sgd_pack_step) and
        the confidence-loss gate epoch > pretrain_num_epochs (region_loss.py:156).  adjust_learning_rate (train.py:34-46) rewrites
        param_groups every batch and the gate flips once per run: a replay with stale values would silently train wrong."""
        g = self.optimizer.param_groups[0]
        gate = self.epoch > getattr(self.criterion, "pretrain_num_epochs", -1)
        return (float(g["lr"]), float(g.get("momentum", 0.0)), float(g.get("weight_decay", 0.0)), bool(gate))

    def set_epoch(self, epoch):
        self.epoch = epoch

    def _ensure_current(self):
        if self.graph is None or self._captured != self._hyper():
            self.capture(warmup=0 if self.graph is not None else None)
        eng = self.model._engine
        if self._sgd_repacks:
            eng.pack_weights()      # no-op unless the weights changed outside the graph (load_weights, load_state_dict): the
                                    # captured step has no re-pack of its own, FlatSGD rewrites the operand planes as it updates

    def _after_replay(self):
        if not self._sgd_repacks:
            self.model._engine.invalidate_packed_weights()     # the replayed SGD moved the master weights past the packed copies

    def _step(self):
        self.optimizer.zero_grad()
        out = self.model(self.x)
        loss = self.criterion(out, self.t, self.epoch)
        loss.backward()
        if self.all_reduce:
            self.optimizer.all_reduce_grads()
        self.optimizer.step()
        return loss

    def capture(self, warmup=None):
        verbose, self.criterion.verbose = getattr(self.criterion, "verbose", False), False
        eng = self.model._engine
        prof, eng.profile = eng.profile, None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(self._warmup if warmup is None else warmup):          # allocations, cudaFuncSetAttribute, optimizer state: all before capture
                self._step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        self.optimizer.zero_grad()
        if self._sgd_repacks:
            eng.pack_weights()                     # FlatSGD rewrites the operand planes itself: start the graph from current ones
        else:
            eng.invalidate_packed_weights()        # the weight re-pack must be part of the captured step
        with torch.cuda.graph(g):
            self.loss = self._step()
        self.graph = g
        self._captured = self._hyper()
        self.criterion.verbose = verbose
        eng.profile = prof
        return self

    # ---- input prefetch: the PCIe copy of the NEXT batch overlaps the replay of the current one ----
    def stage(self, x, target):
        """enqueue host(pinned)->device copies of the next batch on a side stream"""
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream()
            self._x_stage, self._t_stage = torch.empty_like(self.x), torch.empty_like(self.t)
            self._staged, self._consumed = torch.cuda.Event(), torch.cuda.Event()
            self._consumed.record()
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._consumed)        # the previous staged batch has been moved into the static buffers
            self._x_stage.copy_(x, non_blocking=True)
            self._t_stage.copy_(target, non_blocking=True)
            self._staged.record()

    def run_staged(self):
        """replay on the batch passed to the last stage() call"""
        self._ensure_current()
        cur = torch.cuda.current_stream()
        cur.wait_event(self._staged)
        self.x.copy_(self._x_stage, non_blocking=True)          # device-to-device, ~0.1 ms
        self.t.copy_(self._t_stage, non_blocking=True)
        self._consumed.record()
        self.graph.replay()
        self._after_replay()
        return self.loss

    def __call__(self, x, target):
        """x, target: host (pinned) or device tensors of the captured shapes -> loss tensor (device, 0-dim)."""
        self._ensure_current()
        self.x.copy_(x, non_blocking=True)
        self.t.copy_(target, non_blocking=True)
        self.graph.replay()
        self._after_replay()
        return self.loss
