"""Fused optimizer step on ONE flat bucket (SURVEY §8f rank 3).

The reference builds ``torch.optim.Adagrad(model.parameters(), lr=0.1, lr_decay=1e-4, weight_decay=0)``
(reference train_triplet.py:369-383, defaults :70-77) and calls ``optimizer.step()`` after ``loss.backward()``
(:224,291).  ``FusedAdagrad`` keeps that call surface (``zero_grad() / step() / state_dict() / load_state_dict()``,
``param_groups``) but lays parameters, gradients and the running sum of squares out as three flat fp32 buffers with the
same offsets: ``p.data`` and ``p.grad`` of every parameter become views into them, the data-parallel gradient
allreduce is a single collective on the gradient buffer, and the update is ONE kernel over 11.6 M elements
(``dsk_adagrad_step``) that also applies the post-allreduce division by ``world`` (or by ``max(sum_k, 1e-30)`` for the
weighted hard-triplet branch, ``GradBucket.allreduce_weighted_mean``'s arithmetic) — instead of ~6 foreach kernels
over 38 tensors.  Same operation order as torch's foreach Adagrad: the parameters and sums are bit-identical to
``torch.optim.Adagrad`` (CUDA, foreach) stepping on the summed gradient divided by that divisor as a CUDA tensor
(tests/test_gpu_fp32_head_ops.py, tests/test_gpu_head.py).  ``GradBucket.allreduce_mean`` divides BEFORE its sum, as
DDP's default hook does; at world sizes that are not powers of two it differs from this step in the last bit.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import _lib as L


class FusedAdagrad:
    def __init__(self, params, lr=1e-2, lr_decay=0.0, weight_decay=0.0, initial_accumulator_value=0.0, eps=1e-10,
                 process_group=None):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("FusedAdagrad needs at least one parameter")
        dev = self.params[0].device
        if dev.type != "cuda":
            raise RuntimeError("FusedAdagrad runs on CUDA parameters only (no CPU fallback)")
        for p in self.params:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("all parameters must be fp32 on one CUDA device")
        self.device = dev
        self.group = process_group
        self.defaults = dict(lr=lr, lr_decay=lr_decay, weight_decay=weight_decay, eps=eps,
                             initial_accumulator_value=initial_accumulator_value)
        self.param_groups = [dict(self.defaults, params=self.params)]
        # every parameter starts on a 16-byte boundary of the flat buffers (vectorised kernel; TMA-friendly views)
        self.offsets, off = [], 0
        for p in self.params:
            self.offsets.append(off)
            off += (p.numel() + 3) // 4 * 4
        self.numel = off
        # one extra slot after the gradients carries the rank's weight through the same allreduce (weighted mean)
        self._grad_ext = torch.zeros(self.numel + 4, dtype=torch.float32, device=dev)
        self.flat_grad = self._grad_ext[:self.numel]
        self.flat_param = torch.zeros(self.numel, dtype=torch.float32, device=dev)
        self.flat_sum = torch.full((self.numel,), float(initial_accumulator_value), dtype=torch.float32, device=dev)
        for p, o in zip(self.params, self.offsets):
            view = self.flat_param[o:o + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view                                               # parameters now live in the flat buffer
            p.grad = self.flat_grad[o:o + p.numel()].view_as(p)         # autograd accumulates in place into the view
            p._dsk_bucket_grad = p.grad                                 # lets TripletForwardFn add into the bucket directly
        self.step_count = 0
        self.collectives = 0
        self._weighted = False

    # -- torch.optim.Optimizer surface ----------------------------------------------------------------
    def zero_grad(self, set_to_none: bool = False):
        """train_triplet.py:222,289.  Keeps the views (``set_to_none`` is ignored: the bucket is the storage)."""
        self._grad_ext.zero_()
        self._weighted = False

    def allreduce(self, weight: torch.Tensor | None = None, async_op: bool = False):
        """The ONE gradient collective of a data-parallel step (sum over ranks); the division happens inside
        ``step()``.  ``weight`` (device scalar, e.g. the rank's number of selected hard triplets): gradients must
        already be those of ``weight * local_mean_loss``; the weights travel in the same buffer and ``step()`` divides
        by their sum, which yields the mean over the global set of selected triplets (SURVEY §8e)."""
        world = dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1
        if weight is not None:
            self._grad_ext[self.numel] = weight.detach().reshape(()).float()
            self._weighted = True
        if world == 1:
            return None
        self.collectives += 1
        buf = self._grad_ext if self._weighted else self.flat_grad
        return dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)

    @torch.no_grad()
    def step(self):
        g = self.param_groups[0]
        self.step_count += 1
        world = dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1
        denom = self._grad_ext[self.numel:self.numel + 1] if self._weighted else None
        div = 1.0 if self._weighted else float(world)
        with torch.cuda.device(self.device):
            L.check(L.load().dsk_adagrad_step(self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.flat_sum.data_ptr(),
                                              self.numel, float(g["lr"]), float(g["lr_decay"]), float(g["weight_decay"]),
                                              float(g["eps"]), self.step_count, div, L.ptr(denom), L.cur_stream()),
                    "dsk_adagrad_step")
        # the kernel wrote through raw pointers: tell autograd / the engine's repack check that the parameters changed
        torch.autograd.graph.increment_version(self.params)

    # -- checkpoints in torch.optim.Adagrad's format (train_triplet.py:177-186,325-327) ---------------------
    def state_dict(self):
        state = {i: {"step": torch.tensor(float(self.step_count)),
                     "sum": self.flat_sum[o:o + p.numel()].view_as(p).clone()}
                 for i, (p, o) in enumerate(zip(self.params, self.offsets))}
        grp = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        grp.update(foreach=None, maximize=False, differentiable=False, fused=None, params=list(range(len(self.params))))
        return {"state": state, "param_groups": [grp]}

    def load_state_dict(self, sd):
        for i, (p, o) in enumerate(zip(self.params, self.offsets)):
            st = sd["state"].get(i, sd["state"].get(str(i)))
            if st is None:
                continue
            self.flat_sum[o:o + p.numel()].view_as(p).copy_(st["sum"])
            self.step_count = int(float(st["step"]))
        for k in ("lr", "lr_decay", "weight_decay", "eps"):
            if k in sd["param_groups"][0]:
                self.param_groups[0][k] = sd["param_groups"][0][k]
