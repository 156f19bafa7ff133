"""Utterance-sharded data parallelism: one process per GPU, ONE allreduce per step.

The reference is single-device (reference train_triplet.py:97); SURVEY §8e adds exactly one
strategy: every rank runs the triplet step on its own shard of the batch, and the gradients of the 38
differentiated parameters are averaged with a single ``all_reduce`` over one flat fp32 bucket
(11 624 128 elements, 46.5 MB).  BatchNorm statistics stay per replica, as in the reference (no SyncBN).

``torch.distributed`` (NCCL over NVLink on the GPU box, gloo in the CPU tests) is plumbing here.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


class GradBucket:
    """Makes every ``p.grad`` of ``params`` a view into one flat fp32 buffer and reduces it in one collective."""

    def __init__(self, params, process_group=None):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("GradBucket needs at least one parameter")
        dev = self.params[0].device
        self.numel = sum(p.numel() for p in self.params)
        # one extra slot after the gradients carries the rank's weight through the same collective (weighted mean)
        self._ext = torch.zeros(self.numel + 1, dtype=torch.float32, device=dev)
        self.flat = self._ext[:self.numel]
        self.group = process_group
        off = 0
        for p in self.params:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("all bucketed parameters must be fp32 on one device")
            p.grad = self.flat[off:off + p.numel()].view_as(p)   # autograd accumulates in place into the view
            p._dsk_bucket_grad = p.grad                          # lets TripletForwardFn add into the bucket directly
            off += p.numel()
        self.collectives = 0

    def zero(self):
        """optimizer.zero_grad() replacement that keeps the views (train_triplet.py:222)."""
        self.flat.zero_()

    def allreduce_mean(self, async_op: bool = False):
        """Sum over ranks then divide by the world size: the gradient of the mean loss over the global batch
        when every rank holds the same number of triplets."""
        if not (dist.is_available() and dist.is_initialized()):
            return None
        world = dist.get_world_size(self.group)
        if world == 1:
            return None
        self.flat.div_(world)
        self.collectives += 1
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)

    def allreduce_weighted_mean(self, weight):
        """Hard-triplet branch (train_triplet.py:262-291): rank r holds the gradient of the MEAN loss over its own k_r
        selected triplets, and k_r differs per rank.  The gradient of the mean over the global selection is
        sum_r k_r g_r / sum_r k_r: the bucket is scaled by k_r, k_r itself rides in the extra slot of the same buffer,
        and ONE sum-allreduce delivers numerator and denominator together (SURVEY §8e).  ``weight``: python number or
        0-d tensor (stays on the device: no host synchronisation).  A rank with k_r = 0 contributes zeros."""
        w = torch.as_tensor(weight, dtype=torch.float32, device=self.flat.device).reshape(())
        self.flat.mul_(w)
        self._ext[self.numel] = w
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1:
            self.collectives += 1
            dist.all_reduce(self._ext, op=dist.ReduceOp.SUM, group=self.group)
        self.flat.div_(self._ext[self.numel].clamp_min(1e-30))
        return self._ext[self.numel]


def path_parameters(module):
    """The parameters that receive gradients on the triplet path (everything but the classifier, SURVEY §0 fact 5)."""
    return [p for n, p in module.named_parameters() if not n.startswith("model.classifier")]


def broadcast_parameters(module, src: int = 0, process_group=None):
    """Step-0 synchronisation of parameters and BatchNorm buffers."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(process_group) == 1:
        return
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src=src, group=process_group)


def shard(batch: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """Contiguous utterance shard of a global batch (global batch must divide by the world size)."""
    n = batch.shape[0]
    if n % world:
        raise ValueError(f"global batch {n} is not divisible by world size {world}")
    per = n // world
    return batch[rank * per:(rank + 1) * per]
