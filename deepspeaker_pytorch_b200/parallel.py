"""Utterance-sharded data parallelism: one process per GPU, ONE allreduce per step.

The reference is single-device (reference train_triplet.py:97); SURVEY §8e adds exactly one
strategy: every rank runs the triplet step on its own shard of the batch, and the gradients of the 38
differentiated parameters are averaged with a single ``all_reduce`` over one flat fp32 bucket
(11 624 128 elements, 46.5 MB).  By default BatchNorm statistics stay per replica, as in the reference;
``DeepSpeakerModel.sync_batchnorm(process_group)`` synchronises them over the ranks instead (``gather_records``).

``torch.distributed`` (NCCL over NVLink on the GPU box, gloo in the CPU tests) is plumbing here.

Batch-hard mining over the global batch (``GlobalBatchHardTripletLoss``, ``batch_hard_step(..., across_ranks=True)``)
adds three small all_gathers per step: the labels, the fp32 embeddings and the selection records.  The gradient
reduction stays the one all-reduce.

GE2E over the global batch (``GlobalGE2ELoss``, ``ge2e_step(..., across_ranks=True)``) adds the same labels gather, two
all_gathers in the forward (the fp32 embeddings, the row losses) and one in the backward (each row's dcos and the target
column's dcos).  The gradient reduction stays the one all-reduce.

Synchronised BatchNorm adds one all_gather of per-utterance records at each of the 12 BatchNorm layers of a forward
and at 13 points of its backward (the loss scale, then the 12 layers); see ``gather_records`` for the record sizes.

The sharded AAM-softmax head (``ShardedAAMSoftmaxLoss``, ``steps.sharded_aam_softmax_step``) is model parallel in its
classes: rank r holds the contiguous class range ``class_shards(C, R)[r]`` of the (C K, D) weight, its gradient and
its optimizer state, and the weight leaves the gradient all-reduce.  Per forward it adds four all_gathers (the fp32
embeddings, the top-k candidate keys, the row maxima, the per-block partial sums) and per backward one all_to_all of
the embedding rows' gradients; see ``ShardedAAMSoftmaxLoss`` for the sizes.
"""
from __future__ import annotations

import math

import torch
import torch.distributed as dist

from . import engine as _engine


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


# ---- batch-hard mining over the global batch --------------------------------------------------------------------------
# Rank r holds the contiguous shard [r n, (r + 1) n) of a global batch of N = R n utterances (what ``shard`` produces).
# EVERY RANK MUST HOLD THE SAME n: the gathers below are all_gather_into_tensor, which assumes equal sizes (with unequal
# sizes NCCL waits forever rather than raising).

def _distributed(process_group=None) -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1


def gather_labels(local_labels, process_group=None) -> torch.Tensor:
    """The global batch's labels (N,) int64 in rank order, from every rank's (n,) shard: one all_gather_into_tensor.
    Under NCCL CPU labels are moved to the current CUDA device first.  Without a process group (or at world size 1)
    the labels are returned as given."""
    lab = torch.as_tensor(local_labels, dtype=torch.int64).reshape(-1)
    if not _distributed(process_group):
        return lab
    if not lab.is_cuda and dist.get_backend(process_group) == "nccl":
        lab = lab.to(torch.cuda.current_device())
    lab = lab.contiguous()
    out = lab.new_empty(dist.get_world_size(process_group) * lab.numel())
    dist.all_gather_into_tensor(out, lab, group=process_group)
    return out


# The selection of one anchor travels as a 25-byte record: pos_idx, neg_idx (int64), d_ap, d_an (fp32), valid (1 byte).
# A rank's n records are laid out field by field - (8 + 8 + 4 + 4 + 1) n bytes, every field aligned to its size - so
# packing is one cat of byte views and unpacking one strided copy per field.
_SELECTION_FIELDS = ((8, torch.int64), (8, torch.int64), (4, torch.float32), (4, torch.float32), (1, torch.bool))
SELECTION_RECORD_BYTES = sum(b for b, _ in _SELECTION_FIELDS)


def _pack_selection(pos, neg, d_ap, d_an, valid) -> torch.Tensor:
    """(n,) each -> uint8 (25 n,)."""
    return torch.cat([t.contiguous().view(torch.uint8) for t in (pos, neg, d_ap, d_an, valid)])


def _unpack_selection(records, n):
    """uint8 (R, 25 n), one row per rank -> (pos_idx, neg_idx, d_ap, d_an, valid), each (R n,) in rank order."""
    out, lo = [], 0
    for size, dtype in _SELECTION_FIELDS:
        out.append(records[:, lo * n:(lo + size) * n].contiguous().view(dtype).reshape(-1))
        lo += size
    return tuple(out)


class _GlobalBatchHardFn(torch.autograd.Function):
    """Forward: all_gather of the fp32 embeddings, selection of this rank's anchor rows, all_gather of the selection
    records, the mean over all N anchors.  Backward: this rank's rows of the gradient; no collective."""

    @staticmethod
    def forward(ctx, local_emb, global_labels, margin, exact_cuda_cores, group):
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        x = local_emb.detach().float().contiguous()
        n = x.shape[0]
        E = x.new_empty(world * n, x.shape[1])
        dist.all_gather_into_tensor(E, x, group=group)
        row0 = rank * n
        E, *sel = _engine.batch_hard_select_rows(E, global_labels, row0, n, exact_cuda_cores)
        rec = _pack_selection(*sel)
        records = rec.new_empty(world * rec.numel())
        dist.all_gather_into_tensor(records, rec, group=group)
        pos, neg, d_ap, d_an, valid = _unpack_selection(records.view(world, -1), n)
        loss = _engine.batch_hard_mean(d_ap, d_an, valid, margin)
        ctx.save_for_backward(E, pos, neg, d_ap, d_an, valid)
        ctx.margin, ctx.row0, ctx.n = margin, row0, n
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, pos, neg, d_ap, d_an, valid = ctx.saved_tensors
        g = _engine.batch_hard_backward_rows(E, pos, neg, d_ap, d_an, valid, ctx.row0, ctx.n, ctx.margin, gl)
        return g, None, None, None, None


class GlobalBatchHardTripletLoss:
    """``BatchHardTripletLoss`` over the GLOBAL batch under data parallelism: every anchor takes its hardest positive
    and negative among all N = R n utterances, not only its own rank's n.  The loss is the same device scalar on every
    rank and bit-identical to ``BatchHardTripletLoss`` on the gathered embeddings; its gradient w.r.t. ``local_emb`` is
    this rank's rows of that loss's gradient.  Summed over ranks (the mean all-reduce of the gradients scaled by R, as
    ``batch_hard_step(..., across_ranks=True)`` does) that is the gradient of the global loss.

    Collectives per forward: two all_gathers (embeddings N·D·4 bytes, selection 25 bytes per anchor); none in the
    backward.  The labels are an input: gather them once per batch with ``gather_labels``.  Precondition: every rank
    holds the same n.  Without a process group, or at world size 1, this is exactly ``BatchHardTripletLoss`` and issues
    no collective."""

    def __init__(self, margin, process_group=None, exact_cuda_cores=False):
        self.margin = margin
        self.group = process_group
        self.exact_cuda_cores = exact_cuda_cores

    def forward(self, local_emb, global_labels):
        """local_emb (n, D) this rank's shard, global_labels (N,) int64 of the whole batch -> 0-dim loss."""
        if not _distributed(self.group):
            return _engine.BatchHardTripletFn.apply(local_emb, global_labels, float(self.margin), self.exact_cuda_cores)
        world = dist.get_world_size(self.group)
        if global_labels.shape != (world * local_emb.shape[0],):
            raise ValueError(f"expected global labels of shape ({world * local_emb.shape[0]},) for {world} ranks of "
                             f"{local_emb.shape[0]} embeddings, got {tuple(global_labels.shape)}")
        return _GlobalBatchHardFn.apply(local_emb, global_labels, float(self.margin), self.exact_cuda_cores, self.group)

    __call__ = forward


# ---- GE2E over the global batch -----------------------------------------------------------------------------------------
# Same layout and precondition as batch-hard: rank r holds the rows [r n, (r + 1) n) of N = R n, every rank the same n.

class _GlobalGE2EFn(torch.autograd.Function):
    """Forward: all_gather of the fp32 embeddings, this rank's rows of the GE2E op against the centroids of all N rows,
    all_gather of the row losses, the mean over the global V.  Backward: this rank's dcos rows, ONE all_gather of (dcos,
    tdc) rows, this rank's rows of gE; gw and gb are this rank's shares."""

    @staticmethod
    def forward(ctx, local_emb, w, b, csr, V, method, group):
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        x = local_emb.detach().float().contiguous()
        n = x.shape[0]
        E = x.new_empty(world * n, x.shape[1])
        dist.all_gather_into_tensor(E, x, group=group)
        row0 = rank * n
        wc, bc = (t.detach().float().reshape(1).contiguous() for t in (w, b))
        E, cos, rec, row_loss = _engine.ge2e_rows(E, csr, V, wc, bc, method, row0, n)
        losses = row_loss.new_empty(world * n)
        dist.all_gather_into_tensor(losses, row_loss.contiguous(), group=group)
        loss = _engine.ge2e_mean(losses, V)
        ctx.save_for_backward(E, wc, bc, cos, rec, *csr)
        ctx.V, ctx.method, ctx.group, ctx.row0, ctx.n = V, method, group, row0, n
        ctx.shapes = (w.shape, b.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        E, w, b, cos, rec, *csr = ctx.saved_tensors
        dcos, tdc, gw, gb = _engine.ge2e_dcos_rows(cos, rec, csr, ctx.V, w, b, ctx.method, ctx.row0, ctx.n, gl)
        world, P = dist.get_world_size(ctx.group), dcos.shape[1]
        rows = torch.cat([dcos, tdc.reshape(-1, 1)], dim=1)             # (n, P + 1): one record per row
        out = rows.new_empty(world * ctx.n, P + 1)
        dist.all_gather_into_tensor(out, rows, group=ctx.group)
        gE = _engine.ge2e_backward_rows(E, csr, out[:, :P], out[:, P], ctx.row0, ctx.n)
        ni = ctx.needs_input_grad
        return (gE if ni[0] else None, gw.reshape(ctx.shapes[0]) if ni[1] else None,
                gb.reshape(ctx.shapes[1]) if ni[2] else None, None, None, None, None)


class GlobalGE2ELoss:
    """``GE2ELoss`` over the GLOBAL batch under data parallelism: every utterance is scored against the centroids of all
    N = R n utterances, and its own speaker's leave-one-out centroid takes that speaker's rows from every rank, so a
    speaker may span any number of ranks.  The loss is the same device scalar on every rank and bit-identical to
    ``loss`` on the gathered embeddings with the global labels; its gradient w.r.t. ``local_emb`` is this rank's rows of
    that loss's gradient, bit for bit.  The gradients of ``loss.w`` and ``loss.b`` are this rank's shares: summed over
    ranks (the mean all-reduce of the gradients scaled by R, as ``ge2e_step(..., across_ranks=True)`` does) they are
    the global loss's, to ~1e-7 relative.

    Collectives: two all_gathers in the forward (embeddings N·D·4 bytes, row losses N·4 bytes) and one in the backward
    (dcos rows and the target column's dcos, N·(P + 1)·4 bytes).  The labels are an input: gather them once per batch
    with ``gather_labels``; they are read on the host to build the speaker lists (CPU labels need no device
    synchronisation).  Precondition: every rank holds the same n.  Without a process group, or at world size 1, this is
    exactly ``loss(local_emb, global_labels)`` and issues no collective."""

    def __init__(self, loss, process_group=None):
        self.loss = loss
        self.group = process_group

    def forward(self, local_emb, global_labels):
        """local_emb (n, D) this rank's shard, global_labels (N,) int of the whole batch -> 0-dim loss."""
        from .model import ge2e_batch, ge2e_csr_to

        if not _distributed(self.group):
            return self.loss(local_emb, global_labels)
        world = dist.get_world_size(self.group)
        if tuple(global_labels.shape) != (world * local_emb.shape[0],):
            raise ValueError(f"expected global labels of shape ({world * local_emb.shape[0]},) for {world} ranks of "
                             f"{local_emb.shape[0]} embeddings, got {tuple(global_labels.shape)}")
        order, offsets, col, V = ge2e_batch(global_labels)
        if V == 0:
            raise ValueError("GlobalGE2ELoss: no utterance of the global batch contributes to the loss (it needs >= 2 "
                             "speakers, one of them with >= 2 utterances)")
        dev = local_emb.device
        if self.loss.w.device != dev:
            raise RuntimeError("GlobalGE2ELoss: move the loss to the embeddings' device (loss.to(device))")
        csr = ge2e_csr_to(order, offsets, col, dev)
        return _GlobalGE2EFn.apply(local_emb, self.loss.w, self.loss.b, csr, V, self.loss.method, self.group)

    __call__ = forward


# ---- synchronised BatchNorm --------------------------------------------------------------------------------------------
# Per utterance and stage: a forward record is 4 (3C + 1) bytes (pivot, sum and sum of squares per channel, the pixel
# count), 34.6 kB over the 12 layers (2880 channels); a backward record is 8C bytes (23 kB over the layers) and the
# loss-scale record 4 bytes.  Every rank must hold the same number of utterances.

def gather_records(local, process_group=None):
    """The exchange of one synchronised-BatchNorm stage: ``local`` is a list of this rank's record tensors (uint8, one
    per forward in lockstep); returns, for each, the records of all ranks concatenated in rank order.  All sets travel in
    ONE all_gather_into_tensor.  Without a process group (or at world size 1) the local records are the global ones."""
    if not _distributed(process_group):
        return list(local)
    world = dist.get_world_size(process_group)
    flat = torch.cat([t.reshape(-1) for t in local])      # a copy: the library's buffer is reused by the next stage
    out = flat.new_empty(world * flat.numel())
    dist.all_gather_into_tensor(out, flat, group=process_group)
    rows, parts, off = out.view(world, -1), [], 0
    for t in local:
        parts.append(rows[:, off:off + t.numel()].reshape(-1))
        off += t.numel()
    return parts


# ---- the class-sharded AAM-softmax head ------------------------------------------------------------------------------
SHARD_BLOCK = 128   # classes per block of a shard boundary and of the forward's partial sums (dsk_aam_shard_partials)


def class_shards(C: int, R: int):
    """The contiguous class ranges [(c0, c1)] of R ranks over C classes: interior boundaries on multiples of 128
    classes, range sizes that differ by at most 128 (the ranges holding one block more are the last ones, so the last
    range's partial block does not widen the spread).  All K sub-centres of a class stay with its rank (a class's cosine
    is the max over them).  ValueError when C < 128 R."""
    for v, name in ((C, "C"), (R, "R")):
        if isinstance(v, bool) or not isinstance(v, int):
            raise ValueError(f"{name} must be an int, got {v!r}")
    if R < 1 or C < SHARD_BLOCK * R:
        raise ValueError(f"class_shards: {R} ranks need R >= 1 and at least {SHARD_BLOCK} classes each (C >= "
                         f"{SHARD_BLOCK * max(R, 1)}), got C = {C}")
    nb = -(-C // SHARD_BLOCK)
    base, extra = divmod(nb, R)
    out, c0 = [], 0
    for r in range(R):
        c1 = min(c0 + (base + (r >= R - extra)) * SHARD_BLOCK, C)
        out.append((c0, c1))
        c0 = c1
    return out


def shard_record_blocks(C: int, R: int) -> int:
    """Blocks per row of a rank's partial-sum record: the largest range's ceil(size / 128), the same on every rank."""
    return max(-(-(c1 - c0) // SHARD_BLOCK) for c0, c1 in class_shards(C, R))


def emulated_gather(local):
    """The forward exchange of R ranks emulated in one process: every rank receives the concatenation, in rank order,
    of all ranks' records (what ``gather_records`` delivers under a process group)."""
    cat = torch.cat([t.reshape(-1) for t in local])
    return [cat] * len(local)


def emulated_all_to_all(local):
    """The backward exchange of R ranks emulated in one process: ``local[q]`` is rank q's (N, D) partial gradient of
    all N = R n rows; rank r receives rows [r n, (r + 1) n) of every rank's partial, in rank order."""
    R = len(local)
    n = local[0].shape[0] // R
    return [torch.cat([p[r * n:(r + 1) * n] for p in local]) for r in range(R)]


def _all_to_all_rows(local, process_group=None):
    """The backward exchange of a process group: ``all_to_all_single`` of each (N, D) partial (rows [q n, (q + 1) n)
    to rank q), (R n, D) back in rank order.  Without a process group the local partials are returned."""
    if not _distributed(process_group):
        return list(local)
    outs = []
    for t in local:
        t = t.contiguous()
        out = torch.empty_like(t)
        dist.all_to_all_single(out, t, group=process_group)
        outs.append(out)
    return outs


class _ShardState:
    """What the sharded forward leaves for its backward (all caller-owned device tensors)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class _ShardedAAMFn(torch.autograd.Function):
    """Forward: the four exchanged stages of ``ShardedAAMSoftmaxLoss.forward_stages``.  Backward: the shard's gW and
    partial gE^, the all_to_all, this rank's rows of gE."""

    @staticmethod
    def forward(ctx, local_emb, weight, global_labels, head):
        from .train import run_lockstep

        st = run_lockstep([head.forward_stages(local_emb, global_labels)],
                          lambda local: gather_records(local, head.group))[0]
        ctx.head, ctx.st = head, st
        return st.loss.reshape(())

    @staticmethod
    def backward(ctx, gl):
        from .train import run_lockstep

        head = ctx.head
        gE, gW = run_lockstep([head.backward_stages(ctx.st, gl)], lambda local: _all_to_all_rows(local, head.group))[0]
        ni = ctx.needs_input_grad
        return (gE if ni[0] else None), (gW if ni[1] else None), None, None


class ShardedAAMSoftmaxLoss:
    """``AAMSoftmaxLoss`` (sub-centres, inter-top-k penalty) with its classes sharded over the ranks of
    ``process_group``: a model-parallel classifier.  Rank r holds ``.weight``, the ``nn.Parameter`` W_r = rows
    [c0 K, c1 K) of the (C K, D) weight for its ``.class_range`` (c0, c1) = ``class_shards(C, R)[r]``; no rank holds
    the others.  Every rank holds the same n utterances (the precondition of ``GlobalGE2ELoss``).

    ``forward(local_emb, global_labels)`` (labels from ``gather_labels``) returns the loss of ``AAMSoftmaxLoss`` on the
    gathered batch with the full weight, a 0-dim device scalar with the same bits on every rank and for every R and
    split; ``cos``, ``sub`` and ``top`` are the whole op's bits.  Its gradient w.r.t. ``local_emb`` is this rank's rows
    of the global loss's gradient (the shards' parts added in rank order: within ~1e-6 of any other split) and w.r.t.
    ``.weight`` the global loss's gradient for the shard (the same bits for every split).  Without a process group, or
    at world size 1, the same stages run with R = 1, so a one-GPU run reproduces a multi-GPU run bit for bit.

    ``weight_full_or_shape``: the full (C K, D) weight (this rank copies its rows: e.g. ``model.model.classifier.weight``
    at K = 1), or its shape, for a weight drawn from N(0, 1/D) with the generator seeded by ``seed`` (the same on every
    rank).  ``shard=(rank, R)`` without a process group runs the stages as rank ``rank`` of R emulated ranks: the caller
    then drives ``forward_stages`` / ``backward_stages`` of all R heads with ``train.run_lockstep`` and the exchanges
    ``emulated_gather`` / ``emulated_all_to_all``.

    Collectives per step, N = R n rows, topk = k, nb = ``shard_record_blocks(C, R)``, bytes received per rank: forward
    all_gathers of the embeddings (N D 4), the top-k keys (R N k 8, none at k = 0), the row maxima (R N 4) and the
    partial-sum records (R N (2 nb + 2) 4, about N C / 16 bytes: R nb ~ C / 128 blocks of two floats per row); backward
    one all_to_all of the embedding rows' gradients (n D 4 bytes per pair of ranks).  Each rank sends records for all N
    rows, hence the factor R.  The weight, its gradient and its optimizer state never travel."""

    def __init__(self, weight_full_or_shape, margin, scale, *, subcentres=1, topk=0, topk_margin=0.0,
                 process_group=None, shard=None, seed=0, device=None):
        if isinstance(weight_full_or_shape, torch.Tensor):
            full = weight_full_or_shape.detach()
            if full.dim() != 2:
                raise ValueError(f"expected a (C * subcentres, D) weight, got shape {tuple(full.shape)}")
            rows, D = full.shape
        else:
            full = None
            rows, D = (int(v) for v in weight_full_or_shape)
        self.C = _engine.aam_subcentre_args(rows, subcentres, topk, topk_margin)
        for v, name in ((margin, "margin"), (scale, "scale")):
            if not math.isfinite(float(v)):
                raise ValueError(f"{name} must be finite, got {v!r}")
        if float(margin) < 0.0 or not float(scale) > 0.0:
            raise ValueError(f"need margin >= 0 and scale > 0, got {margin!r}, {scale!r}")
        if D < 64 or D % 64:
            raise ValueError(f"the embedding size must be a positive multiple of 64, got {D}")
        self.margin, self.scale = float(margin), float(scale)
        self.subcentres, self.topk, self.topk_margin = subcentres, topk, float(topk_margin)
        self.group = process_group
        if _distributed(process_group):
            if shard is not None:
                raise ValueError("shard= emulates ranks without a process group; the group gives the rank")
            self.rank, self.world = dist.get_rank(process_group), dist.get_world_size(process_group)
        elif shard is not None:
            self.rank, self.world = (int(v) for v in shard)
            if not 0 <= self.rank < self.world:
                raise ValueError(f"shard must be (rank, R) with 0 <= rank < R, got {shard!r}")
        else:
            self.rank, self.world = 0, 1
        self.shards = class_shards(self.C, self.world)
        self.class_range = self.shards[self.rank]
        self.record_blocks = shard_record_blocks(self.C, self.world)
        c0, c1 = self.class_range
        K = subcentres
        if (c1 - c0) * K > _engine.L.DSK_AAM_MAX_C:
            raise ValueError(f"the shard holds {(c1 - c0) * K} weight rows, above the per-rank cap "
                             f"{_engine.L.DSK_AAM_MAX_C}: use more ranks or fewer sub-centres")
        if device is None:
            device = full.device if full is not None and full.is_cuda else torch.device("cuda", torch.cuda.current_device())
        if full is None:
            gen = torch.Generator().manual_seed(int(seed))
            full = torch.randn(rows, D, generator=gen) / D ** 0.5
        self.weight = torch.nn.Parameter(full[c0 * K:c1 * K].to(device=device, dtype=torch.float32).clone())

    # -- the weight ---------------------------------------------------------------------------------------------------
    def full_weight(self) -> torch.Tensor:
        """The full (C K, D) weight in class order: an all_gather of the shards (for checkpoints, or to hand the weight
        to a one-GPU ``AAMSoftmaxLoss``).  Collective: every rank must call it."""
        w = self.weight.detach()
        if not _distributed(self.group):
            if self.world > 1:
                raise RuntimeError("full_weight needs the process group; emulated shards hold only their own rows")
            return w.clone()
        K, D = self.subcentres, w.shape[1]
        most = max(c1 - c0 for c0, c1 in self.shards) * K
        pad = w.new_zeros(most, D)
        pad[:w.shape[0]] = w
        out = w.new_empty(self.world * most, D)
        dist.all_gather_into_tensor(out, pad, group=self.group)
        out = out.view(self.world, most, D)
        return torch.cat([out[r, :(c1 - c0) * K] for r, (c0, c1) in enumerate(self.shards)])

    @torch.no_grad()
    def load_full_weight(self, W):
        """Copies this rank's rows of the full (C K, D) weight W into ``.weight``."""
        c0, c1 = self.class_range
        K = self.subcentres
        if tuple(W.shape) != (self.C * K, self.weight.shape[1]):
            raise ValueError(f"expected a ({self.C * K}, {self.weight.shape[1]}) weight, got {tuple(W.shape)}")
        self.weight.copy_(W[c0 * K:c1 * K])

    # -- the stages -----------------------------------------------------------------------------------------------
    def forward_stages(self, local_emb, global_labels):
        """Generator of this rank's forward: yields its records four times (the fp32 embeddings, the top-k keys unless
        topk = 0, the row maxima, the partial-sum records), each time receiving every rank's, concatenated in rank
        order; returns the state ``backward_stages`` reads (StopIteration.value), with ``.loss`` (1,), ``.lse``,
        ``.row_loss``, ``.cos``, ``.sub``, ``.top``."""
        x = local_emb.detach().float().contiguous()
        n, D = x.shape
        E = (yield x).reshape(-1, D).contiguous()
        labels = torch.as_tensor(global_labels).to(device=E.device, dtype=torch.int64).contiguous()
        if labels.shape != (E.shape[0],):
            raise ValueError(f"expected global labels of shape ({E.shape[0]},), got {tuple(labels.shape)}")
        W = self.weight.detach().contiguous()
        if W.device != E.device:
            raise RuntimeError("ShardedAAMSoftmaxLoss: the weight and the embeddings must be on one device")
        c0, c1 = self.class_range
        R, C, K, k, nb = self.world, self.C, self.subcentres, self.topk, self.record_blocks
        margins = (self.margin, self.scale, self.topk_margin)
        cos, sub, keys = _engine.aam_shard_cos(E, W, labels, C, c0, c1, K, k)
        keys_all = (yield keys) if k > 0 else None
        top, thr, mloc = _engine.aam_shard_merge(cos, labels, keys_all, R, C, c0, c1, k, *margins)
        maxima = yield mloc
        m, rec = _engine.aam_shard_partials(cos, labels, thr, maxima, R, C, c0, c1, k, nb, *margins)
        rec_all = yield rec
        loss, lse, row_loss, den = _engine.aam_shard_finish(rec_all, m, labels, R, C, nb)
        return _ShardState(E=E, W=W, labels=labels, n=n, cos=cos, sub=sub, top=top, thr=thr, m=m, den=den, loss=loss,
                           lse=lse, row_loss=row_loss)

    def backward_stages(self, st, grad_loss):
        """Generator of this rank's backward from the forward's state: yields the shard's (N, D) partial gradient of
        the normalised rows once and receives this rank's n rows of every rank's partial, (R n, D) in rank order;
        returns (gE (n, D), gW of the shard), scaled by the device scalar ``grad_loss``."""
        c0, c1 = self.class_range
        gW, part = _engine.aam_shard_backward(st.E, st.W, st.labels, st.cos, st.sub, st.thr, st.m, st.den, self.C, c0,
                                              c1, self.margin, self.scale, self.subcentres, self.topk, self.topk_margin,
                                              grad_loss)
        parts = yield part
        r0 = self.rank * st.n
        gE = _engine.aam_shard_backward_rows(st.E[r0:r0 + st.n].contiguous(), parts, self.world)
        return gE, gW

    def forward(self, local_emb, global_labels):
        """local_emb (n, D) this rank's shard of the batch, global_labels (N,) int64 of the whole batch -> 0-dim
        loss."""
        if self.world > 1 and not _distributed(self.group):
            raise RuntimeError("an emulated shard runs through forward_stages / backward_stages, not forward")
        if local_emb.dim() != 2 or local_emb.shape[1] != self.weight.shape[1]:
            raise ValueError(f"expected embeddings (n, {self.weight.shape[1]}), got {tuple(local_emb.shape)}")
        if not local_emb.is_cuda:
            raise RuntimeError("the sharded AAM-softmax loss needs CUDA tensors; there is no CPU fallback")
        if tuple(global_labels.shape) != (self.world * local_emb.shape[0],):
            raise ValueError(f"expected global labels of shape ({self.world * local_emb.shape[0]},) for {self.world} "
                             f"ranks of {local_emb.shape[0]} embeddings, got {tuple(global_labels.shape)}")
        return _ShardedAAMFn.apply(local_emb, self.weight, global_labels, self)

    __call__ = forward
