"""The per-batch body of the reference's ``train()`` loop (reference train_triplet.py:208-299) on the H100 engine.

``train_step`` restates both branches of the loop with the drop-in classes and the repo's kernels:

* branch A (``epoch > min_softmax_epoch``, :217-224): triplet loss over all triplets, backward, optimizer step;
* branch B (:251-291): margin mask -> hard-triplet indices, triplet loss on the detached selected embeddings,
  second train-mode forward of the selected inputs through ``forward_classifier``, cross-entropy over
  ``cat[cls_a, cls_p, cls_n]`` vs ``cat[label_p, label_p, label_n]``, ``loss = CE + loss_ratio * triplet``.

What differs from the reference is only where things run: the mask, the ascending index list and every gather stay on
the device (``dsk_margin_select`` / ``dsk_gather_rows``); the reference makes six device->host->device round trips
through numpy (:253-274).  ONE host synchronisation remains - reading the number of selected triplets k, which sizes the
second forward (and implements ``if len(hard_triplets[0]) == 0: continue``, :263-264).

The second forward is NOT replaced by re-using the first one's activations: in train mode its BatchNorm layers normalise
with the statistics of the k SELECTED utterances (and update the running statistics three more times), so its logits are
a different function of the parameters than anything the first forward computed.

Data parallelism (SURVEY §8e): pass ``bucket`` (``parallel.GradBucket``) or a ``FusedAdagrad`` optimizer; branch A
averages gradients over ranks, branch B weights each rank's mean gradient by its own k (``k_r / sum k``) through the
same single allreduce.  With synchronised BatchNorm (``DeepSpeakerModel.sync_batchnorm``) branch A runs unchanged and
branch B raises ``ValueError`` before any collective.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import engine as _engine
from . import train as _train
from .head import CrossEntropyLoss
from .model import (AAMSoftmaxLoss, BatchHardTripletLoss, PairwiseDistance, SupConLoss, TripletMarginLoss,
                    batch_hard_valid_count, select_hard_triplets, supcon_valid_count)
from .optim import FusedAdagrad
from .parallel import GlobalBatchHardTripletLoss, GlobalGE2ELoss, GradBucket, _distributed, gather_labels

_l2 = PairwiseDistance(2)   # train_triplet.py:119


def _reduce_and_step(optimizer, bucket, weight):
    """backward has filled the gradients: the step's one collective, then optimizer.step() (:224, :291)."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        weight = None      # one process: the local mean IS the global mean (and the update stays bit-identical to torch's)
    if isinstance(optimizer, FusedAdagrad):
        if weight is not None:
            optimizer.flat_grad.mul_(weight)     # gradients of k_r * (local mean loss); step() divides by sum_r k_r
        optimizer.allreduce(weight=weight)
    elif bucket is not None:
        if weight is None:
            bucket.allreduce_mean()
        else:
            bucket.allreduce_weighted_mean(weight)
    optimizer.step()


def train_step(model, optimizer, data_a, data_p, data_n, label_p, label_n, *, margin, epoch, min_softmax_epoch=2,
               loss_ratio=2.0, bucket=None):
    """One batch of train_triplet.py:208-299.  Returns a dict of device scalars (``loss``, ``triplet``, ``ce``),
    ``selected`` (python int: triplets that entered the loss) and the bookkeeping distances ``d_p`` / ``d_n``
    (:238-245, :251-252); ``None`` when branch B selects nothing (the reference's ``continue``)."""
    if not model.training:
        raise RuntimeError("train_step needs model.train() (train_triplet.py:203)")
    if epoch <= min_softmax_epoch and _train.sync_bn_setting(model)[0]:
        # branch B re-forwards the k_r selected utterances, and k_r differs per rank: the synchronised stages would
        # gather unequal record sets.  Every rank decides this from the same epoch, before any collective.
        raise ValueError("train_step: the hard-triplet branch (epoch <= min_softmax_epoch) is not supported with "
                         "synchronised BatchNorm; call model.sync_batchnorm(False) for it")
    out_a, out_p, out_n = model.forward_triplet(data_a, data_p, data_n)                 # :215
    crit = TripletMarginLoss(margin)
    if epoch > min_softmax_epoch:
        triplet = crit.forward(out_a, out_p, out_n)                                     # :218
        loss = triplet                                                                  # :219
        optimizer.zero_grad()                                                           # :221
        loss.backward()                                                                 # :222
        _reduce_and_step(optimizer, bucket, None)                                       # :223
        with torch.no_grad():
            d_n = _l2.forward(out_a.detach(), out_n.detach())                           # :237
            d_p = _l2.forward(out_a.detach(), out_p.detach())                           # :242
        return {"loss": loss.detach(), "triplet": triplet.detach(), "ce": None, "selected": int(out_a.shape[0]),
                "d_p": d_p, "d_n": d_n}
    # ---- choose the hard negatives (:250-274) -----------------------------------------------------------------------
    with torch.no_grad():
        d_p = _l2.forward(out_a.detach(), out_p.detach())                               # :251
        d_n = _l2.forward(out_a.detach(), out_n.detach())                               # :252
        idx, cnt = select_hard_triplets(d_p, d_n, margin)                               # :253-262 (device)
    k = int(cnt.item())                                                                 # the branch's one host sync
    if k == 0:
        return None                                                                     # :263-264
    with torch.no_grad():
        g = lambda t: _engine.gather_rows(t, idx, cnt)[:k]                              # :265-274 (device gathers)
        sel_a, sel_p, sel_n = g(out_a), g(out_p), g(out_n)
        xa, xp, xn = g(data_a), g(data_p), g(data_n)
        hard = idx[:k]
        true = torch.cat([label_p.to(hard.device)[hard], label_p.to(hard.device)[hard], label_n.to(hard.device)[hard]])  # :283
    triplet = crit.forward(sel_a, sel_p, sel_n)                                         # :275 (constant w.r.t. the parameters)
    cls_a = model.forward_classifier(xa)                                                # :277
    cls_p = model.forward_classifier(xp)                                                # :278
    cls_n = model.forward_classifier(xn)                                                # :279
    ce = CrossEntropyLoss()(torch.cat([cls_a, cls_p, cls_n]), true)                     # :281-285
    loss = ce + triplet * loss_ratio                                                    # :287
    optimizer.zero_grad()                                                               # :289
    loss.backward()                                                                     # :290
    _reduce_and_step(optimizer, bucket, cnt.to(torch.float32).reshape(()))              # :291 (k_r-weighted under DP)
    return {"loss": loss.detach(), "triplet": triplet.detach(), "ce": ce.detach(), "selected": k, "d_p": d_p, "d_n": d_n,
            "hard": hard}


def _labels_to(labels, device):
    labels = torch.as_tensor(labels, dtype=torch.int64)
    if not labels.is_cuda:   # a pageable copy would wait for the stream; a pinned one is queued like a kernel
        labels = labels.pin_memory().to(device, non_blocking=True)
    return labels


def _no_valid_anchor():
    return ValueError("batch_hard_step: no valid anchor in the batch (it needs >= 2 speakers, one of them with "
                      ">= 2 utterances)")


def batch_hard_step(model, optimizer, data, labels, *, margin, bucket=None, across_ranks=False):
    """One batch-hard training step on a P speakers x K utterances batch: ONE train-mode forward of all N utterances
    (BatchNorm statistics over the whole batch), ``BatchHardTripletLoss`` (hardest positive and negative of every anchor
    inside the batch), backward through all N embeddings, optimizer step.  Under data parallelism each rank's gradient
    is weighted by its number of valid anchors V_r (the mechanism of branch B), so the update is that of the mean over
    the union of valid anchors.  V comes from the labels on the host: with CPU labels the step reads nothing back from
    the device.  Returns ``{"loss": device scalar, "valid": V}``; raises ValueError for a batch with V = 0 (no speaker
    with two utterances, or a single speaker).

    ``across_ranks=True`` (data parallelism, ``data`` / ``labels`` this rank's shard, the same size on every rank):
    anchors are mined over the GLOBAL batch with ``parallel.GlobalBatchHardTripletLoss``, so the loss and the selected
    triplets do not depend on the number of ranks.  The labels are gathered first and read back to the host for the
    global V - the step's one host synchronisation; every rank then sees the same V, so on V = 0 all ranks raise before
    any other collective.  The backward is seeded with R: the unchanged mean all-reduce of the gradients (/R) then sums
    the ranks' gradients, which is the gradient of the global loss (exactly so for power-of-two R).  The ranks are
    those of the optimizer's (``FusedAdagrad``) or the bucket's process group.  BatchNorm statistics stay per replica
    by default; on a model with ``sync_batchnorm(group)`` they are those of the global batch too, and the step's forward
    and loss are then those of the single-device step on the gathered batch.  ``valid`` is the global V.  Without a
    process group this is the step with ``across_ranks=False``."""
    if not model.training:
        raise RuntimeError("batch_hard_step needs model.train()")
    if across_ranks:
        return _global_batch_hard_step(model, optimizer, data, labels, margin, bucket)
    V = batch_hard_valid_count(labels)
    if V == 0:
        raise _no_valid_anchor()
    labels = _labels_to(labels, data.device)
    emb = model(data)
    loss = BatchHardTripletLoss(margin).forward(emb, labels)
    optimizer.zero_grad()
    loss.backward()
    _reduce_and_step(optimizer, bucket, torch.tensor(float(V)))
    return {"loss": loss.detach(), "valid": V}


def _global_batch_hard_step(model, optimizer, data, labels, margin, bucket):
    group = optimizer.group if isinstance(optimizer, FusedAdagrad) else (bucket.group if bucket is not None else None)
    if not _distributed(group):
        return batch_hard_step(model, optimizer, data, labels, margin=margin, bucket=bucket)
    world = dist.get_world_size(group)
    global_labels = gather_labels(_labels_to(labels, data.device), group)   # behind the last step's all-reduce
    V = batch_hard_valid_count(global_labels.cpu())                          # the step's one host synchronisation
    if V == 0:
        raise _no_valid_anchor()
    emb = model(data)
    loss = GlobalBatchHardTripletLoss(margin, group).forward(emb, global_labels)
    optimizer.zero_grad()
    loss.backward(torch.full_like(loss, float(world)))       # R x this rank's share; the mean all-reduce divides by R
    _reduce_and_step(optimizer, bucket, None)
    return {"loss": loss.detach(), "valid": V}


def aam_softmax_step(model, optimizer, data, labels, *, margin, scale, bucket=None, weight=None, subcentres=1, topk=0,
                     topk_margin=0.0):
    """One classification step with the additive angular margin softmax (``AAMSoftmaxLoss`` on
    ``model.model.classifier.weight``): ONE train-mode forward of all N utterances, the loss, backward, optimizer step.
    Returns ``{"loss": device scalar}``.  Every row of the loss depends only on its own embedding and the class weights,
    so under data parallelism (``bucket`` or a ``FusedAdagrad`` optimizer, the same n on every rank) the plain mean
    all-reduce of the gradients is the gradient of the global mean loss; the loss itself needs no collective.  Runs
    unchanged on a model with ``sync_batchnorm()``.

    Sub-centres and the inter-top-k penalty (``AAMSoftmaxLoss``'s ``subcentres``, ``topk``, ``topk_margin``) need a
    (C * subcentres, E) weight: pass it as ``weight``, a parameter the optimizer (or ``bucket``) holds beside the
    model's.  The model's ``state_dict`` keys stay as they are, and with a separate ``weight`` the step leaves
    ``classifier.weight`` and ``classifier.bias`` untouched.  A row of the sub-centre loss still depends only on its own
    embedding, its label and the weight, so the same single mean all-reduce is right under data parallelism.
    ``weight=None`` is ``model.model.classifier.weight``."""
    if not model.training:
        raise RuntimeError("aam_softmax_step needs model.train()")
    if weight is None:
        weight = model.model.classifier.weight
    crit = AAMSoftmaxLoss(weight, margin, scale, subcentres=subcentres, topk=topk, topk_margin=topk_margin)
    labels = _labels_to(labels, data.device)
    emb = model(data)
    loss = crit.forward(emb, labels)
    optimizer.zero_grad()
    loss.backward()
    _reduce_and_step(optimizer, bucket, None)
    return {"loss": loss.detach()}


def _held(opt):
    if opt is None:
        return []
    if isinstance(opt, (FusedAdagrad, GradBucket)):
        return list(opt.params)
    return [p for g in opt.param_groups for p in g["params"]]


def sharded_aam_softmax_step(model, optimizer, data, labels, *, head, head_optimizer, bucket=None):
    """One AAM-softmax step with the class-sharded head ``head`` (``parallel.ShardedAAMSoftmaxLoss``): ONE train-mode
    forward of this rank's n utterances, the sharded loss over the global batch, backward seeded with R, the network's
    gradient reduction and step, then the shard's own step.  Returns ``{"loss": device scalar}``, the same on every
    rank.

    A step of its own rather than a ``head=`` argument of ``aam_softmax_step``: the two differ in everything after the
    forward.  Here the labels are gathered, the loss issues collectives of its own, the backward is seeded with R, and
    a second optimizer steps the shard with no collective; ``aam_softmax_step`` keeps its one all-reduce over the whole
    weight and its signature.

    ``optimizer`` (``FusedAdagrad`` or a torch optimizer with ``bucket``) holds the network's parameters and takes the
    unchanged single mean all-reduce; ``head_optimizer`` holds ``head.weight`` only and steps it locally.  The backward's
    seed R makes the shard's gradient R times the global loss's; the step undoes it: ``FusedAdagrad.step()`` without
    ``allreduce()`` divides by R (build it with ``process_group=head.group``), and a torch optimizer gets the gradient
    divided by R.  Both are exact at power-of-two R.  ValueError, on every rank before any collective, when
    ``head.weight`` is in ``optimizer`` or ``bucket`` or not in ``head_optimizer``.  Runs unchanged on a model with
    ``sync_batchnorm(group)``; without a process group it is the one-GPU step with R = 1."""
    if not model.training:
        raise RuntimeError("sharded_aam_softmax_step needs model.train()")
    W = head.weight
    if any(p is W for p in _held(optimizer) + _held(bucket)):
        raise ValueError("sharded_aam_softmax_step: head.weight must not be in the network optimizer or the bucket "
                         "(it is stepped by head_optimizer, with no collective)")
    if not any(p is W for p in _held(head_optimizer)):
        raise ValueError("sharded_aam_softmax_step: head_optimizer must hold head.weight")
    world = head.world
    if isinstance(head_optimizer, FusedAdagrad):
        opt_world = dist.get_world_size(head_optimizer.group) if (dist.is_available() and dist.is_initialized()) else 1
        if opt_world != world:
            raise ValueError(f"sharded_aam_softmax_step: head_optimizer divides by its group's size {opt_world}, the "
                             f"head has {world} ranks (build it with process_group=head.group)")
    global_labels = gather_labels(_labels_to(labels, data.device), head.group)
    emb = model(data)
    loss = head.forward(emb, global_labels)
    optimizer.zero_grad()
    head_optimizer.zero_grad()
    loss.backward(torch.full_like(loss, float(world)))       # R x this rank's share; the mean all-reduce divides by R
    _reduce_and_step(optimizer, bucket, None)
    if not isinstance(head_optimizer, FusedAdagrad):
        W.grad.div_(world)
    head_optimizer.step()
    return {"loss": loss.detach()}


def _no_valid_ge2e_row():
    return ValueError("ge2e_step: no utterance contributes to the loss (it needs >= 2 speakers, one of them with "
                      ">= 2 utterances)")


def ge2e_step(model, optimizer, data, labels, *, loss, bucket=None, across_ranks=False):
    """One step with the generalised end-to-end loss ``loss`` (a ``GE2ELoss``) on a P speakers x M utterances batch:
    ONE train-mode forward of all N utterances, the loss against the batch's speaker centroids, backward, optimizer step.
    The optimizer (or ``bucket``) must hold ``loss.parameters()`` beside the model's: ``w`` and ``b`` are then reduced
    in the same single all-reduce.  Returns ``{"loss": device scalar, "valid": V}``; raises ValueError for a batch with
    V = 0 (fewer than 2 speakers, or no speaker with 2 utterances).  With CPU labels the step reads nothing back from the
    device.  Runs unchanged on a model with ``sync_batchnorm()``.

    Data parallelism (``bucket`` or a ``FusedAdagrad`` optimizer; ``data`` / ``labels`` this rank's shard, the same size
    on every rank) has two forms:

    * ``across_ranks=False`` (the default): each rank computes GE2E on its own shard, against the centroids of the
      speakers in that shard only, and its gradient is weighted by its number of valid utterances V_r, as in
      ``batch_hard_step``.  The objective then depends on the number of ranks R: a softmax over R times fewer speakers,
      and a speaker split over two ranks gets two smaller centroids.
    * ``across_ranks=True``: GE2E over the GLOBAL batch with ``parallel.GlobalGE2ELoss``.  Every utterance is scored
      against the centroids of all N = R n utterances and a speaker may span any number of ranks, so the loss does not
      depend on R: it is bit-identical to ``GE2ELoss`` on the gathered embeddings.  The labels are gathered first and
      read back to the host for the speaker lists and the global V - the step's one host synchronisation; every rank
      then sees the same V, so on V = 0 all ranks raise before any other collective.  The backward is seeded with R:
      the unchanged mean all-reduce of the gradients (/R, ``loss.parameters()`` in the same bucket) then sums the
      ranks' gradients, which is the gradient of the global loss (exactly so for the embeddings at power-of-two R; w
      and b are summed from per-rank shares).  The ranks are those of the optimizer's (``FusedAdagrad``) or the
      bucket's process group.  BatchNorm statistics stay per replica by default; on a model with
      ``sync_batchnorm(group)`` they are those of the global batch too, and the step's forward and loss are then those
      of the single-device step on the gathered batch.  ``valid`` is the global V.  Without a process group this is
      the step with ``across_ranks=False``."""
    if not model.training:
        raise RuntimeError("ge2e_step needs model.train()")
    if across_ranks:
        return _global_ge2e_step(model, optimizer, data, labels, loss, bucket)
    labels = torch.as_tensor(labels).detach().cpu()     # CUDA labels: the one read-back
    V = batch_hard_valid_count(labels)
    if V == 0:
        raise _no_valid_ge2e_row()
    emb = model(data)
    out = loss(emb, labels)
    optimizer.zero_grad()
    out.backward()
    _reduce_and_step(optimizer, bucket, torch.tensor(float(V)))
    return {"loss": out.detach(), "valid": V}


def _global_ge2e_step(model, optimizer, data, labels, loss, bucket):
    group = optimizer.group if isinstance(optimizer, FusedAdagrad) else (bucket.group if bucket is not None else None)
    if not _distributed(group):
        return ge2e_step(model, optimizer, data, labels, loss=loss, bucket=bucket)
    world = dist.get_world_size(group)
    global_labels = gather_labels(_labels_to(labels, data.device), group)   # behind the last step's all-reduce
    global_labels = global_labels.cpu()                                      # the step's one host synchronisation
    V = batch_hard_valid_count(global_labels)
    if V == 0:
        raise _no_valid_ge2e_row()
    emb = model(data)
    out = GlobalGE2ELoss(loss, group).forward(emb, global_labels)
    optimizer.zero_grad()
    out.backward(torch.full_like(out, float(world)))         # R x this rank's share; the mean all-reduce divides by R
    _reduce_and_step(optimizer, bucket, None)
    return {"loss": out.detach(), "valid": V}


def supcon_step(model, optimizer, data, labels, *, temperature, bucket=None):
    """One supervised-contrastive step (``SupConLoss``): ONE train-mode forward of all N crops, the loss over the batch's
    cosine matrix at ``temperature``, backward, optimizer step.  Returns ``{"loss": device scalar, "valid": V}``; raises
    ValueError for a batch in which no row has a positive (V = 0).  V comes from the labels on the host: with CPU labels
    the step reads nothing back from the device.  Runs unchanged on a model with ``sync_batchnorm()``.  Under data
    parallelism (``bucket`` or a ``FusedAdagrad`` optimizer; ``data`` / ``labels`` this rank's shard, the same size on
    every rank) each rank contrasts within its own shard and its gradient is weighted by its V_r, as in ``ge2e_step``.

    Self-supervised training (SimCLR's NT-Xent; no speaker labels) takes two independently augmented views of each of
    B utterances and labels each view with its utterance.  With a ``WaveBank`` ``bank``, a numpy generator ``g`` and
    the utterance ids ``u`` (B,) of the batch::

        utt = torch.cat([u, u])                                   # 2B examples, view v of utterance b at v B + b
        L = segment_samples(T)
        plan = augment_plan(2 * B, L, g, rir_bank=rirs, noise_bank=noises, noise_groups=groups, speeds=(0.9, 1.0, 1.1))
        start = bank.random_starts(utt, L, g, plan)               # every example draws its own start and augmentation
        x = bank.augmented_crops(utt, start, T, plan, rirs, noises)
        supcon_step(model, opt, x, torch.arange(B).repeat(2), temperature=0.1)

    With speaker labels instead, every pair of rows of one speaker is a positive."""
    if not model.training:
        raise RuntimeError("supcon_step needs model.train()")
    crit = SupConLoss(temperature)
    labels = torch.as_tensor(labels).detach().cpu()     # CUDA labels: the one read-back
    V = supcon_valid_count(labels)
    if V == 0:
        raise ValueError("supcon_step: no row has a positive (every label occurs once)")
    emb = model(data)
    loss = crit.forward(emb, labels)
    optimizer.zero_grad()
    loss.backward()
    _reduce_and_step(optimizer, bucket, torch.tensor(float(V)))
    return {"loss": loss.detach(), "valid": V}
