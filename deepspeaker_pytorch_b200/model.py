"""Drop-in mirror of reference model.py for the hot path, backed by libdsk.so (sm_90a CUDA).

Same names, constructor arguments, submodule tree and ``state_dict`` keys as the reference:

* ``DeepSpeakerModel(embedding_size, num_classes, feature_dim=64)`` — model.py:153-223
* ``TripletMarginLoss(margin).forward(anchor, positive, negative)`` — model.py:19-33
* ``PairwiseDistance(p).forward(x1, x2)`` — model.py:8-18

The ``nn`` submodules below only *hold* parameters/buffers (so ``.cuda()``, ``parameters()``,
``state_dict()``, ``load_state_dict()``, optimizers and checkpoints work exactly as with the
reference, train_triplet.py:168-186,325,372-382); the arithmetic runs in the CUDA engine.  There is no
PyTorch/CPU fallback: non-CUDA inputs or a missing extension raise ``RuntimeError``.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from . import engine as _engine
from . import head as _head


class ReLU(nn.Hardtanh):
    """Clipped ReLU, Hardtanh(0, 20) — model.py:36-44 (parameter-free; fused into the conv epilogues)."""

    def __init__(self, inplace=False):
        super().__init__(0, 20, inplace)

    def __repr__(self):
        return self.__class__.__name__ + " (" + ("inplace" if self.inplace else "") + ")"


def conv3x3(in_planes, out_planes, stride=1):
    """3x3 convolution with padding — model.py:47-50."""
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class BasicBlock(nn.Module):
    """Parameter holder with the reference's attribute names — model.py:53-82."""

    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride


class myResNet(nn.Module):
    """Parameter holder for the 4-stage ResCNN — model.py:85-147 (layers=[1,1,1,1], :162)."""

    def __init__(self, block=BasicBlock, layers=(1, 1, 1, 1), num_classes=1000):
        super().__init__()
        self.relu = ReLU(inplace=True)
        chans = (64, 128, 256, 512)
        cin = 1
        for s, ch in enumerate(chans):
            setattr(self, f"conv{s + 1}", nn.Conv2d(cin, ch, kernel_size=5, stride=2, padding=2, bias=False))
            setattr(self, f"bn{s + 1}", nn.BatchNorm2d(ch))
            setattr(self, f"layer{s + 1}", nn.Sequential(*[block(ch, ch) for _ in range(layers[s])]))
            cin = ch
        self.avgpool = nn.AdaptiveAvgPool2d((1, None))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():  # model.py:114-120
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()


class DeepSpeakerModel(nn.Module):
    """ResCNN speaker-embedding network — model.py:153-223 — running on the H100 engine.

    Extra keyword ``operand_dtype`` ("fp16" default, or "bf16") selects the 16-bit tensor-core operand
    format; accumulation, BatchNorm, pooling, fc and the L2-norm are fp32 either way.
    """

    def __init__(self, embedding_size, num_classes, feature_dim=64, operand_dtype="fp16"):
        super().__init__()
        if feature_dim != 64:
            # model.py:165-166: the feature_dim==40 branch does not match the 4-stage net (SURVEY §8b)
            raise ValueError("only feature_dim=64 is supported")
        if operand_dtype not in ("fp16", "bf16"):
            raise ValueError("operand_dtype must be 'fp16' or 'bf16'")
        self.embedding_size = embedding_size
        self.operand_dtype = operand_dtype
        self.model = myResNet(BasicBlock, [1, 1, 1, 1])
        self.model.fc = nn.Linear(512 * 4, self.embedding_size)          # model.py:163-164
        self.model.classifier = nn.Linear(self.embedding_size, num_classes)  # :167
        self._engine = None
        self._sync_bn = None          # (process group,) while BatchNorm statistics are synchronised

    def sync_batchnorm(self, process_group=None):
        """Synchronise the train-mode BatchNorm statistics over the ranks of ``process_group`` (the default group
        when None and torch.distributed is initialised), as ``nn.SyncBatchNorm.convert_sync_batchnorm`` does for torch
        modules; ``sync_batchnorm(False)`` returns to per-replica statistics (the default).  Returns the model.

        Once on, every train-mode ``model(x)`` / ``forward_triplet`` normalises each layer with the statistics of the
        global batch, combined from per-utterance records in global utterance order: the embeddings, the batch
        statistics and the running statistics a rank computes for its own utterances are bit-identical for every split
        of the batch over ranks, one rank (or no process group) included - that path is the same staged one.  The
        forward exchanges records at each of the 12 BatchNorm layers and the backward at 13 points, so ``backward()``
        issues collectives and every rank must run the same forwards and backwards in the same order, each with the
        same batch size.  Eval mode is unchanged (it uses the running statistics)."""
        if process_group is False:
            self._sync_bn = None
        else:
            if process_group is None:
                import torch.distributed as dist

                if dist.is_available() and dist.is_initialized():
                    process_group = dist.group.WORLD
            self._sync_bn = (process_group,)
        return self

    # -- engine plumbing -------------------------------------------------------------------------
    def _get_engine(self, device):
        if self._engine is None or self._engine.device != device:
            self._engine = _engine.Engine(self, device, self.operand_dtype)
        return self._engine

    def refresh_weights(self):
        """Tell the engine(s) that parameters / BatchNorm buffers were modified through ``.data`` (which PyTorch's
        version counter does not see): the packed 16-bit weights and the folded BN affine are rebuilt at the next
        forward.  In-place updates of the parameters themselves (optimizers, ``load_state_dict``) are detected
        automatically."""
        if self._engine is not None:
            self._engine.invalidate()

    def l2_norm(self, input):
        """model.py:172-183 (kept for API parity; the engine fuses it into the tail kernel)."""
        input_size = input.size()
        buffer = torch.pow(input, 2)
        normp = torch.sum(buffer, 1).add_(1e-10)
        norm = torch.sqrt(normp)
        _output = torch.div(input, norm.view(-1, 1).expand_as(input))
        return _output.view(input_size)

    def forward(self, x):
        """model.py:185-218: x (B,1,T,64) float CUDA tensor -> (B, embedding_size), L2 norm 10."""
        if not x.is_cuda:
            raise RuntimeError("DeepSpeakerModel (H100 engine) needs CUDA tensors; there is no CPU fallback")
        if x.dim() != 4 or x.size(1) != 1 or x.size(3) != 64:
            raise RuntimeError(f"expected input (B,1,T,64), got {tuple(x.shape)}")
        eng = self._get_engine(x.device)
        self.features = eng.forward(x, self.training)
        return self.features

    def forward_triplet(self, anchor, positive, negative):
        """The three forwards of a triplet step, ``model(data_a), model(data_p), model(data_n)``
        (reference train_triplet.py:215), issued together: same three results (bit-identical embeddings, batch
        statistics per call, running statistics updated in the order a, p, n), but in train mode the calls run on three
        streams and overlap - as do their backwards.  In eval mode it is simply three forwards.  ``self.features`` is
        left at the negative's embeddings, as after the reference's third call."""
        xs = (anchor, positive, negative)
        for x in xs:
            if not x.is_cuda:
                raise RuntimeError("DeepSpeakerModel (H100 engine) needs CUDA tensors; there is no CPU fallback")
            if x.dim() != 4 or x.size(1) != 1 or x.size(3) != 64:
                raise RuntimeError(f"expected input (B,1,T,64), got {tuple(x.shape)}")
        if not self.training:
            outs = [self.forward(x) for x in xs]
        else:
            from . import train as _train

            eng = self._get_engine(anchor.device)
            with torch.cuda.device(anchor.device):
                outs = _train.forward_train_many(eng, list(xs))
        self.features = outs[-1]
        return tuple(outs)

    def forward_classifier(self, x):
        """model.py:220-223: embeddings -> ``model.classifier`` logits (B, num_classes), on the repo's fp32 GEMM
        kernels (``dsk_linear_forward/backward``); ``model.classifier`` only holds the parameters."""
        features = self.forward(x)
        c = self.model.classifier
        return _head.LinearFn.apply(features, c.weight, c.bias)


class PairwiseDistance:
    """model.py:8-18 — ``.forward(x1, x2)`` is called directly (train_triplet.py:119,238,251,...)."""

    def __init__(self, p):
        if p != 2:
            raise ValueError("only the L2 distance (p=2) used by the reference hot path is implemented")
        self.norm = p

    def forward(self, x1, x2):
        assert x1.size() == x2.size()
        return _engine.PairwiseDistanceFn.apply(x1, x2)

    __call__ = forward


class TripletMarginLoss:
    """model.py:19-33 — ``TripletMarginLoss(margin).forward(a, p, n)`` (train_triplet.py:219,275)."""

    def __init__(self, margin):
        self.margin = margin
        self.pdist = PairwiseDistance(2)

    def forward(self, anchor, positive, negative):
        return _engine.TripletLossFn.apply(anchor, positive, negative, float(self.margin))

    __call__ = forward


class BatchHardTripletLoss:
    """In-batch hard-triplet mining (no reference implementation; built from PairwiseDistance and the hinge of
    TripletMarginLoss): over a batch of P speakers x K utterances, each anchor takes its farthest same-label embedding
    and its nearest different-label embedding; ``loss = mean over valid anchors of clamp(margin + d_ap - d_an, 0)``.
    An anchor is valid when the batch holds another utterance of its speaker and one of another speaker.
    ``exact_cuda_cores=True`` forces the all-fp32 distance matrix; the default tensor-core path returns the same bits."""

    def __init__(self, margin, exact_cuda_cores=False):
        self.margin = margin
        self.exact_cuda_cores = exact_cuda_cores

    def forward(self, embeddings, labels):
        """embeddings (N, D) CUDA, labels (N,) int -> 0-dim device scalar; back-propagates into every embedding."""
        return _engine.BatchHardTripletFn.apply(embeddings, labels, float(self.margin), self.exact_cuda_cores)

    __call__ = forward

    @torch.no_grad()
    def mine(self, embeddings, labels):
        """(pos_idx int64, neg_idx int64, d_ap fp32, d_an fp32, valid bool), each (N,) on the device.  Anchors without
        a positive have pos_idx -1, d_ap 0; without a negative, neg_idx -1, d_an +inf."""
        _, _, pos, neg, d_ap, d_an, valid = _engine.batch_hard_mine(embeddings, labels, float(self.margin),
                                                                     self.exact_cuda_cores)
        return pos, neg, d_ap, d_an, valid


class AAMSoftmaxLoss:
    """Additive angular margin softmax (ArcFace / AAM-softmax; no reference implementation - the usual modern form of the
    reference's softmax over ``model.classifier``, train_triplet.py:277-287).  Cosines between the L2-normalised
    embeddings and the L2-normalised rows of ``weight`` (C, E), margin ``m`` added to the angle of the target class
    (``cos - sin(pi - m) m`` past pi - m), logits times ``scale``, cross-entropy averaged over the batch.  Pass
    ``model.model.classifier.weight``: parameters, ``state_dict`` keys and optimizer buckets stay as they are, and the
    classifier's bias is not used.  ``margin = 0`` is the normalised softmax (NormFace); a margin warm-up passes a
    different ``margin`` per step.

    Sub-centres and the inter-top-k penalty (Deng et al., "Sub-center ArcFace", ECCV 2020; Zhao et al., ICASSP 2022;
    no reference implementation, parity unpinned): with ``subcentres`` K > 1 the weight is (C K, E), row c K + k being
    sub-centre k of class c (as ``reshape(C, K, E)``), and a class's cosine is the largest of its K; with ``topk`` > 0
    the ``topk`` hardest non-target classes of each row get the logit s cos(theta - ``topk_margin``).  The defaults
    (K = 1, topk = 0) are the plain loss above, bit for bit.  The weight must have C K rows, 1 <= K <= 16,
    0 <= topk <= min(C - 1, 64), and ``topk_margin`` must be finite and >= 0; anything else raises ValueError."""

    def __init__(self, weight, margin, scale, *, subcentres=1, topk=0, topk_margin=0.0):
        _engine.aam_subcentre_args(weight.shape[0] if weight.dim() == 2 else 0, subcentres, topk, topk_margin)
        self.weight = weight
        self.margin = margin
        self.scale = scale
        self.subcentres, self.topk, self.topk_margin = subcentres, topk, topk_margin

    def forward(self, embeddings, labels):
        """embeddings (N, E) CUDA, labels (N,) int in [0, C) -> 0-dim device scalar; back-propagates into the
        embeddings and the weight."""
        return _engine.AAMSoftmaxFn.apply(embeddings, self.weight, labels, float(self.margin), float(self.scale),
                                          self.subcentres, self.topk, float(self.topk_margin))

    __call__ = forward


def ge2e_batch(labels):
    """The speaker lists of a GE2E batch, built on the host from int64 labels of any values: (order, offsets, col, V)
    as int64 numpy arrays and an int.  Speakers are the distinct labels in ascending order (``identification.
    speaker_csr``'s order): speaker k's rows are order[offsets[k]:offsets[k+1]] in ascending row order, col[i] is row
    i's speaker, and V (``batch_hard_valid_count``'s rule) counts the rows whose speaker has >= 2 rows, provided the
    batch holds >= 2 speakers.  A CUDA tensor is read back to the host (one device synchronisation)."""
    from .identification import speaker_csr

    lab = torch.as_tensor(labels).detach().cpu().reshape(-1)
    if lab.dtype.is_floating_point or lab.dtype == torch.bool:
        raise ValueError(f"GE2E labels must be integers, got {lab.dtype}")
    order, offsets, _ = speaker_csr(lab.to(torch.int64))
    counts = np.diff(offsets)
    col = np.empty(order.size, np.int64)
    col[order] = np.repeat(np.arange(counts.size, dtype=np.int64), counts)
    V = int(counts[counts >= 2].sum()) if counts.size >= 2 else 0
    return order, offsets, col, V


def ge2e_csr_to(order, offsets, col, device):
    """``ge2e_batch``'s speaker lists as int64 tensors (order, offsets, col) on ``device``: to a CUDA device one pinned
    copy, queued on the stream like a kernel."""
    host = torch.from_numpy(np.concatenate([order, offsets, col]))
    flat = host.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else host
    N, P = order.size, offsets.size - 1
    return flat[:N], flat[N:N + P + 1], flat[N + P + 1:]


class GE2ELoss(nn.Module):
    """Generalised end-to-end loss (Wan et al., "Generalized End-to-End Loss for Speaker Verification", ICASSP 2018; no
    reference implementation) over a batch of P speakers x M utterances.  Every utterance is scored against every
    speaker's centroid in the batch (the mean of its normalised embeddings), its own speaker's with the utterance left
    out; the cosines pass through ``max(w, 1e-6) cos + b`` and then a softmax over the speakers (``method="softmax"``)
    or the paper's contrast loss (``"contrast"``: 1 - sigmoid(own) + the largest sigmoid of another speaker).  The
    loss is the mean over the utterances whose speaker has >= 2 of them; a singleton speaker's utterance adds no term
    but its centroid is a column for every other one.  The definition is stated in full in ``include/dsk.h``.

    ``w`` and ``b`` are learnable parameters: pass ``loss.parameters()`` to the optimizer (or bucket) with the model's.
    With ``softmax`` the gradient of ``b`` is exactly 0 (b cancels out of the loss), so ``b`` never moves."""

    def __init__(self, init_w=10.0, init_b=-5.0, method="softmax"):
        super().__init__()
        _engine._ge2e_method(method)
        self.method = method
        self.w = nn.Parameter(torch.tensor(float(init_w)))
        self.b = nn.Parameter(torch.tensor(float(init_b)))

    def extra_repr(self):
        return f"method={self.method!r}"

    def forward(self, embeddings, labels):
        """embeddings (N, D) CUDA (D a multiple of 64), labels (N,) int -> 0-dim device scalar; back-propagates into the
        embeddings, ``w`` and ``b``.  With CPU labels, as a data loader yields them, the speaker lists are built on the
        host and the step reads nothing back from the device; CUDA labels are read back once.  Raises ValueError when no
        utterance can contribute (V = 0: fewer than 2 speakers, or no speaker with 2 utterances), before any launch."""
        order, offsets, col, V = ge2e_batch(labels)
        if V == 0:
            raise ValueError("GE2ELoss: no utterance contributes to the loss (it needs >= 2 speakers, one of them with "
                             ">= 2 utterances)")
        if not embeddings.is_cuda:
            raise RuntimeError("GE2ELoss needs CUDA embeddings; there is no CPU fallback")
        if order.size != embeddings.shape[0]:
            raise RuntimeError(f"GE2ELoss: {order.size} labels for {embeddings.shape[0]} embeddings")
        dev = embeddings.device
        if self.w.device != dev:
            raise RuntimeError("GE2ELoss: move the loss to the embeddings' device (loss.to(device))")
        csr = ge2e_csr_to(order, offsets, col, dev)
        return _engine.GE2EFn.apply(embeddings, self.w, self.b, csr, V, self.method)


def batch_hard_valid_count(labels):
    """V, the number of valid anchors of a batch-hard loss, from the labels alone (host-side: no device sync when the
    labels are a CPU tensor, as a data loader yields them): anchors whose speaker has >= 2 utterances, provided the
    batch holds >= 2 speakers."""
    lab = torch.as_tensor(labels).detach().cpu().reshape(-1)
    _, counts = torch.unique(lab, return_counts=True)
    if counts.numel() < 2:
        return 0
    return int(counts[counts >= 2].sum())


def supcon_valid_count(labels):
    """V, the number of valid rows of a supervised-contrastive loss, from the labels alone (host-side: no device sync
    when the labels are a CPU tensor): rows whose label occurs at least twice.  Unlike ``batch_hard_valid_count`` a
    batch of one label counts in full.  ValueError for non-integer labels."""
    lab = torch.as_tensor(labels).detach().cpu().reshape(-1)
    if lab.dtype.is_floating_point or lab.dtype == torch.bool:
        raise ValueError(f"supervised-contrastive labels must be integers, got {lab.dtype}")
    _, counts = torch.unique(lab, return_counts=True)
    return int(counts[counts >= 2].sum())


class SupConLoss:
    """Supervised-contrastive loss (Khosla et al., "Supervised Contrastive Learning", NeurIPS 2020, the L_out form; no
    reference implementation) over the batch's own cosine matrix at temperature ``temperature``: for each row with
    another row of its label, the log-softmax over every other row of cos / temperature, averaged over the row's
    positives; the loss is the mean over those rows.  A row whose label occurs once adds no term but is a negative in
    every other row.  The definition is stated in full in ``include/dsk.h``.

    With labels = the utterance index of each view (two augmented crops of each of B utterances, labels
    ``arange(B).repeat(2)``) it is the NT-Xent loss of SimCLR (Chen et al., ICML 2020): self-supervised training
    without speaker labels (see ``steps.supcon_step``).  With speaker labels it takes every positive pair in the batch.
    ``temperature`` must be finite and > 0 (ValueError)."""

    def __init__(self, temperature=0.1):
        t = float(temperature)
        if not math.isfinite(t) or t <= 0.0:
            raise ValueError(f"SupConLoss: temperature must be finite and > 0, got {temperature!r}")
        self.temperature = t

    def forward(self, embeddings, labels):
        """embeddings (N, D) CUDA (D a multiple of 64), labels (N,) int -> 0-dim device scalar; back-propagates into the
        embeddings.  V comes from the labels on the host: with CPU labels, as a data loader yields them, nothing is read
        back from the device; CUDA labels are read back once.  Raises ValueError when no row has a positive (V = 0) and
        RuntimeError for a label count that does not match the embeddings, before any launch."""
        V = supcon_valid_count(labels)
        if V == 0:
            raise ValueError("SupConLoss: no row has a positive (every label occurs once)")
        n = torch.as_tensor(labels).numel()
        if embeddings.dim() != 2 or n != embeddings.shape[0]:
            raise RuntimeError(f"SupConLoss: {n} labels for embeddings of shape {tuple(embeddings.shape)}")
        if not embeddings.is_cuda:
            raise RuntimeError("SupConLoss needs CUDA embeddings; there is no CPU fallback")
        return _engine.SupConFn.apply(embeddings, labels, V, self.temperature)

    __call__ = forward


def select_hard_triplets(d_p, d_n, margin):
    """Device-side restatement of train_triplet.py:251-262: returns (idx int64 (B,), count int32 (1,)) on the
    GPU; idx[:count] equals np.where((d_n - d_p < margin) == 1)[0].  No host synchronisation."""
    return _engine.margin_select(d_p, d_n, margin)


def allpairs_topk(E, labels, k, exact_cuda_cores=False):
    """BASELINE config 4: per-row k nearest different-label embeddings (idx int64 (N,k), dist fp32 (N,k)).
    Default: wgmma Gram GEMM + exact fp32 refinement (bit-identical to the all-fp32 path, `exact_cuda_cores=True`)."""
    return _engine.allpairs_topk(E, labels, k, exact_cuda_cores)
