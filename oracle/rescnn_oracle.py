"""CPU oracle for the Deep Speaker hot path — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product (deepspeaker_pytorch_b200/) never does.

It is a plain-PyTorch fp32 CPU restatement of the reference's algorithm for the path, function by
function, each citing the reference file:line it follows.  The conv / batch-norm / linear
arithmetic itself lives in PyTorch (un-vendored third-party dependency of the reference, no pinned
version; this container has torch 2.11 CPU kernels), exactly as it does for the reference.

Pinning: tests/golden/*.npz hold outputs of the *reference's own* model.py
(reference model.py imported unmodified by tools/make_golden.py in the build container);
tests/test_oracle_golden.py checks this restatement against them.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

STAGE_CH = (64, 128, 256, 512)
BN_EPS = 1e-5        # torch.nn.BatchNorm2d default, model.py:59
BN_MOMENTUM = 0.1    # torch.nn.BatchNorm2d default
CLIP_HI = 20.0       # Hardtanh(0, 20), model.py:36-39
ALPHA = 10.0         # model.py:211-213


def conv_names():
    """(conv weight key, bn prefix, ksize, stride) of the 12 conv+bn pairs in forward order
    (model.py:187-205 and BasicBlock.forward :66-82)."""
    out = []
    for s in range(4):
        out.append((f"model.conv{s + 1}.weight", f"model.bn{s + 1}", 5, 2))
        out.append((f"model.layer{s + 1}.0.conv1.weight", f"model.layer{s + 1}.0.bn1", 3, 1))
        out.append((f"model.layer{s + 1}.0.conv2.weight", f"model.layer{s + 1}.0.bn2", 3, 1))
    return out


def make_state_dict(seed: int = 0, num_classes: int = 16, embedding_size: int = 512,
                    randomize_bn: bool = True) -> "OrderedDict[str, torch.Tensor]":
    """Deterministic parameters with the reference's state_dict keys (SURVEY §3.4).

    Conv weights follow the reference init N(0, sqrt(2/(k*k*cout))) (model.py:114-117).  BN affine
    and running stats are randomised (the reference's gamma=1, beta=0 init, model.py:118-120, would
    hide scale/bias bugs); fc/classifier use U(-1/sqrt(fan_in), 1/sqrt(fan_in)) like nn.Linear.
    """
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    cin = 1
    for s, ch in enumerate(STAGE_CH):
        def bn(prefix, c):
            if randomize_bn:
                sd[prefix + ".weight"] = torch.empty(c).uniform_(0.5, 1.5, generator=g)
                sd[prefix + ".bias"] = torch.empty(c).normal_(0, 0.1, generator=g)
                sd[prefix + ".running_mean"] = torch.empty(c).normal_(0, 0.1, generator=g)
                sd[prefix + ".running_var"] = torch.empty(c).uniform_(0.5, 1.5, generator=g)
            else:
                sd[prefix + ".weight"] = torch.ones(c)
                sd[prefix + ".bias"] = torch.zeros(c)
                sd[prefix + ".running_mean"] = torch.zeros(c)
                sd[prefix + ".running_var"] = torch.ones(c)
            sd[prefix + ".num_batches_tracked"] = torch.tensor(0, dtype=torch.long)

        sd[f"model.conv{s + 1}.weight"] = torch.empty(ch, cin, 5, 5).normal_(0, math.sqrt(2.0 / (25 * ch)), generator=g)
        bn(f"model.bn{s + 1}", ch)
        for k in (1, 2):
            sd[f"model.layer{s + 1}.0.conv{k}.weight"] = torch.empty(ch, ch, 3, 3).normal_(
                0, math.sqrt(2.0 / (9 * ch)), generator=g)
            bn(f"model.layer{s + 1}.0.bn{k}", ch)
        cin = ch
    b = 1.0 / math.sqrt(2048)
    sd["model.fc.weight"] = torch.empty(embedding_size, 2048).uniform_(-b, b, generator=g)
    sd["model.fc.bias"] = torch.empty(embedding_size).uniform_(-b, b, generator=g)
    b = 1.0 / math.sqrt(embedding_size)
    sd["model.classifier.weight"] = torch.empty(num_classes, embedding_size).uniform_(-b, b, generator=g)
    sd["model.classifier.bias"] = torch.empty(num_classes).uniform_(-b, b, generator=g)
    return sd


def make_input(B: int, T: int = 160, seed: int = 0, scale: float = 1.0) -> torch.Tensor:
    """Synthetic fbank batch (B,1,T,64): time on H, 64 bins on W (SURVEY §0 fact 1)."""
    return scale * torch.randn(B, 1, T, 64, generator=torch.Generator().manual_seed(seed))


def clipped_relu(x):
    """ReLU = Hardtanh(0, 20), model.py:36-44."""
    return torch.clamp(x, 0.0, CLIP_HI)


def _bn(x, sd, prefix, train, stats_out):
    """nn.BatchNorm2d forward (model.py:59,62,94,...). train=True uses batch statistics and returns the
    updated running stats (unbiased variance, momentum 0.1) in stats_out."""
    w, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
    if not train:
        return F.batch_norm(x, sd[prefix + ".running_mean"], sd[prefix + ".running_var"], w, b, False, BN_MOMENTUM, BN_EPS)
    rm = sd[prefix + ".running_mean"].clone()
    rv = sd[prefix + ".running_var"].clone()
    y = F.batch_norm(x, rm, rv, w, b, True, BN_MOMENTUM, BN_EPS)
    if stats_out is not None:
        stats_out[prefix + ".running_mean"] = rm
        stats_out[prefix + ".running_var"] = rv
    return y


def l2_norm(x):
    """DeepSpeakerModel.l2_norm, model.py:172-183."""
    normp = torch.sum(torch.pow(x, 2), 1).add_(1e-10)
    norm = torch.sqrt(normp)
    return torch.div(x, norm.view(-1, 1).expand_as(x))


class _ClipForcedMask(torch.autograd.Function):
    """clamp(x, 0, 20) whose backward passes the gradient where `mask` says so instead of where 0 < x < 20.
    Test-only: lets a test differentiate the oracle with the SAME pass-through set as the implementation under test.
    The clip gradient is discontinuous, so an element whose pre-activation lies within rounding distance of 0 or 20
    flips between implementations, and ONE flipped element moves every upstream gradient by ~1/sqrt(#elements)
    (2.5e-3 at batch 6: fp32 vs fp64 of this very oracle differ by that much, tests/test_oracle_golden.py)."""

    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        return torch.clamp(x, 0.0, CLIP_HI)

    @staticmethod
    def backward(ctx, g):
        (mask,) = ctx.saved_tensors
        return g * mask.to(g.dtype), None


def _ste(t, dtype):
    """Round to `dtype` in the forward, identity in the backward (straight-through)."""
    return t if dtype is None else t + (t.to(dtype).to(t.dtype) - t).detach()


def forward(sd, x, train: bool = False, stats_out=None, taps=None, storage=None, masks=None):
    """DeepSpeakerModel.forward, model.py:185-218. x (B,1,T,64) fp32 -> (B,E), ||.|| = 10.
    taps: optional dict collecting per-layer activations (NCHW) keyed by conv index 0..11.
    storage: None = the reference's fp32 arithmetic.  torch.float16 / torch.bfloat16 = additionally round what
    the CUDA engine stores in 16 bit (tensor-core conv weights and every post-activation tensor; conv1, the
    pre-BN conv outputs and the tail stay fp32).  Only used by tests that need the same ReLU/clip masks as the
    engine to validate its backward kernels in isolation.
    masks: optional {conv index 0..11: bool NCHW tensor}: the clip of that layer back-propagates through exactly these
    elements (see _ClipForcedMask); forward values are unaffected.  Works in fp64 when sd and x are fp64."""
    q = lambda t: _ste(t, storage)
    clip = lambda t, i: clipped_relu(t) if masks is None else _ClipForcedMask.apply(t, masks[i])
    h = x
    for s in range(4):
        pre = f"model.layer{s + 1}.0"
        w_in = sd[f"model.conv{s + 1}.weight"]
        h = F.conv2d(h, w_in if s == 0 else q(w_in), None, 2, 2)              # model.py:187,192,197,202
        h = q(clip(_bn(h, sd, f"model.bn{s + 1}", train, stats_out), 3 * s))  # :188-189
        if taps is not None:
            taps[3 * s] = h
        res = h                                                                # BasicBlock.forward :66-82
        t = F.conv2d(h, q(sd[pre + ".conv1.weight"]), None, 1, 1)
        t = q(clip(_bn(t, sd, pre + ".bn1", train, stats_out), 3 * s + 1))
        if taps is not None:
            taps[3 * s + 1] = t
        t = F.conv2d(t, q(sd[pre + ".conv2.weight"]), None, 1, 1)
        t = _bn(t, sd, pre + ".bn2", train, stats_out)
        h = q(clip(t + res, 3 * s + 2))                                        # :79-80
        if taps is not None:
            taps[3 * s + 2] = h
    h = h.mean(dim=2, keepdim=True)                                            # AdaptiveAvgPool2d((1,None)) :111,207
    h = h.reshape(h.size(0), -1)                                               # :208  (index = c*4 + w)
    h = F.linear(h, sd["model.fc.weight"], sd["model.fc.bias"])               # :209
    return l2_norm(h) * ALPHA                                                  # :210-213


def forward_classifier(sd, x, train: bool = False, stats_out=None):
    """DeepSpeakerModel.forward_classifier, model.py:220-223."""
    return F.linear(forward(sd, x, train, stats_out), sd["model.classifier.weight"], sd["model.classifier.bias"])


def pairwise_distance(x1, x2, p: int = 2):
    """PairwiseDistance.forward, model.py:13-18."""
    assert x1.size() == x2.size()
    eps = 1e-4 / x1.size(1)
    diff = torch.abs(x1 - x2)
    out = torch.pow(diff, p).sum(dim=1)
    return torch.pow(out + eps, 1.0 / p)


def triplet_margin_loss(a, p, n, margin: float):
    """TripletMarginLoss.forward, model.py:27-33."""
    d_p = pairwise_distance(a, p)
    d_n = pairwise_distance(a, n)
    return torch.mean(torch.clamp(margin + d_p - d_n, min=0.0))


def margin_select(d_p, d_n, margin: float) -> np.ndarray:
    """"Choose the hard negatives", train_triplet.py:251-262: ascending indices with d_n - d_p < margin."""
    allm = (d_n - d_p < margin).cpu().data.numpy().flatten()
    return np.where(allm == 1)[0].astype(np.int64)


def allpairs_topk(E, labels, k: int):
    """BASELINE config 4 — NOT in the reference (parity unpinned, SURVEY §0 fact 3 / §8c).
    D[i,j] = PairwiseDistance(2)(e_i, e_j) (model.py:13-18); candidates have a different label;
    k smallest, ties -> lower index."""
    N, D = E.shape
    eps = np.float32(1e-4 / D)
    En = E.numpy().astype(np.float32)
    idx = np.zeros((N, k), dtype=np.int64)
    val = np.zeros((N, k), dtype=np.float32)
    lab = labels.numpy()
    for i in range(N):
        diff = En[i][None, :] - En
        # sequential-in-d fp32 accumulation is restated exactly in oracle/dsk_oracle.c; numpy's pairwise
        # summation differs in the last ulps, which is below every tolerance used with this function.
        s = np.sum(diff * diff, axis=1, dtype=np.float32)
        d = np.sqrt(s + eps)
        d[lab == lab[i]] = np.inf
        order = np.lexsort((np.arange(N), d))[:k]
        idx[i] = order
        val[i] = d[order]
    return idx, val


def triplet_step_branch_a(sd, xa, xp, xn, margin: float, stats_out=None, storage=None, masks=None, taps=None):
    """Branch A of the training step (epoch > min_softmax_epoch), train_triplet.py:215-224:
    three separate train-mode forwards (BN statistics per call, running stats updated three times),
    triplet loss over all triplets, backward.  Returns (loss, grads dict, out_a, out_p, out_n).
    masks / taps: optional lists of three per-call dicts (see forward()).  Works in fp64 when sd and inputs are fp64."""
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items() if v.dtype.is_floating_point
              and "running" not in k}
    cur = dict(sd)
    cur.update(params)
    outs = []
    for j, x in enumerate((xa, xp, xn)):                      # train_triplet.py:215
        st = {}
        outs.append(forward(cur, x, True, st, storage=storage, masks=None if masks is None else masks[j],
                            taps=None if taps is None else taps[j]))
        cur.update(st)                                        # running stats carry across the three calls
    loss = triplet_margin_loss(outs[0], outs[1], outs[2], margin)   # :219
    loss.backward()                                           # :223
    grads = {k: (v.grad if v.grad is not None else None) for k, v in params.items()}
    if stats_out is not None:
        for k in cur:
            if "running" in k:
                stats_out[k] = cur[k]
    return loss.detach(), grads, outs[0].detach(), outs[1].detach(), outs[2].detach()


def triplet_step_branch_b(sd, xa, xp, xn, label_p, label_n, margin: float, loss_ratio: float = 2.0, hard=None):
    """Branch B of the training step (epoch <= min_softmax_epoch), train_triplet.py:215,251-291: three train-mode
    forwards, margin mask -> hard indices, triplet loss on the DETACHED selected embeddings (constant w.r.t. the
    parameters, SURVEY §0 fact 5), second forward of the selected inputs through forward_classifier, cross-entropy over
    cat[cls_a, cls_p, cls_n] against cat[label_p, label_p, label_n] (:283), loss = CE + loss_ratio * triplet (:287).
    `hard` overrides the selection (used to compare implementations on identical indices).
    Returns dict(hard, triplet, ce, loss, grads) or None when no triplet is selected (:263-264)."""
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items() if v.dtype.is_floating_point
              and "running" not in k}
    cur = dict(sd)
    cur.update(params)
    outs = []
    for x in (xa, xp, xn):                                                     # :215
        st = {}
        outs.append(forward(cur, x, True, st))
        cur.update(st)
    d_p = pairwise_distance(outs[0], outs[1])                                  # :251
    d_n = pairwise_distance(outs[0], outs[2])                                  # :252
    if hard is None:
        hard = margin_select(d_p, d_n, margin)                                 # :253-262
    if len(hard) == 0:
        return None                                                            # :263-264
    h = torch.from_numpy(np.asarray(hard))
    sel = [o.detach()[h] for o in outs]                                        # :265-267 (numpy round trip detaches)
    triplet = triplet_margin_loss(sel[0], sel[1], sel[2], margin)              # :275
    logits = []
    for x in (xa, xp, xn):                                                     # :277-279
        st = {}
        logits.append(forward_classifier(cur, x[h], True, st))
        cur.update(st)
    true = torch.cat([label_p[h], label_p[h], label_n[h]])                     # :283
    ce = F.cross_entropy(torch.cat(logits), true)                              # :281-285
    loss = ce + triplet * loss_ratio                                           # :287
    loss.backward()                                                            # :290
    grads = {k: v.grad for k, v in params.items()}
    stats = {k: v for k, v in cur.items() if "running" in k}
    return {"hard": np.asarray(hard), "triplet": triplet.detach(), "ce": ce.detach(), "loss": loss.detach(),
            "grads": grads, "stats": stats}
