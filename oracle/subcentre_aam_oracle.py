"""fp64 restatement of the sub-centre AAM-softmax with the inter-top-k penalty — TEST INFRASTRUCTURE ONLY (the product
never imports this module).

Sub-center ArcFace (Deng et al., ECCV 2020) with the inter-top-k penalty (Zhao et al., ICASSP 2022), as open toolkits
ship the two as one head; no published implementation is available to the project, so parity with one is unpinned.
For embeddings E (N, D), weight W (C K, D) whose row c K + k is sub-centre k of class c, labels y in [0, C), margin m,
scale s, topk and m':

* e^, w^ as F.normalize; g = e^ w^T (N, C K);
* class cosine cos_ic = max_k g_{i,cK+k}, sub_ic its argmax: ties to the lowest k, a NaN sub-centre cosine wins (the
  lowest such k) and makes cos_ic NaN;
* T_i = the topk non-target classes first in the order (-cos, c) with NaN last;
* logits s phi(cos) on the target (``aam_softmax_oracle.phi``), s psi(cos) on T_i with
  psi(c) = c cos m' + sqrt(clamp(1 - c^2, 0, 1)) sin m' = cos(theta - m'), s cos elsewhere;
* loss = (1/N) sum_i (logsumexp_c logit_ic - logit_{i, y_i}).

K = 1, topk = 0 is ``aam_softmax_oracle``, bit for bit.  ``backward`` states the gradients explicitly (the class
gradient goes to column c K + sub_ic only); ``loss_autograd`` is the textbook form for torch autograd.  The forward and
backward can take the engine's own ``cos`` / ``sub`` / ``top`` pinned, to isolate the arithmetic that follows them.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import aam_softmax_oracle as A


def psi(c, topk_margin):
    sn = torch.sqrt(torch.clamp(1.0 - c * c, 0.0, 1.0))
    return c * math.cos(topk_margin) + sn * math.sin(topk_margin)


def dpsi(c, topk_margin):
    """d psi / d cos, with the finite value cos m' at sin = 0 (as ``aam_softmax_oracle.dphi``)."""
    sn = torch.sqrt(torch.clamp(1.0 - c * c, 0.0, 1.0))
    safe = torch.where(sn > 0, sn, torch.ones_like(sn))
    return torch.where(sn > 0, math.cos(topk_margin) - math.sin(topk_margin) * c / safe,
                       torch.full_like(c, math.cos(topk_margin)))


def subcentre_max(g, K):
    """g (N, C K) -> (cos (N, C), sub (N, C) int64): the max over each class's K columns and its argmax, ties to the
    lowest k, NaN winning (the lowest NaN k)."""
    g = torch.as_tensor(g)
    N = g.shape[0]
    v = g.reshape(N, -1, K)
    best, sub = v[..., 0].clone(), torch.zeros(v.shape[:2], dtype=torch.int64)
    for k in range(1, K):
        x = v[..., k]
        upd = ~torch.isnan(best) & (torch.isnan(x) | (x > best))
        best = torch.where(upd, x, best)
        sub = torch.where(upd, torch.full_like(sub, k), sub)
    return best, sub


def select_topk(cos, labels, topk):
    """(N, topk) int64: each row's topk non-target classes in the order (-cos, c), NaN after every number, -0 == +0."""
    c = np.asarray(torch.as_tensor(cos).double().cpu())
    N, C = c.shape
    nan = np.isnan(c).astype(np.int64)
    nan[np.arange(N), np.asarray(torch.as_tensor(labels).cpu())] = 2           # the target is never selected
    cols = np.broadcast_to(np.arange(C), (N, C))
    order = np.lexsort((cols, -np.where(np.isnan(c), 0.0, c) + 0.0, nan), axis=-1)
    return torch.from_numpy(np.ascontiguousarray(order[:, :topk]))


def _membership(top, N, C):
    inT = torch.zeros(N, C, dtype=torch.bool)
    if top is not None and top.shape[1] > 0:
        inT[torch.arange(N)[:, None], top] = True
    return inT


def _logits(cos, labels, inT, margin, scale, topk_margin):
    ar = torch.arange(cos.shape[0])
    logits = scale * cos.clone()
    logits[inT] = scale * psi(cos[inT], topk_margin)
    logits[ar, labels] = scale * A.phi(cos[ar, labels], margin)
    return logits


def _class_cosines(E, W, K, cos, sub):
    if cos is None or sub is None:
        e, _ = A._normalize(torch.as_tensor(E).double().cpu())
        w, _ = A._normalize(torch.as_tensor(W).double().cpu())
        c64, s64 = subcentre_max(e @ w.T, K)
        cos = c64 if cos is None else cos
        sub = s64 if sub is None else sub
    return torch.as_tensor(cos).double().cpu(), torch.as_tensor(sub).to(torch.int64).cpu()


def forward(E, W, labels, K, margin, scale, topk=0, topk_margin=0.0, cos=None, sub=None, top=None):
    """-> (loss, cos (N, C), lse (N,), sub (N, C), top (N, topk)) in fp64.  ``cos`` / ``sub`` / ``top`` given: those
    are used (the selection is taken from ``cos`` when ``top`` is not given)."""
    labels = torch.as_tensor(labels, dtype=torch.int64).cpu()
    cos, sub = _class_cosines(E, W, K, cos, sub)
    N, C = cos.shape
    top = select_topk(cos, labels, topk) if top is None else torch.as_tensor(top).to(torch.int64).cpu()
    logits = _logits(cos, labels, _membership(top, N, C), margin, scale, topk_margin)
    lse = torch.logsumexp(logits, dim=1)
    rows = lse - logits[torch.arange(N), labels]
    return rows.sum() / N, cos, lse, sub, top


def backward(E, W, labels, K, margin, scale, topk=0, topk_margin=0.0, grad_loss=1.0, cos=None, sub=None, top=None):
    """-> (gE (N, D), gW (C K, D)) in fp64, the explicit gradients; ``cos`` / ``sub`` / ``top`` as in ``forward``."""
    labels = torch.as_tensor(labels, dtype=torch.int64).cpu()
    e, ne = A._normalize(torch.as_tensor(E).double().cpu())
    w, nw = A._normalize(torch.as_tensor(W).double().cpu())
    cos, sub = _class_cosines(E, W, K, cos, sub)
    N, C = cos.shape
    top = select_topk(cos, labels, topk) if top is None else torch.as_tensor(top).to(torch.int64).cpu()
    inT = _membership(top, N, C)
    ar = torch.arange(N)
    p = torch.softmax(_logits(cos, labels, inT, margin, scale, topk_margin), dim=1)
    d = p.clone()
    d[ar, labels] -= 1.0
    d *= scale * grad_loss / N
    d[inT] *= dpsi(cos[inT], topk_margin)
    d[ar, labels] *= A.dphi(cos[ar, labels], margin)
    dx = torch.zeros(N, C * K, dtype=torch.float64)
    dx[ar[:, None], torch.arange(C)[None, :] * K + sub] = d            # the chosen sub-centre only
    ge, gw = dx @ w, dx.T @ e
    gE = (ge - e * (e * ge).sum(1, keepdim=True)) / ne
    gW = (gw - w * (w * gw).sum(1, keepdim=True)) / nw
    return gE, gW


def loss_autograd(E, W, labels, K, margin, scale, topk=0, topk_margin=0.0):
    """The textbook form (F.normalize, a max over the sub-centres, torch.topk on the detached class cosines,
    cross_entropy) for torch autograd, in E's dtype."""
    labels = torch.as_tensor(labels, dtype=torch.int64)
    g = F.normalize(E) @ F.normalize(W).T
    cos = g.reshape(E.shape[0], -1, K).max(dim=2).values
    onehot = F.one_hot(labels, cos.shape[1]).bool()
    inT = torch.zeros_like(onehot)
    if topk > 0:
        inT.scatter_(1, cos.detach().masked_fill(onehot, -math.inf).topk(topk, dim=1).indices, True)
    logits = scale * torch.where(onehot, A.phi(cos, margin), torch.where(inT, psi(cos, topk_margin), cos))
    return F.cross_entropy(logits, labels)
