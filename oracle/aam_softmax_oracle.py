"""fp64 restatement of the additive angular margin softmax (ArcFace / AAM-softmax) — TEST INFRASTRUCTURE ONLY (the
product never imports this module).

The common ArcFace formulation with the non-"easy" margin; no reference implementation exists, so parity with one is
unpinned.  For embeddings E (N, D), class weights W (C, D), labels y, margin m and scale s:

* e^ = E / max(||E||, 1e-12), w^ likewise (F.normalize); cos = e^ w^T;
* target column: sin = sqrt(clamp(1 - cos^2, 0, 1)), phi = cos cos m - sin sin m if cos > cos(pi - m), else
  cos - sin(pi - m) m;  logits = s * (phi on the target column, cos elsewhere);
* loss = (1/N) sum_i (logsumexp_c logit_ic - logit_{i, y_i}).

``backward`` states the gradients explicitly (the softmax, the margin's chain rule with the finite value cos m at
sin = 0, the two products and the F.normalize Jacobians); ``loss_autograd`` is the textbook formula for torch autograd.
"""
import math

import torch
import torch.nn.functional as F


def _consts(margin):
    return math.cos(margin), math.sin(margin), math.cos(math.pi - margin), math.sin(math.pi - margin) * margin


def phi(c, margin):
    cos_m, sin_m, th, mm = _consts(margin)
    sn = torch.sqrt(torch.clamp(1.0 - c * c, 0.0, 1.0))
    return torch.where(c > th, c * cos_m - sn * sin_m, c - mm)


def dphi(c, margin):
    cos_m, sin_m, th, _ = _consts(margin)
    sn = torch.sqrt(torch.clamp(1.0 - c * c, 0.0, 1.0))
    safe = torch.where(sn > 0, sn, torch.ones_like(sn))
    return torch.where(c > th, torch.where(sn > 0, cos_m + sin_m * c / safe, torch.full_like(c, cos_m)),
                       torch.ones_like(c))


def _normalize(X):
    n = X.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return X / n, n


def _logits(cos, labels, margin, scale):
    ar = torch.arange(cos.shape[0])
    logits = scale * cos.clone()
    logits[ar, labels] = scale * phi(cos[ar, labels], margin)
    return logits


def forward(E, W, labels, margin, scale, cos=None):
    """-> (loss, cos (N, C), lse (N,)) in fp64.  ``cos`` given: the loss of those cosines."""
    labels = torch.as_tensor(labels, dtype=torch.int64).cpu()
    if cos is None:
        e, _ = _normalize(torch.as_tensor(E).double().cpu())
        w, _ = _normalize(torch.as_tensor(W).double().cpu())
        cos = e @ w.T
    cos = torch.as_tensor(cos).double().cpu()
    logits = _logits(cos, labels, margin, scale)
    lse = torch.logsumexp(logits, dim=1)
    rows = lse - logits[torch.arange(cos.shape[0]), labels]
    return rows.sum() / cos.shape[0], cos, lse


def backward(E, W, labels, margin, scale, grad_loss=1.0, cos=None):
    """-> (gE (N, D), gW (C, D)) in fp64, the explicit gradients.  ``cos`` given: the softmax and the margin's chain
    rule are taken at those cosines (the engine's own, to isolate the backward's arithmetic)."""
    labels = torch.as_tensor(labels, dtype=torch.int64).cpu()
    e, ne = _normalize(torch.as_tensor(E).double().cpu())
    w, nw = _normalize(torch.as_tensor(W).double().cpu())
    if cos is None:
        cos = e @ w.T
    cos = torch.as_tensor(cos).double().cpu()
    N = cos.shape[0]
    ar = torch.arange(N)
    p = torch.softmax(_logits(cos, labels, margin, scale), dim=1)
    d = p.clone()
    d[ar, labels] -= 1.0
    d *= scale * grad_loss / N
    d[ar, labels] *= dphi(cos[ar, labels], margin)
    ge, gw = d @ w, d.T @ e
    gE = (ge - e * (e * ge).sum(1, keepdim=True)) / ne
    gW = (gw - w * (w * gw).sum(1, keepdim=True)) / nw
    return gE, gW


def loss_autograd(E, W, labels, margin, scale):
    """The textbook formula (F.normalize, torch.where, cross_entropy) for torch autograd, in E's dtype."""
    labels = torch.as_tensor(labels, dtype=torch.int64)
    cos = F.normalize(E) @ F.normalize(W).T
    onehot = F.one_hot(labels, W.shape[0]).bool()
    logits = scale * torch.where(onehot, phi(cos, margin), cos)
    return F.cross_entropy(logits, labels)
