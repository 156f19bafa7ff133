"""fp64 restatement of the generalised end-to-end (GE2E) loss — TEST INFRASTRUCTURE ONLY (the product never imports
this module).

Wan et al., "Generalized End-to-End Loss for Speaker Verification" (ICASSP 2018), with the centroids taken over the
normalised rows; no reference implementation exists, so parity with one is unpinned and this module defines the op.
For embeddings E (N, D), int64 labels y of any values, learnable scalars w, b and a method ``softmax`` or ``contrast``:

* e^_i = e_i / max(||e_i||, 1e-12) (F.normalize).  Speakers are the distinct labels in ascending order; speaker k has
  the members S_k (n_k of them) and is column k of every output.
* inclusive centroid c_k = (1/n_k) sum_{u in S_k} e^_u; exclusive centroid c_k^(-i) = (1/(n_k - 1)) sum_{u in S_k,
  u != i} e^_u for a row i of speaker k with n_k >= 2; c^ = c / max(||c||, 1e-12).
* cos_ik = e^_i . c^_k for k != y_i, cos_{i,y_i} = e^_i . c^_{y_i}^(-i) (a singleton speaker's row keeps the
  inclusive cosine there); S_ik = max(w, 1e-6) cos_ik + b.
* row i is valid when n_{y_i} >= 2 and the batch holds >= 2 speakers; V = the number of valid rows.
* softmax: L_i = logsumexp_k S_ik - S_{i,y_i};  contrast: L_i = 1 - sigmoid(S_{i,y_i}) + max_{k != y_i} sigmoid(S_ik),
  ties in the max to the lowest column.  loss = (1/V) sum over valid i of L_i.

``backward`` states the gradients explicitly (the three paths into e^: direct, through the inclusive centroids and
through the exclusive centroids, then the F.normalize Jacobian; gb exactly 0 for softmax); ``loss_autograd`` is the
textbook formula as torch ops for autograd.
"""
import numpy as np
import torch
import torch.nn.functional as F


def speakers(labels):
    """(col (N,) int64 tensor: each row's speaker index, P, n (P,) members per speaker)."""
    lab = torch.as_tensor(labels, dtype=torch.int64).cpu().reshape(-1)
    ids, col, n = torch.unique(lab, sorted=True, return_inverse=True, return_counts=True)
    return col, ids.numel(), n


def _normalize(X):
    n = X.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return X / n, n


def centroids(E, labels):
    """-> (e^ (N, D), ||e|| clamped (N, 1), c (P, D) inclusive, cx (N, D) exclusive (zero rows where n_k < 2), col, n,
    valid (N,) bool) in fp64."""
    col, P, n = speakers(labels)
    e, ne = _normalize(torch.as_tensor(E).double().cpu())
    onehot = F.one_hot(col, P).double()                    # (N, P)
    c = (onehot.T @ e) / n.double()[:, None]
    same = onehot @ onehot.T - torch.eye(col.numel(), dtype=torch.float64)   # same speaker, j != i
    nk = n[col]
    valid = (nk >= 2) & (P >= 2)
    cx = (same @ e) / torch.clamp(nk - 1, min=1).double()[:, None]
    cx[~valid] = 0.0
    return e, ne, c, cx, col, n, valid


def _scores(cos, w, b):
    return max(float(w), 1e-6) * cos + float(b)


def _argmax_other(S, col):
    """argmax over k != y of sigmoid(S), ties to the lowest column."""
    sig = torch.sigmoid(S).masked_fill(F.one_hot(col, S.shape[1]).bool(), -1.0)
    m = sig.max(dim=1, keepdim=True).values
    return torch.argmax((sig == m).to(torch.int8), dim=1)  # first maximal column


def forward(E, labels, w, b, method, cos=None):
    """-> (loss, cos (N, P), rec (N,)) in fp64; rec = logsumexp_k S_ik (softmax) or the contrast argmax column.
    ``cos`` given: the loss of those cosines."""
    e, _, c, cx, col, n, valid = centroids(E, labels)
    N = col.numel()
    ar = torch.arange(N)
    if cos is None:
        ch, _ = _normalize(c)
        cxh, _ = _normalize(cx)
        cos = e @ ch.T
        cos[ar[valid], col[valid]] = (e * cxh).sum(1)[valid]
    cos = torch.as_tensor(cos).double().cpu()
    S = _scores(cos, w, b)
    if method == "softmax":
        rec = torch.logsumexp(S, dim=1)
        rows = rec - S[ar, col]
    elif method == "contrast":
        rec = _argmax_other(S, col)
        sig = torch.sigmoid(S)
        rows = 1.0 - sig[ar, col] + sig[ar, rec]
    else:
        raise ValueError(method)
    V = int(valid.sum())
    return rows[valid].sum() / V, cos, rec


def score_grads(cos, labels, w, b, method, grad_loss=1.0, argmax=None):
    """dS (N, P) = grad_loss / V * dL_i / dS_ik on valid rows, 0 elsewhere, in fp64 at the given cosines (and contrast
    argmax)."""
    col, P, n = speakers(labels)
    cos = torch.as_tensor(cos).double().cpu()
    ar = torch.arange(col.numel())
    valid = (n[col] >= 2) & (P >= 2)
    S = _scores(cos, w, b)
    if method == "softmax":
        dS = torch.softmax(S, dim=1) - F.one_hot(col, P).double()
    else:
        k = _argmax_other(S, col) if argmax is None else torch.as_tensor(argmax).long().cpu()
        sig = torch.sigmoid(S)
        dS = torch.zeros_like(S)
        dS[ar, col] = -sig[ar, col] * (1 - sig[ar, col])
        dS[ar, k] = sig[ar, k] * (1 - sig[ar, k])
    dS = dS * (grad_loss / int(valid.sum()))
    dS[~valid] = 0.0
    return dS


def backward(E, labels, w, b, method, grad_loss=1.0, cos=None, argmax=None):
    """-> (gE (N, D), gw, gb) in fp64, the explicit gradients.  ``cos`` (and, for contrast, ``argmax``) given: the
    row derivatives are taken at those values (the engine's own, to isolate the backward's arithmetic)."""
    e, ne, c, cx, col, n, valid = centroids(E, labels)
    N, P = col.numel(), n.numel()
    ar = torch.arange(N)
    ch, cn = _normalize(c)
    cxh, cxn = _normalize(cx)
    if cos is None:
        cos = e @ ch.T
        cos[ar[valid], col[valid]] = (e * cxh).sum(1)[valid]
    cos = torch.as_tensor(cos).double().cpu()
    onehot = F.one_hot(col, P).bool()
    dS = score_grads(cos, labels, w, b, method, grad_loss, argmax)
    gw = float((dS * cos).sum()) if float(w) >= 1e-6 else 0.0
    gb = 0.0 if method == "softmax" else float(dS.sum())
    dcos = max(float(w), 1e-6) * dS
    t = dcos[ar, col]                                      # target column
    d = dcos.masked_fill(onehot, 0.0)
    ge = d @ ch + t[:, None] * cxh                         # direct
    gch = d.T @ e                                          # through the inclusive centroids
    gc = (gch - ch * (ch * gch).sum(1, keepdim=True)) / cn
    ge = ge + gc[col] / n[col].double()[:, None]
    v = t[:, None] * e                                     # through the exclusive centroids
    gcx = (v - cxh * (cxh * v).sum(1, keepdim=True)) / cxn
    term = gcx / torch.clamp(n[col] - 1, min=1).double()[:, None]
    term[~valid] = 0.0
    same = onehot.double() @ onehot.double().T - torch.eye(N, dtype=torch.float64)
    ge = ge + same @ term
    gE = (ge - e * (e * ge).sum(1, keepdim=True)) / ne
    return gE, gw, gb


def loss_autograd(E, labels, w, b, method):
    """The textbook formula (F.normalize, per-speaker means, clamp, logsumexp / sigmoid) for torch autograd in E's
    dtype; ``w`` and ``b`` are tensors."""
    col, P, n = speakers(labels)
    col, n = col.to(E.device), n.to(E.device)
    N = col.numel()
    e = F.normalize(E)
    onehot = F.one_hot(col, P).bool()
    sums = onehot.to(E.dtype).T @ e
    c = sums / n.to(E.dtype)[:, None]
    valid = (n[col] >= 2) & (P >= 2)
    cx = (sums[col] - e) / torch.clamp(n[col] - 1, min=1).to(E.dtype)[:, None]   # leave-one-out means
    cx = torch.where(valid[:, None], cx, c[col])
    cos = e @ F.normalize(c).T
    tgt = (e * F.normalize(cx)).sum(1)
    cos = torch.where(onehot & valid[:, None], tgt[:, None].expand(-1, P), cos)
    S = torch.clamp(w, min=1e-6) * cos + b
    ar = torch.arange(N, device=E.device)
    if method == "softmax":
        rows = torch.logsumexp(S, dim=1) - S[ar, col]
    else:
        sig = torch.sigmoid(S)
        rows = 1 - sig[ar, col] + sig.masked_fill(onehot, -1.0).max(dim=1).values
    return rows[valid].sum() / int(valid.sum())


def host_csr(labels):
    """(order, offsets, col) as numpy int64: the stable argsort of the labels, the speakers' bounds, each row's speaker."""
    lab = np.asarray(torch.as_tensor(labels).cpu().numpy()).reshape(-1)
    order = np.argsort(lab, kind="stable").astype(np.int64)
    ids, inv, counts = np.unique(lab, return_inverse=True, return_counts=True)
    return order, np.concatenate(([0], np.cumsum(counts))).astype(np.int64), inv.astype(np.int64).reshape(-1)
