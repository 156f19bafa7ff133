"""fp64 restatement of the supervised-contrastive loss — TEST INFRASTRUCTURE ONLY (the product never imports this module).

Khosla et al., "Supervised Contrastive Learning" (NeurIPS 2020), the L_out form; with labels equal to the utterance
index of each view it is the NT-Xent loss of SimCLR (Chen et al., ICML 2020).  No reference implementation exists, so
parity with one is unpinned and this module defines the op.  For embeddings E (N, D), int64 labels y of any values and
a temperature tau:

* e^_i = e_i / max(||e_i||, 1e-12) (F.normalize);  cos_ij = e^_i . e^_j;  s_ij = cos_ij / tau.
* P(i) = {j != i : y_j = y_i};  row i is valid iff P(i) is non-empty;  V = the number of valid rows.
* lse_i = log sum_{j != i} exp(s_ij);  l_i = lse_i - (1/|P(i)|) sum_{p in P(i)} s_ip;  loss = (1/V) sum_{valid i} l_i.

``backward`` states the gradient explicitly (dS = softmax minus the positives' 1/|P(i)| on valid rows, g^ = dC e^ +
dC^T e^, then the F.normalize Jacobian); ``loss_autograd`` is the textbook formula as torch ops for autograd.
"""
import torch
import torch.nn.functional as F


def _normalize(X):
    n = X.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return X / n, n


def masks(labels, device="cpu"):
    """(pos (N, N) bool: j != i with y_j = y_i, |P(i)| (N,) int64, valid (N,) bool) on ``device``."""
    y = torch.as_tensor(labels, dtype=torch.int64).to(device).reshape(-1)
    pos = (y[:, None] == y[None, :]) & ~torch.eye(y.numel(), dtype=torch.bool, device=device)
    cnt = pos.sum(1)
    return pos, cnt, cnt > 0


def valid_count(labels):
    """V by brute force: the rows with another row of the same label."""
    return int(masks(labels)[2].sum())


def forward(E, labels, tau, cos=None):
    """-> (loss, cos (N, N), lse (N,), row_loss (N,): l_i on valid rows, 0 elsewhere) in fp64, on the device of E (or
    of ``cos``).  ``cos`` given: the loss of those cosines (their diagonal is not read)."""
    if cos is None:
        e, _ = _normalize(torch.as_tensor(E).double())
        cos = e @ e.T
    cos = torch.as_tensor(cos).double()
    N, dev = cos.shape[0], cos.device
    pos, cnt, valid = masks(labels, dev)
    s = cos / float(tau)
    lse = torch.logsumexp(s.masked_fill(torch.eye(N, dtype=torch.bool, device=dev), float("-inf")), dim=1)
    rows = lse - torch.where(pos, s, torch.zeros_like(s)).sum(1) / cnt.clamp_min(1).double()
    rows = torch.where(valid, rows, torch.zeros_like(rows))
    return rows.sum() / int(valid.sum()), cos, lse, rows


def score_grads(cos, labels, tau, grad_loss=1.0):
    """dS (N, N) = grad_loss / V * (exp(s_ij - lse_i) - [j in P(i)] / |P(i)|) on valid rows, 0 on the diagonal and on
    invalid rows, in fp64 at the given cosines, on their device."""
    cos = torch.as_tensor(cos).double()
    N, dev = cos.shape[0], cos.device
    pos, cnt, valid = masks(labels, dev)
    eye = torch.eye(N, dtype=torch.bool, device=dev)
    p = torch.softmax((cos / float(tau)).masked_fill(eye, float("-inf")), dim=1)
    dS = (p - pos.double() / cnt.clamp_min(1).double()[:, None]) * (grad_loss / int(valid.sum()))
    dS[~valid] = 0.0
    return dS.masked_fill(eye, 0.0)


def backward(E, labels, tau, grad_loss=1.0, cos=None):
    """-> gE (N, D) in fp64, the explicit gradient.  ``cos`` given: the row derivatives are taken at those cosines (the
    engine's own, to isolate the backward's arithmetic; the engine's saved lse needs no pinning, since the probabilities
    are normalised by their own sum and lse cancels out of them).  Computed on E's device."""
    e, ne = _normalize(torch.as_tensor(E).double())
    cos = e @ e.T if cos is None else torch.as_tensor(cos).to(e.device)
    dC = score_grads(cos, labels, tau, grad_loss) / float(tau)
    g = dC @ e + dC.T @ e
    return (g - e * (e * g).sum(1, keepdim=True)) / ne


def loss_autograd(E, labels, tau):
    """The textbook formula (F.normalize, the Gram matrix, a masked logsumexp and the mean over the positives) for torch
    autograd in E's dtype and on E's device."""
    pos, cnt, valid = masks(labels, E.device)
    N = E.shape[0]
    e = F.normalize(E)
    s = (e @ e.T) / tau
    eye = torch.eye(N, dtype=torch.bool, device=E.device)
    lse = torch.logsumexp(s.masked_fill(eye, float("-inf")), dim=1)
    rows = lse - (s * pos.to(E.dtype)).sum(1) / cnt.clamp_min(1).to(E.dtype)
    return rows[valid].sum() / int(valid.sum())
