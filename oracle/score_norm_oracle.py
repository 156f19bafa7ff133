"""fp64 restatement of cosine scoring with adaptive score normalisation (AS-norm) and of the exact EER / minDCF —
TEST INFRASTRUCTURE ONLY (the product never imports this module).  The torch functions compute on their inputs'
device (fp64 on a GPU is still fp64).

No reference implementation exists (the reference scores Euclidean distances on a fixed threshold grid,
eval_metrics.py:5-50).  Definitions:

* x^ = x / max(||x||, 1e-12) (F.normalize); cos = a^ b^T;
* cohort statistics of a row: the k largest values (torch.topk; which tied copies are taken does not change the
  values), their mean and unbiased standard deviation; a row with a NaN gives NaN;
* raw trial score s = x^_e . x^_t; AS-norm 0.5 ((s - mu_e) / sigma_e + (s - mu_t) / sigma_t); an index outside
  [0, U) gives NaN;
* EER / minDCF by brute force: one mask per operating point (the sorted distinct scores plus +inf),
  P_miss(t) = #{target, s < t} / n_tar, P_fa(t) = #{non-target, s >= t} / n_non; the EER interpolates
  P_miss - P_fa linearly from the point before the first one where P_miss >= P_fa and averages the two rates there;
  minDCF = min_t (c_miss P_miss p + c_fa P_fa (1 - p)) / min(c_miss p, c_fa (1 - p)).
"""
import numpy as np
import torch


def normalize(X):
    X = torch.as_tensor(X).detach().double()
    return X / X.norm(dim=1, keepdim=True).clamp_min(1e-12)


def cosine_matrix(A, B):
    """(M, Nc) fp64."""
    return normalize(A) @ normalize(B).T


def topk_mean_std(S, k):
    """(mean, std) (rows,) fp64 of the k largest values of every row of S."""
    S = torch.as_tensor(S).detach().double()
    top = torch.topk(S, k, dim=1).values
    mean, std = top.mean(dim=1), top.std(dim=1, unbiased=True)
    nan = torch.isnan(S).any(dim=1)
    mean[nan] = float("nan")
    std[nan] = float("nan")
    return mean, std


def cohort_stats(E, cohort, k):
    return topk_mean_std(cosine_matrix(E, cohort), k)


def score_trials(X, trials, mean=None, std=None):
    """(raw, normed) (T,) fp64; ``mean`` / ``std`` are taken as given (e.g. the engine's fp32 statistics)."""
    Xn = normalize(X)
    U = Xn.shape[0]
    tr = torch.as_tensor(trials).to(device=Xn.device, dtype=torch.int64)
    ok = ((tr >= 0) & (tr < U)).all(dim=1)
    e, t = tr[:, 0].clamp(0, U - 1), tr[:, 1].clamp(0, U - 1)
    raw = (Xn[e] * Xn[t]).sum(dim=1)
    raw[~ok] = float("nan")
    if mean is None:
        return raw, None
    mu = torch.as_tensor(mean).detach().to(device=Xn.device, dtype=torch.float64)
    sd = torch.as_tensor(std).detach().to(device=Xn.device, dtype=torch.float64)
    normed = 0.5 * ((raw - mu[e]) / sd[e] + (raw - mu[t]) / sd[t])
    normed[~ok] = float("nan")
    return raw, normed


def eer_min_dcf(scores, targets, p_target=0.01, c_miss=1.0, c_fa=1.0):
    """Brute force, O(n * points)."""
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    y = np.asarray(targets).astype(bool).reshape(-1)
    n_tar, n_non = int(y.sum()), int((~y).sum())
    points = np.concatenate((np.unique(s), [np.inf]))
    below = s[None, :] < points[:, None]
    p_miss = (below & y[None, :]).sum(1) / n_tar
    p_fa = (~below & ~y[None, :]).sum(1) / n_non
    diff = p_miss - p_fa
    i = int(np.flatnonzero(diff >= 0)[0])
    w = -diff[i - 1] / (diff[i] - diff[i - 1]) if diff[i] != diff[i - 1] else 0.0
    eer = (p_miss[i - 1] + w * (p_miss[i] - p_miss[i - 1]) + p_fa[i - 1] + w * (p_fa[i] - p_fa[i - 1])) / 2
    dcf = (c_miss * p_miss * p_target + c_fa * p_fa * (1 - p_target)) / min(c_miss * p_target, c_fa * (1 - p_target))
    return float(eer), float(dcf.min())
