"""Verification loop of the reference's ``test()`` (reference train_triplet.py:330-366) on the H100 engine, plus
the derived equal error rate (SURVEY §8f rank 1: the reference sweeps thresholds for best accuracy,
reference eval_metrics.py:5-50, and has no EER function).

Distances come from the CUDA kernels (eval forward + PairwiseDistance).  ``evaluate`` is the drop-in for
``eval_metrics.evaluate`` (called at train_triplet.py:361): its two threshold sweeps (3 000 + 30 000 thresholds, one
numpy pass over the distance array each in the reference) are ONE counting kernel launch each (``dsk_threshold_counts``,
exact numpy comparison semantics); the handful of scalar operations that follow (argmax, the interpolation of the FAR
curve) stay on the host as in the reference.  ``sweep`` (accuracy + the derived EER) keeps its numpy form for host arrays.

For embeddings scored by cosine similarity (higher = same speaker, e.g. trained with ``AAMSoftmaxLoss``):
``cosine_matrix``, ``cohort_stats`` and ``score_trials`` (AS-norm against an impostor cohort) run on the GPU, and
``eer_min_dcf`` computes the exact EER and minDCF over every distinct score on the host.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib as L
from . import engine
from .model import PairwiseDistance


@torch.no_grad()
def verification_distances(model, data_a: torch.Tensor, data_p: torch.Tensor) -> torch.Tensor:
    """data_* (P, crops, T, 64): `crops` random crops per file (train_triplet.py:339-340 resizes them to
    (crops*P, 1, T, 64)); returns the per-pair distance averaged over crops ("length normalization", :348-350)."""
    if model.training:
        raise RuntimeError("verification runs in eval mode (train_triplet.py:332)")
    P, crops, T, F = data_a.shape
    a = data_a.reshape(P * crops, 1, T, F)
    p = data_p.reshape(P * crops, 1, T, F)
    out_a, out_p = model(a), model(p)
    d = PairwiseDistance(2).forward(out_a, out_p)
    return d.reshape(P, crops).mean(dim=1)


def sweep(distances, labels, thresholds=None):
    """(best-threshold accuracy, EER).  Accuracy follows eval_metrics.py:16-50 (thresholds 0..30 step 0.01, first
    argmax); EER is the FAR == FRR crossing of the same sweep."""
    d = np.asarray(distances, dtype=np.float64)
    same = np.asarray(labels).astype(bool)
    if thresholds is None:
        thresholds = np.arange(0, 30, 0.01)
    below = d[None, :] < thresholds[:, None]
    tp = (below & same[None, :]).sum(1)
    fp = (below & ~same[None, :]).sum(1)
    tn = (~below & ~same[None, :]).sum(1)
    fn = (~below & same[None, :]).sum(1)
    acc = (tp + tn) / d.size
    far = fp / max(1, int((~same).sum()))
    frr = fn / max(1, int(same.sum()))
    diff = far - frr
    i = int(np.argmax(diff >= 0))
    if i == 0:
        eer = float((far[0] + frr[0]) / 2)
    else:
        w = -diff[i - 1] / (diff[i] - diff[i - 1]) if diff[i] != diff[i - 1] else 0.0
        eer = float((far[i - 1] + w * (far[i] - far[i - 1]) + frr[i - 1] + w * (frr[i] - frr[i - 1])) / 2)
    return float(acc[int(np.argmax(acc))]), eer


def threshold_counts(distances: torch.Tensor, labels: torch.Tensor, thresholds):
    """tp[t] = #{same & d < t}, fp[t] = #{different & d < t} for every threshold, on the GPU (exact: fp32 distances are
    compared as doubles with the double thresholds, like np.less in eval_metrics.py:41,76).  Returns int64 numpy arrays."""
    if not distances.is_cuda:
        raise RuntimeError("threshold_counts needs CUDA tensors; there is no CPU fallback")
    d = distances.detach().float().contiguous().reshape(-1)
    same = labels.to(device=d.device).reshape(-1).ne(0).to(torch.uint8).contiguous()
    if same.numel() != d.numel():
        raise RuntimeError("distances and labels differ in length")
    th = torch.as_tensor(np.asarray(thresholds, dtype=np.float64), device=d.device)
    tp = torch.empty(th.numel(), dtype=torch.int32, device=d.device)
    fp = torch.empty_like(tp)
    with torch.cuda.device(d.device):
        L.check(L.load().dsk_threshold_counts(d.data_ptr(), same.data_ptr(), d.numel(), th.data_ptr(), th.numel(),
                                              tp.data_ptr(), fp.data_ptr(), L.cur_stream()), "dsk_threshold_counts")
    return tp.cpu().numpy().astype(np.int64), fp.cpu().numpy().astype(np.int64)


def evaluate(distances: torch.Tensor, labels: torch.Tensor, far_target: float = 1e-3):
    """Drop-in for ``eval_metrics.evaluate(distances, labels)`` (reference eval_metrics.py:5-13) on CUDA tensors:
    returns (tpr, fpr, accuracy, val, far) — tpr / fpr / accuracy at the best-accuracy threshold of arange(0, 30, 0.01)
    (first argmax, :16-37), and VAL / FAR at the threshold where the FAR curve over arange(0, 30, 0.001) crosses
    ``far_target`` (:53-88).

    The reference interpolates the FAR curve with ``scipy.interpolate.interp1d(far_train, thresholds, 'slinear')``,
    which raises on the duplicate x values every real FAR curve has under current scipy (the reference's own
    ``evaluate`` fails here; tools/make_golden.py records that); the threshold is taken as the linear interpolation
    over the strictly increasing points of the curve (the first threshold of each FAR level), which is what 'slinear'
    computes on a duplicate-free curve."""
    n = distances.numel()
    same_np = labels.detach().cpu().numpy().reshape(-1).astype(bool)
    n_same, n_diff = int(same_np.sum()), int((~same_np).sum())
    # ---- calculate_roc ----
    th1 = np.arange(0, 30, 0.01)
    tp, fp = threshold_counts(distances, labels, th1)
    fn, tn = n_same - tp, n_diff - fp
    acc = (tp + tn) / float(n)
    best = int(np.argmax(acc))
    tpr = 0.0 if n_same == 0 else float(tp[best]) / float(n_same)
    fpr = 0.0 if n_diff == 0 else float(fp[best]) / float(n_diff)
    # ---- calculate_val ----
    th2 = np.arange(0, 30, 0.001)
    tp2, fp2 = threshold_counts(distances, labels, th2)
    far_train = np.zeros(len(th2)) if n_same == 0 else fp2 / float(max(n_diff, 1))
    threshold = val_threshold(far_train, th2, far_target)
    tpv, fpv = threshold_counts(distances, labels, np.array([threshold], dtype=np.float64))
    if n_same == 0:
        val, far = 0.0, 0.0
    else:
        val, far = float(tpv[0]) / float(n_same), float(fpv[0]) / float(max(n_diff, 1))
    return tpr, fpr, float(acc[best]), val, far


def val_threshold(far_train, thresholds, far_target):
    """eval_metrics.py:65-69: the threshold at which FAR == far_target (0.0 if the curve never reaches it)."""
    if np.max(far_train) < far_target:
        return 0.0
    keep = np.concatenate(([True], np.diff(far_train) > 0))       # first threshold of every FAR level
    x, y = far_train[keep], thresholds[keep]
    if far_target <= x[0]:
        return float(y[0])
    return float(np.interp(far_target, x, y))


# ---------------------------------------------------------------------------------------------------
# Cosine scoring with adaptive score normalisation (AS-norm) and exact EER / minDCF: the usual evaluation of embeddings
# trained with a cosine classifier (AAMSoftmaxLoss), where a higher score means the same speaker.
# ---------------------------------------------------------------------------------------------------
def cosine_matrix(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """(M, Nc) fp32 cosines between the rows of A (M, D) and B (Nc, D) (CUDA tensors; D a multiple of 64)."""
    return engine.cosine_matrix(A, B)


def cohort_stats(emb: torch.Tensor, cohort: torch.Tensor, topk: int = 300):
    """(mean, std), (M,) fp32 on the device: mean and standard deviation (divisor topk - 1) of the ``topk`` largest
    cosines of each row of ``emb`` (M, D) against the impostor cohort (Nc, D); 2 <= topk <= Nc (topk = Nc: S-norm)."""
    return engine.cohort_stats(emb, cohort, topk)


def score_trials(emb: torch.Tensor, trials, cohort: torch.Tensor = None, topk: int = 300):
    """(raw, normed) (T,) fp32 scores of trials (T, 2) of row indices (enrolment, test) into the embedding table ``emb``
    (U, D): raw = the cosine, normed = its AS-norm 0.5 ((s - mu_e) / sigma_e + (s - mu_t) / sigma_t) with every row's
    statistics against ``cohort`` (``cohort_stats``); normed is None without a cohort.  An index outside [0, U) gives
    NaN."""
    mean = std = None
    if cohort is not None:
        mean, std = engine.cohort_stats(emb, cohort, topk)
    return engine.score_trials(emb, trials, mean, std)


def eer_min_dcf(scores, targets, p_target: float = 0.01, c_miss: float = 1.0, c_fa: float = 1.0):
    """(EER, minDCF) of ``scores`` (higher = same speaker) with boolean ``targets``, exact over every distinct score.

    The operating points are the sorted distinct scores plus +inf; P_miss(t) = #{target, s < t} / n_tar and
    P_fa(t) = #{non-target, s >= t} / n_non.  EER interpolates P_miss - P_fa as ``sweep`` does: at the first point where
    P_miss >= P_fa, linearly from the previous point, and averages the two interpolated rates.  minDCF is the minimum over
    the same points of (c_miss P_miss p + c_fa P_fa (1 - p)) / min(c_miss p, c_fa (1 - p)).  Host numpy, one sort.
    Raises ValueError without target or non-target trials, or for a score that is not finite."""
    s = (scores.detach().cpu().double().numpy() if isinstance(scores, torch.Tensor)
         else np.asarray(scores, dtype=np.float64)).reshape(-1)
    y = (targets.detach().cpu().numpy() if isinstance(targets, torch.Tensor) else np.asarray(targets)).reshape(-1)
    y = y.astype(bool)
    if s.shape != y.shape:
        raise ValueError(f"scores and targets differ in length ({s.size} and {y.size})")
    if not np.isfinite(s).all():
        raise ValueError("every score must be finite")
    n_tar = int(y.sum())
    n_non = y.size - n_tar
    if n_tar == 0 or n_non == 0:
        raise ValueError(f"need target and non-target trials (got {n_tar} and {n_non})")
    if not (0.0 < p_target < 1.0) or not (c_miss > 0.0) or not (c_fa > 0.0):
        raise ValueError("need 0 < p_target < 1, c_miss > 0 and c_fa > 0")
    order = np.argsort(s, kind="stable")
    s, y = s[order], y[order]
    cum_tar = np.concatenate(([0], np.cumsum(y)))                # targets among the i lowest scores
    first = np.flatnonzero(np.concatenate(([True], s[1:] != s[:-1])))
    idx = np.concatenate((first, [s.size]))                      # scores below each operating point; +inf last
    p_miss = cum_tar[idx] / n_tar
    p_fa = (n_non - (idx - cum_tar[idx])) / n_non
    diff = p_miss - p_fa                                         # -1 at the lowest score, +1 at +inf
    i = int(np.argmax(diff >= 0))
    w = -diff[i - 1] / (diff[i] - diff[i - 1]) if diff[i] != diff[i - 1] else 0.0
    eer = float((p_miss[i - 1] + w * (p_miss[i] - p_miss[i - 1]) + p_fa[i - 1] + w * (p_fa[i] - p_fa[i - 1])) / 2)
    dcf = (c_miss * p_miss * p_target + c_fa * p_fa * (1.0 - p_target)) / min(c_miss * p_target, c_fa * (1.0 - p_target))
    return eer, float(dcf.min())
