"""Oracle for spectral clustering with NME-SC speaker counting (tests only; numpy / scipy fp64, no GPU).

NME-SC (Park, Han, Kumar, Narayanan, "Auto-tuning spectral clustering for speaker diarization using normalized maximum
eigengap", IEEE SPL 2020) reads only the ranks of each row's similarities:

  1. ``ranks``: per row i, the columns j != i sorted by S[i][j] descending, ties to the lower column (the search order
     of dsk_topk_indices); rank[i][j] is j's 0-based position.  The diagonal is never read or ranked (a window is not
     its own neighbour).  Both triangles are read.  A non-finite off-diagonal value is a ValueError.
  2. ``affinity``: A_p[i][j] = ([rank[i][j] < p] + [rank[j][i] < p]) / 2 off the diagonal, 0 on it;
     L_p = diag(A_p 1) - A_p.
  3. ``spectral_cluster``: per p, the eigenvalues lambda_1 <= ... of L_p (dense ``eigh``); the count k_p is the first
     i in 1 .. m - 1 maximising lambda_{i+1} - lambda_i (or the given count), g_p = (lambda_{k+1} - lambda_k) /
     (lambda_N + 1e-10) and r_p = (p / N) / (g_p + 1e-10); p-hat is the first p of least r_p.
  4. ``kmeans``: on the rows of the eigenvectors of lambda_1 .. lambda_k of L_p-hat: maximin initialisation (the row
     farthest from the mean row, then the row farthest from its nearest chosen centre, ties to the lower row), Lloyd
     iterations (ties to the lower centre, an emptied centre keeps its place) until no assignment changes or
     ``iters``; labels numbered by each cluster's smallest member.  Row distances do not change under a rotation of the
     eigenbasis, so the partition does not depend on the basis ``eigh`` returns for a repeated eigenvalue.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np


def p_grid(N, p_max_frac=0.25, p_steps=30):
    """The default grid of pruning levels: unique integers of linspace(1, max(1, floor(p_max_frac (N - 1))), p_steps)."""
    top = max(1, int(np.floor(p_max_frac * (N - 1))))
    return np.unique(np.linspace(1, top, int(p_steps)).astype(np.int64))


def ranks(S):
    """(N, N) int64 ranks of step 1; the diagonal holds N - 1 (it is never read)."""
    S = np.asarray(S, np.float32)
    N = S.shape[0]
    off = ~np.eye(N, dtype=bool)
    if not np.isfinite(S[off]).all():
        raise ValueError("spectral: a non-finite off-diagonal similarity")
    key = S.astype(np.float64) + 0.0          # -0 ranks as +0
    key[~off] = -np.inf                      # the diagonal sorts last, at position N - 1
    order = np.argsort(-key, axis=1, kind="stable")   # descending value, equal values in ascending column
    R = np.empty((N, N), np.int64)
    np.put_along_axis(R, order, np.broadcast_to(np.arange(N), (N, N)), axis=1)
    return R


def affinity(R, p):
    """A_p of step 2 from the ranks R."""
    B = (R < p).astype(np.float64)
    np.fill_diagonal(B, 0.0)
    return 0.5 * (B + B.T)


def laplacian(R, p):
    A = affinity(R, p)
    return np.diag(A.sum(1)) - A


def count_and_ratio(lam, lam_max, p, N, num_speakers=None):
    """(k_p, r_p) of step 4 from lam = lambda_1 .. lambda_m."""
    if num_speakers is None:
        k = int(np.argmax(np.diff(lam))) + 1
    else:
        k = int(num_speakers)
    g = (lam[k] - lam[k - 1]) / (lam_max + 1e-10)
    return k, (p / N) / (g + 1e-10)


def kmeans(Y, k, iters=100):
    """Step 6 on the rows of Y (N, >= k) fp64 -> (N,) int32 labels numbered by each cluster's smallest member."""
    Y = np.asarray(Y, np.float64)[:, :k]
    N = Y.shape[0]
    if k <= 1:
        return np.zeros(N, np.int32)

    def sqdist(c):
        return ((Y - c) ** 2).sum(1)

    first = int(np.argmax(sqdist(Y.mean(0))))
    idx = [first]
    near = sqdist(Y[first])
    for _ in range(1, k):
        j = int(np.argmax(near))
        idx.append(j)
        near = np.minimum(near, sqdist(Y[j]))
    C = Y[idx].copy()
    lab = None
    for _ in range(int(iters)):
        D = np.stack([sqdist(C[c]) for c in range(k)], 1)
        new = np.argmin(D, 1)
        if lab is not None and np.array_equal(new, lab):
            break
        lab = new
        for c in range(k):
            mem = lab == c
            if mem.any():
                C[c] = Y[mem].mean(0)
    return renumber(lab)


def renumber(lab):
    """Labels numbered from 0 in the order of each cluster's smallest member."""
    lab = np.asarray(lab).reshape(-1)
    _, first, inv = np.unique(lab, return_index=True, return_inverse=True)
    return np.argsort(np.argsort(first))[inv].astype(np.int32)


class Result(NamedTuple):
    labels: np.ndarray      # (N,) int32
    k: int
    p_index: int
    eigenvalues: np.ndarray  # (n_p, m) fp64
    lambda_max: np.ndarray   # (n_p,)
    ratio: np.ndarray        # (n_p,)
    ks: np.ndarray           # (n_p,) the count at every p
    embedding: np.ndarray    # (N, k) eigenvectors of L_p-hat


def spectral_cluster(S, p_values, max_speakers=8, num_speakers=None, kmeans_iters=100, subset=None):
    """Steps 1-6 on S (N, N).  ``subset``: compute only these indices into p_values (eigenvalue checks at sizes where
    a dense eigh per grid point is slow); the selection then runs over them alone."""
    from scipy.linalg import eigh

    S = np.asarray(S, np.float32)
    N = S.shape[0]
    pv = np.asarray(p_values, np.int64)
    m = min(max_speakers + 1, N) if num_speakers is None else int(num_speakers) + 1
    R = ranks(S)
    which = range(pv.size) if subset is None else subset
    lam = np.full((pv.size, m), np.nan)
    lmax = np.full(pv.size, np.nan)
    ratio = np.full(pv.size, np.inf)
    ks = np.zeros(pv.size, np.int64)
    for t in which:
        L = laplacian(R, int(pv[t]))
        w = eigh(L, eigvals_only=True)
        lam[t] = w[:m]
        lmax[t] = w[-1]
        ks[t], ratio[t] = count_and_ratio(w[:m], w[-1], int(pv[t]), N, num_speakers)
    t = int(np.argmin(ratio))
    k = int(ks[t])
    _, V = eigh(laplacian(R, int(pv[t])), subset_by_index=[0, k - 1])
    return Result(kmeans(V, k, kmeans_iters), k, t, lam, lmax, ratio, ks, V)
