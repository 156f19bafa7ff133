"""fp64 restatement of speaker identification (enrolment centroids, exact top-k search, top-k accuracy) — TEST
INFRASTRUCTURE ONLY (the product never imports this module).

No reference implementation exists.  Definitions:

* x^ = x / max(||x||, 1e-12) in fp64 (F.normalize); the centroid of a class is the fp64 mean of its rows' x^;
* the search order of a row of values: larger first, ties to the lower column, -0 == +0, NaN below every number
  (-inf included); ``topk`` takes the k first columns under that order by np.lexsort((column, -value, isnan));
* top-k accuracy: a query is correct at k when one of its first k gallery rows carries its label.
"""
import numpy as np
import torch


def normalize(X):
    X = np.asarray(torch.as_tensor(X).detach().cpu().double().numpy())
    return X / np.maximum(np.linalg.norm(X, axis=1, keepdims=True), 1e-12)


def cosine_matrix(Q, G):
    """(M, Ng) fp64."""
    return normalize(Q) @ normalize(G).T


def centroids(X, labels):
    """(centroids (S, D) fp64, ids (S,)) with ids the sorted distinct labels."""
    Xn = normalize(X)
    lab = np.asarray(labels).reshape(-1)
    ids = np.unique(lab)
    return np.stack([Xn[lab == s].mean(axis=0) for s in ids]), ids


def topk(S, k):
    """(idx int64 (rows, k), val (rows, k)) of every row of S in the search order; val keeps S's dtype and bits."""
    S = np.asarray(S)
    idx = np.empty((S.shape[0], k), dtype=np.int64)
    cols = np.arange(S.shape[1])
    for r in range(S.shape[0]):
        v = S[r].astype(np.float64)
        nan = np.isnan(v)
        key = np.where(nan, 0.0, -v) + 0.0                    # -(-0) + 0 = +0
        idx[r] = np.lexsort((cols, key, nan))[:k]
    return idx, np.take_along_axis(S, idx, axis=1)


def topk_keys(S, k):
    """``topk`` restated for large torch matrices on any device: each entry's place in the search order as one unique
    int64 (its order-preserving key above its reversed column), so torch.topk is exact.  Columns < 2^21."""
    S = torch.as_tensor(S)
    bits = S.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    bits = torch.where(S == 0, torch.zeros_like(bits), bits)                      # -0 -> +0
    key = torch.where(bits >= 2 ** 31, (~bits) & 0xFFFFFFFF, bits | 2 ** 31)
    key = torch.where(torch.isnan(S), torch.zeros_like(key), key)                 # NaN below -inf (0x007fffff)
    cols = torch.arange(S.shape[1], device=S.device, dtype=torch.int64)
    idx = torch.topk(key * 2 ** 21 + (2 ** 21 - 1 - cols), k, dim=1).indices
    return idx, torch.gather(S, 1, idx)


def search(Q, G, k):
    """The accuracy target: topk of the fp64 cosines."""
    return topk(cosine_matrix(Q, G), k)


def accuracy(idx, gallery_labels, query_labels, ks=(1, 5)):
    """Brute force: one query and one k at a time."""
    idx = np.asarray(idx)
    gl, ql = np.asarray(gallery_labels).reshape(-1), np.asarray(query_labels).reshape(-1)
    out = {}
    for k in ks:
        hits = sum(any(gl[j] == ql[i] for j in idx[i, :k]) for i in range(idx.shape[0]))
        out[k] = hits / idx.shape[0]
    return out
