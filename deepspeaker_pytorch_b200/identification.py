"""Speaker identification: which enrolled speaker is this utterance?  (The Deep Speaker paper reports identification
accuracy beside EER; the reference has no identification code.)

``enroll`` averages each speaker's normalised utterance embeddings into one centroid, ``search`` finds the k gallery
rows of largest cosine for every query, exactly and with indices, against a gallery of any size, and ``accuracy``
scores the result against labels.  The gallery may be the centroids or the utterances themselves.

The search order is total: higher cosine first, ties to the lower gallery row, and NaN last, so a corrupt gallery
embedding never becomes every query's top-1.  The returned score is exactly the fp32 cosine ``verification.
cosine_matrix`` gives for the pair, and a query's result does not depend on the other queries of the call.
"""
from __future__ import annotations

import numpy as np
import torch

from . import engine


def speaker_csr(speakers):
    """(order, offsets, speaker_ids) on the host: the rows of each distinct label, in ascending label order and, within
    a label, in row order (a stable argsort); offsets (S + 1,) delimit them.  No segment is empty."""
    lab = np.asarray(torch.as_tensor(speakers).cpu().numpy() if isinstance(speakers, torch.Tensor) else speakers)
    lab = lab.reshape(-1)
    if lab.size == 0:
        raise ValueError("enroll: no utterances")
    order = np.argsort(lab, kind="stable").astype(np.int64)
    ids, counts = np.unique(lab, return_counts=True)
    offsets = np.concatenate(([0], np.cumsum(counts))).astype(np.int64)
    return order, offsets, ids


def enroll(emb, speakers):
    """(centroids (S, D) fp32 on emb's device, speaker_ids np.ndarray (S,)): centroid s is the mean of the normalised
    embeddings of the utterances labelled speaker_ids[s] (speaker_ids ascending), summed in fp64 in utterance order.
    ``emb`` (U, D) is a CUDA tensor, ``speakers`` (U,) CPU labels (a numpy array, list or CPU tensor)."""
    if not isinstance(emb, torch.Tensor) or not emb.is_cuda:
        raise RuntimeError("enroll needs a CUDA embedding tensor; there is no CPU fallback")
    if isinstance(speakers, torch.Tensor) and speakers.is_cuda:
        raise RuntimeError("enroll: speakers must be CPU labels (the enrolment lists are built on the host)")
    order, offsets, ids = speaker_csr(speakers)
    if order.size != emb.shape[0]:
        raise ValueError(f"enroll: {order.size} labels for {emb.shape[0]} embeddings")
    cent = engine.class_centroids(emb, torch.from_numpy(order).to(emb.device), torch.from_numpy(offsets).to(emb.device))
    return cent, ids


def search(queries, gallery, k):
    """(idx int64 (M, k), score fp32 (M, k)) on the device: the k gallery rows of largest cosine for every query, best
    first.  ``queries`` (M, D) and ``gallery`` (Ng, D) are CUDA tensors, D a multiple of 64, 1 <= k <= 1024, Ng >= k."""
    return engine.cosine_topk(queries, gallery, k)


def accuracy(idx, gallery_labels, query_labels, ks=(1, 5)):
    """{k: fraction of queries whose label is among the labels of their first k gallery rows} for every k in ``ks``,
    in host numpy.  ``idx`` (M, >= max(ks)) as ``search`` returns it; ``gallery_labels`` (Ng,) label every gallery row
    (the ``speaker_ids`` of ``enroll`` for a centroid gallery, the utterances' labels for an utterance gallery)."""
    idx = np.asarray(idx.cpu().numpy() if isinstance(idx, torch.Tensor) else idx)
    gl = np.asarray(gallery_labels.cpu().numpy() if isinstance(gallery_labels, torch.Tensor) else gallery_labels)
    ql = np.asarray(query_labels.cpu().numpy() if isinstance(query_labels, torch.Tensor) else query_labels)
    gl, ql = gl.reshape(-1), ql.reshape(-1)
    if idx.ndim != 2 or idx.shape[0] != ql.size or idx.shape[0] == 0:
        raise ValueError(f"accuracy: idx {idx.shape} does not match {ql.size} query labels")
    ks = tuple(int(k) for k in ks)
    if not ks or min(ks) < 1 or max(ks) > idx.shape[1]:
        raise ValueError(f"accuracy: every k must lie in [1, {idx.shape[1]}], got {ks}")
    if idx.size and (idx.min() < 0 or idx.max() >= gl.size):
        raise ValueError("accuracy: an index lies outside the gallery")
    hit = gl[idx] == ql[:, None]
    first = np.where(hit.any(axis=1), hit.argmax(axis=1), idx.shape[1])   # rank of the first correct row
    return {k: float((first < k).mean()) for k in ks}
