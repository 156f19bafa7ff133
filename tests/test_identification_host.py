"""Speaker identification without a GPU: the oracle's search order against a pure-Python brute force, top-k accuracy
and the host enrolment lists against brute force, and argument rejection by the C ABI."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import identification as I
from oracle import identification_oracle as O


def _ranks_above(a, b):
    """The search order on (value, column) pairs, written out case by case: True when a comes first."""
    (va, ca), (vb, cb) = a, b
    na, nb = math.isnan(va), math.isnan(vb)
    if na != nb:
        return nb
    if not na and va != vb:                             # -0.0 == 0.0 here
        return va > vb
    return ca < cb


def _brute_topk(row, k):
    pairs = [(float(v), c) for c, v in enumerate(row)]
    cmp = lambda a, b: -1 if _ranks_above(a, b) else (1 if _ranks_above(b, a) else 0)
    return [c for _, c in sorted(pairs, key=functools.cmp_to_key(cmp))[:k]]


def _adversarial_rows(cols, seed):
    rng = np.random.default_rng(seed)
    rows = [np.round(rng.standard_normal(cols) * 4) / 4,                                   # quantised ties
            np.full(cols, 0.5),                                                               # all equal
            np.where(rng.random(cols) < 0.5, -0.0, 0.0),                                      # signed zeros
            rng.choice([np.inf, -np.inf, np.nan, 1.0, -1.0, 0.0, -0.0], cols),                # specials
            np.full(cols, np.nan)]
    r = rng.standard_normal(cols)
    r[cols // 2:] = r[: cols - cols // 2]                                                     # duplicated columns
    rows.append(r)
    return np.stack(rows).astype(np.float32)


@pytest.mark.parametrize("cols", [1, 2, 7, 64, 300])
def test_oracle_order_matches_brute_force(cols):
    S = _adversarial_rows(cols, seed=cols)
    for k in sorted({1, min(3, cols), cols}):
        idx, val = O.topk(S, k)
        for r in range(S.shape[0]):
            assert idx[r].tolist() == _brute_topk(S[r], k), (cols, k, r)
        assert np.array_equal(val.view(np.int32), np.take_along_axis(S, idx, 1).view(np.int32))


def test_oracle_key_form_matches_lexsort():
    S = np.concatenate([_adversarial_rows(300, seed=s) for s in range(3)])
    for k in (1, 10, 300):
        i1, v1 = O.topk(S, k)
        i2, v2 = O.topk_keys(torch.from_numpy(S), k)
        assert np.array_equal(i1, i2.numpy()) and np.array_equal(v1.view(np.int32), v2.numpy().view(np.int32))


def test_oracle_nan_ranks_below_minus_inf_and_zeros_tie():
    row = np.array([np.nan, -np.inf, -0.0, 0.0, np.inf, -0.0], dtype=np.float32)
    idx, _ = O.topk(row[None], 6)
    assert idx[0].tolist() == [4, 2, 3, 5, 1, 0]


def _brute_accuracy(idx, gl, ql, ks):
    out = {}
    for k in ks:
        out[k] = np.mean([ql[i] in {gl[j] for j in idx[i, :k]} for i in range(idx.shape[0])])
    return out


@pytest.mark.parametrize("gallery", ["centroids", "utterances"])
def test_accuracy_matches_brute_force(gallery):
    rng = np.random.default_rng(3)
    M, Ng, k = 500, 60 if gallery == "centroids" else 600, 10
    gl = np.arange(Ng) if gallery == "centroids" else rng.integers(0, 40, Ng)
    ql = rng.integers(0, 40, M)
    idx = np.stack([rng.permutation(Ng)[:k] for _ in range(M)])
    idx[:50, 0] = [int(np.flatnonzero(gl == q)[0]) if (gl == q).any() else 0 for q in ql[:50]]   # some top-1 hits
    ks = (1, 5, 10)
    got = I.accuracy(torch.from_numpy(idx), gl, torch.from_numpy(ql), ks)
    assert got == _brute_accuracy(idx, gl, ql, ks) == O.accuracy(idx, gl, ql, ks)
    assert got[1] >= 0.1 and got[1] <= got[5] <= got[10]


def test_accuracy_rejects_bad_arguments():
    idx = np.zeros((4, 3), dtype=np.int64)
    for bad in (lambda: I.accuracy(idx, np.arange(5), np.arange(4), ks=(4,)),
                lambda: I.accuracy(idx, np.arange(5), np.arange(4), ks=(0,)),
                lambda: I.accuracy(idx, np.arange(5), np.arange(3)),
                lambda: I.accuracy(idx + 5, np.arange(5), np.arange(4), ks=(1,))):
        with pytest.raises(ValueError):
            bad()


def test_enrolment_lists_match_brute_force():
    rng = np.random.default_rng(5)
    labels = rng.choice(np.array([17, 3, 99, 42, -1, 8]), 1000)
    order, offsets, ids = I.speaker_csr(torch.from_numpy(labels))
    assert ids.tolist() == sorted(set(labels.tolist()))
    assert offsets[0] == 0 and offsets[-1] == labels.size and (np.diff(offsets) > 0).all()
    for s, sid in enumerate(ids):
        assert order[offsets[s]:offsets[s + 1]].tolist() == np.flatnonzero(labels == sid).tolist()
    names = np.array([f"spk{v}" for v in labels])
    order2, offsets2, ids2 = I.speaker_csr(names.tolist())                            # string labels, a list
    assert ids2.tolist() == sorted(set(names.tolist()))
    for s, sid in enumerate(ids2):
        assert order2[offsets2[s]:offsets2[s + 1]].tolist() == np.flatnonzero(names == sid).tolist()


P = ctypes.c_void_p(256)                                 # never dereferenced: the arguments are checked first


def _rejected(rc, what):
    assert rc == -1, (what, rc)
    assert b"bad arguments" in L.load().dsk_last_error(), what


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    # dsk_topk_indices(S, rows, cols, ld, k, idx, val, stream)
    for what, a in {"null S": (None, 4, 100, 100, 5, P, P), "null idx": (P, 4, 100, 100, 5, None, P),
                    "null val": (P, 4, 100, 100, 5, P, None), "rows = 0": (P, 0, 100, 100, 5, P, P),
                    "cols = 0": (P, 4, 0, 0, 1, P, P), "cols > 65536": (P, 4, 65537, 65537, 5, P, P),
                    "ld < cols": (P, 4, 100, 99, 5, P, P), "k = 0": (P, 4, 100, 100, 0, P, P),
                    "k > cols": (P, 4, 100, 100, 101, P, P), "k > 1024": (P, 4, 2000, 2000, 1025, P, P)}.items():
        _rejected(lib.dsk_topk_indices(*a, None), "topk_indices " + what)
    # dsk_cosine_topk(h, Q, M, G, Ng, D, k, idx, val, stream)
    for what, a in {"null Q": (None, 10, P, 100, 128, 5, P, P), "null G": (P, 10, None, 100, 128, 5, P, P),
                    "null idx": (P, 10, P, 100, 128, 5, None, P), "null val": (P, 10, P, 100, 128, 5, P, None),
                    "M = 0": (P, 0, P, 100, 128, 5, P, P), "k = 0": (P, 10, P, 100, 128, 0, P, P),
                    "k > 1024": (P, 10, P, 5000, 128, 1025, P, P), "Ng < k": (P, 10, P, 4, 128, 5, P, P),
                    "D % 64": (P, 10, P, 100, 96, 5, P, P), "D = 0": (P, 10, P, 100, 0, 5, P, P)}.items():
        _rejected(lib.dsk_cosine_topk(P, *a, None), "cosine_topk " + what)
    # dsk_class_centroids(X, U, D, order, offsets, S, out, stream)
    for what, a in {"null X": (None, 10, 64, P, P, 3, P), "null order": (P, 10, 64, None, P, 3, P),
                    "null offsets": (P, 10, 64, P, None, 3, P), "null out": (P, 10, 64, P, P, 3, None),
                    "U = 0": (P, 0, 64, P, P, 3, P), "D = 0": (P, 10, 0, P, P, 3, P),
                    "S = 0": (P, 10, 64, P, P, 0, P)}.items():
        _rejected(lib.dsk_class_centroids(*a, None), "class_centroids " + what)


def test_gpu_entry_points_raise_on_cpu_tensors():
    Q, G = torch.randn(8, 64), torch.randn(10, 64)
    with pytest.raises(RuntimeError):
        I.search(Q, G, 3)
    with pytest.raises(RuntimeError):
        I.enroll(Q, np.arange(8) % 3)
    from deepspeaker_pytorch_b200 import engine as EN

    with pytest.raises(RuntimeError):
        EN.topk_indices(G, 3)
    with pytest.raises(RuntimeError):
        EN.class_centroids(Q, torch.arange(8), torch.tensor([0, 8]))
