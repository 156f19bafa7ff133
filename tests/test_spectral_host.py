"""Spectral clustering without a GPU: the NME-SC oracle on textbook graphs, its k-means under a rotation of the
eigenbasis, the default grid, and the argument checks of dsk_spectral_cluster and the Python entry points."""
import ctypes

import numpy as np
import pytest

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import diarization as DZ
from oracle import spectral_oracle as SO


def _cliques(sizes):
    """Similarities of disjoint cliques: 1 inside a clique, -1 across (ties everywhere: the lower column wins)."""
    lab = np.repeat(np.arange(len(sizes)), sizes)
    S = np.where(lab[:, None] == lab[None, :], 1.0, -1.0)
    return S.astype(np.float32), lab


def test_disjoint_cliques_give_k_zero_eigenvalues_and_k():
    for sizes in ([6, 6, 6], [5, 9, 7, 8], [12, 10], [8, 8, 8, 8]):
        S, lab = _cliques(sizes)
        k = len(sizes)
        R = SO.ranks(S)
        p = min(sizes) - 1                              # every window's p nearest lie in its clique
        w = np.linalg.eigvalsh(SO.laplacian(R, p))
        assert np.all(np.abs(w[:k]) < 1e-10) and w[k] > 1e-3
        if len(set(sizes)) == 1:                        # complete cliques: the spectrum is {0 x k, n x (N - k)}
            res = SO.spectral_cluster(S, [p])
            assert res.k == k
            assert np.array_equal(res.labels, SO.renumber(lab))


def test_affinity_matches_explicit_loops():
    rng = np.random.default_rng(1)
    N = 17
    S = rng.standard_normal((N, N)).astype(np.float32)
    R = SO.ranks(S)
    for p in (1, 3, 8, 16):
        A = np.zeros((N, N))
        for i in range(N):
            for j in range(N):
                if i != j:
                    A[i, j] = (int(R[i, j] < p) + int(R[j, i] < p)) / 2
        assert np.array_equal(A, SO.affinity(R, p))
        L_ = SO.laplacian(R, p)
        assert np.array_equal(np.diag(L_), A.sum(1))


def test_ties_go_to_the_lower_column():
    rng = np.random.default_rng(2)
    N = 40
    S = (np.round(rng.random((N, N)) * 8) / 8).astype(np.float32)
    S[3] = S[5]                                     # duplicated rows
    np.fill_diagonal(S, np.nan)                     # the diagonal is never read
    R = SO.ranks(S)
    for i in range(N):
        cols = [j for j in range(N) if j != i]
        order = sorted(cols, key=lambda j: (-float(S[i, j]), j))
        assert [int(R[i, j]) for j in order] == list(range(N - 1))
    S2 = S.copy()
    S2[0, 1] = np.inf
    with pytest.raises(ValueError):
        SO.ranks(S2)


def test_default_grid():
    assert SO.p_grid(2).tolist() == [1]
    assert SO.p_grid(3).tolist() == [1]
    g = SO.p_grid(10_000)
    assert g[0] == 1 and g[-1] == int(np.floor(0.25 * 9999)) and g.size == 30 and np.all(np.diff(g) > 0)
    for N in (2, 3, 10, 10_000):
        assert np.array_equal(SO.p_grid(N), DZ.p_grid(N))


def test_kmeans_partition_is_rotation_invariant():
    rng = np.random.default_rng(3)
    k = 4
    centres = 3 * rng.standard_normal((k, k))
    Y = centres[rng.integers(0, k, 200)] + 0.3 * rng.standard_normal((200, k))
    Q, _ = np.linalg.qr(rng.standard_normal((k, k)))
    a = SO.kmeans(Y, k)
    b = SO.kmeans(Y @ Q, k)
    assert np.array_equal(a, b)
    assert SO.kmeans(Y, 1).tolist() == [0] * 200


P = ctypes.c_void_p(16)  # never dereferenced: every call below fails validation first


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    k, t = ctypes.c_int32(0), ctypes.c_int32(0)
    pv = np.array([1, 2, 3], np.int32)
    bad_order = np.array([1, 3, 2], np.int32)
    zero = np.array([0, 1], np.int32)
    high = np.array([1, 10], np.int32)

    def call(S=P, N=10, ld=10, p=pv, n_p=3, ms=8, ns=0, it=100, labels=P, k_=True, t_=True, eig=P, lmax=P, ratio=P):
        pp = p.ctypes.data_as(ctypes.c_void_p) if isinstance(p, np.ndarray) else p
        return lib.dsk_spectral_cluster(S, N, ld, pp, n_p, ms, ns, it, labels, ctypes.byref(k) if k_ else None,
                                        ctypes.byref(t) if t_ else None, eig, lmax, ratio, None, None)

    cases = {"N = 1": dict(N=1, ld=1), "N > max": dict(N=32769, ld=32769), "ld < N": dict(ld=9),
             "n_p = 0": dict(n_p=0), "n_p > max": dict(n_p=65), "p not increasing": dict(p=bad_order),
             "p = 0": dict(p=zero, n_p=2), "p = N": dict(p=high, n_p=2), "max_speakers 0": dict(ms=0),
             "max_speakers > max": dict(ms=33), "num_speakers < 0": dict(ns=-1), "num_speakers = N": dict(ns=10),
             "num_speakers > max": dict(N=40, ld=40, ns=33), "kmeans_iters 0": dict(it=0),
             "null S": dict(S=None), "null p": dict(p=None), "null labels": dict(labels=None),
             "null k": dict(k_=False), "null p_index": dict(t_=False), "null eigenvalues": dict(eig=None),
             "null lambda_max": dict(lmax=None), "null ratio": dict(ratio=None)}
    for what, kw in cases.items():
        assert call(**kw) == -1, what
        assert b"dsk_spectral_cluster: bad arguments" in lib.dsk_last_error(), what


def test_python_entry_points_raise_value_errors():
    class Model:
        training = False

    for kw in (dict(spectral={}, threshold=0.5), dict(spectral={}, vbx={}, num_speakers=2),
               dict(spectral={"p_max": 0.3}), dict(spectral=[("p_steps", 3)])):
        with pytest.raises(ValueError):
            DZ.diarize(Model(), None, [0], **kw)
    with pytest.raises(ValueError):
        DZ.diarize(Model(), None, [0])                 # AHC still needs a count or a threshold
    S = np.zeros((4, 4), np.float32)
    with pytest.raises(ValueError):
        DZ.spectral(S, p_max_frac=0.0)
    with pytest.raises(ValueError):
        DZ.spectral(S, num_speakers=0)
    with pytest.raises(ValueError, match="DSK_SC_MAX_SPEAKERS"):
        DZ.spectral(S, max_speakers=L.DSK_SC_MAX_SPEAKERS + 1)
    with pytest.raises(ValueError, match="DSK_SC_MAX_SPEAKERS"):
        DZ.spectral(np.zeros((40, 40), np.float32), num_speakers=33)
