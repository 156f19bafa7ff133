"""Diarization without a GPU: the clustering oracle against scipy, the replay validator against seeded defects,
argument rejection by dsk_ahc, and the frame-label / segment assembly and RTTM lines against brute force."""
import ctypes

import numpy as np
import pytest
from scipy.cluster.hierarchy import linkage as scipy_linkage
from scipy.spatial.distance import squareform

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import frontend as F
from oracle import ahc_oracle as O


def _similarities(N, seed, clustered):
    rng = np.random.default_rng(seed)
    if clustered:
        C = rng.standard_normal((4, 32))
        X = C[rng.integers(0, 4, N)] + 0.6 * rng.standard_normal((N, 32))
    else:
        X = rng.standard_normal((N, 32))
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return (X @ X.T).astype(np.float32)


def scipy_tree(d, method):
    return scipy_linkage(squareform(d, checks=False), method=method)


@pytest.mark.parametrize("N", [2, 3, 40, 150])
@pytest.mark.parametrize("clustered", [False, True])
def test_naive_oracle_matches_scipy(N, clustered):
    d = O.distances(_similarities(N, N, clustered))
    for method in ("complete", "average"):
        Zo, _ = O.naive_ahc(d, method)
        Zs = scipy_tree(d, method)
        if method == "complete":
            assert np.array_equal(Zo, Zs)
        else:
            assert np.array_equal(Zo[:, [0, 1, 3]], Zs[:, [0, 1, 3]])
            np.testing.assert_allclose(Zo[:, 2], Zs[:, 2], rtol=1e-12, atol=0)


def test_naive_oracle_early_stops_match_fcluster():
    from scipy.cluster.hierarchy import fcluster

    d = O.distances(_similarities(120, 7, True))
    Zf = scipy_tree(d, "average")
    for k in (1, 2, 4, 17, 120):
        Z, lab = O.naive_ahc(d, "average", stop_k=k)
        assert Z.shape[0] == 120 - k and np.array_equal(Z[:, [0, 1, 3]], Zf[:120 - k, [0, 1, 3]])
        assert _same_partition(lab, fcluster(Zf, k, "maxclust"))
    for t in (0.2, 0.7, 1.1):
        Z, lab = O.naive_ahc(d, "average", stop_height=t)
        assert np.all(Z[:, 2] <= t) and Z.shape[0] == int(np.sum(Zf[:, 2] <= t))
        assert _same_partition(lab, fcluster(Zf, t, "distance"))


def _same_partition(a, b):
    a, b = np.asarray(a), np.asarray(b)
    pairs = set(zip(a.tolist(), b.tolist()))
    return len(pairs) == len(set(a.tolist())) == len(set(b.tolist()))


@pytest.mark.parametrize("method", ["average", "complete"])
def test_replay_accepts_scipy_and_rejects_defects(method):
    d = O.distances(_similarities(60, 3, True))
    Z = scipy_tree(d, method)
    assert O.replay(Z, d, method) is None
    bad = Z.copy()
    bad[[5, 6]] = bad[[6, 5]]                                 # swapped merge order (heights no longer least)
    if Z[5, 2] != Z[6, 2]:
        assert O.replay(bad, d, method) is not None
    bad = Z.copy()
    bad[10, 2] *= 1 + 1e-9                                    # wrong height
    assert "height" in O.replay(bad, d, method)
    bad = Z.copy()
    bad[10, 3] += 1                                           # wrong size
    assert "size" in O.replay(bad, d, method)
    bad = Z.copy()
    r = next(i for i in range(20, 59) if Z[i, 0] >= 60 or Z[i, 1] >= 60)
    dead = next(int(x) for x in Z[:r, :2].reshape(-1) if x not in Z[r, :2])   # merged before row r
    bad[r, 0] = min(dead, Z[r, 1])
    bad[r, 1] = max(dead, Z[r, 1])
    assert "live" in O.replay(bad, d, method)


def test_replay_accepts_tie_heavy_oracle_runs():
    rng = np.random.default_rng(11)
    S = np.round(rng.uniform(-1, 1, (50, 50)) * 8) / 8
    S[10:20] = S[0:10]
    S[:, 10:20] = S[:, 0:10]
    for S_ in (S.astype(np.float32), np.full((30, 30), 0.25, np.float32)):
        d = O.distances(S_)
        for method in ("average", "complete"):
            Z, _ = O.naive_ahc(d, method)
            assert O.replay(Z, d, method) is None


P = ctypes.c_void_p(256)                                  # never dereferenced: the arguments are checked first


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    m, r = ctypes.c_int32(0), ctypes.c_int32(0)
    inf = float("inf")
    # dsk_ahc(S, N, ld, linkage, stop_k, stop_height, Z, n_merges, labels, n_rounds, stream)
    cases = {"null S": (None, 10, 10, 0, 1, inf, P, ctypes.byref(m), P),
             "null Z": (P, 10, 10, 0, 1, inf, None, ctypes.byref(m), P),
             "null n_merges": (P, 10, 10, 0, 1, inf, P, None, P),
             "null labels": (P, 10, 10, 0, 1, inf, P, ctypes.byref(m), None),
             "N = 1": (P, 1, 1, 0, 1, inf, P, ctypes.byref(m), P),
             "N > max": (P, 32769, 32769, 0, 1, inf, P, ctypes.byref(m), P),
             "ld < N": (P, 10, 9, 0, 1, inf, P, ctypes.byref(m), P),
             "linkage 2": (P, 10, 10, 2, 1, inf, P, ctypes.byref(m), P),
             "linkage -1": (P, 10, 10, -1, 1, inf, P, ctypes.byref(m), P),
             "stop_k = 0": (P, 10, 10, 0, 0, inf, P, ctypes.byref(m), P),
             "stop_k > N": (P, 10, 10, 1, 11, inf, P, ctypes.byref(m), P),
             "NaN height": (P, 10, 10, 0, 1, float("nan"), P, ctypes.byref(m), P)}
    for what, a in cases.items():
        rc = lib.dsk_ahc(*a, ctypes.byref(r), None)
        assert rc == -1, (what, rc)
        assert b"bad arguments" in lib.dsk_last_error(), what


def test_python_entry_points_reject_bad_arguments():
    import torch

    from deepspeaker_pytorch_b200 import engine as EN

    S = torch.zeros(4, 4)
    with pytest.raises(RuntimeError):
        EN.ahc(S)                                             # CPU tensor
    with pytest.raises(ValueError):
        EN.ahc(S, linkage="single")
    with pytest.raises(ValueError):
        EN.ahc(S, num_clusters=2, threshold=0.5)

    class _Eval:
        training = False

    for kw in ({}, {"num_speakers": 2, "threshold": 0.5}):
        with pytest.raises(ValueError):
            DZ.diarize(_Eval(), None, [0], **kw)

    class _Train:
        training = True

    with pytest.raises(RuntimeError):
        DZ.diarize(_Train(), None, [0], num_speakers=2)


def _assembly_cases():
    rng = np.random.default_rng(2)
    for n, T, hop in ((1000, 160, 40), (1000, 160, 80), (161, 160, 40), (203, 160, 40), (100, 160, 40),
                      (160, 160, 40), (977, 150, 33), (50, 20, 5), (41, 20, 10), (7, 3, 1), (1, 160, 40)):
        _, ws, _ = F.sliding_windows([n], [0], T, hop)
        labels = rng.integers(0, 3, ws.numel()).astype(np.int32)
        yield n, T, ws.numpy(), labels


def test_frame_labels_and_segments_match_brute_force():
    for n, T, ws, wl in _assembly_cases():
        got = DZ.frame_labels(ws, wl, n, T)
        ref = O.frame_labels_brute(ws, wl, n, T)
        assert np.array_equal(got, ref), (n, T)
        assert DZ.segments(got) == O.segments_brute(ref), (n, T)


def test_frame_label_ties_go_to_the_earlier_window():
    # T even, hop odd: frame centres fall exactly half way between two window centres
    ws = np.array([0, 3, 6, 9])
    wl = np.array([0, 1, 2, 3])
    got = DZ.frame_labels(ws, wl, 13, 4)
    assert np.array_equal(got, O.frame_labels_brute(ws, wl, 13, 4))
    # frame 3 (centre 3.5): windows 0 (centre 2) and 1 (centre 5) are 1.5 away -> window 0
    assert got[3] == 0
    # the tail window of sliding_windows starts off the hop grid: it wins only the frames nearest to it
    _, ws2, _ = F.sliding_windows([170], [0], 160, 40)
    assert ws2.tolist() == [0, 10]
    got = DZ.frame_labels(ws2.numpy(), np.array([4, 7]), 170, 160)
    assert np.array_equal(got, O.frame_labels_brute(ws2.numpy(), np.array([4, 7]), 170, 160))
    assert got[:85].tolist() == [4] * 85 and got[85:].tolist() == [7] * 85


def test_rttm_lines():
    segs = DZ.segments(np.array([0, 0, 1, 1, 1, 0], np.int32))
    assert segs == [(0.0, 0.02, 0), (0.02, 0.05, 1), (0.05, 0.06, 0)]
    txt = DZ.to_rttm(segs, "rec1")
    assert txt == ("SPEAKER rec1 1 0.000 0.020 <NA> <NA> spk0 <NA> <NA>\n"
                   "SPEAKER rec1 1 0.020 0.030 <NA> <NA> spk1 <NA> <NA>\n"
                   "SPEAKER rec1 1 0.050 0.010 <NA> <NA> spk0 <NA> <NA>\n")
    for line in txt.splitlines():
        assert len(line.split()) == 10
    with pytest.raises(ValueError):
        DZ.to_rttm(segs, "rec 1")
