"""Cosine scoring without a GPU: the exact EER / minDCF against the brute-force oracle, its errors, and argument
rejection by the C ABI of the scoring ops."""
import ctypes

import numpy as np
import pytest

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import verification as V
from oracle import score_norm_oracle as O


def _random(n, p_tar, seed):
    rng = np.random.default_rng(seed)
    y = rng.random(n) < p_tar
    y[:2] = [True, False]
    s = rng.standard_normal(n) + 2.0 * y
    return s, y


def _close(got, ref):
    assert abs(got[0] - ref[0]) <= 1e-12 and abs(got[1] - ref[1]) <= 1e-12, (got, ref)


@pytest.mark.parametrize("p_target", [0.01, 0.05])
@pytest.mark.parametrize("p_tar", [0.5, 0.1])
def test_random_scores_match_brute_force(p_target, p_tar):
    s, y = _random(2000, p_tar, seed=int(1000 * p_target + 10 * p_tar))
    _close(V.eer_min_dcf(s, y, p_target), O.eer_min_dcf(s, y, p_target))
    _close(V.eer_min_dcf(s, y, p_target, c_miss=10.0, c_fa=1.0), O.eer_min_dcf(s, y, p_target, 10.0, 1.0))


@pytest.mark.parametrize("p_target", [0.01, 0.05])
def test_tie_heavy_scores_match_brute_force(p_target):
    s, y = _random(2000, 0.3, seed=7)
    s = np.round(s, 1)
    assert np.unique(s).size < 100
    _close(V.eer_min_dcf(s, y, p_target), O.eer_min_dcf(s, y, p_target))


def test_perfectly_separated_scores():
    s, y = _random(500, 0.2, seed=3)
    s = np.where(y, 10.0 + s, s - 10.0)
    got = V.eer_min_dcf(s, y)
    _close(got, O.eer_min_dcf(s, y))
    assert got == (0.0, 0.0)


def test_all_equal_scores():
    _, y = _random(300, 0.4, seed=4)
    s = np.full(y.size, 0.25)
    got = V.eer_min_dcf(s, y)
    _close(got, O.eer_min_dcf(s, y))
    assert got == (0.5, 1.0)


def test_strictly_monotone_transform_gives_identical_results():
    s, y = _random(2000, 0.2, seed=5)
    s = np.round(s, 2)                                  # keep ties, which the transform must preserve
    ref = V.eer_min_dcf(s, y)
    for f in (lambda x: np.exp(x), lambda x: 3.0 * x - 7.0, lambda x: np.arctan(x)):
        assert V.eer_min_dcf(f(s), y) == ref
        assert V.eer_min_dcf(f(s), y, 0.05) == V.eer_min_dcf(s, y, 0.05)


def test_torch_and_float32_inputs():
    import torch

    s, y = _random(1000, 0.2, seed=6)
    s32 = s.astype(np.float32)
    ref = O.eer_min_dcf(s32.astype(np.float64), y)
    _close(V.eer_min_dcf(torch.from_numpy(s32), torch.from_numpy(y)), ref)
    _close(V.eer_min_dcf(s32, y.astype(np.int64)), ref)


def test_bad_inputs_raise_value_error():
    s, y = _random(100, 0.3, seed=8)
    with pytest.raises(ValueError):
        V.eer_min_dcf(s, np.ones_like(y))               # no non-targets
    with pytest.raises(ValueError):
        V.eer_min_dcf(s, np.zeros_like(y))              # no targets
    for bad in (np.nan, np.inf, -np.inf):
        s2 = s.copy()
        s2[5] = bad
        with pytest.raises(ValueError):
            V.eer_min_dcf(s2, y)
    with pytest.raises(ValueError):
        V.eer_min_dcf(s[:50], y)
    with pytest.raises(ValueError):
        V.eer_min_dcf(s, y, p_target=0.0)


P = ctypes.c_void_p(256)                                 # never dereferenced: the arguments are checked first


def _rejected(rc, what):
    assert rc == -1, (what, rc)
    assert b"bad arguments" in L.load().dsk_last_error(), what


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    M, Nc, D, k = 10, 100, 128, 20
    cases = {
        "null E": (None, M, P, Nc, D, k),
        "null cohort": (P, M, None, Nc, D, k),
        "M = 0": (P, 0, P, Nc, D, k),
        "k = 1": (P, M, P, Nc, D, 1),
        "k > Nc": (P, M, P, Nc, D, Nc + 1),
        "Nc = 1": (P, M, P, 1, D, 1),
        "Nc > 65536": (P, M, P, 65537, D, k),
        "D % 64": (P, M, P, Nc, 96, k),
        "D = 0": (P, M, P, Nc, 0, k),
    }
    for what, (e, m, c, nc, d, kk) in cases.items():
        _rejected(lib.dsk_cohort_stats(P, e, m, c, nc, d, kk, P, P, None), what)
    _rejected(lib.dsk_cohort_stats(P, P, M, P, Nc, D, k, None, P, None), "null mean")
    _rejected(lib.dsk_cohort_stats(P, P, M, P, Nc, D, k, P, None, None), "null std")
    _rejected(lib.dsk_cosine_matrix(P, P, M, P, Nc, D, None, None), "null cos")
    _rejected(lib.dsk_cosine_matrix(P, P, M, P, 65537, D, P, None), "cosine Nc > 65536")
    _rejected(lib.dsk_cosine_matrix(P, P, M, P, Nc, 100, P, None), "cosine D % 64")
    # the selection kernel's own entry point
    _rejected(lib.dsk_topk_mean_std(None, 4, 100, 100, 5, P, P, None), "null S")
    _rejected(lib.dsk_topk_mean_std(P, 4, 100, 100, 1, P, P, None), "topk k = 1")
    _rejected(lib.dsk_topk_mean_std(P, 4, 100, 100, 101, P, P, None), "topk k > cols")
    _rejected(lib.dsk_topk_mean_std(P, 4, 65537, 65537, 5, P, P, None), "topk cols > 65536")
    _rejected(lib.dsk_topk_mean_std(P, 4, 100, 99, 5, P, P, None), "topk ld < cols")
    # trial scoring
    _rejected(lib.dsk_score_trials(P, 10, 64, None, 5, None, None, P, None, None), "null trials")
    _rejected(lib.dsk_score_trials(P, 10, 64, P, 0, None, None, P, None, None), "T = 0")
    _rejected(lib.dsk_score_trials(P, 10, 64, P, 5, P, None, P, P, None), "mean without std")
    _rejected(lib.dsk_score_trials(P, 10, 64, P, 5, P, P, P, None, None), "stats without normed")


def test_gpu_entry_points_raise_on_cpu_tensors():
    import torch

    E, C = torch.randn(8, 64), torch.randn(10, 64)
    with pytest.raises(RuntimeError):
        V.cosine_matrix(E, C)
    with pytest.raises(RuntimeError):
        V.cohort_stats(E, C, 5)
    with pytest.raises(RuntimeError):
        V.score_trials(E, torch.zeros(3, 2, dtype=torch.int64))
