"""Frame-energy VAD on the host: the vectorised oracle against its frame-by-frame loop, the runs and select oracles
against numpy boolean indexing, the parameter checks, the default threshold's arithmetic and the window counting behind
diarize's hop search."""
import math

import numpy as np
import pytest

from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import frontend as F
from oracle import vad_oracle as VO


def _energies(lens, seed):
    g = np.random.default_rng(seed)
    E = np.exp(g.normal(-4.0, 3.0, int(np.sum(lens)))).astype(np.float32)
    E[g.random(E.size) < 0.05] = np.float32(2.220446049250313e-16)        # exact-zero frames, as the engine stores them
    return E, np.concatenate(([0], np.cumsum(lens))).astype(np.int64)


CASES = [
    ({}, [1, 1, 1, 5, 40, 2, 3]),                              # 1-frame utterances among others
    ({"context": 7}, [1, 3, 7, 8, 15, 16, 100]),                # c >= n_u and c < n_u
    ({"context": 0}, [1, 9, 30]),
    ({"proportion": 0.0}, [1, 4, 60]),                          # every frame speech
    ({"proportion": 1.5}, [1, 4, 60]),                          # no frame speech
    ({"proportion": 1.0, "context": 1}, [2, 50]),
    ({"mean_scale": 0.0, "energy_threshold": -4.0}, [33, 7]),
    ({"mean_scale": -0.7, "energy_threshold": 2.0, "context": 3, "proportion": 0.5}, [64, 3]),
]


@pytest.mark.parametrize("params,lens", CASES)
def test_decide_matches_the_loop(params, lens):
    for seed in range(3):
        E, off = _energies(lens, seed)
        p = {**VO.DEFAULTS, **params}
        got, thr, le = VO.decide(E, off, **p)
        assert np.array_equal(got, VO.decide_brute(E, off, **p)), (params, lens, seed)
        assert thr.shape == (len(lens),) and le.shape == E.shape
        if p["proportion"] == 0.0:
            assert got.all()
        if p["proportion"] > 1.0:
            assert not got.any()


def test_ties_at_the_threshold_are_not_above():
    """e_g > thr is strict: four equal energies with energy_threshold 0 and mean_scale 1 put thr exactly on e."""
    E = np.full(4, 0.25, np.float32)                     # ln 0.25 sums and divides by 4 exactly
    off = [0, 4]
    got, thr, le = VO.decide(E, off, energy_threshold=0.0, mean_scale=1.0, context=2, proportion=0.01)
    assert thr[0] == le[0] and not got.any()
    assert np.array_equal(got, VO.decide_brute(E, off, energy_threshold=0.0, mean_scale=1.0, context=2, proportion=0.01))
    got, _, _ = VO.decide(E, off, energy_threshold=-1e-12, mean_scale=1.0, context=2, proportion=0.01)
    assert got.all()


def test_default_threshold_arithmetic():
    want = 5.5 - 0.5 * 31 * math.log(2.0)
    assert F.VAD_ENERGY_THRESHOLD == pytest.approx(want, abs=1e-14)
    assert VO.DEFAULT_ENERGY_THRESHOLD == pytest.approx(want, abs=1e-14)
    assert round(F.VAD_ENERGY_THRESHOLD, 4) == -5.2438
    assert F.VAD_DEFAULTS == {"energy_threshold": F.VAD_ENERGY_THRESHOLD, "mean_scale": 0.5, "context": 2,
                              "proportion": 0.12}
    # shifting every ln E by -D and the constant by -(1 - mean_scale) D leaves every decision unchanged
    E, off = _energies([50, 70], 1)
    D = 31 * math.log(2.0)
    a, _, _ = VO.decide(E.astype(np.float64), off, energy_threshold=5.5)
    b, _, _ = VO.decide(E.astype(np.float64) * 2.0 ** -31, off, energy_threshold=5.5 - 0.5 * D)
    assert np.array_equal(a, b)


def test_vad_params():
    assert F.vad_params({}) == F.VAD_DEFAULTS and F.vad_params(None) == F.VAD_DEFAULTS
    assert F.vad_params({"context": 3.0})["context"] == 3
    for bad in ({"context": -1}, {"context": 1.5}, {"context": True}, {"context": 2 ** 31}, {"proportion": -0.1},
                {"proportion": float("nan")}, {"mean_scale": float("inf")}, {"energy_threshold": float("-inf")},
                {"threshold": 1.0}):
        with pytest.raises(ValueError):
            F.vad_params(bad)


def _runs_numpy(mask, off, utt):
    out = []
    for j, u in enumerate(utt):
        m = np.asarray(mask[off[u]:off[u + 1]], np.int8)
        d = np.diff(np.concatenate(([0], m, [0])))
        out += [(j, int(a), int(b)) for a, b in zip(np.flatnonzero(d == 1), np.flatnonzero(d == -1))]
    return out


def test_runs_and_select_oracles_match_numpy():
    g = np.random.default_rng(5)
    lens = np.array([1, 2, 3, 17, 1, 40, 5])
    off = np.concatenate(([0], np.cumsum(lens)))
    n = int(off[-1])
    feats = g.standard_normal((n, 64)).astype(np.float32)
    masks = [np.zeros(n, bool), np.ones(n, bool), np.arange(n) % 2 == 0, g.random(n) < 0.6]
    m = np.zeros(n, bool)
    m[off[3] - 1:off[3] + 2] = True                          # straddles the boundary of utterances 2 and 3
    masks.append(m)
    for mask in masks:
        for utt in (range(lens.size), [5, 0, 5, 3]):
            assert VO.runs_brute(mask, off, list(utt)) == _runs_numpy(mask, off, list(utt))
        rows, new = VO.select_brute(feats, off, mask)
        assert np.array_equal(rows, feats[mask])
        assert np.array_equal(np.diff(new), [int(mask[off[u]:off[u + 1]].sum()) for u in range(lens.size)])
    assert VO.runs_brute(m, off, [2, 3]) == [(0, 2, 3), (1, 0, 2)]   # one run each side of the boundary


def test_run_window_counts_and_hop_search():
    g = np.random.default_rng(2)
    rlen = np.concatenate(([1, 159, 160, 161, 199, 200, 201], g.integers(1, 5000, 200)))
    last = np.maximum(rlen - 160, 0)
    for hop in (1, 7, 40, 80, 160, 4999):
        _, _, wo = F.sliding_windows(rlen, np.arange(rlen.size), 160, hop)
        assert np.array_equal(DZ._window_counts(last, hop), np.diff(wo.numpy())), hop
    rec = np.sort(g.integers(0, 3, rlen.size))
    h = DZ._smallest_hop(last, rec, 3, 1)
    counts = lambda hh: np.bincount(rec, DZ._window_counts(last, hh), minlength=3).max()   # noqa: E731
    if h is not None and h > 1:
        assert counts(h) <= DZ.MAX_WINDOWS < counts(h - 1)
    big = np.full(40000, 1000)                                # 40 000 runs in one recording: no hop fits
    assert DZ._smallest_hop(big - 160, np.zeros(big.size, np.int64), 1, 1) is None
    one = np.array([400000 - 160])
    h = DZ._smallest_hop(one, np.zeros(1, np.int64), 1, 1)
    assert DZ._window_counts(one, h)[0] <= DZ.MAX_WINDOWS < DZ._window_counts(one, h - 1)[0]
