"""Speed perturbation, host side: the filter table against its fp64 formula, the oracle against an independent
polyphase evaluation (scipy.signal.upfirdn), the resampler's tone response, augmentation plans with speeds, start
bounds, speed labels, and argument rejection.  No GPU needed."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import frontend as F
from oracle import speed_oracle as S

FACTORS = [Fraction(1, 2), Fraction(9, 10), Fraction(19, 20), Fraction(11, 10), Fraction(2)]


@pytest.mark.parametrize("alpha", FACTORS, ids=str)
def test_filter_table_is_fp32_of_the_fp64_formula(alpha):
    got = F.speed_filter(alpha)
    assert got.shape == (alpha.denominator, 50) and got.dtype == np.float32
    assert np.array_equal(got.view(np.int32), S.taps(alpha).view(np.int32))
    # the 50 taps cover the support |tau| <= Z_s: the next tap on either side would be 0
    fc = 0.5 * 0.99 * min(1.0, 1 / alpha)
    zs = 12 / (2 * fc)
    assert zs <= 24.25 and all(S.h(r / alpha.denominator - d, alpha) == 0.0
                               for r in range(alpha.denominator) for d in (-25, 26))
    # every phase sums to about 1 (unit DC gain)
    assert np.abs(got.astype(np.float64).sum(1) - 1).max() < 1e-3


def _upfirdn_reference(x, alpha, table):
    """y[i] = sum_m g[i p - m q + K0] x[m] with g the table's taps laid out at step 1/q: g[K0 + j] = h(j / q), j = r - d q."""
    from scipy.signal import upfirdn

    p, q = alpha.numerator, alpha.denominator
    c = -(-25 * q // p)
    K0 = c * p
    g = np.zeros(K0 + 25 * q)
    for j in range(-25 * q, 25 * q):
        r = j % q
        d = (r - j) // q
        g[K0 + j] = table[r, d + 24]
    return upfirdn(g, x.astype(np.float64), up=q, down=p)[c:]


@pytest.mark.parametrize("alpha", FACTORS, ids=str)
def test_oracle_matches_upfirdn_on_an_interior_segment(alpha):
    g = np.random.default_rng(int(alpha * 100))
    x = g.integers(-32768, 32768, 9000).astype(np.int16)
    s0, L_ = 1000, 3000
    tab = S.taps(alpha)
    acc, _ = S.resample_sum(x, alpha, s0, L_, tab)
    want = _upfirdn_reference(x[s0:], alpha, tab)
    i = np.arange(L_)
    m = i * alpha.numerator // alpha.denominator
    inner = (m >= 24) & (m + 25 < x.size - s0)
    assert inner.sum() > 1000
    err = np.abs(acc[inner] - want[:L_][inner]) / 32768.0
    assert err.max() <= 1e-12, err.max()
    # the wrap: start 0 reads the end of the utterance for negative indices
    acc0, _ = S.resample_sum(x, alpha, 0, 5, tab)
    xx = np.concatenate([x[-100:], x])
    acc1, _ = S.resample_sum(xx, alpha, 100, 5, tab)
    assert np.array_equal(acc0, acc1)


@pytest.mark.parametrize("alpha", FACTORS, ids=str)
def test_tone_response(alpha):
    fc = 0.5 * 0.99 * min(1.0, float(1 / alpha))
    tab = S.taps(alpha)
    n = 30000
    L_ = int(n / alpha) - 200
    for rel in (0.05, 0.3, 0.6, 0.8, 1.1, 1.2, 1.3):
        f = rel * fc
        if f >= 0.5:
            continue                                  # above the input's Nyquist frequency
        x = 1000.0 * np.cos(2 * np.pi * f * np.arange(n) + 0.3)
        acc, _ = S.resample_sum(x, alpha, 0, L_, tab)
        y = acc[100:L_ - 100]
        gain = 10 * np.log10(np.mean(y ** 2) / np.mean(x ** 2))
        if rel <= 0.8:
            assert abs(gain) <= 0.05, (rel, gain)
            # the output is the tone at alpha f
            t = np.arange(100, L_ - 100)
            basis = np.stack([np.cos(2 * np.pi * f * float(alpha) * t), np.sin(2 * np.pi * f * float(alpha) * t)], 1)
            coef, *_ = np.linalg.lstsq(basis, y, rcond=None)
            resid = y - basis @ coef
            assert 10 * np.log10(np.mean(resid ** 2) / np.mean(y ** 2)) < -60, rel
        elif rel <= 1.1:
            assert gain <= -25, (rel, gain)
        else:
            assert gain <= -50, (rel, gain)


class _Bank:
    def __init__(self, lengths):
        self.lengths = np.asarray(lengths, np.int64)
        self.num_utterances = self.num_rirs = self.lengths.size


def test_plan_with_speeds_keeps_the_other_draws():
    rirs, noise = _Bank([4000] * 7), _Bank([100000, 20000, 30000, 5000])
    groups = [([0, 1], (0.0, 15.0), (1, 1), 1.0), ([2, 3], (13.0, 20.0), (2, 4), 1.0)]
    B, Ls = 3000, 25840
    g0, g1, g2 = (np.random.default_rng(5) for _ in range(3))
    p0 = F.augment_plan(B, Ls, g0, rirs, 0.4, noise, groups, 0.7)
    p1 = F.augment_plan(B, Ls, g1, rirs, 0.4, noise, groups, 0.7, speeds=None)
    p2 = F.augment_plan(B, Ls, g2, rirs, 0.4, noise, groups, 0.7, speeds=[0.9, 1.0, 1.1], speed_weights=[1, 2, 1])
    assert set(p0) == set(p1) == {"rir_idx", "noise_idx", "noise_start", "snr_db"}
    for k in p0:
        assert torch.equal(p0[k], p1[k]) and torch.equal(p0[k], p2[k])
    assert g0.integers(1 << 62) == g1.integers(1 << 62)         # speeds=None consumes the generator as before
    assert p2["speeds"] == (Fraction(9, 10), Fraction(1), Fraction(11, 10))
    k = p2["speed_idx"].numpy()
    assert k.dtype == np.int64 and k.shape == (B,)
    assert np.allclose(np.bincount(k, minlength=3) / B, [0.25, 0.5, 0.25], atol=0.04)
    # speeds are taken exactly, floats through their decimal form
    p3 = F.augment_plan(4, Ls, np.random.default_rng(0), p_reverb=0, p_noise=0, speeds=[0.95, Fraction(3, 2), 2])
    assert p3["speeds"] == (Fraction(19, 20), Fraction(3, 2), Fraction(2))
    for bad in ([2.5], [0.49], [Fraction(34, 33)], [0.9, 0.9], [], list(np.linspace(0.5, 2, 9)), [float("nan")], ["1"]):
        with pytest.raises(ValueError):
            F.augment_plan(4, Ls, None, p_reverb=0, p_noise=0, speeds=bad)
    for w in ([1, 1], [-1, 1, 1], [0, 0, 0], [np.nan, 1, 1]):
        with pytest.raises(ValueError):
            F.augment_plan(4, Ls, None, p_reverb=0, p_noise=0, speeds=[0.9, 1.0, 1.1], speed_weights=w)
    with pytest.raises(ValueError):
        F.augment_plan(4, Ls, None, p_reverb=0, p_noise=0, speed_weights=[1.0])


def test_starts_leave_room_for_the_perturbed_span():
    bank = _Bank([30000, 26000, 25840, 20000, 100000])
    Ls = 25840
    B = 4000
    g = np.random.default_rng(2)
    utt = g.integers(0, 5, B)
    plan = F.augment_plan(B, Ls, g, p_reverb=0, p_noise=0, speeds=[0.5, 0.9, 1.0, 1.1, 2.0])
    plan["speed_idx"][:7] = torch.tensor([-1, 0, 1, 2, 3, 4, -1])
    st = F.WaveBank.random_starts(bank, utt, Ls, g, plan).numpy()
    alpha = np.array([1.0] + [float(a) for a in plan["speeds"]])[plan["speed_idx"].numpy() + 1]
    need = np.array([-(-int(a * 1000) * Ls // 1000) for a in alpha])          # the factors are exact in 1/1000
    hi = np.maximum(bank.lengths[utt] - need, 0)
    assert np.all(st >= 0) and np.all(st <= hi)
    assert np.all(st[hi == 0] == 0) and (hi == 0).sum() > 100 and st.max() > 50000
    # without a plan (or a plan without speeds) the draws are those of random_starts
    a = F.WaveBank.random_starts(bank, utt, Ls, np.random.default_rng(9))
    b = F.random_starts(bank.lengths, utt, Ls, np.random.default_rng(9))
    c = F.WaveBank.random_starts(bank, utt, Ls, np.random.default_rng(9), {"rir_idx": torch.full((B,), -1)})
    assert torch.equal(a, b) and torch.equal(a, c)
    # with a plan whose factors are all 1 the bounds are random_starts' (and so are the draws)
    ones = {"speed_idx": torch.zeros(B, dtype=torch.int64), "speeds": (1,)}
    assert torch.equal(F.WaveBank.random_starts(bank, utt, Ls, np.random.default_rng(9), ones), b)
    bad = dict(plan, speed_idx=plan["speed_idx"].clone())
    bad["speed_idx"][0] = 5
    with pytest.raises(ValueError):
        F.WaveBank.random_starts(bank, utt, Ls, g, bad)


def test_speed_labels_extend_the_classes():
    plan = {"speed_idx": torch.tensor([-1, 0, 1, 2, 3, 0, 2]), "speeds": (Fraction(11, 10), 1, 0.9, 2)}
    lab = torch.tensor([0, 1, 2, 3, 4, 5, 6])
    C = 10
    # non-unit factors by value: 0.9 -> 1, 1.1 -> 2, 2 -> 3
    assert F.speed_labels(lab, plan, C).tolist() == [0, 1 + 2 * C, 2, 3 + C, 4 + 3 * C, 5 + 2 * C, 6 + C]
    assert torch.equal(F.speed_labels(lab, None, C), lab)
    assert torch.equal(F.speed_labels(lab, {"rir_idx": torch.zeros(7)}, C), lab)
    with pytest.raises(ValueError):
        F.speed_labels(lab, dict(plan, speed_idx=torch.tensor([4, 0, 0, 0, 0, 0, 0])), C)
    with pytest.raises(ValueError):
        F.speed_labels(lab, plan, 0)
    with pytest.raises(ValueError):
        F.speed_labels(lab[:3], plan, C)


def test_abi_rejects_bad_speed_arguments_without_a_gpu():
    lib = L.load()
    taps = np.empty((32, 50), np.float32)
    tp = taps.ctypes.data_as(ctypes.c_void_p)
    for p, q in ((9, 10), (1, 2), (2, 1), (1, 1), (63, 32), (33, 32)):
        assert lib.dsk_speed_filter(p, q, tp) == 0, (p, q)
    for p, q in ((18, 20), (1, 3), (3, 1), (1, 33), (0, 1), (1, 0), (-9, 10), (65, 32)):
        assert lib.dsk_speed_filter(p, q, tp) < 0, (p, q)
        assert b"dsk_speed_filter" in lib.dsk_last_error()
    assert lib.dsk_speed_filter(9, 10, None) < 0
    d = np.zeros(64, np.int64)
    p = d.ctypes.data_as(ctypes.c_void_p)

    def call(K=1, ratio=p, tab=p, idx=p, B=4):
        return lib.dsk_wave_augment_speed(p, p, 1, p, p, B, 1000, None, None, 0, 1, None, None, None, 0, 0, None, None,
                                          None, ratio, tab, K, idx, p, None)

    for kw in ({"K": 9}, {"K": -1}, {"ratio": None}, {"tab": None}, {"idx": None}, {"B": 0}):
        assert call(**kw) < 0, kw
        assert b"dsk_wave_augment" in lib.dsk_last_error()
    with pytest.raises(ValueError):
        F.speed_filter(Fraction(1, 3))
    assert F.speed_filter(Fraction(18, 20)).shape == (10, 50)             # 18/20 is 9/10
