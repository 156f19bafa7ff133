"""Waveform augmentation, host side: the fp64 oracle, segment lengths, augmentation plans, ABI limits, and a self-test
of the reverberation error checker the GPU tests use (see tests/test_gpu_augment.py for the bound).  No GPU needed."""
import ctypes

import numpy as np
import pytest

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import frontend as F
from oracle import augment_oracle as A


def test_oracle_fft_convolution_matches_np_convolve():
    g = np.random.default_rng(0)
    for L_, lh in ((1, 1), (100, 1), (100, 250), (3000, 1024), (25840, 16000), (4096, 65536)):
        s, h = g.normal(size=L_), g.normal(size=lh)
        want = np.convolve(s, h)[:L_]
        got = A.reverb(s, h)
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want))), (L_, lh)
    assert np.array_equal(A.reverb(s, None), s)


def test_oracle_mix_achieves_the_requested_snr():
    g = np.random.default_rng(1)
    r = g.normal(0, 0.1, 25840)
    for snr in (-5.0, 0.0, 7.3, 20.0, 40.0):
        n = g.normal(0, 0.3, 25840)
        (gain,) = A.gains(r, [n], [snr])
        achieved = 10 * np.log10(A.power(r) / A.power(gain * n))
        assert abs(achieved - snr) <= 1e-9
    assert A.gains(r, [np.zeros(100)], [10.0]) == [0.0]


@pytest.mark.parametrize("sr", [8000, 16000])
def test_segment_length_gives_exactly_T_frames(sr):
    lib = L.load()
    for T in range(16, 801):
        assert lib.dsk_fbank_num_frames(F.segment_samples(T, sr), sr) == T
    assert F.segment_samples(160, 16000) == 25840


class _Bank:
    def __init__(self, lengths):
        self.lengths = np.asarray(lengths, np.int64)
        self.num_utterances = self.num_rirs = self.lengths.size


def test_augment_plan_bounds_groups_and_reproducibility():
    rirs, noise = _Bank([4000] * 7), _Bank([100000, 20000, 30000, 5000, 400000, 60000, 26000, 90000])
    groups = [([0, 1, 2], (0.0, 15.0), (1, 1), 1.0), ([3, 4], (5.0, 15.0), (1, 1), 1.0), ([5, 6, 7], (13.0, 20.0), (3, 8), 2.0)]
    B, Ls = 4000, 25840
    p = F.augment_plan(B, Ls, np.random.default_rng(3), rirs, 0.4, noise, groups, 0.7)
    q = F.augment_plan(B, Ls, np.random.default_rng(3), rirs, 0.4, noise, groups, 0.7)
    assert all(np.array_equal(p[k].numpy(), q[k].numpy()) for k in p)
    ri, ni, ns, sd = (p[k].numpy() for k in ("rir_idx", "noise_idx", "noise_start", "snr_db"))
    assert ri.shape == (B,) and ni.shape == ns.shape == sd.shape == (B, 8) and sd.dtype == np.float64
    assert ri.min() == -1 and ri.max() == 6 and abs(np.mean(ri >= 0) - 0.4) < 0.04
    noisy = ni[:, 0] >= 0
    assert abs(noisy.mean() - 0.7) < 0.04
    # -1 padding after the used sources; none at all without noise
    cnt = (ni >= 0).sum(1)
    assert np.all(ni[np.arange(8)[None, :] >= cnt[:, None]] == -1) and np.all(cnt[~noisy] == 0)
    assert np.all(ns[ni < 0] == 0) and np.all(sd[ni < 0] == 0)
    # each group: its utterances, SNR range, count range; weights 1 : 1 : 2
    grp = np.where(np.isin(ni[:, 0], [0, 1, 2]), 0, np.where(np.isin(ni[:, 0], [3, 4]), 1, 2))[noisy]
    for gi, (ids, (lo, hi), (clo, chi), _) in enumerate(groups):
        rows = np.nonzero(noisy)[0][grp == gi]
        assert np.all(np.isin(ni[rows][ni[rows] >= 0], ids))
        s = sd[rows][ni[rows] >= 0]
        assert s.min() >= lo and s.max() <= hi
        assert cnt[rows].min() == clo and cnt[rows].max() == chi
    frac = np.bincount(grp, minlength=3) / grp.size
    assert np.allclose(frac, [0.25, 0.25, 0.5], atol=0.04)
    # starts in [0, n - L], 0 when n < L (utterance 3 has 5000 < L samples)
    used = ni >= 0
    n = noise.lengths[ni[used]]
    assert np.all(ns[used] >= 0) and np.all(ns[used] <= np.maximum(n - Ls, 0))
    assert np.all(ns[used][n < Ls] == 0)
    # p = 0 / 1
    z = F.augment_plan(50, Ls, np.random.default_rng(0), rirs, 0.0, noise, groups, 0.0)
    assert np.all(z["rir_idx"].numpy() == -1) and np.all(z["noise_idx"].numpy() == -1)
    o = F.augment_plan(50, Ls, np.random.default_rng(0), rirs, 1.0, noise, groups, 1.0)
    assert np.all(o["rir_idx"].numpy() >= 0) and np.all(o["noise_idx"].numpy()[:, 0] >= 0)
    e = F.augment_plan(5, Ls, np.random.default_rng(0), p_reverb=0.0, p_noise=0.0)
    assert e["noise_idx"].shape == (5, 0) and np.all(e["rir_idx"].numpy() == -1)
    with pytest.raises(ValueError):
        F.augment_plan(5, Ls, None, None, 0.5)
    with pytest.raises(ValueError):
        F.augment_plan(5, Ls, None, rirs, 0.5, noise, [([0], (0, 1), (1, 9), 1.0)], 0.5)
    with pytest.raises(ValueError):
        F.augment_plan(5, Ls, None, rirs, 0.5, noise, [([8], (0, 1), (1, 1), 1.0)], 0.5)


def test_abi_rejects_out_of_range_limits_without_a_gpu():
    lib = L.load()
    d = np.zeros(64, np.int64)
    p = d.ctypes.data_as(ctypes.c_void_p)

    def call(B=4, L_=1000, M=1, max_rir=16000, speech=p, rir_idx=p):
        return lib.dsk_wave_augment(speech, p, 1, p, p, B, L_, p, p, 1, max_rir, rir_idx, p, p, 1, M, p, p, p, p, None)

    for kw in ({"M": 9}, {"M": -1}, {"max_rir": 65537}, {"max_rir": 0}, {"B": 0}, {"L_": 0}, {"L_": (1 << 24) + 1},
               {"speech": None}):
        assert call(**kw) < 0, kw
        assert b"dsk_wave_augment" in lib.dsk_last_error()
    assert lib.dsk_wave_augment(p, p, 1, p, p, 4, 1000, None, None, 0, 1, p, p, p, 1, 0, p, p, p, p, None) < 0
    assert lib.dsk_wave_augment(p, p, 1, p, p, 4, 1000, p, p, 1, 1, None, None, None, 1, 2, None, p, p, p, None) < 0
    assert lib.dsk_fbank_segments(None, 1, 1000, 16000, 1, 1, p, None, 0, None, 0, p, None) < 0
    assert lib.dsk_fbank_segments(p, 0, 1000, 16000, 1, 1, p, None, 0, None, 0, p, None) < 0
    assert lib.dsk_fbank_segments(p, 1, 1000, 16000, 1, 1, p, None, 2, None, 0, p, None) < 0
    assert lib.dsk_fbank_filterbank(16000, None) < 0


def test_filterbank_matches_the_published_construction():
    from oracle import fbank_oracle as FO

    lib = L.load()
    for sr in (8000, 16000):
        fb = np.empty((64, 257), np.float32)
        assert lib.dsk_fbank_filterbank(sr, fb.ctypes.data_as(ctypes.c_void_p)) == 0
        assert np.array_equal(fb, FO.get_filterbanks(64, 512, sr).astype(np.float32))


def test_bank_constructors_reject_bad_input():
    import torch

    with pytest.raises(ValueError):                          # pageable CPU memory
        F.WaveBank(torch.zeros(100, dtype=torch.int16), [0, 100])
    with pytest.raises(ValueError):
        F.WaveBank.from_waveforms([np.array([0.1, 0.2], np.float32)])   # not k / 32768
    with pytest.raises(ValueError):
        F.WaveBank.from_waveforms([np.array([1, 2], np.int32)])
    with pytest.raises(ValueError):
        F.RirBank.from_arrays([np.zeros(10)])
    with pytest.raises(ValueError):
        F.RirBank.from_arrays([np.ones(65537)])


# ---- self-test of the reverberation checker ---------------------------------------------------------------------------
def _speech(L_, seed):
    g = np.random.default_rng(seed)
    t = np.arange(L_) / 16000
    x = 0.3 * np.sin(2 * np.pi * 220 * t) * (1 + np.sin(2 * np.pi * 3 * t)) + g.normal(0, 0.05, L_)
    return (np.clip(np.round(x * 32768), -32768, 32767) / 32768).astype(np.float32)


def _rir(lh, kind, seed):
    g = np.random.default_rng(seed)
    h = g.normal(size=lh)
    if kind == "decay":
        h *= np.exp(-np.arange(lh) / 800.0)       # 50 ms decay constant at 16 kHz
    return (h / np.linalg.norm(h)).astype(np.float32)


@pytest.mark.parametrize("kind", ["flat", "decay"])
@pytest.mark.parametrize("L_,lh", [(25840, 16000), (25840, 1025), (4096, 8000), (3000, 2048)])
def test_reverb_checker_passes_the_fp32_emulation_and_fails_seeded_defects(kind, L_, lh):
    s, h = _speech(L_, lh), _rir(lh, kind, L_)
    r, _, _ = A.partitioned_convolve(s, h)
    elem, blk = A.reverb_error_ratios(r, s, h)
    assert elem <= 1.0 and blk <= 1.0, (elem, blk)
    for defect in A.DEFECTS:
        rd, _, _ = A.partitioned_convolve(s, h, defect=defect)
        elem, blk = A.reverb_error_ratios(rd, s, h)
        assert elem > 1.0 and blk > 1.0, (defect, elem, blk)
