"""Feature-bank front-end, host side: frame offsets of a batch, sliding windows, crop starts and SpecAugment masks.
No GPU needed."""
import math

import numpy as np
import pytest

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import frontend as F
from oracle import fbank_oracle as FO


def _lengths(sr):
    flen, step = FO.round_half_up(0.025 * sr), FO.round_half_up(0.01 * sr)
    return [1, flen - 1, flen, flen + 1, flen + step, 3 * sr + 7, 16000, 48000, 100003]


@pytest.mark.parametrize("sr", [8000, 16000])
def test_frame_offsets_match_the_single_utterance_count(sr):
    lib = L.load()
    lens = _lengths(sr)
    off = F.fbank_frame_offsets(lens, sr)
    want = np.concatenate(([0], np.cumsum([lib.dsk_fbank_num_frames(n, sr) for n in lens])))
    assert off.dtype == np.int64 and np.array_equal(off, want)
    flen, step = FO.round_half_up(0.025 * sr), FO.round_half_up(0.01 * sr)
    assert np.array_equal(np.diff(off), [1 if n <= flen else 1 + int(math.ceil((n - flen) / step)) for n in lens])


def test_frame_offsets_reject_a_zero_length():
    with pytest.raises(ValueError):
        F.fbank_frame_offsets([400, 0, 16000], 16000)
    with pytest.raises(ValueError):
        F.fbank_frame_offsets([], 16000)
    # the C entry point itself, without the Python check
    lib = L.load()
    soff = np.array([0, 400, 400, 16400], np.int64)
    foff = np.zeros(4, np.int64)
    assert lib.dsk_fbank_frame_offsets(F._ptr64(soff), 3, 16000, F._ptr64(foff)) < 0
    assert b"utterance 1" in lib.dsk_last_error()
    assert lib.dsk_fbank_batch(None, F._ptr64(soff), 3, 16000, 1, 1, None, None) < 0
    assert lib.dsk_fbank_crops(None, None, 1, None, None, 1, 1, None, 0, None, 0, None, None) < 0


@pytest.mark.parametrize("T,hop", [(160, 80), (160, 160), (160, 37), (7, 3), (5, 1)])
def test_windows_cover_every_frame(T, hop):
    rng = np.random.default_rng(T * 1000 + hop)
    lens = np.concatenate(([1, T - 1, T, T + 1, T + hop, T + hop - 1, 2 * T, 2 * T + 1], rng.integers(1, 2000, 200)))
    utt = rng.permutation(lens.size)[:150]
    wu, ws, wo = F.sliding_windows(lens, utt, T, hop)
    wu, ws, wo = wu.numpy(), ws.numpy(), wo.numpy()
    assert wo[0] == 0 and wo[-1] == wu.size == ws.size and np.all(np.diff(wo) >= 1)
    for i, u in enumerate(utt):
        n = lens[u]
        st = ws[wo[i]:wo[i + 1]]
        assert np.all(wu[wo[i]:wo[i + 1]] == u)
        if n < T:
            assert st.tolist() == [0]
            continue
        covered = np.zeros(n, bool)
        for s in st:
            assert 0 <= s <= n - T
            covered[s:s + T] = True
        assert covered.all(), (n, st)
        assert st[0] == 0 and st[-1] + T == n
        assert np.all(np.diff(st) >= 1) and np.all(np.diff(st) <= hop)
        brute = list(range(0, n - T + 1, hop))
        if brute[-1] != n - T:
            brute.append(n - T)
        assert st.tolist() == brute


def test_random_starts_in_bounds_and_reproducible():
    rng = np.random.default_rng(0)
    lens = np.concatenate(([1, 159, 160, 161], rng.integers(1, 2000, 500)))
    utt = rng.integers(0, lens.size, 4000)
    a = F.random_starts(lens, utt, 160, np.random.default_rng(7)).numpy()
    b = F.random_starts(lens, utt, 160, np.random.default_rng(7)).numpy()
    assert a.dtype == np.int64 and np.array_equal(a, b)
    hi = np.maximum(lens[utt] - 160, 0)
    assert np.all(a >= 0) and np.all(a <= hi)
    assert np.all(a[lens[utt] <= 160] == 0)
    # the last start n - T is reachable (the reference's randrange(9, n - 23) never picks it)
    one = F.random_starts([170], np.zeros(20000, np.int64), 160, np.random.default_rng(1)).numpy()
    assert set(one.tolist()) == set(range(11))
    with pytest.raises(ValueError):
        F.random_starts(lens, [lens.size], 160, np.random.default_rng(0))


def test_spec_augment_masks_in_bounds_and_reproducible():
    tm, fm = F.spec_augment_masks(384, 160, 2, 20, 3, 8, np.random.default_rng(3))
    tm2, fm2 = F.spec_augment_masks(384, 160, 2, 20, 3, 8, np.random.default_rng(3))
    assert tm.shape == (384, 2, 2) and fm.shape == (384, 3, 2)
    assert str(tm.dtype) == "torch.int32" and str(fm.dtype) == "torch.int32"
    assert np.array_equal(tm.numpy(), tm2.numpy()) and np.array_equal(fm.numpy(), fm2.numpy())
    for m, mx, ext in ((tm.numpy(), 20, 160), (fm.numpy(), 8, 64)):
        s, w = m[..., 0], m[..., 1]
        assert w.min() == 0 and w.max() == mx                     # both ends of [0, max] are drawn
        assert s.min() >= 0 and np.all(s + w <= ext)
    tm0, fm0 = F.spec_augment_masks(4, 160, 0, 20, 0, 8, np.random.default_rng(0))
    assert tm0.shape == (4, 0, 2) and fm0.shape == (4, 0, 2)
    with pytest.raises(ValueError):
        F.spec_augment_masks(4, 160, 1, 161, 1, 8)
    with pytest.raises(ValueError):
        F.spec_augment_masks(4, 160, 1, 10, 1, 65)


def test_bank_needs_cuda_features():
    import torch

    with pytest.raises(RuntimeError):
        F.FeatureBank(torch.zeros(10, 64), [0, 4, 10])
    with pytest.raises(RuntimeError):
        F.mk_mfb_batch(torch.zeros(100), [100])
