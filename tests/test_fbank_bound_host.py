"""The log-fbank gate of tests/fbank_bound.py on the CPU: an fp32 numpy emulation of ``fbank_kernel`` with its operation
order passes it on every signal of the GPU test, and eight seeded defects each fail it; the filterbank facts the signals
rely on; and the sample rates every fbank entry point accepts."""
import ctypes

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import frontend as F
from oracle import fbank_oracle as FO
from tests import fbank_bound as FB

RATES = (50, 100, 8000, 11025, 12000, 16000, 20499)
f32 = np.float32


def _bitrev9(i):
    return int(f"{i:09b}"[::-1], 2)


REV = np.array([_bitrev9(i) for i in range(FB.NFFT)])


def _twiddles(half, defect):
    """fp32 (cos, sin) of -pi pos / half, correctly rounded (within the kernel's 1-ulp sincospif)."""
    pos = np.arange(half)
    th = -np.pi * pos / half
    cs, sn = np.cos(th), np.sin(th)
    if defect == "twiddle_2^-11":                       # twiddles accurate to 2^-11 only
        cs, sn = np.round(cs * 2048) / 2048, np.round(sn * 2048) / 2048
    return cs.astype(f32), sn.astype(f32)


def emulate(audio, lengths, sr, defect=None):
    """fp32 emulation of dsk_fbank_batch(_vad) on the concatenated ``audio`` -> per utterance a dict of 'lin', 'log'
    (un-subtracted), 'lin_sub', 'log_sub' (F, 64) and 'energy' (F,)."""
    flen, step = FB.geometry(sr)
    W32 = FB.filterbank(sr).astype(f32)
    if defect == "mel_skips_last_weight":
        for j in range(FB.NMEL):
            nz = np.flatnonzero(W32[j])
            if nz.size:
                W32[j, nz[-1]] = 0
    W64 = W32.astype(np.float64)
    a = f32(0.97)
    soff = np.concatenate(([0], np.cumsum(lengths)))
    out = []
    for u, n in enumerate(lengths):
        nf = FB.num_frames(n, sr)
        s = np.arange(nf)[:, None] * step + np.arange(flen)[None, :]
        gidx = soff[u] + s
        live = s < n if defect != "reads_past_end" else gidx < audio.size
        gi = np.minimum(gidx, audio.size - 1)
        prev = np.where(s > 0, audio[np.maximum(gi - 1, 0)], f32(0))
        if defect == "preemph_frame_start":             # x[s-1] taken as 0 at each frame's first sample
            prev[:, 0] = 0
        v = np.where(s == 0, audio[gi], audio[gi] - a * prev).astype(f32)
        v = np.where(live, v, f32(0))
        re = np.zeros((nf, FB.NFFT), f32)
        re[:, REV[:flen]] = v
        im = np.zeros_like(re)
        for st in range(1, 10):
            half = 1 << (st - 1)
            b = np.arange(FB.NFFT // 2)
            grp, pos = b // half, b % half
            i0 = grp * 2 * half + pos
            i1 = i0 + half
            cs, sn = _twiddles(half, defect)
            cs, sn = cs[pos], sn[pos]
            if defect == "last_stage_sine_sign" and st == 9:
                sn = sn.copy()
                sn[37] = -sn[37]
            ax, ay, cx, cy = re[:, i0], im[:, i0], re[:, i1], im[:, i1]
            wx = cx * cs - cy * sn
            wy = cx * sn + cy * cs
            re[:, i0], im[:, i0] = ax + wx, ay + wy
            re[:, i1], im[:, i1] = ax - wx, ay - wy
        zr, zi = re[:, :FB.BINS], im[:, :FB.BINS]
        p = (zr * zr + zi * zi) * f32(1.0 / FB.NFFT)
        acc = np.zeros((nf, FB.NMEL), f32)
        p64 = p.astype(np.float64)
        for k in range(FB.BINS):                         # fmaf(p_k, w_k, acc): the product is exact in fp64
            acc = (acc.astype(np.float64) + p64[:, k:k + 1] * W64[None, :, k]).astype(f32)
        e = np.zeros(nf, f32)
        for k in range(FB.BINS - (defect == "energy_drops_nyquist")):
            e = e + p[:, k]
        e = np.where(e == 0, f32(FB.EPS32), e)
        lin = acc if defect == "no_eps" else np.where(acc == 0, f32(FB.EPS32), acc)
        log = (f32(20) * np.log10(np.maximum(lin, f32(1e-5)).astype(np.float64)).astype(f32)).astype(f32)
        res = {"lin": lin, "log": log, "energy": e}
        for key in ("lin", "log"):
            g = res[key]
            nblk = -(-nf // 4)
            rows = np.zeros((nblk * 4, FB.NMEL), f32)
            rows[:nf] = g
            part = np.zeros((nblk, FB.NMEL), f32)
            for r in range(4):
                part = part + rows[r::4]
            div = nblk * 4 if defect == "mean_rounds_count_up" else nf
            mean = (part.astype(np.float64).sum(0) / div).astype(f32)
            res[key + "_sub"] = g - mean
        out.append(res)
    return out


def ratios(utts, sr, res):
    """Max err / bound per stage over the batch."""
    worst = {}
    for (_, x), r in zip(utts, res):
        R = FB.Reference(x, sr)
        for stage, val in (("mel", FB.mel_ratio(r["lin"], R)), ("log", FB.log_ratio(r["log"], R)),
                           ("mean_lin", FB.mean_ratio(r["lin_sub"], r["lin"])),
                           ("mean_log", FB.mean_ratio(r["log_sub"], r["log"])),
                           ("energy", FB.energy_ratio(r["energy"], R)), ("power_iso", FB.iso_ratio(r["lin"], R))):
            worst[stage] = max(worst.get(stage, 0.0), float(val.max()) if val.size else 0.0)
    return worst


def _run(sr, defect=None):
    utts = FB.batch(sr, long=False)
    audio = np.concatenate([x for _, x in utts])
    return ratios(utts, sr, emulate(audio, [x.size for _, x in utts], sr, defect))


@pytest.mark.parametrize("sr", RATES)
def test_the_emulated_kernel_passes_the_gate(sr):
    worst = _run(sr)
    print(f"\n{sr} Hz emulation, max err/bound: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("defect,stages", [
    ("preemph_frame_start", ("mel", "log")),
    ("reads_past_end", ("mel", "log")),
    ("last_stage_sine_sign", ("mel", "log")),
    ("twiddle_2^-11", ("mel", "log")),
    ("mel_skips_last_weight", ("mel", "log")),
    ("mean_rounds_count_up", ("mean_lin", "mean_log")),
    ("energy_drops_nyquist", ("energy",)),
    ("no_eps", ("mel",)),
])
def test_each_seeded_defect_fails_the_gate(defect, stages):
    worst = _run(16000, defect)
    print(f"\n{defect}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert all(worst[s] > 1.0 for s in stages), (defect, worst)


@pytest.mark.parametrize("sr", RATES)
def test_filterbank_facts_the_signals_rely_on(sr):
    W = FB.filterbank(sr)
    assert np.all(W[:, 256] == 0)                       # only the energy sees the Nyquist bin
    if sr in (8000, 16000):
        assert W[:, 0].any() == (sr == 16000)            # bin 0 (DC) is in filter 0 at 16 kHz only
    lib = L.load()
    fb = np.empty((64, 257), np.float32)
    assert lib.dsk_fbank_filterbank(sr, fb.ctypes.data_as(ctypes.c_void_p)) == 0
    assert np.array_equal(fb, W.astype(np.float32))


def test_isolated_filters_at_16k():
    iso = FB.isolated_filters(16000)
    assert len(iso) >= 1 and all(FB.filterbank(16000)[j, k] == 1.0 for j, k in iso)


REJECTED = (1, 19, 20, 49, 20500, 0, -16000)


def test_sample_rates_outside_50_to_20499_are_rejected_by_every_entry_point():
    lib = L.load()
    d = np.zeros(4096, np.int64)
    p = d.ctypes.data_as(ctypes.c_void_p)
    soff = np.array([0, 1000, 3000], np.int64)
    foff = np.full(3, -7, np.int64)
    po, pf = soff.ctypes.data_as(ctypes.c_void_p), foff.ctypes.data_as(ctypes.c_void_p)
    for sr in REJECTED:
        assert lib.dsk_fbank_num_frames(1000, sr) == 0, sr
        # pointers to host memory: a call that got past the checks would fail on the device, not with DSK_ERR_INVALID
        calls = {
            "dsk_fbank_frame_offsets": lambda: lib.dsk_fbank_frame_offsets(po, 2, sr, pf),
            "dsk_fbank_filterbank": lambda: lib.dsk_fbank_filterbank(sr, p),
            "dsk_fbank": lambda: lib.dsk_fbank(p, 1000, sr, 1, 1, p, None),
            "dsk_fbank_batch": lambda: lib.dsk_fbank_batch(p, po, 2, sr, 1, 1, p, None),
            "dsk_fbank_batch_vad": lambda: lib.dsk_fbank_batch_vad(p, po, 2, sr, 1, 1, -5.0, 0.5, 2, 0.12, p, p, p, None),
            "dsk_fbank_segments": lambda: lib.dsk_fbank_segments(p, 2, 1000, sr, 1, 1, p, None, 0, None, 0, p, None),
        }
        for name, call in calls.items():
            assert call() == -1, (name, sr)                                    # DSK_ERR_INVALID
            assert b"sample_rate must lie in [50, 20499] Hz" in lib.dsk_last_error(), (name, sr)
        assert np.all(foff == -7)
        for fn in (lambda: F.segment_samples(160, sr), lambda: F.fbank_frame_offsets([1000], sr),
                   lambda: F.mk_mfb_batch(torch.zeros(1000), [1000], sr),
                   lambda: F.WaveBank.augmented_crops(None, [0], [0], 160, sample_rate=sr)):   # checked before the bank
            with pytest.raises(ValueError, match=r"\[50, 20499\]"):
                fn()


@pytest.mark.parametrize("sr", [50, 20499])
def test_sample_rates_at_the_ends_of_the_header_range_are_accepted(sr):
    lib = L.load()
    flen, step = FB.geometry(sr)
    assert (flen, step) == {50: (1, 1), 20499: (512, 205)}[sr]
    lens = np.array([1, flen - 1, flen, flen + 1, flen + step, 1000, 100003])
    lens = lens[lens >= 1]
    for n in lens:
        want = 1 if n <= flen else 1 + int(np.ceil((n - flen) / step))
        assert lib.dsk_fbank_num_frames(int(n), sr) == want == FB.num_frames(int(n), sr), (sr, n)
        assert FO.fbank(np.full(int(n), 1e-3, np.float32), samplerate=sr, nfilt=64)[0].shape[0] == want
    foff = F.fbank_frame_offsets(lens, sr)
    assert np.array_equal(np.diff(foff), [FB.num_frames(int(n), sr) for n in lens])
    assert lib.dsk_fbank_num_frames(F.segment_samples(160, sr), sr) == 160
    # the range is exactly the rates with a step of at least one sample and a frame of at most 512
    ok = [r for r in range(1, 30000) if FB.geometry(r)[1] >= 1 and FB.geometry(r)[0] <= 512]
    assert (ok[0], ok[-1], len(ok)) == (L.DSK_FBANK_MIN_RATE, L.DSK_FBANK_MAX_RATE,
                                        L.DSK_FBANK_MAX_RATE - L.DSK_FBANK_MIN_RATE + 1)
