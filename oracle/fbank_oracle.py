"""CPU restatement of the reference's log-fbank front-end - TEST INFRASTRUCTURE ONLY.

reference audio_processing.py:9-36 (`mk_MFB`) calls ``python_speech_features.fbank`` (package not vendored in the
reference, no pinned version, absent from this image: **parity against the package itself is unpinned**).  Its published
algorithm (python_speech_features 0.6, base.py ``fbank`` / ``get_filterbanks`` and sigproc.py ``preemphasis`` /
``framesig`` / ``powspec``) is restated here in numpy with the same operation order and dtypes (float64 from the framing
on), followed by the reference's own ``20*log10(max(., 1e-5))`` (:16-17) and ``normalize_frames(Scale=False)`` (:29,88-92).
"""
import decimal
import math

import numpy as np


def round_half_up(number):
    return int(decimal.Decimal(number).quantize(decimal.Decimal("1"), rounding=decimal.ROUND_HALF_UP))


def hz2mel(hz):
    return 2595 * np.log10(1 + hz / 700.0)


def mel2hz(mel):
    return 700 * (10 ** (mel / 2595.0) - 1)


def get_filterbanks(nfilt=20, nfft=512, samplerate=16000, lowfreq=0, highfreq=None):
    highfreq = highfreq or samplerate / 2
    melpoints = np.linspace(hz2mel(lowfreq), hz2mel(highfreq), nfilt + 2)
    bin = np.floor((nfft + 1) * mel2hz(melpoints) / samplerate)
    fbank = np.zeros([nfilt, nfft // 2 + 1])
    for j in range(0, nfilt):
        for i in range(int(bin[j]), int(bin[j + 1])):
            fbank[j, i] = (i - bin[j]) / (bin[j + 1] - bin[j])
        for i in range(int(bin[j + 1]), int(bin[j + 2])):
            fbank[j, i] = (bin[j + 2] - i) / (bin[j + 2] - bin[j + 1])
    return fbank


def fbank(signal, samplerate=16000, winlen=0.025, winstep=0.01, nfilt=26, nfft=512, lowfreq=0, highfreq=None, preemph=0.97):
    """python_speech_features.fbank with its default rectangular window.  Returns (features, energy)."""
    signal = np.append(signal[0], signal[1:] - preemph * signal[:-1])            # sigproc.preemphasis
    frame_len, frame_step = round_half_up(winlen * samplerate), round_half_up(winstep * samplerate)
    slen = len(signal)
    numframes = 1 if slen <= frame_len else 1 + int(math.ceil((1.0 * slen - frame_len) / frame_step))
    padlen = int((numframes - 1) * frame_step + frame_len)
    padsignal = np.concatenate((signal, np.zeros((padlen - slen,))))            # float64 from here on
    idx = np.tile(np.arange(0, frame_len), (numframes, 1)) + np.tile(np.arange(0, numframes * frame_step, frame_step), (frame_len, 1)).T
    frames = padsignal[idx.astype(np.int32)]
    pspec = 1.0 / nfft * np.square(np.absolute(np.fft.rfft(frames, nfft)))       # sigproc.powspec
    energy = np.sum(pspec, 1)
    energy = np.where(energy == 0, np.finfo(float).eps, energy)
    feat = np.dot(pspec, get_filterbanks(nfilt, nfft, samplerate, lowfreq, highfreq).T)
    feat = np.where(feat == 0, np.finfo(float).eps, feat)
    return feat, energy


def mk_mfb(audio, sample_rate=16000, use_logscale=True):
    """audio_processing.py:9-36 with the reference's constants (FILTER_BANK 64, USE_LOGSCALE, no delta, no scale)."""
    fb, _ = fbank(np.asarray(audio), samplerate=sample_rate, nfilt=64, winlen=0.025)
    if use_logscale:
        fb = 20 * np.log10(np.maximum(fb, 1e-5))
    return fb - np.mean(fb, axis=0)
