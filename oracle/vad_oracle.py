"""Oracle for the frame-energy VAD, the runs of kept frames and the speech-only diarization assembly (tests only; numpy
fp64, no GPU).

  * ``decide``: the decision rule of include/dsk.h (Kaldi's compute-vad restated) on given frame energies, vectorised;
    ``decide_brute`` is the same rule frame by frame.  ``vad`` feeds ``decide`` the fp64 energies of
    ``fbank_oracle.fbank``.
  * ``runs_brute`` / ``select_brute``: the runs of kept frames and the selected bank, by loops.
  * ``frame_labels_runs_brute``: per-run frame labels (``ahc_oracle.frame_labels_brute`` on every run), -1 elsewhere.
"""
from __future__ import annotations

import numpy as np

from oracle import ahc_oracle, fbank_oracle

DEFAULT_ENERGY_THRESHOLD = 5.5 - 0.5 * np.log(2.0 ** 31)
DEFAULTS = {"energy_threshold": DEFAULT_ENERGY_THRESHOLD, "mean_scale": 0.5, "context": 2, "proportion": 0.12}


def decide(energy, offsets, energy_threshold=DEFAULT_ENERGY_THRESHOLD, mean_scale=0.5, context=2, proportion=0.12):
    """(speech (F,) bool, thr (U,) fp64, ln E (F,) fp64) of the frame energies ``energy`` (F,) of the utterances
    ``offsets`` (U + 1)."""
    E = np.asarray(energy, np.float64).reshape(-1)
    off = np.asarray(offsets, np.int64)
    le = np.log(E)
    speech = np.zeros(E.size, bool)
    thr = np.empty(off.size - 1)
    c = int(context)
    for u in range(off.size - 1):
        a, b = int(off[u]), int(off[u + 1])
        e = le[a:b]
        n = b - a
        thr[u] = energy_threshold + mean_scale * (np.sum(e) / n)
        cum = np.concatenate(([0], np.cumsum(e > thr[u])))
        f = np.arange(n)
        lo, hi = np.maximum(f - c, 0), np.minimum(f + c, n - 1)
        speech[a:b] = (cum[hi + 1] - cum[lo]).astype(np.float64) >= proportion * (hi - lo + 1).astype(np.float64)
    return speech, thr, le


def decide_brute(energy, offsets, energy_threshold=DEFAULT_ENERGY_THRESHOLD, mean_scale=0.5, context=2,
                 proportion=0.12):
    E = [float(x) for x in np.asarray(energy, np.float64).reshape(-1)]
    off = [int(x) for x in offsets]
    out = []
    for u in range(len(off) - 1):
        e = [float(np.log(x)) for x in E[off[u]:off[u + 1]]]
        n = len(e)
        thr = energy_threshold + mean_scale * (sum(e) / n)
        for f in range(n):
            win = [g for g in range(n) if abs(g - f) <= context]
            votes = sum(1 for g in win if e[g] > thr)
            out.append(votes >= proportion * len(win))
    return np.array(out, bool)


def vad(signal, samplerate=16000, **params):
    """(speech, thr, ln E) of one waveform from the fp64 energies of ``fbank_oracle.fbank``."""
    _, E = fbank_oracle.fbank(np.asarray(signal), samplerate=samplerate, nfilt=64, winlen=0.025)
    return decide(E, [0, E.size], **{**DEFAULTS, **params})


def runs_brute(mask, offsets, utt):
    """[(j, first, end)]: the runs of kept frames of the utterances utt[j], in list order."""
    m = np.asarray(mask, bool)
    off = np.asarray(offsets, np.int64)
    out = []
    for j, u in enumerate(utt):
        a, b = int(off[u]), int(off[u + 1])
        f = 0
        while f < b - a:
            if m[a + f]:
                g = f
                while g < b - a and m[a + g]:
                    g += 1
                out.append((j, f, g))
                f = g
            else:
                f += 1
    return out


def select_brute(feats, offsets, mask):
    """(rows, offsets) of each utterance's kept rows, in order."""
    m = np.asarray(mask, bool)
    off = np.asarray(offsets, np.int64)
    rows, new = [], [0]
    for u in range(off.size - 1):
        keep = [i for i in range(int(off[u]), int(off[u + 1])) if m[i]]
        rows.extend(keep)
        new.append(new[-1] + len(keep))
    return np.asarray(feats)[rows], np.array(new, np.int64)


def frame_labels_runs_brute(runs, run_win_start, run_win_labels, n_frames, T):
    """(n_frames,) int32: frames of run (first, end) labelled by ``ahc_oracle.frame_labels_brute`` over that run's
    windows (starts relative to the run), every other frame -1."""
    out = np.full(n_frames, -1, np.int32)
    for (first, end), ws, wl in zip(runs, run_win_start, run_win_labels):
        out[first:end] = ahc_oracle.frame_labels_brute(ws, wl, end - first, T)
    return out
