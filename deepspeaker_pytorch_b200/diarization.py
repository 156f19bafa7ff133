"""Speaker diarization: who spoke when in one recording.

``diarize`` embeds the sliding windows of every recording with the eval forward (one batched pass over all of them,
``frontend.window_embeddings``), builds each recording's window-by-window cosine matrix on the tensor cores
(``engine.cosine_matrix``) and clusters it by agglomerative clustering on the device (``engine.ahc``, average linkage
by default), cut at a known number of speakers or at a distance threshold.  Each 10 ms frame then takes the speaker of
the covering window whose centre is nearest, and runs of equal frame labels become segments.  ``to_rttm`` writes them
in the RTTM format scoring tools read.

With ``plda`` (a fitted ``plda.PLDA`` backend) the affinity is the PLDA log-likelihood ratio of the windows instead of
their cosine, as in the Kaldi diarization recipe.

With ``speech`` (an (F,) mask over the bank's rows: ``bank.speech`` from the frame-energy VAD of
``FeatureBank.from_waveforms(..., vad={})``, or oracle speech from reference annotations) only speech is diarized: every
run of speech frames is cut into windows of its own (``FeatureBank.runs``; a run shorter than T gets one window that
wraps inside the run), all windows of a recording are clustered together, each speech frame takes the label of the
nearest window centre within its run and every other frame is -1, which no segment or RTTM line covers.  Without it,
every frame gets a speaker, silence included.

With ``plda`` and ``vbx`` (a dict of ``vbx`` options, ``{}`` for the defaults) the AHC labels are only the start:
``vbx`` refines every recording's window labels with VBx, a variational-Bayes HMM whose states are speakers and whose
emission model is the PLDA itself (Landini et al., 2022), so neighbouring windows tend to share a speaker and surplus
initial clusters lose their windows.  ``der`` scores per-frame labels against a reference.

With ``spectral`` (a dict of ``spectral`` options, ``{}`` for the defaults) every recording is clustered by spectral
clustering instead of AHC, with the number of speakers estimated by the normalised maximum eigengap (NME-SC, Park et
al., IEEE SPL 2020) unless ``num_speakers`` fixes it: no threshold and no PLDA are needed, since NME-SC reads only
the ranks of each window's affinities (cosines, or PLDA LLRs with ``plda``).  ``engine.spectral_cluster`` solves the
eigenproblems of every pruning level of the grid in one call on the device.

Overlapped speech and re-segmentation are not part of this module: a frame gets at most one speaker.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import _lib as L
from . import engine
from . import frontend

FRAME_SHIFT_S = 0.01   # the fbank's 10 ms frame shift, at every sample rate
MAX_WINDOWS = L.DSK_AHC_MAX_N


class Recording(NamedTuple):
    """The diarization of one recording: ``segments`` [(start_s, end_s, speaker)], ``frame_labels`` (n_frames,)
    int32, ``window_labels`` (W,) int32 and ``Z`` the linkage matrix of the windows (scipy's format; the first rows of
    the full tree)."""
    segments: list
    frame_labels: np.ndarray
    window_labels: np.ndarray
    Z: np.ndarray


def frame_labels(win_start, win_labels, n_frames: int, T: int) -> np.ndarray:
    """Host: (n_frames,) int32, frame f taking the label of the covering window whose centre is nearest to the frame's
    centre, ties to the earlier window.  Windows start at ``win_start`` (ascending, as ``frontend.sliding_windows``
    gives them, so every frame is covered) and span T frames; a recording shorter than T has one window.  With equal
    window lengths the nearest centre overall covers the frame, so a search over the centres suffices."""
    s = np.asarray(win_start, np.int64).reshape(-1)
    lab = np.asarray(win_labels).reshape(-1)
    if s.size == 0 or s.size != lab.size:
        raise ValueError(f"frame_labels: {s.size} window starts for {lab.size} labels")
    c2 = 2 * s + int(T)                                # doubled centres, in half frames
    q = 2 * np.arange(int(n_frames), dtype=np.int64) + 1
    hi = np.clip(np.searchsorted(c2, q, side="left"), 0, s.size - 1)
    lo = np.clip(hi - 1, 0, s.size - 1)
    w = np.where(np.abs(q - c2[lo]) <= np.abs(c2[hi] - q), lo, hi)
    return lab[w].astype(np.int32)


def segments(labels, frame_shift: float = FRAME_SHIFT_S) -> list:
    """Host: runs of equal frame labels -> [(start_s, end_s, speaker)]; frame f covers [f, f + 1) * frame_shift."""
    lab = np.asarray(labels).reshape(-1)
    if lab.size == 0:
        return []
    cut = np.flatnonzero(lab[1:] != lab[:-1]) + 1
    starts = np.concatenate(([0], cut))
    ends = np.concatenate((cut, [lab.size]))
    return [(float(a * frame_shift), float(b * frame_shift), int(lab[a])) for a, b in zip(starts, ends)]


def to_rttm(segs, recording_id: str) -> str:
    """RTTM ``SPEAKER`` lines (one per segment, newline-terminated): onset and duration in seconds to the millisecond,
    speaker ``spk<label>``."""
    rid = str(recording_id)
    if not rid or any(ch.isspace() for ch in rid):
        raise ValueError(f"to_rttm: the recording id must be non-empty without white space, got {rid!r}")
    return "".join(f"SPEAKER {rid} 1 {a:.3f} {b - a:.3f} <NA> <NA> spk{k} <NA> <NA>\n" for a, b, k in segs)


class VBxResult(NamedTuple):
    """The VBx refinement of R recordings' windows: ``labels`` (W,) int32 numpy, renumbered per recording in the order
    of first window (-1 for a recording with a non-finite embedding); ``gamma`` (W, S) and ``pi`` (R, S) fp64, ``elbo``
    (R, max_iters) fp64 (NaN past a recording's last iteration) and ``iters`` (R,) int32, device tensors whose speaker
    columns are the initial labels' (not renumbered)."""
    labels: np.ndarray
    gamma: torch.Tensor
    pi: torch.Tensor
    elbo: torch.Tensor
    iters: torch.Tensor


VBX_OPTIONS = ("Fa", "Fb", "loop_p", "init_smoothing", "max_iters", "epsilon")


def _plda_space(plda, E):
    """The PLDA-space rows P (y - m_bar) of raw embeddings E, y their length-normalised LDA outputs (PLDA.transform
    without the scoring normalisation)."""
    m = plda._on(E.device)
    y = engine.affine_norm_f64(E, m["lda"], m["mu"], mode="length")
    return engine.affine_norm_f64(y, m["plda_transform"], m["plda_mean"], mode="none")


def _renumber(labels, offsets):
    """Labels renumbered per recording offsets[r] .. offsets[r + 1] in the order of first appearance; -1 stays."""
    out = np.asarray(labels, np.int32).copy()
    for a, b in zip(offsets[:-1], offsets[1:]):
        seg = out[a:b]
        keep = seg >= 0
        _, first, inv = np.unique(seg[keep], return_index=True, return_inverse=True)
        seg[keep] = np.argsort(np.argsort(first))[inv]
    return out


def vbx(plda, E, offsets, init_labels, Fa: float = 0.3, Fb: float = 17.0, loop_p: float = 0.99,
        init_smoothing: float = 5.0, max_iters: int = 40, epsilon: float = 1e-4) -> VBxResult:
    """Refine the initial speaker labels of the window embeddings E (W, D) (raw, a CUDA tensor) of R recordings
    (``offsets`` (R + 1,): recording r is rows offsets[r] .. offsets[r + 1], in time order) with VBx on the PLDA
    model ``plda``.  ``init_labels`` (W,): each recording's initial clusters numbered from 0 (``engine.ahc`` labels,
    over-clustered), at most DSK_VBX_MAX_SPEAKERS per recording.

    The rows are taken into the PLDA space without the scoring normalisation, where the within-speaker covariance is
    I and the across-speaker one diag(psi); ``engine.vbx`` then runs the iteration of oracle/vbx_oracle.py on all
    recordings in one call.  Fa scales the acoustic likelihoods, Fb the speaker-model prior, loop_p is the
    probability of staying with the same speaker from one window to the next, init_smoothing the softmax temperature
    of the initial labels; a recording stops when its ELBO gains less than epsilon.  The defaults are starting values
    common in the VBx literature for x-vectors every 0.25 s; they are NOT tuned for this model or for other hops."""
    if not isinstance(E, torch.Tensor) or not E.is_cuda:
        raise RuntimeError("vbx needs a CUDA embedding tensor; there is no CPU fallback")
    off = np.asarray(offsets, np.int64).reshape(-1)
    X = _plda_space(plda, E)
    gamma, pi, elbo, iters, lab = engine.vbx(X, off, init_labels, plda._on(E.device)["psi"], Fa, Fb, loop_p,
                                             init_smoothing, max_iters, epsilon)
    return VBxResult(_renumber(lab.cpu().numpy(), off), gamma, pi, elbo, iters)


class DER(NamedTuple):
    """``der``'s result: fractions of the reference's speech frames, and the speaker mapping."""
    der: float
    miss: float
    false_alarm: float
    confusion: float
    mapping: dict


def der(ref, hyp):
    """Host: the frame-level diarization error of per-frame labels ``hyp`` against ``ref`` (equal lengths; -1 is
    non-speech) -> (der, miss, false_alarm, confusion, mapping): the three errors are fractions of the reference's
    speech frames and der is their sum; mapping {hyp speaker: ref speaker} is the one-to-one mapping that maximises the
    frames both label alike (Hungarian algorithm), listing matched pairs that share frames.

    Frames are scored one speaker each, with no forgiveness collar around reference boundaries: this is NOT the
    md-eval / dscore DER (no collar, no overlap, 10 ms frames).  ValueError on a length mismatch or a reference without
    speech."""
    from scipy.optimize import linear_sum_assignment

    r = np.asarray(ref).reshape(-1)
    h = np.asarray(hyp).reshape(-1)
    if r.size != h.size:
        raise ValueError(f"der: {r.size} reference frames and {h.size} hypothesis frames")
    speech = r >= 0
    n = int(speech.sum())
    if n == 0:
        raise ValueError("der: the reference has no speech")
    miss = int((speech & (h < 0)).sum())
    fa = int((~speech & (h >= 0)).sum())
    both = speech & (h >= 0)
    r_ids, ri = np.unique(r[both], return_inverse=True)
    h_ids, hi = np.unique(h[both], return_inverse=True)
    C = np.zeros((h_ids.size, r_ids.size), np.int64)
    np.add.at(C, (hi, ri), 1)
    rows, cols = linear_sum_assignment(C, maximize=True)
    conf = int(both.sum()) - int(C[rows, cols].sum())
    mapping = {int(h_ids[i]): int(r_ids[j]) for i, j in zip(rows, cols) if C[i, j] > 0}
    return DER((miss + fa + conf) / n, miss / n, fa / n, conf / n, mapping)


class SpectralResult(NamedTuple):
    """``spectral``'s result: ``labels`` (N,) int32 device tensor numbered by each cluster's smallest member, ``k`` the
    number of speakers, ``p`` the index of the chosen pruning level into ``p_values`` (None when no eigenproblem was
    solved), ``eigenvalues`` (n_p, m) fp64 the m smallest eigenvalues of every level's Laplacian, ``lambda_max`` and
    ``ratio`` (n_p,) its largest eigenvalue and NME ratio r_p."""
    labels: torch.Tensor
    k: int
    p: int
    p_values: np.ndarray
    eigenvalues: np.ndarray
    lambda_max: np.ndarray
    ratio: np.ndarray


SPECTRAL_OPTIONS = ("max_speakers", "p_max_frac", "p_steps", "kmeans_iters")


def p_grid(N: int, p_max_frac: float = 0.25, p_steps: int = 30) -> np.ndarray:
    """The pruning levels tried for N items: the unique integers of linspace(1, max(1, floor(p_max_frac (N - 1))),
    p_steps)."""
    top = max(1, int(np.floor(float(p_max_frac) * (int(N) - 1))))
    return np.unique(np.linspace(1, top, int(p_steps)).astype(np.int64))


def spectral(S, max_speakers: int = 8, num_speakers=None, p_max_frac: float = 0.25, p_steps: int = 30,
             kmeans_iters: int = 100) -> SpectralResult:
    """Spectral clustering of N items from their similarities S (N, N) fp32 CUDA (cosines or PLDA LLRs; only each
    row's ranks matter) with NME-SC speaker counting (oracle/spectral_oracle.py): for every pruning level p of
    ``p_grid(N, p_max_frac, p_steps)`` the graph keeping each item's p nearest neighbours, the eigengap count and the
    NME ratio r_p; the level of least r_p gives the count (at most ``max_speakers``, or ``num_speakers`` when given)
    and the k-means partition of its spectral embedding.  ``num_speakers >= N`` gives one speaker per item without
    solving anything; a count or ``max_speakers`` above DSK_SC_MAX_SPEAKERS (32) is otherwise a ValueError.  The defaults are the starting values of NeMo's diarization configs; they are NOT tuned for
    this model."""
    N = int(S.shape[0])
    if not 0 < p_max_frac <= 1 or int(p_steps) < 1:
        raise ValueError(f"spectral: need 0 < p_max_frac <= 1 and p_steps >= 1, got {p_max_frac}, {p_steps}")
    if num_speakers is not None and int(num_speakers) < 1:
        raise ValueError(f"spectral: num_speakers must be >= 1, got {num_speakers}")
    if not 1 <= int(max_speakers) <= L.DSK_SC_MAX_SPEAKERS:
        raise ValueError(f"spectral: max_speakers must be in [1, {L.DSK_SC_MAX_SPEAKERS}] (DSK_SC_MAX_SPEAKERS), got "
                         f"{max_speakers}")
    if num_speakers is not None and L.DSK_SC_MAX_SPEAKERS < int(num_speakers) < N:
        raise ValueError(f"spectral: num_speakers must be <= {L.DSK_SC_MAX_SPEAKERS} (DSK_SC_MAX_SPEAKERS) or >= the "
                         f"{N} items, got {num_speakers}")
    pv = p_grid(N, p_max_frac, p_steps)
    if N < 2 or (num_speakers is not None and int(num_speakers) >= N):
        empty = np.zeros((0,), np.float64)
        return SpectralResult(torch.arange(N, dtype=torch.int32, device=S.device), N, None, pv,
                              np.zeros((0, 0)), empty, empty)
    lab, k, t, eig, lmax, ratio = engine.spectral_cluster(S, pv, max_speakers, num_speakers, kmeans_iters)
    return SpectralResult(lab, k, t, pv, eig, lmax, ratio)


def _spectral_options(spectral, threshold, vbx):
    if spectral is None:
        return None
    if not isinstance(spectral, dict):
        raise ValueError(f"diarize: spectral must be None or a dict of options, got {type(spectral).__name__}")
    unknown = sorted(set(spectral) - set(SPECTRAL_OPTIONS))
    if unknown:
        raise ValueError(f"diarize: unknown spectral options {unknown}; known: {list(SPECTRAL_OPTIONS)}")
    if threshold is not None:
        raise ValueError("diarize: spectral clustering takes no threshold (it estimates the count, or num_speakers "
                         "fixes it)")
    if vbx is not None:
        raise ValueError("diarize: give at most one of vbx and spectral")
    return dict(spectral)


def _vbx_options(vbx, plda):
    if vbx is None:
        return None
    if plda is None:
        raise ValueError("diarize: vbx needs a PLDA backend (plda=)")
    if not isinstance(vbx, dict):
        raise ValueError(f"diarize: vbx must be None or a dict of options, got {type(vbx).__name__}")
    unknown = sorted(set(vbx) - set(VBX_OPTIONS))
    if unknown:
        raise ValueError(f"diarize: unknown vbx options {unknown}; known: {list(VBX_OPTIONS)}")
    return dict(vbx)


def _refine(plda, emb, spans, wls, opts):
    """VBx on every recording of more than one window (rows spans[r] of emb, AHC labels wls[r]), in one call; the
    window labels of those recordings are replaced in place."""
    multi = [r for r, (a, b) in enumerate(spans) if b - a > 1]
    if not multi:
        return
    most = max(int(wls[r].max()) + 1 for r in multi)
    if most > L.DSK_VBX_MAX_SPEAKERS:
        raise ValueError(f"diarize: AHC gave {most} initial clusters, more than VBx takes "
                         f"({L.DSK_VBX_MAX_SPEAKERS}); use a higher threshold or fewer speakers")
    lens = [spans[r][1] - spans[r][0] for r in multi]
    off = np.concatenate(([0], np.cumsum(lens)))
    E = torch.cat([emb[spans[r][0]:spans[r][1]] for r in multi])
    res = vbx(plda, E, off, np.concatenate([wls[r] for r in multi]), **opts)
    for i, r in enumerate(multi):
        wls[r] = res.labels[off[i]:off[i + 1]]


def _per_recording(x, n, what):
    if isinstance(x, (list, tuple, np.ndarray)):
        if len(x) != n:
            raise ValueError(f"diarize: {len(x)} values of {what} for {n} recordings")
        return list(x)
    return [x] * n


def _window_counts(last, hop):
    """Windows per run of ``sliding_windows`` at ``hop``, from each run's last start n - T (clipped at 0)."""
    return np.where(last > 0, -(-last // hop) + 1, 1)


def _smallest_hop(last, rec, R, hop):
    """The smallest hop >= ``hop`` at which no recording (``rec``: each run's recording, of R) has more than
    MAX_WINDOWS windows, or None.  The counts do not grow with the hop, so a binary search finds it."""
    def fits(h):
        return np.bincount(rec, _window_counts(last, h), minlength=R).max() <= MAX_WINDOWS

    hi = int(max(last.max(), 1)) + 1                      # past the longest run every run has at most 2 windows
    if not fits(hi):
        return None
    lo = int(hop)
    while lo < hi:
        mid = (lo + hi) // 2
        if fits(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def _cluster(E, plda, threshold, linkage, k, sc_opts=None):
    """AHC of one recording's window embeddings E: on their cosines, or with a PLDA backend on the LLRs of their
    transformed rows (a threshold on LLRs s is the threshold 1 - s on ahc's distance 1 - S).  With ``spectral``
    options ``sc_opts``, spectral clustering of the same affinity instead (k None: estimated), and an empty linkage matrix."""
    if plda is None:
        S = engine.cosine_matrix(E, E)
    else:
        Y = plda.transform(E)
        S = plda.score_matrix(Y, Y)
        if threshold is not None:
            threshold = 1.0 - float(threshold)
    if sc_opts is not None:
        return np.zeros((0, 4)), spectral(S, num_speakers=k, **sc_opts).labels
    if threshold is not None:
        return engine.ahc(S, linkage, threshold=threshold)
    return engine.ahc(S, linkage, num_clusters=k)


def _count(ks, r, W):
    return None if ks[r] is None else min(int(ks[r]), W)


def _diarize_speech(model, bank, u, speech, T, hop, ks, threshold, linkage, batch, plda, vbx, spectral):
    R = u.size
    table, runs, run_off, kept = bank._run_table(speech, u, "diarize")
    rec, first, end = table[:, 0], table[:, 1], table[:, 2]
    rlen = end - first
    if rec.size:
        wcount = np.bincount(rec, _window_counts(np.maximum(rlen - int(T), 0), int(hop)), minlength=R)
        if wcount.max() > MAX_WINDOWS:
            need = _smallest_hop(np.maximum(rlen - int(T), 0), rec, R, hop)
            fix = f"use hop >= {need}" if need is not None else "no hop fits: the recording has too many speech runs"
            raise ValueError(f"diarize: a recording's speech runs have {int(wcount.max())} windows at hop {hop}, more "
                             f"than {MAX_WINDOWS}; {fix}")
        run_bank = frontend.FeatureBank(bank._gather(runs, run_off, rec.size, kept, u),
                                        np.concatenate(([0], np.cumsum(rlen))))
        emb, _, win_start, win_off = frontend.window_embeddings(model, run_bank, np.arange(rec.size), T, hop, batch,
                                                                "diarize")
        win_off = win_off.numpy()
    run_off_rec = np.searchsorted(rec, np.arange(R + 1))     # runs of recording r: run_off_rec[r] .. [r + 1]
    spans, wls, Zs = [], [], []
    for r in range(R):
        r0, r1 = int(run_off_rec[r]), int(run_off_rec[r + 1])
        a, b = (int(win_off[r0]), int(win_off[r1])) if r0 < r1 else (0, 0)
        W = b - a
        if W == 0:
            wl, Z = np.zeros(0, np.int32), np.zeros((0, 4))
        elif W == 1:
            wl, Z = np.zeros(1, np.int32), np.zeros((0, 4))
        else:
            Z, lab = _cluster(emb[a:b], plda, threshold, linkage, _count(ks, r, W), spectral)
            wl = lab.cpu().numpy()
        spans.append((a, b))
        wls.append(wl)
        Zs.append(Z)
    if vbx is not None:
        _refine(plda, emb, spans, wls, vbx)
    out = []
    for r in range(R):
        fl = np.full(int(bank.lengths[u[r]]), -1, np.int32)
        r0, r1 = int(run_off_rec[r]), int(run_off_rec[r + 1])
        a, wl = spans[r][0], wls[r]
        for i in range(r0, r1):
            w0, w1 = int(win_off[i]), int(win_off[i + 1])
            fl[first[i]:end[i]] = frame_labels(win_start[w0:w1].numpy(), wl[w0 - a:w1 - a], int(rlen[i]), T)
        out.append(Recording([sg for sg in segments(fl) if sg[2] >= 0] if r0 < r1 else [], fl, wl, Zs[r]))
    return out


def diarize(model, bank: frontend.FeatureBank, utt, T: int = 160, hop: int = 40, num_speakers=None, threshold=None,
            linkage: str = "average", batch: int = 256, speech=None, plda=None, vbx=None, spectral=None) -> list:
    """Diarize the recordings ``utt`` (indices into ``bank``) -> [Recording] in the order of ``utt``.  Give exactly
    one of ``num_speakers`` (an int, or one per recording; a recording with fewer windows gets one speaker per window)
    and ``threshold`` (a cosine distance 1 - cos: windows merge while the linkage distance is <= threshold), else
    ValueError.  Windows of T frames every ``hop`` frames; a recording needing more than ``MAX_WINDOWS`` windows is a
    ValueError naming the smallest hop that fits.  RuntimeError on a model in train mode.

    ``speech``: None (every frame gets a speaker), or an (F,) bool mask over the bank's rows (CPU or CUDA, such as
    ``bank.speech``): the windows are cut per run of speech frames, non-speech frames are labelled -1 and lie in no
    segment, and a recording without speech has no windows, no segments and only -1 frames.

    ``plda``: None (the affinity is the windows' cosine), or a fitted ``plda.PLDA``: the affinity is then the PLDA
    log-likelihood ratio of the transformed window embeddings (``plda.score_matrix(plda.transform(E), ...)``), and
    ``threshold`` is an LLR: windows merge while the linkage of LLRs is >= threshold (``engine.ahc`` gets
    1 - threshold, its distance being 1 - S, and ``Z``'s heights are 1 - LLR).

    ``vbx``: None, or a dict of options of ``vbx`` (``{}`` for its defaults; needs ``plda``, else ValueError, as is an
    unknown key).  The AHC cut (``threshold`` or ``num_speakers``) is then the initial over-clustering, and one ``vbx``
    call refines the window labels of every recording of more than one window (with ``speech``, all speech windows of
    a recording in time order form one sequence).  ``window_labels`` are VBx's, renumbered by first window; frame
    labels and segments follow from them as above; ``Z`` stays the AHC tree.  More than DSK_VBX_MAX_SPEAKERS initial
    clusters in a recording is a ValueError.

    ``spectral``: None (AHC, as above), or a dict of options of ``spectral`` (``{}`` for its defaults): every recording
    of more than one window is then clustered by spectral clustering of the same affinity (cosines, or PLDA LLRs with
    ``plda``), with or without ``speech``.  ``num_speakers`` becomes optional: None estimates each recording's count,
    an int or a per-recording list fixes it.  ``threshold`` or ``vbx`` with ``spectral``, and an unknown option, are
    ValueErrors.  ``Z`` is then an empty (0, 4) array."""
    spectral = _spectral_options(spectral, threshold, vbx)
    if spectral is None and (num_speakers is None) == (threshold is None):
        raise ValueError("diarize: give exactly one of num_speakers and threshold")
    if linkage not in engine.LINKAGES:
        raise ValueError(f"diarize: linkage must be one of {sorted(engine.LINKAGES)}, got {linkage!r}")
    vbx = _vbx_options(vbx, plda)
    if model.training:
        raise RuntimeError("diarize needs model.eval() (train-mode BatchNorm would use batch statistics)")
    u = np.asarray(utt, np.int64).reshape(-1)
    if u.size == 0:
        raise ValueError("diarize: no recordings")
    ks = _per_recording(num_speakers, u.size, "num_speakers")
    if num_speakers is not None and any(int(k) < 1 for k in ks):
        raise ValueError(f"diarize: num_speakers must be >= 1, got {num_speakers}")
    if speech is not None:
        return _diarize_speech(model, bank, u, speech, T, hop, ks, threshold, linkage, batch, plda, vbx, spectral)
    _, _, win_off = bank.windows(u, T, hop)
    counts = np.diff(win_off.numpy())
    if counts.max() > MAX_WINDOWS:
        n = int(bank.lengths[u[int(counts.argmax())]])
        need = -(-max(n - int(T), 1) // (MAX_WINDOWS - 2))
        raise ValueError(f"diarize: a recording of {n} frames has {int(counts.max())} windows at hop {hop}, more than "
                         f"{MAX_WINDOWS}; use hop >= {need}")
    emb, _, win_start, win_off = frontend.window_embeddings(model, bank, u, T, hop, batch, "diarize")
    spans, wls, Zs = [], [], []
    for r in range(u.size):
        a, b = int(win_off[r]), int(win_off[r + 1])
        W = b - a
        if W == 1:
            wl, Z = np.zeros(1, np.int32), np.zeros((0, 4))
        else:
            Z, lab = _cluster(emb[a:b], plda, threshold, linkage, _count(ks, r, W), spectral)
            wl = lab.cpu().numpy()
        spans.append((a, b))
        wls.append(wl)
        Zs.append(Z)
    if vbx is not None:
        _refine(plda, emb, spans, wls, vbx)
    out = []
    for r in range(u.size):
        a, b = spans[r]
        fl = frame_labels(win_start[a:b].numpy(), wls[r], int(bank.lengths[u[r]]), T)
        out.append(Recording(segments(fl), fl, wls[r], Zs[r]))
    return out
