"""GPU log-fbank front-end: the reference's ``mk_MFB`` (reference audio_processing.py:9-36 with constants.py) on the
device, written directly in the ``(T, 64)`` layout the network's ``(B, 1, T, 64)`` input is cropped from (SURVEY §8f-4),
and the input stage that feeds training and scoring from it.

The reference computes the features once per wav file on the CPU (python_speech_features + librosa) and stores ``.npy``
files; here one launch does pre-emphasis, framing, a 512-point FFT per frame in shared memory, the 64 mel filters and
``20*log10(max(., 1e-5))``, a second pair the per-bin mean subtraction.  ``mk_mfb_batch`` does it for many waveforms in
one call (one host synchronisation per call, not per file); ``mk_mfb`` is its one-waveform call.  python_speech_features
is not vendored in the reference: parity is against the numpy restatement of its published algorithm
(oracle/fbank_oracle.py), unpinned against the package itself.

``FeatureBank`` keeps the features of a whole dataset on the device as one CSR bank (the frames of all utterances
concatenated, plus frame offsets).  ``bank.crops`` cuts a step's ``(B, 1, T, 64)`` input from it in one launch, with
SpecAugment time and frequency masks; ``random_starts`` and ``spec_augment_masks`` draw the crop positions and masks on
the host.  ``bank.windows`` and ``embed_utterances`` turn whole utterances into utterance-level embeddings through the
fixed-shape eval forward: the mean of the unit embeddings of sliding windows.

``mk_mfb_batch_vad`` adds a frame-energy voice activity decision (Kaldi's ``compute-vad`` rule on the fbank's own
frame energies); ``FeatureBank.from_waveforms(..., vad={})`` keeps it as ``bank.speech``.  ``bank.select(mask)`` keeps
each utterance's speech frames (``embed_utterances(model, bank.select(bank.speech), utt)`` embeds speech only) and
``bank.runs(mask, utt)`` cuts every run of kept frames into an utterance of its own (what ``diarize`` windows).

``WaveBank`` keeps int16 waveforms (on the device or in pinned host memory) for training on augmented speech:
``augmented_crops`` gathers each step's segments, reverberates them by a ``RirBank`` RIR, mixes noise sources at target
SNRs (``augment_plan`` draws them on the host) and computes their features, all on the device with no host
synchronisation.  Training features then subtract the segment's own mean; ``FeatureBank`` subtracts the utterance's.
``augment_plan(..., speeds=(0.9, 1.0, 1.1))`` adds speed perturbation in front of the reverb (a windowed-sinc resampler
on the device), and ``speed_labels`` gives each perturbed copy of a speaker a class of its own.
"""
from __future__ import annotations

import ctypes
from fractions import Fraction

import numpy as np
import torch

from . import _lib       # for methods whose segment-length argument is named L
from . import _lib as L

N_MELS = 64


def _host_int64(x, what):
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    if a.dtype.kind not in "iu":
        raise ValueError(f"{what}: expected integers, got dtype {a.dtype}")
    return np.ascontiguousarray(a.reshape(-1), dtype=np.int64)


def _ptr64(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _fbank_step(sample_rate, what="fbank"):
    """(flen, step) of ``sample_rate``; ValueError unless it is an integer in
    [DSK_FBANK_MIN_RATE, DSK_FBANK_MAX_RATE]."""
    sr = float(sample_rate)
    if not sr.is_integer() or not L.DSK_FBANK_MIN_RATE <= sr <= L.DSK_FBANK_MAX_RATE:
        raise ValueError(f"{what}: sample_rate must be an integer in [{L.DSK_FBANK_MIN_RATE}, {L.DSK_FBANK_MAX_RATE}] Hz "
                         f"(a 10 ms step of at least one sample, a 25 ms frame of at most 512), got {sample_rate}")
    return int(np.floor(0.025 * sr + 0.5)), int(np.floor(0.01 * sr + 0.5))


def fbank_frame_offsets(lengths, sample_rate: int = 16000) -> np.ndarray:
    """Host only: frame offsets (U + 1,) int64 of utterances of ``lengths`` samples; utterance u gets
    ``dsk_fbank_num_frames(lengths[u], sample_rate)`` frames.  ValueError for an empty list, a length outside
    [1, 2^31) or a sample rate outside [DSK_FBANK_MIN_RATE, DSK_FBANK_MAX_RATE]."""
    _fbank_step(sample_rate, "fbank_frame_offsets")
    lens = _host_int64(lengths, "fbank_frame_offsets")
    if lens.size == 0:
        raise ValueError("fbank_frame_offsets: no utterances")
    if lens.min() < 1 or lens.max() >= 2 ** 31:
        raise ValueError(f"fbank_frame_offsets: every length must lie in [1, 2^31), got min {lens.min()}, max {lens.max()}")
    soff = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    foff = np.empty(lens.size + 1, np.int64)
    L.check(L.load().dsk_fbank_frame_offsets(_ptr64(soff), lens.size, int(sample_rate), _ptr64(foff)),
            "dsk_fbank_frame_offsets")
    return foff


def _fbank_batch(audio, lengths, sample_rate, use_logscale, subtract_mean, vad, what):
    _fbank_step(sample_rate, what)
    if not isinstance(audio, torch.Tensor) or not audio.is_cuda:
        raise RuntimeError(f"{what} needs a CUDA tensor; there is no CPU fallback")
    if isinstance(lengths, torch.Tensor) and lengths.is_cuda:
        raise RuntimeError(f"{what}: lengths must be on the host (they size the output)")
    a = audio.detach().reshape(-1).float().contiguous()
    lens = _host_int64(lengths, what)
    if lens.size and int(lens.sum()) != a.numel():
        raise ValueError(f"{what}: lengths add up to {int(lens.sum())} samples, audio has {a.numel()}")
    foff = fbank_frame_offsets(lens, sample_rate)
    soff = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    feat = torch.empty(int(foff[-1]), N_MELS, device=a.device, dtype=torch.float32)
    with torch.cuda.device(a.device):
        if vad is None:
            L.check(L.load().dsk_fbank_batch(a.data_ptr(), _ptr64(soff), lens.size, int(sample_rate), int(use_logscale),
                                             int(subtract_mean), feat.data_ptr(), L.cur_stream()), "dsk_fbank_batch")
            return feat, torch.from_numpy(foff)
        energy = torch.empty(int(foff[-1]), device=a.device, dtype=torch.float32)
        speech = torch.empty(int(foff[-1]), device=a.device, dtype=torch.bool)
        L.check(L.load().dsk_fbank_batch_vad(a.data_ptr(), _ptr64(soff), lens.size, int(sample_rate), int(use_logscale),
                                             int(subtract_mean), vad["energy_threshold"], vad["mean_scale"],
                                             vad["context"], vad["proportion"], feat.data_ptr(), energy.data_ptr(),
                                             speech.data_ptr(), L.cur_stream()), "dsk_fbank_batch_vad")
    return feat, torch.from_numpy(foff), energy, speech


def mk_mfb_batch(audio: torch.Tensor, lengths, sample_rate: int = 16000, use_logscale: bool = True,
                 subtract_mean: bool = True):
    """``audio``: 1-D fp32 CUDA tensor, U waveforms concatenated; ``lengths`` (U,) samples per waveform, on the host
    -> ``(feats (F, 64) fp32 CUDA, offsets (U + 1,) int64 CPU)``: rows ``offsets[u]:offsets[u+1]`` are utterance u's,
    bit-identical to ``mk_mfb`` on that waveform alone.  One launch sequence and one host synchronisation per call.
    RuntimeError for a CPU tensor; ValueError for a zero length, lengths that do not add up to ``audio`` or a sample
    rate outside [DSK_FBANK_MIN_RATE, DSK_FBANK_MAX_RATE] = [50, 20499] Hz, before any launch."""
    return _fbank_batch(audio, lengths, sample_rate, use_logscale, subtract_mean, None, "mk_mfb_batch")


# Kaldi's compute-vad threshold 5.5 is set against ln of an int16-scale sum of squares over the frame.  Float samples
# are 2^-15 of int16 ones (2^-30 in energy) and bins 0..256 of |rfft|^2 / 512 hold about half the frame's sum of
# squares (Parseval), so every e_f here is about ln(2^31) lower.  Lowering every e_f by D lowers the mean term by
# mean_scale * D = 0.5 D, so the same decisions need the constant lowered by the other 0.5 D: 5.5 - 0.5 ln(2^31).
# Pre-emphasis is not corrected for.
VAD_ENERGY_THRESHOLD = 5.5 - 0.5 * float(np.log(2.0 ** 31))
VAD_DEFAULTS = {"energy_threshold": VAD_ENERGY_THRESHOLD, "mean_scale": 0.5, "context": 2, "proportion": 0.12}


def vad_params(vad=None, **kw) -> dict:
    """The VAD parameters of a dict (``{}`` or None: the defaults ``VAD_DEFAULTS``) plus keyword overrides, checked:
    ValueError for an unknown key, a non-finite value, a context that is not an integer in [0, 2^31) or a negative
    proportion."""
    p = dict(VAD_DEFAULTS)
    for src in (vad or {}, kw):
        for k, v in src.items():
            if k not in VAD_DEFAULTS:
                raise ValueError(f"vad: unknown parameter {k!r} (known: {sorted(VAD_DEFAULTS)})")
            p[k] = v
    for k in ("energy_threshold", "mean_scale", "proportion"):
        p[k] = float(p[k])
        if not np.isfinite(p[k]):
            raise ValueError(f"vad: {k} must be finite, got {p[k]}")
    c = p["context"]
    if isinstance(c, bool) or not float(c).is_integer() or not 0 <= float(c) < 2 ** 31:
        raise ValueError(f"vad: context must be an integer in [0, 2^31), got {c!r}")
    p["context"] = int(c)
    if p["proportion"] < 0:
        raise ValueError(f"vad: proportion must be >= 0, got {p['proportion']}")
    return p


def mk_mfb_batch_vad(audio: torch.Tensor, lengths, sample_rate: int = 16000, use_logscale: bool = True,
                     subtract_mean: bool = True, energy_threshold: float = VAD_ENERGY_THRESHOLD,
                     mean_scale: float = 0.5, context: int = 2, proportion: float = 0.12):
    """``mk_mfb_batch`` plus a frame-energy voice activity decision on the same frames -> ``(feats, offsets, energy,
    speech)``: ``feats`` and ``offsets`` bit-identical to ``mk_mfb_batch``'s, ``energy`` (F,) fp32 CUDA the frame
    energy E_f (the sum over bins 0..256 of the frame's power spectrum, added in fp32 in bin order; 0 becomes
    2.220446049250313e-16; python_speech_features' ``energy``), ``speech`` (F,) bool CUDA.

    The rule is Kaldi's ``compute-vad``: with e_f = ln E_f in fp64 and thr_u = energy_threshold + mean_scale * mean_f
    e_f over the utterance, frame f is speech iff at least ``proportion`` of the frames within ``context`` frames of it
    (clipped to the utterance) have e_g > thr_u.  The defaults are Kaldi's VoxCeleb ``vad.conf`` (0.5, 2, 0.12) with its
    threshold 5.5 moved to float samples and this energy: 5.5 - 0.5 ln(2^31) ~ -5.2438.  **That threshold is not
    calibrated on labelled speech**; check it on your data.  Each utterance's energies and decisions are bit-identical
    whatever the other utterances of the batch.  ValueError for bad parameters (``vad_params``)."""
    vad = vad_params(energy_threshold=energy_threshold, mean_scale=mean_scale, context=context, proportion=proportion)
    return _fbank_batch(audio, lengths, sample_rate, use_logscale, subtract_mean, vad, "mk_mfb_batch_vad")


def mk_mfb(audio: torch.Tensor, sample_rate: int = 16000, use_logscale: bool = True, subtract_mean: bool = True) -> torch.Tensor:
    """audio: 1-D float CUDA tensor (mono samples, as ``librosa.load(..., sr=sample_rate, mono=True)`` yields) ->
    ``(frames, 64)`` fp32 features: the one-waveform call of ``mk_mfb_batch``.  No CPU fallback."""
    if not audio.is_cuda:
        raise RuntimeError("mk_mfb needs a CUDA tensor; there is no CPU fallback")
    if audio.numel() == 0:
        raise RuntimeError("mk_mfb: empty signal")
    return mk_mfb_batch(audio, [audio.numel()], sample_rate, use_logscale, subtract_mean)[0]


# ---- host-side sampling -----------------------------------------------------------------------------------------------
def _rng(generator):
    return np.random.default_rng() if generator is None else generator


def random_starts(lengths, utt, T: int, generator=None) -> torch.Tensor:
    """Host: one crop start per entry of ``utt``, uniform in [0, n_u - T] (every start whose crop ends inside the
    utterance, the last one included), or 0 when n_u < T (the crop then wraps).  ``generator`` is a
    ``numpy.random.Generator``; the same generator state gives the same starts.  The reference draws
    ``randrange(9, n - 23)`` (audio_processing.py:66), which never picks the last start."""
    lens = _host_int64(lengths, "random_starts")
    u = _host_int64(utt, "random_starts")
    if u.size and (u.min() < 0 or u.max() >= lens.size):
        raise ValueError(f"random_starts: utterance index outside [0, {lens.size})")
    hi = np.maximum(lens[u] - int(T), 0)
    return torch.from_numpy(_rng(generator).integers(0, hi + 1, dtype=np.int64) if u.size else np.zeros(0, np.int64))


def spec_augment_masks(B: int, T: int, n_time: int, max_time: int, n_freq: int, max_freq: int, generator=None):
    """Host: SpecAugment time and frequency masks (Park et al. 2019, masking only) for ``bank.crops``:
    ``(time_masks (B, n_time, 2), freq_masks (B, n_freq, 2))`` int32 (start, width) pairs.  Each width is uniform in
    [0, max] and each start uniform in [0, T - width] (time) or [0, 64 - width] (frequency); ``generator`` is a
    ``numpy.random.Generator``."""
    if not (0 <= max_time <= T and 0 <= max_freq <= N_MELS and n_time >= 0 and n_freq >= 0 and B >= 0):
        raise ValueError(f"spec_augment_masks: need 0 <= max_time <= T ({max_time}, {T}), 0 <= max_freq <= 64 "
                         f"({max_freq}), n_time, n_freq, B >= 0")
    g = _rng(generator)

    def draw(n, max_w, extent):
        w = g.integers(0, max_w + 1, size=(B, n), dtype=np.int64)
        s = g.integers(0, extent - w + 1, dtype=np.int64)
        return torch.from_numpy(np.stack([s, w], axis=-1).astype(np.int32))

    return draw(n_time, max_time, T), draw(n_freq, max_freq, N_MELS)


def sliding_windows(lengths, utt, T: int, hop: int):
    """Host: the sliding windows of the utterances ``utt``: ``(win_utt, win_start, win_off)`` int64, windows
    ``win_off[i]:win_off[i+1]`` belong to ``utt[i]``.  Starts are 0, hop, 2 hop, ... up to n - T, plus n - T when the
    last of those does not end at frame n, so every frame is covered; an utterance with n < T gets one window at 0,
    which wraps."""
    if T < 1 or hop < 1:
        raise ValueError(f"sliding_windows: need T >= 1 and hop >= 1, got {T}, {hop}")
    lens = _host_int64(lengths, "sliding_windows")
    u = _host_int64(utt, "sliding_windows")
    if u.size and (u.min() < 0 or u.max() >= lens.size):
        raise ValueError(f"sliding_windows: utterance index outside [0, {lens.size})")
    n = lens[u]
    last = np.maximum(n - T, 0)
    cnt = last // hop + 1 + (last % hop != 0)
    win_off = np.concatenate(([0], np.cumsum(cnt))).astype(np.int64)
    win_utt = np.repeat(u, cnt)
    k = np.arange(win_off[-1], dtype=np.int64) - np.repeat(win_off[:-1], cnt)
    win_start = np.minimum(k * hop, np.repeat(last, cnt))
    return torch.from_numpy(win_utt), torch.from_numpy(win_start), torch.from_numpy(win_off)


# ---- the device-resident bank -----------------------------------------------------------------------------------------
class FeatureBank:
    """The features of many utterances on one device, as one CSR bank: ``feats`` (F, 64) fp32 CUDA, the frames of all
    utterances one after another, and ``offsets`` (U + 1,) int64, utterance u = rows ``offsets[u]:offsets[u+1]``
    (every utterance at least one frame).  The frame counts stay on the host (``lengths``) for sampling."""

    def __init__(self, feats: torch.Tensor, offsets):
        if not isinstance(feats, torch.Tensor) or not feats.is_cuda:
            raise RuntimeError("FeatureBank needs CUDA features; there is no CPU fallback")
        if feats.dim() != 2 or feats.shape[1] != N_MELS or feats.dtype != torch.float32:
            raise ValueError(f"FeatureBank: expected (F, 64) fp32 features, got {tuple(feats.shape)} {feats.dtype}")
        off = _host_int64(offsets, "FeatureBank")
        if off.size < 2 or off[0] != 0 or off[-1] != feats.shape[0] or np.any(np.diff(off) < 1):
            raise ValueError("FeatureBank: offsets must start at 0, end at F and give every utterance >= 1 frame")
        self.feats = feats.contiguous()
        self.lengths = np.diff(off)
        self.offsets = torch.from_numpy(off).to(feats.device)
        self.speech = None      # (F,) bool CUDA voice activity of the rows, when the bank was built with a VAD

    @property
    def num_utterances(self) -> int:
        return int(self.lengths.size)

    @property
    def device(self):
        return self.feats.device

    @classmethod
    def from_waveforms(cls, waveforms, sample_rate: int = 16000, chunk_samples: int = 1 << 26, device=None,
                       use_logscale: bool = True, subtract_mean: bool = True, vad=None):
        """The bank of a list of 1-D waveforms (numpy arrays or tensors), through ``mk_mfb_batch`` in chunks of at most
        ``chunk_samples`` samples (or one waveform, if longer), so only one chunk of audio is on the device at a time.
        ``vad``: a dict of ``mk_mfb_batch_vad``'s VAD parameters (``{}``: the defaults) to also set ``bank.speech``,
        the (F,) bool CUDA speech decision of every row (the features are the same bits either way)."""
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        params = None if vad is None else vad_params(vad)
        lens = np.array([int(np.prod(w.shape)) for w in waveforms], np.int64)
        foff = fbank_frame_offsets(lens, sample_rate)          # ValueError on an empty list or waveform
        feats = torch.empty(int(foff[-1]), N_MELS, device=device, dtype=torch.float32)
        speech = None if params is None else torch.empty(int(foff[-1]), device=device, dtype=torch.bool)
        i = 0
        while i < len(waveforms):
            j, total = i + 1, lens[i]
            while j < len(waveforms) and total + lens[j] <= chunk_samples:
                total += lens[j]
                j += 1
            host = torch.cat([torch.as_tensor(w).reshape(-1).float() for w in waveforms[i:j]])
            out = _fbank_batch(host.to(device), lens[i:j], sample_rate, use_logscale, subtract_mean, params,
                               "FeatureBank.from_waveforms")
            feats[foff[i]:foff[j]].copy_(out[0])
            if speech is not None:
                speech[foff[i]:foff[j]].copy_(out[3])
            i = j
        bank = cls(feats, foff)
        bank.speech = speech
        return bank

    @classmethod
    def from_arrays(cls, arrays, device=None):
        """The bank of a list of (n_u, 64) feature arrays, such as the reference's ``mk_MFB`` / ``read_MFB`` ``.npy``
        files (float64): cast to fp32 on the host and copied to the device in one transfer."""
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        arrs = [np.asarray(a) for a in arrays]
        if not arrs or any(a.ndim != 2 or a.shape[1] != N_MELS or a.shape[0] < 1 for a in arrs):
            raise ValueError("FeatureBank.from_arrays: expected a non-empty list of (n >= 1, 64) arrays")
        host = torch.from_numpy(np.concatenate(arrs).astype(np.float32, copy=False))
        off = np.concatenate(([0], np.cumsum([a.shape[0] for a in arrs]))).astype(np.int64)
        return cls(host.pin_memory().to(device), off)

    def crops(self, utt, start, T: int, time_masks=None, freq_masks=None) -> torch.Tensor:
        """(B, 1, T, 64) fp32: crop b is frames ``start[b]`` .. of utterance ``utt[b]``, wrapping round the utterance
        when it is shorter than T, with the masked frames and bins of ``time_masks`` / ``freq_masks`` ((B, n, 2) int32
        (start, width) pairs, as ``spec_augment_masks`` gives) set to 0, the utterance mean.  One launch.  CPU indices
        are checked on the host (ValueError); CUDA indices are not (a check would synchronise): a crop with an index
        outside the bank or a start outside [0, n_u) comes out NaN."""
        u = torch.as_tensor(utt)
        s = torch.as_tensor(start)
        if u.dim() != 1 or s.shape != u.shape or u.numel() == 0:
            raise ValueError(f"crops: expected 1-D utt and start of one length >= 1, got {tuple(u.shape)}, {tuple(s.shape)}")
        if u.is_floating_point() or s.is_floating_point():
            raise ValueError("crops: utt and start must be integers")
        if T < 1:
            raise ValueError(f"crops: T must be >= 1, got {T}")
        B = u.numel()
        if not u.is_cuda:
            uh, sh = u.to(torch.int64).numpy(), s.cpu().to(torch.int64).numpy()
            if uh.min() < 0 or uh.max() >= self.num_utterances:
                raise ValueError(f"crops: utterance index outside [0, {self.num_utterances})")
            if sh.min() < 0 or np.any(sh >= self.lengths[uh]):
                raise ValueError("crops: a start lies outside [0, n_u)")
        dev = self.device
        u, s = _to_dev(u, torch.int64, dev), _to_dev(s, torch.int64, dev)
        tm, nt = self._masks(time_masks, B, "time_masks")
        fm, nf = self._masks(freq_masks, B, "freq_masks")
        out = torch.empty(B, 1, int(T), N_MELS, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            L.check(L.load().dsk_fbank_crops(self.feats.data_ptr(), self.offsets.data_ptr(), self.num_utterances,
                                             u.data_ptr(), s.data_ptr(), B, int(T), L.ptr(tm), nt, L.ptr(fm), nf,
                                             out.data_ptr(), L.cur_stream()), "dsk_fbank_crops")
        return out

    def _masks(self, m, B, what):
        if m is None:
            return None, 0
        m = torch.as_tensor(m)
        if m.dim() != 3 or m.shape[0] != B or m.shape[2] != 2 or m.is_floating_point():
            raise ValueError(f"crops: {what} must be integer (B, n, 2) with B = {B}, got {tuple(m.shape)} {m.dtype}")
        if m.shape[1] == 0:
            return None, 0
        return _to_dev(m, torch.int32, self.device), int(m.shape[1])

    def random_starts(self, utt, T: int, generator=None) -> torch.Tensor:
        """``random_starts`` over this bank's frame counts (host int64 starts)."""
        return random_starts(self.lengths, utt, T, generator)

    def windows(self, utt, T: int, hop: int):
        """``sliding_windows`` over this bank's frame counts: ``(win_utt, win_start, win_off)`` host int64."""
        return sliding_windows(self.lengths, utt, T, hop)

    def select(self, mask) -> "FeatureBank":
        """The bank of each utterance's kept frames (``mask``: (F,) bool over this bank's rows, CPU or CUDA, such as
        ``bank.speech``), in order: utterance u of the result is the rows of utterance u with ``mask`` set.  The rows
        are copied bit for bit (the features keep the mean of the whole utterance).  ValueError naming every utterance
        left without frames.  One host read (the run count) and one copy of the run table."""
        table, runs, run_off, kept = self._run_table(mask, np.arange(self.num_utterances), "select")
        counts = np.zeros(self.num_utterances, np.int64)
        np.add.at(counts, table[:, 0], table[:, 2] - table[:, 1])
        empty = np.flatnonzero(counts == 0)
        if empty.size:
            raise ValueError(f"select: {empty.size} utterance(s) left without frames: {empty.tolist()}")
        feats = self._gather(runs, run_off, table.shape[0], kept, np.arange(self.num_utterances))
        return FeatureBank(feats, np.concatenate(([0], np.cumsum(counts))))

    def runs(self, mask, utt):
        """Every run of kept frames (``mask`` as for ``select``) of the utterances ``utt`` as an utterance of its own
        -> ``(run_bank, run_utt, run_start)``: run i is frames ``run_start[i]`` .. ``run_start[i] + run_bank.lengths[i]``
        of utterance ``run_utt[i]`` (host int64), in the order of ``utt`` and in frame order within an utterance.
        ValueError when no frame of ``utt`` is kept."""
        u = _host_int64(utt, "runs")
        table, runs, run_off, kept = self._run_table(mask, u, "runs")
        if table.shape[0] == 0:
            raise ValueError("runs: no frame of these utterances is kept")
        feats = self._gather(runs, run_off, table.shape[0], kept, u)
        bank = FeatureBank(feats, np.concatenate(([0], np.cumsum(table[:, 2] - table[:, 1]))))
        return bank, torch.from_numpy(u[table[:, 0]]), torch.from_numpy(table[:, 1].copy())

    def _mask(self, mask, what):
        m = torch.as_tensor(mask)
        if m.shape != (self.feats.shape[0],) or m.is_floating_point() or m.is_complex():
            raise ValueError(f"{what}: expected an (F,) = ({self.feats.shape[0]},) bool mask, got {tuple(m.shape)} {m.dtype}")
        if m.dtype != torch.bool:
            m = m != 0
        return _to_dev(m, torch.bool, self.device)

    def _run_table(self, mask, u, what):
        """(table (n, 3) host int64 rows (j, first, end), runs and run_off on the device, kept frames) of ``dsk_frame_runs``
        over the utterances u (host int64)."""
        m = self._mask(mask, what)
        if u.size == 0 or u.min() < 0 or u.max() >= self.num_utterances:
            raise ValueError(f"{what}: expected utterance indices in [0, {self.num_utterances}), at least one")
        lens = self.lengths[u]
        loff = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
        cap = int(np.sum((lens + 1) // 2))                   # an utterance of n frames has at most ceil(n / 2) runs
        dev = self.device
        runs = torch.empty(cap, 3, device=dev, dtype=torch.int64)
        run_off = torch.empty(cap + 1, device=dev, dtype=torch.int64)
        ud, ld = _to_dev(torch.from_numpy(u), torch.int64, dev), _to_dev(torch.from_numpy(loff), torch.int64, dev)
        counts = np.zeros(2, np.int64)
        with torch.cuda.device(dev):
            L.check(L.load().dsk_frame_runs(m.data_ptr(), self.offsets.data_ptr(), self.num_utterances, ud.data_ptr(),
                                            ld.data_ptr(), u.size, int(loff[-1]), cap, runs.data_ptr(),
                                            run_off.data_ptr(), _ptr64(counts), L.cur_stream()), "dsk_frame_runs")
        n = int(counts[0])
        return runs[:n].cpu().numpy(), runs, run_off, int(counts[1])

    def _gather(self, runs, run_off, n, kept, u):
        out = torch.empty(kept, N_MELS, device=self.device, dtype=torch.float32)
        ud = _to_dev(torch.from_numpy(np.ascontiguousarray(u, np.int64)), torch.int64, self.device)
        with torch.cuda.device(self.device):
            L.check(L.load().dsk_gather_runs(self.feats.data_ptr(), self.offsets.data_ptr(), self.num_utterances,
                                             ud.data_ptr(), runs.data_ptr(), run_off.data_ptr(), n, kept,
                                             out.data_ptr(), L.cur_stream()), "dsk_gather_runs")
        return out


def _to_dev(t, dtype, dev):
    t = t.to(dtype)
    if not t.is_cuda:   # a pageable copy would wait for the stream; a pinned one is queued like a kernel
        return t.contiguous().pin_memory().to(dev, non_blocking=True)
    return t.to(dev).contiguous()


_FB_CACHE = {}


def _filterbank(dev, sample_rate: int) -> torch.Tensor:
    """The (64, 257) fp32 mel filterbank on ``dev`` (``dsk_fbank_filterbank``), uploaded once per (device, rate)."""
    key = (dev.index, int(sample_rate))
    if key not in _FB_CACHE:
        fb = np.empty((N_MELS, 257), np.float32)
        L.check(L.load().dsk_fbank_filterbank(int(sample_rate), fb.ctypes.data_as(ctypes.c_void_p)), "dsk_fbank_filterbank")
        _FB_CACHE[key] = torch.from_numpy(fb).to(dev)
    return _FB_CACHE[key]


def segment_samples(T: int, sample_rate: int = 16000) -> int:
    """Samples L = flen + (T - 1) step of a segment whose log-fbank has exactly T frames (25 840 at 16 kHz, T = 160).
    ValueError for a sample rate outside [DSK_FBANK_MIN_RATE, DSK_FBANK_MAX_RATE] = [50, 20499] Hz."""
    flen, step = _fbank_step(sample_rate, "segment_samples")
    return flen + (int(T) - 1) * step


# ---- waveform augmentation ---------------------------------------------------------------------------------------------
def _bank_samples(samples, dtype, what):
    if not isinstance(samples, torch.Tensor) or samples.dim() != 1 or samples.dtype != dtype or samples.numel() == 0:
        raise ValueError(f"{what}: expected a non-empty 1-D {dtype} tensor")
    if not samples.is_cuda and not (torch.cuda.is_available() and samples.is_pinned()):
        raise ValueError(f"{what}: samples must be a CUDA tensor or page-locked (pinned) CPU memory, not pageable memory")
    return samples.contiguous()


def _bank_offsets(offsets, n, what):
    off = _host_int64(offsets, what)
    if off.size < 2 or off[0] != 0 or off[-1] != n or np.any(np.diff(off) < 1):
        raise ValueError(f"{what}: offsets must start at 0, end at {n} and give every entry >= 1 sample")
    return off


def _bank_device(samples, device):
    if samples.is_cuda:
        return samples.device
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


class WaveBank:
    """Int16 PCM waveforms of many utterances as one CSR bank: ``samples`` (S,) int16, the utterances one after
    another, on the device or in page-locked host memory (read over the bus by the kernels: VoxCeleb2 as 16-bit PCM is
    ~265 GB, more than a card holds), and ``offsets`` (U + 1,) int64, utterance u = ``samples[offsets[u]:offsets[u+1]]``.
    The sample counts stay on the host (``lengths``) for sampling; the offsets are copied to ``device``."""

    def __init__(self, samples: torch.Tensor, offsets, device=None):
        self.samples = _bank_samples(samples, torch.int16, "WaveBank")
        off = _bank_offsets(offsets, self.samples.numel(), "WaveBank")
        self.lengths = np.diff(off)
        self.device = _bank_device(self.samples, device)
        self.offsets = torch.from_numpy(off).to(self.device)

    @property
    def num_utterances(self) -> int:
        return int(self.lengths.size)

    @classmethod
    def from_waveforms(cls, waves, pin: bool = False, device=None):
        """The bank of a list of 1-D waveforms: int16 arrays, or float arrays whose values are exactly k / 32768 (what
        ``librosa.load`` returns for a 16-bit file at its native rate).  ``pin``: keep the samples in page-locked host
        memory rather than on the device.  ValueError for anything else."""
        arrs = []
        for w in waves:
            a = w.detach().cpu().numpy() if isinstance(w, torch.Tensor) else np.asarray(w)
            a = a.reshape(-1)
            if a.size == 0:
                raise ValueError("WaveBank.from_waveforms: empty waveform")
            if a.dtype == np.int16:
                arrs.append(a)
                continue
            if a.dtype.kind != "f":
                raise ValueError(f"WaveBank.from_waveforms: expected int16 or float samples, got {a.dtype}")
            k = a.astype(np.float64) * 32768.0
            if not np.all(np.isfinite(k)) or np.any(k != np.round(k)) or k.min() < -32768 or k.max() > 32767:
                raise ValueError("WaveBank.from_waveforms: float samples must be exactly k / 32768 with k an int16")
            arrs.append(k.astype(np.int16))
        if not arrs:
            raise ValueError("WaveBank.from_waveforms: no waveforms")
        host = torch.from_numpy(np.concatenate(arrs))
        off = np.concatenate(([0], np.cumsum([a.size for a in arrs]))).astype(np.int64)
        if pin:
            return cls(host.pin_memory(), off, device)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        return cls(host.pin_memory().to(dev), off)

    def random_starts(self, utt, L: int, generator=None, plan=None) -> torch.Tensor:
        """``random_starts`` over this bank's sample counts: uniform in [0, n - L], 0 when n < L (host int64).  With a
        ``plan`` that has speeds, example b reads about alpha_b L input samples, so its start is uniform in
        [0, n - ceil(alpha_b L)] (0 when that is negative).  Draw the plan first, then the starts from it: a plan's
        draws do not depend on the starts, and without a plan (or without speeds) the draws are those of
        ``random_starts``.  A CUDA ``speed_idx`` is read back to the host."""
        if plan is None or plan.get("speed_idx") is None:
            return random_starts(self.lengths, utt, L, generator)
        u = _host_int64(utt, "random_starts")
        if u.size and (u.min() < 0 or u.max() >= self.num_utterances):
            raise ValueError(f"random_starts: utterance index outside [0, {self.num_utterances})")
        speeds = _speed_factors(plan.get("speeds"), "random_starts")
        k = _host_int64(plan["speed_idx"], "random_starts")
        if k.shape != u.shape or (k.size and (k.min() < -1 or k.max() >= len(speeds))):
            raise ValueError(f"random_starts: speed_idx must be ({u.size},) in [-1, {len(speeds)})")
        p = np.array([1] + [a.numerator for a in speeds], np.int64)[k + 1]
        q = np.array([1] + [a.denominator for a in speeds], np.int64)[k + 1]
        need = -(-p * int(L) // q)                           # ceil(alpha L)
        hi = np.maximum(self.lengths[u] - need, 0)
        return torch.from_numpy(_rng(generator).integers(0, hi + 1, dtype=np.int64) if u.size else np.zeros(0, np.int64))

    def segments(self, utt, start, L: int, plan=None, rir_bank=None, noise_bank=None) -> torch.Tensor:
        """(B, L) fp32 augmented audio (``dsk_wave_augment_speed``): segment b is samples ``start[b]`` .. of utterance
        ``utt[b]`` (wrapping) times 2^-15, resampled by the speed factor ``plan["speeds"][plan["speed_idx"][b]]`` (-1:
        none), reverberated by RIR ``plan["rir_idx"][b]`` of ``rir_bank`` and mixed with the sources of ``plan`` from
        ``noise_bank`` (see ``augment_plan``).  No plan: the clean segments.  CPU indices are checked on the host
        (ValueError); CUDA ones are not: an example with an index, start, SNR or speed index out of range comes out NaN.
        No host synchronisation once the plan's speed table is on the device."""
        u, s = _index_pair(utt, start, "segments")
        B, L = u.numel(), int(L)
        if not 1 <= L <= 1 << 24:
            raise ValueError(f"segments: L must lie in [1, 2^24], got {L}")
        plan = {} if plan is None else plan
        rir_idx, noise_idx, noise_start, snr = (plan.get(k) for k in ("rir_idx", "noise_idx", "noise_start", "snr_db"))
        if rir_idx is not None and rir_bank is None:
            r = torch.as_tensor(rir_idx)
            if r.is_cuda or bool((r != -1).any()):
                raise ValueError("segments: the plan reverberates but no rir_bank is given")
            rir_idx = None
        M = 0
        if noise_idx is not None:
            noise_idx, noise_start, snr = (torch.as_tensor(x) for x in (noise_idx, noise_start, snr))
            if noise_idx.dim() != 2 or noise_idx.shape[0] != B or noise_start.shape != noise_idx.shape \
                    or snr.shape != noise_idx.shape:
                raise ValueError(f"segments: noise_idx, noise_start, snr_db must be (B, M) with B = {B}")
            M = int(noise_idx.shape[1])
            if M > _lib.DSK_AUG_MAX_SOURCES:
                raise ValueError(f"segments: at most {_lib.DSK_AUG_MAX_SOURCES} noise sources, got {M}")
            if M and noise_bank is None:
                raise ValueError("segments: the plan adds noise but no noise_bank is given")
        speed_idx, K = plan.get("speed_idx"), 0
        if speed_idx is not None:
            speeds = _speed_factors(plan.get("speeds"), "segments")
            K = len(speeds)
            speed_idx = torch.as_tensor(speed_idx)
            if speed_idx.shape != u.shape or speed_idx.is_floating_point():
                raise ValueError(f"segments: speed_idx must be integer (B,) with B = {B}")
            if not speed_idx.is_cuda:
                k = speed_idx.to(torch.int64).numpy()
                if k.min() < -1 or k.max() >= K:
                    raise ValueError(f"segments: speed_idx outside [-1, {K})")
        if not u.is_cuda:
            _check_host_index(u, s, self.lengths, "segments")
        if rir_idx is not None:
            rir_idx = torch.as_tensor(rir_idx)
            if rir_idx.shape != u.shape or rir_idx.is_floating_point():
                raise ValueError(f"segments: rir_idx must be integer (B,) with B = {B}")
            if not rir_idx.is_cuda:
                r = rir_idx.to(torch.int64).numpy()
                if r.min() < -1 or r.max() >= rir_bank.num_rirs:
                    raise ValueError(f"segments: rir_idx outside [-1, {rir_bank.num_rirs})")
        if M and not noise_idx.is_cuda:
            q, st, sn = noise_idx.to(torch.int64).numpy(), noise_start.cpu().to(torch.int64).numpy(), snr.cpu().double().numpy()
            used = q != -1
            if q.min() < -1 or q.max() >= noise_bank.num_utterances:
                raise ValueError(f"segments: noise_idx outside [-1, {noise_bank.num_utterances})")
            if np.any(st[used] < 0) or np.any(st[used] >= noise_bank.lengths[q[used]]):
                raise ValueError("segments: a noise start lies outside [0, n)")
            if not np.all(np.isfinite(sn[used])):
                raise ValueError("segments: a non-finite SNR")
        dev = self.device
        u, s = _to_dev(u, torch.int64, dev), _to_dev(s, torch.int64, dev)
        out = torch.empty(B, L, device=dev, dtype=torch.float32)
        ri = _to_dev(rir_idx, torch.int64, dev) if rir_idx is not None else None
        if M:
            ni, ns = _to_dev(noise_idx, torch.int64, dev), _to_dev(noise_start, torch.int64, dev)
            sd = _to_dev(snr, torch.float64, dev)
        else:
            ni = ns = sd = None
        rb = rir_bank if ri is not None else None
        nb = noise_bank if M else None
        si, ratio, taps = None, None, None
        if K:
            si = _to_dev(speed_idx, torch.int64, dev)
            ratio, taps = _speed_table(dev, speeds)
        ptr = _lib.ptr
        with torch.cuda.device(dev):
            _lib.check(_lib.load().dsk_wave_augment_speed(
                self.samples.data_ptr(), self.offsets.data_ptr(), self.num_utterances, u.data_ptr(), s.data_ptr(), B, L,
                ptr(rb.samples if rb else None), ptr(rb.offsets if rb else None), rb.num_rirs if rb else 0,
                rb.max_len if rb else 1, ptr(ri),
                ptr(nb.samples if nb else None), ptr(nb.offsets if nb else None), nb.num_utterances if nb else 0, M,
                ptr(ni), ptr(ns), ptr(sd), ptr(ratio), ptr(taps), K, ptr(si), out.data_ptr(), _lib.cur_stream()),
                "dsk_wave_augment_speed")
        return out

    def augmented_crops(self, utt, start, T: int, plan=None, rir_bank=None, noise_bank=None, time_masks=None,
                        freq_masks=None, sample_rate: int = 16000, use_logscale: bool = True,
                        subtract_mean: bool = True) -> torch.Tensor:
        """(B, 1, T, 64) fp32 training input: ``mk_mfb`` of each augmented segment of ``segment_samples(T)`` samples
        (``segments``), the mean subtracted over the segment's own T frames, then the SpecAugment masks exactly as
        ``FeatureBank.crops`` applies them.  ``start`` counts samples.  No host synchronisation once the filterbank of
        ``sample_rate`` is on the device.  ValueError for a sample rate outside
        [DSK_FBANK_MIN_RATE, DSK_FBANK_MAX_RATE]."""
        _fbank_step(sample_rate, "augmented_crops")
        Ls = segment_samples(T, sample_rate)
        if T < 1 or L.load().dsk_fbank_num_frames(Ls, int(sample_rate)) != T:
            raise ValueError(f"augmented_crops: no segment length gives T = {T} frames at {sample_rate} Hz")
        audio = self.segments(utt, start, Ls, plan, rir_bank, noise_bank)
        B = audio.shape[0]
        dev = self.device
        tm, nt = _masks(time_masks, B, "time_masks", dev)
        fm, nf = _masks(freq_masks, B, "freq_masks", dev)
        fb = _filterbank(dev, sample_rate)
        out = torch.empty(B, 1, int(T), N_MELS, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            L.check(L.load().dsk_fbank_segments(audio.data_ptr(), B, Ls, int(sample_rate), int(use_logscale),
                                                int(subtract_mean), fb.data_ptr(), L.ptr(tm), nt, L.ptr(fm), nf,
                                                out.data_ptr(), L.cur_stream()), "dsk_fbank_segments")
        return out


class RirBank:
    """Room impulse responses as one CSR bank: ``samples`` (S,) fp32 (device or page-locked host memory), ``offsets``
    (R + 1,) int64.  ``max_len`` (host) is the longest RIR, at most 65 536 taps."""

    def __init__(self, samples: torch.Tensor, offsets, device=None):
        self.samples = _bank_samples(samples, torch.float32, "RirBank")
        off = _bank_offsets(offsets, self.samples.numel(), "RirBank")
        self.lengths = np.diff(off)
        if self.lengths.max() > L.DSK_AUG_MAX_RIR:
            raise ValueError(f"RirBank: a RIR has {self.lengths.max()} taps, more than {L.DSK_AUG_MAX_RIR}")
        self.max_len = int(self.lengths.max())
        self.device = _bank_device(self.samples, device)
        self.offsets = torch.from_numpy(off).to(self.device)

    @property
    def num_rirs(self) -> int:
        return int(self.lengths.size)

    @classmethod
    def from_arrays(cls, rirs, pin: bool = False, device=None):
        """The bank of a list of 1-D RIRs, each normalised to unit energy (in fp64 on the host, rounded once to fp32).
        ValueError for an empty, non-finite or all-zero RIR."""
        arrs = []
        for h in rirs:
            a = np.asarray(h.detach().cpu().numpy() if isinstance(h, torch.Tensor) else h, np.float64).reshape(-1)
            e = float(np.sqrt(np.sum(a * a))) if a.size else 0.0
            if a.size == 0 or not np.isfinite(e) or e == 0.0:
                raise ValueError("RirBank.from_arrays: every RIR must be non-empty, finite and not all zero")
            if a.size > L.DSK_AUG_MAX_RIR:
                raise ValueError(f"RirBank.from_arrays: a RIR has {a.size} taps, more than {L.DSK_AUG_MAX_RIR}")
            arrs.append((a / e).astype(np.float32))
        if not arrs:
            raise ValueError("RirBank.from_arrays: no RIRs")
        host = torch.from_numpy(np.concatenate(arrs))
        off = np.concatenate(([0], np.cumsum([a.size for a in arrs]))).astype(np.int64)
        if pin:
            return cls(host.pin_memory(), off, device)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        return cls(host.pin_memory().to(dev), off)


def augment_plan(B: int, L: int, generator=None, rir_bank=None, p_reverb: float = 0.5, noise_bank=None,
                 noise_groups=(), p_noise: float = 0.5, speeds=None, speed_weights=None):
    """Host: a random augmentation plan for B segments of L samples, as a dict of CPU tensors ``rir_idx`` (B,) int64,
    ``noise_idx``, ``noise_start`` (B, M) int64 and ``snr_db`` (B, M) fp64, M the largest source count of any group and
    unused slots -1 (start 0, SNR 0).  Per example: with probability ``p_reverb`` a uniform RIR of ``rir_bank`` (else
    -1); with probability ``p_noise`` one of ``noise_groups`` chosen by weight, then a uniform source count, uniform
    utterances, uniform starts in [0, n - L] (0 when n < L: the source wraps) and a uniform SNR.  A group is
    ``(utterance ids in noise_bank, (snr_lo_db, snr_hi_db), (count_lo, count_hi), weight)``.  ``generator`` is a
    ``numpy.random.Generator``; the same state gives the same plan.

    ``speeds``: up to 8 distinct speed factors (floats or ``Fraction``s, each taken exactly, 0.9 as 9/10; each a ratio
    p / q with 1/2 <= p / q <= 2 and q <= 32), drawn per example by ``speed_weights`` (default uniform) in one draw
    after all the others, so the other keys are the same with or without speeds for one generator state.  The plan
    then also holds ``speed_idx`` (B,) int64 and ``speeds`` (a tuple of ``Fraction``s, host metadata).  Draw the starts
    after the plan with ``WaveBank.random_starts(utt, L, generator, plan)``, and the labels with ``speed_labels``."""
    g = _rng(generator)
    if speeds is not None:
        speeds = _speed_factors(speeds, "augment_plan")
        if len(set(speeds)) != len(speeds):
            raise ValueError(f"augment_plan: the speed factors must be distinct, got {[str(a) for a in speeds]}")
        sw = np.ones(len(speeds)) if speed_weights is None else np.asarray(speed_weights, np.float64).reshape(-1)
        if sw.shape != (len(speeds),) or not np.all(np.isfinite(sw)) or sw.min() < 0 or sw.sum() <= 0:
            raise ValueError(f"augment_plan: speed_weights must be {len(speeds)} finite weights >= 0 with a positive sum")
    elif speed_weights is not None:
        raise ValueError("augment_plan: speed_weights without speeds")
    B, L = int(B), int(L)
    if B < 0 or L < 1 or not (0.0 <= p_reverb <= 1.0 and 0.0 <= p_noise <= 1.0):
        raise ValueError(f"augment_plan: need B >= 0, L >= 1 and probabilities in [0, 1] (got {B}, {L}, {p_reverb}, {p_noise})")
    groups = []
    for grp in noise_groups:
        ids, (slo, shi), (clo, chi), w = grp
        ids = _host_int64(ids, "augment_plan")
        if noise_bank is None:
            raise ValueError("augment_plan: noise groups need a noise_bank")
        if ids.size == 0 or ids.min() < 0 or ids.max() >= noise_bank.num_utterances:
            raise ValueError(f"augment_plan: a group's utterances must be a non-empty subset of [0, {noise_bank.num_utterances})")
        if not (1 <= clo <= chi <= _lib.DSK_AUG_MAX_SOURCES) or not (np.isfinite(slo) and np.isfinite(shi) and slo <= shi) \
                or w < 0:
            raise ValueError(f"augment_plan: need 1 <= count_lo <= count_hi <= {_lib.DSK_AUG_MAX_SOURCES}, finite "
                             "snr_lo <= snr_hi and weight >= 0")
        groups.append((ids, float(slo), float(shi), int(clo), int(chi), float(w)))
    if p_reverb > 0 and rir_bank is None:
        raise ValueError("augment_plan: p_reverb > 0 needs a rir_bank")
    if p_noise > 0 and not groups:
        raise ValueError("augment_plan: p_noise > 0 needs noise groups")
    weights = np.array([grp[5] for grp in groups], np.float64)
    if groups and weights.sum() <= 0:
        raise ValueError("augment_plan: the group weights add up to 0")
    M = max((grp[4] for grp in groups), default=0)
    rir_idx = np.full(B, -1, np.int64)
    noise_idx = np.full((B, M), -1, np.int64)
    noise_start = np.zeros((B, M), np.int64)
    snr_db = np.zeros((B, M), np.float64)
    for b in range(B):
        if rir_bank is not None and g.random() < p_reverb:
            rir_idx[b] = g.integers(0, rir_bank.num_rirs)
        if groups and g.random() < p_noise:
            ids, slo, shi, clo, chi, _ = groups[g.choice(len(groups), p=weights / weights.sum())]
            c = int(g.integers(clo, chi + 1))
            q = ids[g.integers(0, ids.size, c)]
            noise_idx[b, :c] = q
            noise_start[b, :c] = g.integers(0, np.maximum(noise_bank.lengths[q] - L, 0) + 1)
            snr_db[b, :c] = g.uniform(slo, shi, c)
    plan = {"rir_idx": torch.from_numpy(rir_idx), "noise_idx": torch.from_numpy(noise_idx),
            "noise_start": torch.from_numpy(noise_start), "snr_db": torch.from_numpy(snr_db)}
    if speeds is not None:
        plan["speed_idx"] = torch.from_numpy(g.choice(len(speeds), size=B, p=sw / sw.sum()).astype(np.int64))
        plan["speeds"] = speeds
    return plan


# ---- speed perturbation ------------------------------------------------------------------------------------------------
def speed_factor(a) -> Fraction:
    """The exact ratio of a speed factor: a float through its shortest decimal form (0.9 -> 9/10), an int or a
    ``Fraction`` as is.  ValueError unless 1/2 <= alpha <= 2 with a denominator of at most 32."""
    if isinstance(a, bool) or not isinstance(a, (int, float, Fraction, np.integer, np.floating)):
        raise ValueError(f"speed factor: expected a number, got {a!r}")
    if isinstance(a, (float, np.floating)):
        if not np.isfinite(a):
            raise ValueError(f"speed factor: {a} is not finite")
        f = Fraction(str(float(a)))
    else:
        f = Fraction(a)
    if not (Fraction(1, 2) <= f <= 2) or f.denominator > L.DSK_SPEED_MAX_DEN:
        raise ValueError(f"speed factor {a} = {f}: need 1/2 <= p / q <= 2 and q <= {L.DSK_SPEED_MAX_DEN}")
    return f


def _speed_factors(speeds, what):
    if speeds is None:
        raise ValueError(f"{what}: speed_idx needs the plan's speeds")
    out = tuple(speed_factor(a) for a in speeds)
    if not 1 <= len(out) <= L.DSK_SPEED_MAX_FACTORS:
        raise ValueError(f"{what}: need 1 .. {L.DSK_SPEED_MAX_FACTORS} speed factors, got {len(out)}")
    return out


def speed_filter(alpha) -> np.ndarray:
    """Host: the (q, 50) fp32 polyphase taps of the factor alpha = p / q (``dsk_speed_filter``)."""
    f = speed_factor(alpha)
    taps = np.empty((f.denominator, L.DSK_SPEED_TAPS), np.float32)
    L.check(L.load().dsk_speed_filter(f.numerator, f.denominator, taps.ctypes.data_as(ctypes.c_void_p)),
            "dsk_speed_filter")
    return taps


_SPEED_CACHE = {}


def _speed_table(dev, speeds):
    """(ratio (K, 2) int32, taps (K, 32, 50) fp32) of the factors ``speeds`` on ``dev``, uploaded once per (device,
    factors)."""
    key = (dev.index, tuple(speeds))
    if key not in _SPEED_CACHE:
        ratio = np.array([[a.numerator, a.denominator] for a in speeds], np.int32)
        taps = np.zeros((len(speeds), L.DSK_SPEED_MAX_DEN, L.DSK_SPEED_TAPS), np.float32)
        for k, a in enumerate(speeds):
            taps[k, :a.denominator] = speed_filter(a)
        _SPEED_CACHE[key] = (torch.from_numpy(ratio).to(dev), torch.from_numpy(taps).to(dev))
    return _SPEED_CACHE[key]


def speed_labels(labels, plan, num_speakers: int) -> torch.Tensor:
    """Labels of speed-perturbed examples as new classes ("speed perturb + extend speakers"): labels[b] +
    num_speakers * j_b, j_b = 0 for a unit factor or speed_idx -1, else the 1-based rank (by value) of the example's
    factor among the plan's non-unit factors, so the classifier has num_speakers * (1 + #non-unit factors) classes.  A
    plan without speeds leaves the labels as they are.  On the labels' device; a CPU speed_idx is checked (ValueError),
    a CUDA one is not (an out-of-range example, NaN in ``segments``, keeps its label)."""
    lab = torch.as_tensor(labels)
    if lab.dim() != 1 or lab.is_floating_point() or int(num_speakers) < 1:
        raise ValueError(f"speed_labels: need 1-D integer labels and num_speakers >= 1, got {tuple(lab.shape)} "
                         f"{lab.dtype}, {num_speakers}")
    lab = lab.to(torch.int64)
    if plan is None or plan.get("speed_idx") is None:
        return lab
    speeds = _speed_factors(plan.get("speeds"), "speed_labels")
    ranked = sorted(a for a in speeds if a != 1)
    j = [0] + [0 if a == 1 else 1 + ranked.index(a) for a in speeds]
    k = torch.as_tensor(plan["speed_idx"])
    if k.shape != lab.shape or k.is_floating_point():
        raise ValueError(f"speed_labels: speed_idx must be integer ({lab.numel()},)")
    if not k.is_cuda and k.numel() and (int(k.min()) < -1 or int(k.max()) >= len(speeds)):
        raise ValueError(f"speed_labels: speed_idx outside [-1, {len(speeds)})")
    k = k.to(lab.device, torch.int64) + 1
    lut = torch.tensor(j, dtype=torch.int64, device=lab.device)
    valid = (k >= 0) & (k <= len(speeds))
    return lab + int(num_speakers) * torch.where(valid, lut[k.clamp(0, len(speeds))], 0)


def _index_pair(utt, start, what):
    u = torch.as_tensor(utt)
    s = torch.as_tensor(start)
    if u.dim() != 1 or s.shape != u.shape or u.numel() == 0:
        raise ValueError(f"{what}: expected 1-D utt and start of one length >= 1, got {tuple(u.shape)}, {tuple(s.shape)}")
    if u.is_floating_point() or s.is_floating_point():
        raise ValueError(f"{what}: utt and start must be integers")
    return u, s


def _check_host_index(u, s, lengths, what):
    uh, sh = u.to(torch.int64).numpy(), s.cpu().to(torch.int64).numpy()
    if uh.min() < 0 or uh.max() >= lengths.size:
        raise ValueError(f"{what}: utterance index outside [0, {lengths.size})")
    if sh.min() < 0 or np.any(sh >= lengths[uh]):
        raise ValueError(f"{what}: a start lies outside [0, n_u)")


def _masks(m, B, what, dev):
    if m is None:
        return None, 0
    m = torch.as_tensor(m)
    if m.dim() != 3 or m.shape[0] != B or m.shape[2] != 2 or m.is_floating_point():
        raise ValueError(f"{what} must be integer (B, n, 2) with B = {B}, got {tuple(m.shape)} {m.dtype}")
    if m.shape[1] == 0:
        return None, 0
    return _to_dev(m, torch.int32, dev), int(m.shape[1])


def window_embeddings(model, bank: FeatureBank, utt, T: int = 160, hop: int = 80, batch: int = 256,
                      what: str = "window_embeddings"):
    """(emb (W, D) fp32, win_utt, win_start, win_off): the eval-forward embedding of every sliding window
    ``bank.windows(utt, T, hop)`` of the utterances ``utt`` (windows ``win_off[i]:win_off[i+1]`` are ``utt[i]``'s, host
    int64).  The forward runs over the windows in batches of ``min(batch, W)`` rows, the last one padded, so every
    batch has the same shape and one captured forward serves them all: the rows are those of
    ``model(bank.crops(...))`` over the same windows in the same batches.  RuntimeError on a model in train mode."""
    if model.training:
        raise RuntimeError(f"{what} needs model.eval() (train-mode BatchNorm would use batch statistics)")
    if batch < 1:
        raise ValueError(f"{what}: batch must be >= 1, got {batch}")
    win_utt, win_start, win_off = bank.windows(utt, T, hop)
    W = win_utt.numel()
    if W == 0:
        raise ValueError(f"{what}: no utterances")
    Bb = min(int(batch), W)
    nb = (W + Bb - 1) // Bb
    pad = nb * Bb - W                                   # padded rows repeat the last window and are dropped
    wu = torch.cat([win_utt, win_utt[-1:].expand(pad)])
    ws = torch.cat([win_start, win_start[-1:].expand(pad)])
    emb = None
    with torch.no_grad():
        for i in range(nb):
            e = model(bank.crops(wu[i * Bb:(i + 1) * Bb], ws[i * Bb:(i + 1) * Bb], T))
            if emb is None:
                emb = torch.empty(nb * Bb, e.shape[1], device=e.device, dtype=torch.float32)
            emb[i * Bb:(i + 1) * Bb].copy_(e)
    return emb[:W], win_utt, win_start, win_off


def embed_utterances(model, bank: FeatureBank, utt, T: int = 160, hop: int = 80, batch: int = 256) -> torch.Tensor:
    """(len(utt), D) fp32: one embedding per utterance ``utt[i]`` of ``bank``, the mean of the unit embeddings of its
    sliding windows (``window_embeddings``), summed in fp64 in window order by ``engine.class_centroids``.
    The rows are what ``identification.enroll`` gives for those windows: for cosine scoring (``verification``,
    ``identification``), not of norm 10.  RuntimeError on a model in train mode."""
    from . import engine

    emb, _, _, win_off = window_embeddings(model, bank, utt, T, hop, batch, "embed_utterances")
    order = torch.arange(emb.shape[0], dtype=torch.int64)
    return engine.class_centroids(emb, order, win_off)
