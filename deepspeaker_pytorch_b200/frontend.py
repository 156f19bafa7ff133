"""GPU log-fbank front-end: the reference's ``mk_MFB`` (reference audio_processing.py:9-36 with constants.py) on the
device, written directly in the ``(T, 64)`` layout the network's ``(B, 1, T, 64)`` input is cropped from (SURVEY §8f-4).

The reference computes the features once per wav file on the CPU (python_speech_features + librosa) and stores ``.npy``
files; here one launch does pre-emphasis, framing, a 512-point FFT per frame in shared memory, the 64 mel filters and
``20*log10(max(., 1e-5))``, a second one the per-bin mean subtraction.  python_speech_features is not vendored in the
reference: parity is against the numpy restatement of its published algorithm (oracle/fbank_oracle.py), unpinned
against the package itself.
"""
from __future__ import annotations

import torch

from . import _lib as L


def mk_mfb(audio: torch.Tensor, sample_rate: int = 16000, use_logscale: bool = True, subtract_mean: bool = True) -> torch.Tensor:
    """audio: 1-D float CUDA tensor (mono samples, as ``librosa.load(..., sr=sample_rate, mono=True)`` yields) ->
    ``(frames, 64)`` fp32 features.  No CPU fallback."""
    if not audio.is_cuda:
        raise RuntimeError("mk_mfb needs a CUDA tensor; there is no CPU fallback")
    a = audio.detach().reshape(-1).float().contiguous()
    lib = L.load()
    frames = int(lib.dsk_fbank_num_frames(a.numel(), sample_rate))
    if frames <= 0:
        raise RuntimeError("mk_mfb: empty signal")
    feat = torch.empty(frames, 64, device=a.device, dtype=torch.float32)
    with torch.cuda.device(a.device):
        L.check(lib.dsk_fbank(a.data_ptr(), a.numel(), sample_rate, int(use_logscale), int(subtract_mean), feat.data_ptr(),
                              L.cur_stream()), "dsk_fbank")
    return feat
