"""Frame-energy VAD, select / runs and speech-only diarization: one JSON line with
  * seconds of FeatureBank.from_waveforms over 2 000 synthetic waveforms of 4-12 s at 16 kHz (noise bursts and
    near-silence), without and with vad={} (alternated, best of --iters each), and the fraction of frames kept;
  * milliseconds of bank.select and bank.runs (all utterances) on a 20 000-utterance bank (200-1 200 frames each) with
    a speech-like mask keeping about 60 % of the frames (host clock around calls that end in a device synchronise);
  * milliseconds of diarize on the one-hour synthetic recording of tools/bench_diarize.py (360 000 frames, T = 160,
    hop = 40, 4 speakers), without a mask and with a mask keeping about 60 % of the frames in runs;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_vad.py
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info  # noqa: E402


def speech_mask(n, rng, keep=0.6, mean_run=150):
    """Alternating kept / dropped runs of geometric lengths, about ``keep`` of the frames kept."""
    import numpy as np

    out = np.zeros(n, bool)
    f, on = 0, True
    while f < n:
        m = int(rng.geometric(1.0 / (mean_run if on else mean_run * (1 - keep) / keep)))
        out[f:f + m] = on
        f += m
        on = not on
    return out


def timed(fn, iters):
    import torch

    best = float("inf")
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import diarization as DZ
    from deepspeaker_pytorch_b200 import frontend as F
    from oracle import rescnn_oracle as O

    assert torch.cuda.is_available(), "bench_vad needs a GPU"
    dev = torch.device("cuda:0")
    rec = {"metric": "vad", **gpu_info()}
    rng = np.random.default_rng(0)

    waves = []
    for _ in range(2000):
        n = int(rng.uniform(4, 12) * 16000)
        lab = np.repeat(speech_mask(n // 160 + 1, rng), 160)[:n]
        waves.append((np.where(lab, 0.1, 1e-5) * rng.standard_normal(n)).astype(np.float32))
    rec["waveforms"] = len(waves)
    rec["audio_hours"] = round(sum(w.size for w in waves) / 16000 / 3600, 2)
    F.FeatureBank.from_waveforms(waves[:50], vad={})          # warm-up
    t_plain, t_vad = float("inf"), float("inf")
    for _ in range(args.iters):
        t_plain = min(t_plain, timed(lambda: F.FeatureBank.from_waveforms(waves), 1))
        t_vad = min(t_vad, timed(lambda: F.FeatureBank.from_waveforms(waves, vad={}), 1))
    rec["from_waveforms_s"] = round(t_plain, 3)
    rec["from_waveforms_vad_s"] = round(t_vad, 3)
    bank = F.FeatureBank.from_waveforms(waves, vad={})
    rec["from_waveforms_vad_speech_fraction"] = round(float(bank.speech.float().mean()), 3)
    del bank, waves

    lens = rng.integers(200, 1201, 20000)
    off = np.concatenate(([0], np.cumsum(lens)))
    n = int(off[-1])
    bank = F.FeatureBank(torch.randn(n, 64, device=dev), off)
    mask = speech_mask(n, rng)
    mask[off[:-1]] = True                                    # every utterance keeps a frame
    md = torch.from_numpy(mask).to(dev)
    utt = np.arange(20000)
    bank.select(md)
    bank.runs(md, utt)
    rec["bank_frames"] = n
    rec["bank_kept_fraction"] = round(float(mask.mean()), 3)
    rec["select_ms"] = round(timed(lambda: bank.select(md), args.iters * 3) * 1e3, 2)
    rec["runs_ms"] = round(timed(lambda: bank.runs(md, utt), args.iters * 3) * 1e3, 2)
    rec["runs"] = int(bank.runs(md, utt)[1].numel())
    del bank

    model = dsk.DeepSpeakerModel(512, 16).to(dev)
    model.load_state_dict(O.make_state_dict(0, num_classes=16))
    model.eval()
    bank = F.FeatureBank.from_arrays([rng.standard_normal((360000, 64), dtype=np.float32)])
    sp = torch.from_numpy(speech_mask(360000, rng)).to(dev)
    DZ.diarize(model, bank, [0], num_speakers=4)
    DZ.diarize(model, bank, [0], num_speakers=4, speech=sp)
    rec["diarize_1h_ms"] = round(timed(lambda: DZ.diarize(model, bank, [0], num_speakers=4), args.iters) * 1e3, 1)
    rec["diarize_1h_speech_ms"] = round(
        timed(lambda: DZ.diarize(model, bank, [0], num_speakers=4, speech=sp), args.iters) * 1e3, 1)
    rec["diarize_1h_speech_fraction"] = round(float(sp.float().mean()), 3)
    rec["diarize_1h_speech_windows"] = int(DZ.diarize(model, bank, [0], num_speakers=4, speech=sp)[0].window_labels.size)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
