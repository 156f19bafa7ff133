"""Waveform-augmented training input: ``WaveBank.augmented_crops`` at B = 384, T = 160 (25 840 samples per segment).

Prints one JSON line:
  - ms per call (CUDA events) for clean segments, one noise source, babble x 5, 0.5 s and 1 s RIRs, and everything
    together (1 s RIR + one noise source + babble x 3), with device banks, and the same for the last case with the
    speech, noise and RIR banks in page-locked host memory;
  - a per-kernel split of the "everything" case from a separate torch.profiler run;
  - ``batch_hard_step`` ms (N = 384, T = 160, FusedAdagrad) fed by ``augmented_crops`` (everything) vs
    ``FeatureBank.crops``, alternated;
  - the card's name and power limit (read-only nvidia-smi query in the same run).
Synthetic data from fixed seeds; plans and indices are device-resident.  Writes nothing but stdout.
Run: python tools/bench_augment.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--utts", type=int, default=2000)
    args = ap.parse_args()
    import numpy as np
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import frontend as F
    from oracle import rescnn_oracle as O        # deterministic parameters only

    assert torch.cuda.is_available(), "bench_augment needs a GPU"
    rec = {"metric": "augment", **gpu_info()}
    B, T = 384, 160
    Ls = F.segment_samples(T)
    g = np.random.default_rng(0)

    def pcm(n):
        return np.round(np.clip(g.normal(0, 0.1, n), -1, 32767 / 32768) * 32768).astype(np.int16)

    speech = [pcm(n) for n in g.integers(4 * 16000, 12 * 16000, args.utts)]
    noise = [pcm(n) for n in g.integers(5 * 16000, 30 * 16000, 300)]
    rirs = {lh: [g.normal(size=lh) * np.exp(-np.arange(lh) / 3200.0) for _ in range(100)] for lh in (8000, 16000)}
    sb, nb = F.WaveBank.from_waveforms(speech), F.WaveBank.from_waveforms(noise)
    rb = {lh: F.RirBank.from_arrays(r) for lh, r in rirs.items()}
    sbh, nbh = F.WaveBank.from_waveforms(speech, pin=True), F.WaveBank.from_waveforms(noise, pin=True)
    rbh = F.RirBank.from_arrays(rirs[16000], pin=True)
    rec["speech_bank_gb"] = round(sb.samples.numel() * 2 / 1e9, 3)

    utt = g.integers(0, sb.num_utterances, B)
    start = sb.random_starts(utt, Ls, g).cuda()
    utt = torch.from_numpy(utt).cuda()
    tm, fm = (m.cuda() for m in F.spec_augment_masks(B, T, 2, 20, 2, 8, g))
    allu = range(nb.num_utterances)
    noise1 = [(allu, (0.0, 15.0), (1, 1), 1.0)]

    def plan(rir=None, groups=(), babble=0):
        grp = list(groups) + ([(allu, (13.0, 20.0), (babble, babble), 1.0)] if babble else [])
        p = F.augment_plan(B, Ls, np.random.default_rng(1), rb[rir] if rir else None, 1.0 if rir else 0.0,
                           nb if grp else None, grp, 1.0 if grp else 0.0)
        if grp and babble and groups:          # everything: each example gets one noise source and babble
            p1 = F.augment_plan(B, Ls, np.random.default_rng(2), None, 0.0, nb, list(groups), 1.0)
            p2 = F.augment_plan(B, Ls, np.random.default_rng(3), None, 0.0, nb, grp[-1:], 1.0)
            for k in ("noise_idx", "noise_start", "snr_db"):
                p[k] = torch.cat([p1[k], p2[k]], 1)
        if not rir:
            del p["rir_idx"]
        return {k: v.cuda() for k, v in p.items()}, (rb[rir] if rir else None)

    cases = {"clean": plan(), "noise_x1": plan(groups=noise1), "babble_x5": plan(babble=5),
             "rir_0.5s": plan(rir=8000), "rir_1s": plan(rir=16000), "all": plan(rir=16000, groups=noise1, babble=3)}
    calls = {}
    for name, (p, r) in cases.items():
        calls[name] = (lambda p=p, r=r: sb.augmented_crops(utt, start, T, p, r, nb, tm, fm))
    pa, _ = cases["all"]
    calls["all_host_banks"] = lambda: sbh.augmented_crops(utt, start, T, pa, rbh, nbh, tm, fm)
    ms = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ms[name] = round(time_events(fn, args.iters), 4)
    rec["augmented_crops_ms"] = ms
    rec["fbank_frames_per_call"] = B * T

    # per-kernel split of the "all" case, in a run of its own
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            calls["all"]()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0 and ev.count > 0:
            split[ev.key[:60]] = round(t / 10 / 1000, 4)       # ms per call
    rec["all_kernel_split_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1]))

    # batch_hard_step fed by augmented crops vs feature-bank crops, alternated
    fbank = F.FeatureBank.from_arrays([g.standard_normal((n, 64)) for n in g.integers(400, 1200, args.utts)])
    P, K = 96, 4
    labels = torch.from_numpy(np.repeat(np.arange(P), K))
    su = torch.from_numpy(np.repeat(g.choice(sb.num_utterances, P, replace=False), K)).cuda()
    ss = sb.random_starts(su.cpu(), Ls, g).cuda()
    fu = torch.from_numpy(np.repeat(g.choice(fbank.num_utterances, P, replace=False), K)).cuda()
    fs = fbank.random_starts(fu.cpu(), T, g).cuda()
    model = dsk.DeepSpeakerModel(512, 16).cuda()
    model.load_state_dict(O.make_state_dict(0, num_classes=16))
    model.train()
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
    feeds = {"augmented_crops": lambda: sb.augmented_crops(su, ss, T, pa, rb[16000], nb, tm, fm),
             "feature_bank_crops": lambda: fbank.crops(fu, fs, T, tm, fm)}
    step_ms = {k: [] for k in feeds}
    for _ in range(args.warmup):
        for fn in feeds.values():
            dsk.batch_hard_step(model, opt, fn(), labels, margin=0.1)
    for _ in range(3):
        for k, fn in feeds.items():
            step_ms[k].append(time_events(lambda: dsk.batch_hard_step(model, opt, fn(), labels, margin=0.1), args.steps))
    rec["batch_hard_step_ms"] = {k: round(min(v), 3) for k, v in step_ms.items()}
    rec["batch_hard_step_ms_all_rounds"] = {k: [round(x, 3) for x in v] for k, v in step_ms.items()}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
