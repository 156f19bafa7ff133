"""Speed-perturbed training input: ``WaveBank.augmented_crops`` with and without speed factors {0.9, 1.0, 1.1} at
B = 384, T = 160 (25 840 samples per segment).

Prints one JSON line:
  - ms per call (CUDA events) for clean segments, speed only, everything (1 s RIR + one noise source + babble x 3)
    and everything with speed, with device banks, and the last two with the banks in page-locked host memory;
  - a per-kernel split of the everything-with-speed case, device and pinned banks, from a separate torch.profiler run;
  - the speed kernel's bank reads (the int16 samples each tile stages, computed from the plan) over its profiled time,
    as achieved GB/s;
  - ``aam_softmax_step`` ms (N = 384, T = 160, 1 211 speakers, FusedAdagrad) fed by ``augmented_crops`` (everything)
    without speed (1 211 classes) and with speed (3 633 classes, ``speed_labels``), alternated;
  - the card's name and power limit (read-only nvidia-smi query in the same run).
Synthetic data from fixed seeds; plans and indices are device-resident.  Writes nothing but stdout.
Run: python tools/bench_speed.py
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

    assert torch.cuda.is_available(), "bench_speed needs a GPU"
    rec = {"metric": "speed_perturb", **gpu_info()}
    B, T, C = 384, 160, 1211
    Ls = F.segment_samples(T)
    g = np.random.default_rng(0)

    def pcm(n):
        return np.round(np.clip(g.normal(0, 0.1, n), -1, 32767 / 32768) * 32768).astype(np.int16)

    speech = [pcm(n) for n in g.integers(4 * 16000, 12 * 16000, args.utts)]
    noise = [pcm(n) for n in g.integers(5 * 16000, 30 * 16000, 300)]
    rirs = [g.normal(size=16000) * np.exp(-np.arange(16000) / 3200.0) for _ in range(100)]
    sb, nb, rb = F.WaveBank.from_waveforms(speech), F.WaveBank.from_waveforms(noise), F.RirBank.from_arrays(rirs)
    sbh, nbh = F.WaveBank.from_waveforms(speech, pin=True), F.WaveBank.from_waveforms(noise, pin=True)
    rbh = F.RirBank.from_arrays(rirs, pin=True)

    allu = range(nb.num_utterances)
    groups = [(allu, (0.0, 15.0), (1, 1), 1.0)]
    babble = [(allu, (13.0, 20.0), (3, 3), 1.0)]

    def plan(everything, speed, seed=1):
        p = F.augment_plan(B, Ls, np.random.default_rng(seed), rb if everything else None, 1.0 if everything else 0.0,
                           nb if everything else None, groups if everything else (), 1.0 if everything else 0.0,
                           speeds=(0.9, 1.0, 1.1) if speed else None)
        if everything:                         # each example gets one noise source and babble x 3
            p2 = F.augment_plan(B, Ls, np.random.default_rng(seed + 1), None, 0.0, nb, babble, 1.0)
            for k in ("noise_idx", "noise_start", "snr_db"):
                p[k] = torch.cat([p[k], p2[k]], 1)
        else:
            for k in ("rir_idx", "noise_idx", "noise_start", "snr_db"):
                del p[k]
        return p

    def dev(p):
        return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in p.items()}

    utt_h = g.integers(0, sb.num_utterances, B)
    plans = {"clean": plan(False, False), "speed": plan(False, True), "all": plan(True, False), "all_speed": plan(True, True)}
    starts = {k: sb.random_starts(utt_h, Ls, np.random.default_rng(5), p).cuda() for k, p in plans.items()}
    utt = torch.from_numpy(utt_h).cuda()
    tm, fm = (m.cuda() for m in F.spec_augment_masks(B, T, 2, 20, 2, 8, g))
    dplans = {k: dev(p) for k, p in plans.items()}
    calls = {k: (lambda k=k: sb.augmented_crops(utt, starts[k], T, dplans[k], rb, nb, tm, fm)) for k in plans}
    for k in ("all", "all_speed"):
        calls[k + "_host_banks"] = lambda k=k: sbh.augmented_crops(utt, starts[k], T, dplans[k], rbh, nbh, tm, fm)
    ms = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ms[name] = round(time_events(fn, args.iters), 4)
    rec["augmented_crops_ms"] = ms
    rec["speed_adds_ms"] = {"clean": round(ms["speed"] - ms["clean"], 4), "all": round(ms["all_speed"] - ms["all"], 4),
                            "all_host_banks": round(ms["all_speed_host_banks"] - ms["all_host_banks"], 4)}

    # bank samples the speed kernel stages: per tile of 1024 outputs, m_last - m_first + 50 int16 samples
    sp = plans["all_speed"]
    alpha = [None] + list(sp["speeds"])
    staged = 0
    for k in sp["speed_idx"].numpy():
        a = alpha[k + 1]
        if a is None or a == 1:
            continue
        i0 = np.arange(0, Ls, 1024)
        i1 = np.minimum(i0 + 1023, Ls - 1)
        staged += int(np.sum(i1 * a.numerator // a.denominator - i0 * a.numerator // a.denominator + 50))
    rec["speed_examples"] = int(sum(1 for k in sp["speed_idx"].numpy() if alpha[k + 1] not in (None, 1)))
    rec["speed_bank_bytes_per_call"] = 2 * staged

    # per-kernel split of the everything-with-speed case, in runs of their own
    from torch.profiler import ProfilerActivity, profile

    for name in ("all_speed", "all_speed_host_banks"):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                calls[name]()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t > 0 and ev.count > 0:
                split[ev.key[:60]] = round(t / 10 / 1000, 4)       # ms per call
        rec[name + "_kernel_split_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1]))
        speed_ms = sum(v for k, v in split.items() if "aug_speed_kernel" in k)
        rec[name + "_speed_kernel_bank_gb_s"] = round(2 * staged / (speed_ms * 1e-3) / 1e9, 2) if speed_ms else None

    # aam_softmax_step fed with and without speed, alternated
    P, K = 96, 4
    labels = torch.from_numpy(np.repeat(g.choice(C, P, replace=False), K))
    su = np.repeat(g.choice(sb.num_utterances, P, replace=False), K)
    feeds = {}
    for name, speed in (("without_speed", False), ("with_speed", True)):
        p = plan(True, speed, seed=11)
        st = sb.random_starts(su, Ls, np.random.default_rng(12), p).cuda()
        ncls = C * (3 if speed else 1)
        lab = F.speed_labels(labels, p, C).cuda()
        model = dsk.DeepSpeakerModel(512, ncls).cuda()
        model.load_state_dict(O.make_state_dict(0, num_classes=ncls))
        model.train()
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        dp, u = dev(p), torch.from_numpy(su).cuda()
        feeds[name] = (lambda model=model, opt=opt, dp=dp, st=st, lab=lab, u=u: dsk.aam_softmax_step(
            model, opt, sb.augmented_crops(u, st, T, dp, rb, nb, tm, fm), lab, margin=0.2, scale=30.0))
    for _ in range(args.warmup):
        for fn in feeds.values():
            fn()
    step_ms = {k: [] for k in feeds}
    for _ in range(3):
        for k, fn in feeds.items():
            step_ms[k].append(time_events(fn, args.steps))
    rec["aam_softmax_step_ms"] = {k: round(min(v), 3) for k, v in step_ms.items()}
    rec["aam_softmax_step_ms_all_rounds"] = {k: [round(x, 3) for x in v] for k, v in step_ms.items()}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
