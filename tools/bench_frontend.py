"""Feature-bank front-end: one JSON line with
  (a) files/s and seconds of audio per second of ``mk_mfb_batch`` over 2 000 seeded synthetic waveforms of 4-12 s
      (16 kHz, one call), beside a loop of ``mk_mfb`` over the same waveforms (host clock around work ending in a
      device synchronise, alternated, best of --reps);
  (b) microseconds and GB/s written of ``bank.crops`` at B = 384, T = 160 with 2 time + 2 frequency masks from a bank of
      20 000 utterances (device indices, CUDA events over --iters calls), beside the same crops as torch ops (index
      arithmetic, advanced indexing, masked fill), and the host-fed path a training loop runs (``random_starts`` +
      ``spec_augment_masks`` on the host, then ``crops``);
  (c) ms per ``batch_hard_step`` at N = 384 (96 x 4), T = 160 with FusedAdagrad, fed by ``random_starts`` +
      ``spec_augment_masks`` + ``crops``, against the same step fed a resident tensor, alternated;
  (d) utterances/s of ``embed_utterances`` on 4 874 utterances of 4-20 s (400-2 000 frames) at T = 160, hop 80;
  and the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_frontend.py
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402


def host_time(fn, reps):
    import torch

    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--embed-utts", type=int, default=4874)
    args = ap.parse_args()
    import numpy as np
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import frontend as F
    from oracle import rescnn_oracle as O        # deterministic parameters only

    assert torch.cuda.is_available(), "bench_frontend needs a GPU"
    dev = torch.device("cuda:0")
    rec = {"metric": "frontend", **gpu_info()}
    rng = np.random.default_rng(0)

    # ---- (a) batched fbank vs one call per file
    sr = 16000
    lens = rng.integers(4 * sr, 12 * sr + 1, args.files)
    audio = torch.randn(int(lens.sum()), device=dev, generator=torch.Generator(device=dev).manual_seed(0)) * 0.1
    soff = np.concatenate(([0], np.cumsum(lens)))
    views = [audio[soff[i]:soff[i + 1]] for i in range(args.files)]
    batch = lambda: F.mk_mfb_batch(audio, lens, sr)  # noqa: E731
    loop = lambda: [F.mk_mfb(v, sr) for v in views]  # noqa: E731
    batch(), loop()
    tb = tl = float("inf")
    for _ in range(args.reps):
        tb = min(tb, host_time(batch, 1))
        tl = min(tl, host_time(loop, 1))
    secs = float(lens.sum()) / sr
    rec.update({"fbank_files": args.files, "fbank_audio_s": round(secs, 1),
                "fbank_batch_files_per_s": round(args.files / tb, 1), "fbank_batch_audio_s_per_s": round(secs / tb, 1),
                "fbank_loop_files_per_s": round(args.files / tl, 1), "fbank_loop_audio_s_per_s": round(secs / tl, 1)})
    del audio, views
    torch.cuda.empty_cache()

    # ---- (b) crops from a 20 000-utterance bank
    U, B, T = 20000, 384, 160
    nfr = rng.integers(200, 2001, U)
    off = np.concatenate(([0], np.cumsum(nfr))).astype(np.int64)
    bank = F.FeatureBank(torch.randn(int(off[-1]), 64, device=dev), off)
    utt = rng.integers(0, U, B)
    start = bank.random_starts(utt, T, rng)
    tm, fm = F.spec_augment_masks(B, T, 2, 20, 2, 8, rng)
    du, ds, dtm, dfm = (torch.as_tensor(t).to(dev) for t in (utt, start, tm, fm))
    offd = bank.offsets
    nd = offd[1:] - offd[:-1]
    ar = torch.arange(T, device=dev)
    mel = torch.arange(64, device=dev)

    def torch_crops():
        rows = offd[du][:, None] + (ds[:, None] + ar) % nd[du][:, None]
        x = bank.feats[rows]
        tmask = ((ar[None, None, :] >= dtm[:, :, :1]) & (ar[None, None, :] < dtm[:, :, :1] + dtm[:, :, 1:])).any(1)
        fmask = ((mel[None, None, :] >= dfm[:, :, :1]) & (mel[None, None, :] < dfm[:, :, :1] + dfm[:, :, 1:])).any(1)
        return x.masked_fill(tmask[:, :, None] | fmask[:, None, :], 0.0).unsqueeze(1)

    kern = lambda: bank.crops(du, ds, T, dtm, dfm)  # noqa: E731
    assert torch.equal(kern(), torch_crops())
    gen = np.random.default_rng(1)

    def host_fed():
        u = gen.integers(0, U, B)
        t_m, f_m = F.spec_augment_masks(B, T, 2, 20, 2, 8, gen)
        return bank.crops(torch.from_numpy(u), bank.random_starts(u, T, gen), T, t_m, f_m)

    out_bytes = B * T * 64 * 4
    for key, fn in (("kernel", kern), ("torch_ops", torch_crops)):
        for _ in range(20):
            fn()
        us = 1e3 * time_events(fn, args.iters)
        rec[f"crops_us_{key}"] = round(us, 2)
        rec[f"crops_gbs_written_{key}"] = round(out_bytes / us / 1e3, 1)
    for _ in range(20):
        host_fed()
    rec["crops_us_host_fed"] = round(1e6 * host_time(lambda: [host_fed() for _ in range(args.iters)], 1) / args.iters, 2)
    rec["crops_mb_written"] = round(out_bytes / 1e6, 2)

    # ---- (c) batch_hard_step fed by the bank vs a resident tensor
    P, K = 96, 4
    sd = O.make_state_dict(0, num_classes=16)
    model = dsk.DeepSpeakerModel(512, 16).to(dev).train()
    model.load_state_dict(sd)
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
    labels = torch.arange(P).repeat_interleave(K)
    resident = bank.crops(du, ds, T, dtm, dfm)

    def fed_step():
        spk = gen.choice(U // K, P, replace=False)
        u = (spk[:, None] * K + np.arange(K)).reshape(-1)
        t_m, f_m = F.spec_augment_masks(P * K, T, 2, 20, 2, 8, gen)
        x = bank.crops(torch.from_numpy(u), bank.random_starts(u, T, gen), T, t_m, f_m)
        dsk.batch_hard_step(model, opt, x, labels, margin=0.1)

    res_step = lambda: dsk.batch_hard_step(model, opt, resident, labels, margin=0.1)  # noqa: E731
    for _ in range(args.warmup):
        fed_step()
        res_step()
    tf = tr = float("inf")
    for _ in range(2):
        tr = min(tr, host_time(lambda: [res_step() for _ in range(args.steps)], 1) / args.steps)
        tf = min(tf, host_time(lambda: [fed_step() for _ in range(args.steps)], 1) / args.steps)
    rec.update({"step_ms_resident": round(1e3 * tr, 3), "step_ms_bank_fed": round(1e3 * tf, 3),
                "step_input_share": round((tf - tr) / tf, 4)})
    del bank, resident
    torch.cuda.empty_cache()

    # ---- (d) utterance embeddings
    nfr = rng.integers(400, 2001, args.embed_utts)
    off = np.concatenate(([0], np.cumsum(nfr))).astype(np.int64)
    ebank = F.FeatureBank(torch.randn(int(off[-1]), 64, device=dev), off)
    model.eval()
    every = np.arange(args.embed_utts)
    F.embed_utterances(model, ebank, every[:600], T=160, hop=80, batch=256)
    te = host_time(lambda: F.embed_utterances(model, ebank, every, T=160, hop=80, batch=256), 2)
    wins = ebank.windows(every, 160, 80)[0].numel()
    rec.update({"embed_utts": args.embed_utts, "embed_windows": wins, "embed_utts_per_s": round(args.embed_utts / te, 1),
                "embed_windows_per_s": round(wins / te, 1)})
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
