"""VBx: one JSON line with
  * milliseconds per engine.vbx call and per iteration (CUDA events; the call reads its finished-recordings count once
    per 8 iterations) on the one-hour recording of bench_diarize.py (8 997 windows at hop 40), d = 128 synthetic
    PLDA-space rows, 16 and 64 initial clusters, all 40 iterations forced (epsilon = -inf);
  * the same for 64 ten-minute recordings (1 497 windows each, 16 initial clusters) in one call;
  * a per-kernel split from torch.profiler in a separate run of each of those calls, with the forward-backward's time
    per window (one forward and one backward step);
  * the fp64 oracle's seconds per iteration on the host cores for the one-hour recording (2 iterations timed);
  * diarize(plda=, vbx={}) on a one-hour synthetic recording (360 000 frames of random features, the model of
    bench_diarize.py, a PLDA fitted on synthetic 512-d speakers, lda_dim 128, 16 initial AHC clusters), split into
    window embedding, AHC (transform, LLR matrix, clustering) and VBx;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_vbx.py
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

ITERS = 40


def synthetic(rng, lens, d, clusters):
    """PLDA-space rows of recordings with 4 speakers each (HMM turns, self-loop 0.99) and initial labels over
    ``clusters`` clusters."""
    import numpy as np

    phi = np.sort(rng.gamma(2.0, 1.0, size=d))[::-1].copy()
    X, lab = [], []
    for n in lens:
        Y = rng.normal(size=(4, d))
        z = np.zeros(n, np.int64)
        jump = rng.integers(4, size=n)
        stay = rng.random(n) < 0.99
        for t in range(1, n):
            z[t] = z[t - 1] if stay[t] else jump[t]
        X.append(np.sqrt(phi) * Y[z] + rng.normal(size=(n, d)))
        lab.append((z * (clusters // 4) + rng.integers(0, clusters // 4, size=n)) % clusters)
    return (np.concatenate(X).astype(np.float32), np.concatenate(lab).astype(np.int32), phi,
            np.concatenate(([0], np.cumsum(lens))).astype(np.int64))


def kernel_split(fn):
    """{kernel: ms} summed over one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "vbx" in ev.key:
            name = ev.key.split("vbx_")[1].split("_kernel")[0]
            out[name] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3, help="timed calls per configuration")
    ap.add_argument("--oracle", type=int, default=1, help="1: time the fp64 oracle on the host")
    args = ap.parse_args()
    import numpy as np
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import diarization as DZ
    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200 import frontend as F
    from deepspeaker_pytorch_b200 import plda as P

    assert torch.cuda.is_available(), "bench_vbx needs a GPU"
    dev = torch.device("cuda:0")
    rec = {"metric": "vbx", **gpu_info(), "host_cpus": os.cpu_count(), "iterations": ITERS}
    rng = np.random.default_rng(0)
    configs = [("1h_k16", [8997], 16), ("1h_k64", [8997], 64), ("64x10min_k16", [1497] * 64, 16)]
    for name, lens, k in configs:
        X, lab, phi, off = synthetic(rng, lens, 128, k)
        Xd, ld = torch.from_numpy(X).to(dev), torch.from_numpy(lab).to(dev)

        def call():
            return EN.vbx(Xd, off, ld, phi, 0.3, 17.0, 0.99, 5.0, ITERS, -np.inf)

        res = call()                                                     # warm-up
        assert int(res[3].min()) == ITERS
        ms = time_events(call, args.iters)
        rec[f"vbx_ms_{name}"] = round(ms, 2)
        rec[f"vbx_ms_per_iter_{name}"] = round(ms / ITERS, 3)
        split = kernel_split(call)
        rec[f"vbx_kernel_ms_{name}"] = split
        if "fb" in split:                                                # one warp per recording, all in parallel
            rec[f"vbx_fb_us_per_window_{name}"] = round(split["fb"] * 1e3 / ITERS / lens[0], 4)
        if args.oracle and len(lens) == 1:
            from oracle import vbx_oracle as O

            t0 = time.perf_counter()
            O.vbx(X, phi, lab, max_iters=2, epsilon=-np.inf)
            rec[f"oracle_s_per_iter_{name}"] = round((time.perf_counter() - t0) / 2, 2)

    # diarize with VBx on one hour of audio
    from oracle import rescnn_oracle as RO

    model = dsk.DeepSpeakerModel(512, 16).to(dev)
    model.load_state_dict(RO.make_state_dict(0, num_classes=16))
    model.eval()
    C, n = 400, 10
    centres = rng.normal(size=(C, 512))
    E = torch.from_numpy((np.repeat(centres, n, axis=0) + rng.normal(size=(C * n, 512))).astype(np.float32)).to(dev)
    be = P.fit(E, np.repeat(np.arange(C), n), lda_dim=128)
    bank = F.FeatureBank.from_arrays([rng.standard_normal((360000, 64), dtype=np.float32)])
    T, hop, k = 160, 40, 16
    DZ.diarize(model, bank, [0], T=T, hop=hop, num_speakers=k, plda=be, vbx={})      # warm-up
    times = {"embed": [], "ahc": [], "vbx": [], "total": []}
    for _ in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emb, _, ws, _ = F.window_embeddings(model, bank, [0], T, hop)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        Z, lab = DZ._cluster(emb, be, None, "average", k)
        lab = lab.cpu().numpy()
        t2 = time.perf_counter()
        res = DZ.vbx(be, emb, [0, emb.shape[0]], lab)
        DZ.segments(DZ.frame_labels(ws.numpy(), res.labels, 360000, T))
        t3 = time.perf_counter()
        for key, v in zip(times, (t1 - t0, t2 - t1, t3 - t2, t3 - t0)):
            times[key].append(v * 1e3)
    rec["diarize_vbx_1h_windows"] = int(emb.shape[0])
    rec["diarize_vbx_1h_iterations"] = int(res.iters[0])
    rec["diarize_vbx_1h_speakers"] = int(res.labels.max()) + 1
    for key, v in times.items():
        rec[f"diarize_vbx_1h_ms_{key}"] = round(min(v), 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    DZ.diarize(model, bank, [0], T=T, hop=hop, num_speakers=k, plda=be, vbx={})
    rec["diarize_vbx_1h_ms_call"] = round((time.perf_counter() - t0) * 1e3, 1)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
