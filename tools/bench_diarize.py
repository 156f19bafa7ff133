"""Diarization: one JSON line with
  * milliseconds per engine.ahc call (CUDA events; the call synchronises once per 64 rounds) at N = 4 800 and 20 000
    speaker-clustered cosines (16 speakers, D = 512), average and complete linkage, the full tree and a threshold stop
    (at the height of the full tree's merge N - 16), with the number of merge rounds of each;
  * seconds of scipy.cluster.hierarchy.linkage on the same fp64 distances on the host cores (one call each; the
    condensed matrix is built outside the timed call);
  * the chain input of tests/test_gpu_diarization.py (N = 3 000, one mutual pair per round, N - 1 rounds): ms and
    rounds, the worst case for the number of rounds;
  * diarize on a one-hour synthetic recording (360 000 frames of random features, T = 160, hop = 40: 8 997 windows,
    4 speakers), split into window embedding, affinity (cosine_matrix) and clustering (ahc) plus the host assembly;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_diarize.py
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


def clustered_cosines(N, dev, seed):
    import torch

    from deepspeaker_pytorch_b200 import engine as EN

    g = torch.Generator(device=dev).manual_seed(seed)
    C = torch.randn(16, 512, device=dev, generator=g)
    X = C[torch.randint(0, 16, (N,), device=dev, generator=g)] + 0.8 * torch.randn(N, 512, device=dev, generator=g)
    return EN.cosine_matrix(X, X)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--scipy", type=int, default=1, help="1: time scipy's linkage on the same matrices")
    args = ap.parse_args()
    import numpy as np
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import diarization as DZ
    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200 import frontend as F

    assert torch.cuda.is_available(), "bench_diarize needs a GPU"
    dev = torch.device("cuda:0")
    rec = {"metric": "diarize", **gpu_info(), "host_cpus": os.cpu_count()}

    for N in (4800, 20000):
        S = clustered_cosines(N, dev, N)
        for method in ("average", "complete"):
            Z, _, rounds = EN.ahc(S, method, return_rounds=True)
            t = float(Z[N - 16, 2])
            _, _, rounds_t = EN.ahc(S, method, threshold=t, return_rounds=True)
            rec[f"ahc_ms_{method}_N{N}_full"] = round(time_events(lambda: EN.ahc(S, method), args.iters), 2)
            rec[f"ahc_rounds_{method}_N{N}_full"] = rounds
            rec[f"ahc_ms_{method}_N{N}_threshold"] = round(
                time_events(lambda: EN.ahc(S, method, threshold=t), args.iters), 2)
            rec[f"ahc_rounds_{method}_N{N}_threshold"] = rounds_t
        if args.scipy:
            from scipy.cluster.hierarchy import linkage
            from scipy.spatial.distance import squareform

            d = 1.0 - S.cpu().numpy().astype(np.float64)
            d = np.triu(d, 1)
            cond = squareform(d + d.T, checks=False)
            del d
            for method in ("average", "complete"):
                t0 = time.perf_counter()
                linkage(cond, method)
                rec[f"scipy_linkage_s_{method}_N{N}"] = round(time.perf_counter() - t0, 2)
            del cond
        del S

    # the chain: d(i, j) = (j (N + 1) - i) 2^-24 for i < j, one mutual pair per round (tests/test_gpu_diarization.py)
    N = 3000
    j = np.arange(N, dtype=np.int64)
    d = np.maximum(j[None, :], j[:, None]) * (N + 1) - np.minimum(j[None, :], j[:, None])
    S = torch.from_numpy((1.0 - d * 2.0 ** -24).astype(np.float32)).to(dev)
    for method in ("average", "complete"):
        _, _, rounds = EN.ahc(S, method, return_rounds=True)
        rec[f"chain_ms_{method}_N3000"] = round(time_events(lambda: EN.ahc(S, method), args.iters), 2)
        rec[f"chain_rounds_{method}_N3000"] = rounds

    # one hour of audio
    from oracle import rescnn_oracle as O

    model = dsk.DeepSpeakerModel(512, 16).to(dev)
    model.load_state_dict(O.make_state_dict(0, num_classes=16))
    model.eval()
    rng = np.random.default_rng(0)
    bank = F.FeatureBank.from_arrays([rng.standard_normal((360000, 64), dtype=np.float32)])
    T, hop = 160, 40
    DZ.diarize(model, bank, [0], T=T, hop=hop, num_speakers=4)           # warm-up (plans, graphs)
    times = {"embed": [], "affinity": [], "cluster": [], "total": []}
    for _ in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emb, _, ws, _ = F.window_embeddings(model, bank, [0], T, hop)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        S = EN.cosine_matrix(emb, emb)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        _, lab = EN.ahc(S, "average", num_clusters=4)
        DZ.segments(DZ.frame_labels(ws.numpy(), lab.cpu().numpy(), 360000, T))
        t3 = time.perf_counter()
        for k, v in zip(times, (t1 - t0, t2 - t1, t3 - t2, t3 - t0)):
            times[k].append(v * 1e3)
        del S
    rec["diarize_1h_windows"] = int(emb.shape[0])
    for k, v in times.items():
        rec[f"diarize_1h_ms_{k}"] = round(min(v), 1)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
