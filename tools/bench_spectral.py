"""Spectral clustering with NME-SC on the GPU: ``engine.spectral_cluster`` at N = 4 800 and 8 997 windows (about 40
and 75 minutes of speech at the diarization default hop) on clustered cosines of 5 speakers, with the default
30-point grid of pruning levels and with a single level, so the per-level cost and what solving the grid in the same
launches saves are both visible; a per-kernel split of the N = 4 800 grid call from torch.profiler, the filter's
achieved fp64 rate, ``diarize``'s window embedding, affinity and spectral clustering on the one-hour synthetic
recording of bench_diarize.py (not warmed up: the embedding time includes first-call set-up); and scipy's dense
``eigh`` of one level's Laplacian on the host at N = 4 800, the work a CPU implementation repeats per grid point.
Prints one JSON line with the card's name and power limit (a read-only nvidia-smi query in the same run).

    python tools/bench_spectral.py [--reps R]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_batch_hard import gpu_info  # noqa: E402


def clustered_cosines(N, dev, seed, K=5):
    import torch

    from deepspeaker_pytorch_b200 import engine as EN

    g = torch.Generator(device=dev).manual_seed(seed)
    C = torch.randn(K, 512, device=dev, generator=g)
    X = C[torch.randint(0, K, (N,), device=dev, generator=g)] + 0.8 * torch.randn(N, 512, device=dev, generator=g)
    return EN.cosine_matrix(X, X)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    from scipy.linalg import eigh

    from deepspeaker_pytorch_b200 import diarization as DZ
    from deepspeaker_pytorch_b200 import engine as EN
    from oracle import spectral_oracle as SO

    if not torch.cuda.is_available():
        raise SystemExit("bench_spectral needs a GPU")
    dev = torch.device("cuda")
    out = {"bench": "spectral_cluster", **gpu_info()}
    for N in (4800, 8997):
        S = clustered_cosines(N, dev, N)
        grid = DZ.p_grid(N)
        for name, pv in (("grid", grid), ("one_p", grid[len(grid) // 2:len(grid) // 2 + 1])):
            EN.spectral_cluster(S, pv)                 # warm-up: module load, allocator
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                res = EN.spectral_cluster(S, pv)       # the call synchronises the stream
                times.append(time.perf_counter() - t0)
            out[f"N{N}_{name}_s"] = float(np.median(times))
            out[f"N{N}_{name}_k"] = int(res[1])
        out[f"N{N}_grid_points"] = int(grid.size)
    # per-kernel split of one N = 4 800 grid call, from torch.profiler in a run of its own; the filter's achieved fp64
    # rate from the first matvec launch, in which every problem is active: 2 N^2 sum_q w_q flop (w_q the block width,
    # max(m + 8, 40) for the 30 smallest-eigenvalue problems and 8 for the 30 largest) over its device time
    from torch.profiler import ProfilerActivity, profile

    N = 4800
    S = clustered_cosines(N, dev, N)
    grid = DZ.p_grid(N)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        EN.spectral_cluster(S, grid)
        torch.cuda.synchronize()
    split, first_matvec = {}, None
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "sc_" not in ev.name:
            continue
        name = ev.name.split("sc_")[1].split("_kernel")[0]
        split[name] = split.get(name, 0.0) + ev.device_time / 1e3
        if name == "matvec" and first_matvec is None:
            first_matvec = ev.device_time
    out["N4800_grid_kernel_ms"] = {k: round(v, 1) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}
    flop = 2.0 * N * N * grid.size * (max(9 + 8, 40) + 8)
    out["N4800_filter_first_launch_us"] = round(first_matvec, 1)
    out["N4800_filter_fp64_tflops"] = round(flop / (first_matvec * 1e-6) / 1e12, 2)

    # diarize(spectral={}) on the one-hour synthetic recording of bench_diarize.py
    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import frontend as F
    from oracle import rescnn_oracle as RO

    model = dsk.DeepSpeakerModel(512, 16).to(dev)
    model.load_state_dict(RO.make_state_dict(0, num_classes=16))
    model.eval()
    rng = np.random.default_rng(0)
    bank = F.FeatureBank.from_arrays([rng.standard_normal((360000, 64), dtype=np.float32)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    emb, _, ws, _ = F.window_embeddings(model, bank, [0], 160, 40)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    A = EN.cosine_matrix(emb, emb)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    res = DZ.spectral(A)
    DZ.segments(DZ.frame_labels(ws.numpy(), res.labels.cpu().numpy(), 360000, 160))
    t3 = time.perf_counter()
    out["diarize_1h_windows"] = int(emb.shape[0])
    out["diarize_1h_spectral_k"] = int(res.k)
    out["diarize_1h_s_embed"], out["diarize_1h_s_affinity"], out["diarize_1h_s_cluster"] = (
        round(t1 - t0, 3), round(t2 - t1, 3), round(t3 - t2, 3))
    del A

    S = S.cpu().numpy()
    R = SO.ranks(S)
    grid = DZ.p_grid(N)
    for p in (int(grid[1]), int(grid[-1])):
        L_ = SO.laplacian(R, p)
        t0 = time.perf_counter()
        eigh(L_, eigvals_only=True)
        out[f"scipy_eigh_N{N}_p{p}_s"] = time.perf_counter() - t0
    print(json.dumps(out))


if __name__ == "__main__":
    main()
