"""PLDA backend: one JSON line with
  * ``plda.fit`` at VoxCeleb2-dev size, (N, D, C) = (1 092 009, 512, 5 994), lda_dim 200, 10 EM iterations (seeded
    synthetic speakers): the whole call (host clock around a device synchronise), and its GPU passes timed on their
    own with CUDA events (class sums, Gram of x - mu, the LDA + length-norm transform, Gram of the 200-d outputs) beside
    the host algebra (LDA eigendecompositions, EM, diagonalisation);
  * the Gram's achieved fp64 TFLOP/s, FLOP = 2 N D (D + 1) / 2 (the upper triangle it computes), against the H100 SXM
    data sheet's 67 TFLOP/s FP64 tensor-core rate;
  * ``score_trials`` at 37 720 and 600 000 trials, and ``score_matrix`` at W = 8 997 (a one-hour recording's windows
    at hop 40), d = 200;
  * the same operations as torch fp64 ops on the same card (Gram by one fp64 matmul of the centred rows, the trials by
    gathered rows, the matrix in the same expanded form);
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_plda.py
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

FP64_TC_PEAK = 67.0    # TFLOP/s, H100 SXM data sheet (dense FP64 tensor core), for a card allowed 700 W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1092009)
    ap.add_argument("--D", type=int, default=512)
    ap.add_argument("--C", type=int, default=5994)
    ap.add_argument("--dim", type=int, default=200)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch

    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200 import plda as P
    from deepspeaker_pytorch_b200.identification import speaker_csr

    if not torch.cuda.is_available():
        raise SystemExit("bench_plda needs a GPU")
    dev = torch.device("cuda:0")
    N, D, C, d = args.N, args.D, args.C, args.dim
    g = torch.Generator(device=dev).manual_seed(0)
    lab = np.random.default_rng(0).permutation(np.arange(N) % C)
    scale = torch.linspace(0.3, 1.5, D, device=dev)
    centres = torch.randn(C, D, device=dev, generator=g) * scale
    X = centres[torch.from_numpy(lab).to(dev)] + torch.randn(N, D, device=dev, generator=g) * scale.flip(0) + 0.5
    del centres
    out = {"N": N, "D": D, "C": C, "lda_dim": d}

    # the whole fit (one warm-up call loads the kernels)
    P.fit(X[:20000], lab[:20000], lda_dim=min(d, 99), iters=1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    be = P.fit(X, lab, lda_dim=d, iters=10)
    torch.cuda.synchronize()
    out["fit_s"] = round(time.perf_counter() - t0, 3)

    # its GPU passes on their own
    order, offsets, _ = speaker_csr(lab)
    od, ofd = torch.from_numpy(order).to(dev), torch.from_numpy(offsets).to(dev)
    mu = be.mu.to(dev)
    L = be.lda.to(dev)
    it = args.iters
    passes = {
        "class_sums_ms": time_events(lambda: EN.class_sums_f64(X, od, ofd, mu), it),
        "gram_ms": time_events(lambda: EN.gram_f64(X, mu), it),
        "transform_ms": time_events(lambda: EN.affine_norm_f64(X, L, mu, mode="length"), it),
    }
    Y = EN.affine_norm_f64(X, L, mu, mode="length")
    passes["gram_d_ms"] = time_events(lambda: EN.gram_f64(Y), it)
    passes["class_sums_d_ms"] = time_events(lambda: EN.class_sums_f64(Y, od, ofd), it)
    out["fit_gpu_passes"] = {k: round(v, 3) for k, v in passes.items()}
    gpu_total = (2 * passes["class_sums_ms"] + passes["gram_ms"] + passes["transform_ms"] + passes["gram_d_ms"]
                 + passes["class_sums_d_ms"])
    out["fit_gpu_passes_total_ms"] = round(gpu_total, 2)
    # host algebra, from the same statistics
    counts = np.diff(offsets)
    s = EN.class_sums_f64(X, od, ofd, mu).cpu().numpy()
    G = EN.gram_f64(X, mu).cpu().numpy()
    sy = EN.class_sums_f64(Y, od, ofd).cpu().numpy()
    Gy = EN.gram_f64(Y).cpu().numpy()
    t0 = time.perf_counter()
    P.lda_from_stats(G / N, s.T @ (s / counts[:, None]) / N, d)
    t1 = time.perf_counter()
    means = sy / counts[:, None]
    pw, pb = P.plda_em(Gy - sy.T @ means, means - means.mean(axis=0), counts, 10)
    P.diagonalise(pw, pb)
    t2 = time.perf_counter()
    out["fit_host_ms"] = {"lda": round((t1 - t0) * 1e3, 1), "em_and_diagonalise": round((t2 - t1) * 1e3, 1)}
    flop = 2.0 * N * D * (D + 1) / 2
    out["gram_tflops"] = round(flop / passes["gram_ms"] / 1e9, 2)
    out["gram_share_of_fp64_tc_peak"] = round(flop / passes["gram_ms"] / 1e9 / FP64_TC_PEAK, 3)

    # torch fp64 for comparison: the Gram (the upper triangle is not separable in one matmul: the full D x D)
    def torch_gram():
        Xc = X.double() - mu
        return Xc.T @ Xc

    torch_gram()
    out["torch_fp64_gram_ms"] = round(time_events(torch_gram, it), 3)

    # scoring
    U = 40000
    Ys = be.transform(X[:U])
    psi = be.psi.to(dev)
    rng = np.random.default_rng(1)
    sc = {}
    for T in (37720, 600000):
        trials = torch.from_numpy(rng.integers(0, U, size=(T, 2))).to(dev)
        be.score_trials(Ys, trials)
        sc[f"score_trials_{T}_ms"] = round(time_events(lambda: be.score_trials(Ys, trials), 20), 4)

        def torch_trials():
            e, t = Ys[trials[:, 0]].double(), Ys[trials[:, 1]].double()
            a, v1, v0 = psi / (psi + 1), 1 + psi / (psi + 1), 1 + psi
            return (-0.5 * (torch.log(v1) + (t - a * e) ** 2 / v1) + 0.5 * (torch.log(v0) + t * t / v0)).sum(1).float()

        torch_trials()
        sc[f"torch_fp64_score_trials_{T}_ms"] = round(time_events(torch_trials, 20), 4)
    W = 8997
    Yw = Ys[:W].contiguous()
    be.score_matrix(Yw, Yw)
    sc[f"score_matrix_{W}_ms"] = round(time_events(lambda: be.score_matrix(Yw, Yw), 10), 3)

    def torch_matrix():
        Yd = Yw.double()
        w = -0.5 * psi * psi / ((1 + psi) * (2 * psi + 1))
        k = 0.5 * (torch.log(1 + psi) - torch.log((2 * psi + 1) / (1 + psi))).sum()
        q = (Yd * Yd * w).sum(1)
        return (k + q[:, None] + q[None, :] + (Yd * (psi / (2 * psi + 1))) @ Yd.T).float()

    torch_matrix()
    sc[f"torch_fp64_score_matrix_{W}_ms"] = round(time_events(torch_matrix, 10), 3)
    out.update(sc)
    out.update(gpu_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
