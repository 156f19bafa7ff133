"""Cosine scoring with AS-norm: one JSON line with
  * milliseconds per cohort_stats call at (M, Nc, k, D) = (4874, 5994, 300, 512) and (131072, 5994, 300, 512) (CUDA
    events around --iters back-to-back calls), beside the same statistics as torch ops on the same card (F.normalize,
    fp32 matmul with TF32 off, torch.topk, mean / std, in row chunks of the same 256 MiB bound);
  * a per-kernel split of one call from torch.profiler, in a window of its own: the GEMM (conv_umma_kernel), the
    selection (topk_select_stats_kernel) and the norm / split kernels; the GEMM's achieved tensor TFLOP/s
    (3 * 2 * M * Npad * D: hi/lo operands triple K) and the selection's GB/s (M * Nc * 4 bytes read);
  * milliseconds per score_trials call (AS-norm, statistics given) for 40 000 and 600 000 trials at U = 40 000, beside
    torch ops (gather, fp32 dot, the normalisation);
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_score_norm.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402


def chunk_rows(M, Nc):
    """Rows per chunk of dsk_cohort_stats (include/dsk.h)."""
    Np = (Nc + 127) // 128 * 128
    return min(max(128, (256 << 20) // (Np * 4) // 128 * 128), (M + 127) // 128 * 128)


def kernel_split(fn):
    """Device time (ms) per kernel family of one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"gemm": 0.0, "select": 0.0, "prep": 0.0, "other": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        key = ("gemm" if "conv_umma_kernel" in name else "select" if "topk_select_stats" in name else
               "prep" if ("aam_norm_kernel" in name or "aam_split_kernel" in name) else "other")
        split[key] += us / 1e3
    return {k: round(v, 4) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200 import verification as V

    assert torch.cuda.is_available(), "bench_score_norm needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "score_norm", **gpu_info()}
    Nc, k, D = 5994, 300, 512
    Np = (Nc + 127) // 128 * 128
    cohort = torch.randn(Nc, D, device=dev, generator=g)

    def torch_stats(E):
        Cn = F.normalize(cohort)
        En = F.normalize(E)
        ch = chunk_rows(E.shape[0], Nc)
        means, stds = [], []
        for r0 in range(0, E.shape[0], ch):
            top = torch.topk(En[r0:r0 + ch] @ Cn.T, k, dim=1).values
            means.append(top.mean(dim=1))
            stds.append(top.std(dim=1))
        return torch.cat(means), torch.cat(stds)

    for M in (4874, 131072):
        E = torch.randn(M, D, device=dev, generator=g)
        iters = args.iters * (10 if M < 10000 else 1)
        op = lambda E=E: V.cohort_stats(E, cohort, k)      # noqa: E731
        ref = lambda E=E: torch_stats(E)                    # noqa: E731
        for fn in (op, ref):
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        m_op, m_ref = [], []
        for _ in range(2):                                  # alternated, so both see the same card state
            m_op.append(time_events(op, iters))
            m_ref.append(time_events(ref, max(2, iters // 4)))
        tag = f"M{M}_Nc{Nc}_k{k}_D{D}"
        rec[f"cohort_stats_ms_{tag}"] = [round(t, 4) for t in m_op]
        rec[f"torch_ops_ms_{tag}"] = [round(t, 4) for t in m_ref]
        mo, mt = op(), ref()
        rec[f"max_abs_dmean_vs_torch_{tag}"] = float((mo[0] - mt[0]).abs().max())
        split = kernel_split(op)
        rec[f"kernel_ms_{tag}"] = split
        rec[f"chunks_{tag}"] = -(-M // chunk_rows(M, Nc))
        if split["gemm"] > 0:
            rec[f"gemm_tensor_tflops_{tag}"] = round(3 * 2 * M * Np * D / (split["gemm"] * 1e-3) / 1e12, 1)
        if split["select"] > 0:
            rec[f"select_gb_per_s_{tag}"] = round(M * Nc * 4 / (split["select"] * 1e-3) / 1e9, 1)
        del E

    U = 40000
    X = torch.randn(U, D, device=dev, generator=g)
    mean, std = V.cohort_stats(X, cohort, k)
    for T in (40000, 600000):
        trials = torch.randint(0, U, (T, 2), device=dev, generator=g)
        op = lambda trials=trials: EN.score_trials(X, trials, mean, std)   # noqa: E731

        def ref(trials=trials):
            Xn = F.normalize(X)
            e, t = trials[:, 0], trials[:, 1]
            s = (Xn[e] * Xn[t]).sum(dim=1)
            return s, 0.5 * ((s - mean[e]) / std[e] + (s - mean[t]) / std[t])

        for fn in (op, ref):
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        m_op, m_ref = [], []
        for _ in range(2):
            m_op.append(time_events(op, args.iters * 5))
            m_ref.append(time_events(ref, args.iters * 5))
        rec[f"score_trials_ms_T{T}"] = [round(t, 4) for t in m_op]
        rec[f"torch_ops_ms_T{T}"] = [round(t, 4) for t in m_ref]
    rec["score_trials_shape"] = {"U": U, "D": D}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
