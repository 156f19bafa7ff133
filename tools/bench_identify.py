"""Speaker identification: one JSON line with
  * milliseconds per search call (CUDA events around back-to-back calls) for
      (a) M = 4874 queries (the VoxCeleb1-O test utterances) against Ng = 1 092 009 gallery rows, D = 512, k = 10;
      (b) the same queries against 1251 centroids, k = 5;
      (c) one query against Ng = 1 092 009, k = 10;
    beside, for (a) and (c), the same search as torch ops on the same card (F.normalize, fp32 matmul with TF32 off in the
    same 16384-column chunks, torch.topk, and a torch.topk merge of the running and the new list);
  * (d) milliseconds per enroll of 1 092 009 utterances into 5994 speakers (the host lists included);
  * a per-kernel split of one (a) and one (c) call from torch.profiler, in a window of its own: the GEMM
    (conv_umma_kernel, its tensor TFLOP/s counting the three hi/lo products, 3 * 2 * rows * Npad * D over the padded
    row chunks actually run), the selection (topk_indices_kernel, GB/s of the M * Ng * 4 bytes of cosines it reads),
    the merge and the norm / split kernels;
  * the selection alone on a 4096 x 16384 matrix (rows staged in shared memory) and a 4096 x 65536 one (not staged):
    its GB/s in each regime, which decides the search's column chunk width;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_identify.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402

WIDTH = 16384          # gallery columns per search chunk (include/dsk.h)


def chunk_rows(M, Nc):
    """Query rows per chunk (include/dsk.h, as dsk_cohort_stats)."""
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
    split = {"gemm": 0.0, "select": 0.0, "merge": 0.0, "prep": 0.0, "other": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        key = ("gemm" if "conv_umma_kernel" in name else "select" if "topk_indices" in name else
               "merge" if "topk_merge" in name else
               "prep" if ("aam_norm_kernel" in name or "aam_split_kernel" in name) else "other")
        split[key] += us / 1e3
    return {k: round(v, 4) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F

    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200 import identification as I

    assert torch.cuda.is_available(), "bench_identify needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "identify", **gpu_info()}
    D, Ng, Mq = 512, 1092009, 4874
    G = torch.randn(Ng, D, device=dev, generator=g)
    Q = torch.randn(Mq, D, device=dev, generator=g)

    def torch_search(Qx, k):
        Qn = F.normalize(Qx)
        idx = val = None
        for c0 in range(0, Ng, WIDTH):
            v, i = torch.topk(Qn @ F.normalize(G[c0:c0 + WIDTH]).T, k, dim=1)
            i = i + c0
            if idx is None:
                idx, val = i, v
            else:
                val, j = torch.topk(torch.cat([val, v], 1), k, dim=1)
                idx = torch.gather(torch.cat([idx, i], 1), 1, j)
        return idx, val

    for tag, Qx, k in (("a_M4874_Ng1092009_k10", Q, 10), ("c_M1_Ng1092009_k10", Q[:1], 10)):
        M = Qx.shape[0]
        op = lambda Qx=Qx, k=k: I.search(Qx, G, k)         # noqa: E731
        ref = lambda Qx=Qx, k=k: torch_search(Qx, k)        # noqa: E731
        for fn in (op, ref):
            fn()
        torch.cuda.synchronize()
        m_op, m_ref = [], []
        for _ in range(2):                                  # alternated, so both see the same card state
            m_op.append(time_events(op, args.iters * (1 if M > 1 else 10)))
            m_ref.append(time_events(ref, args.iters * (1 if M > 1 else 10)))
        rec[f"search_ms_{tag}"] = [round(t, 3) for t in m_op]
        rec[f"torch_ops_ms_{tag}"] = [round(t, 3) for t in m_ref]
        (io, vo), (it, vt) = op(), ref()
        rec[f"top1_agree_with_torch_{tag}"] = float((io[:, 0] == it[:, 0]).float().mean())
        rec[f"max_abs_dscore_vs_torch_{tag}"] = float((vo - vt).abs().max())
        split = kernel_split(op)
        rec[f"kernel_ms_{tag}"] = split
        rows_run = -(-M // chunk_rows(M, WIDTH)) * chunk_rows(M, WIDTH)
        if split["gemm"] > 0:
            rec[f"gemm_tensor_tflops_{tag}"] = round(3 * 2 * rows_run * (-(-Ng // WIDTH) * WIDTH) * D
                                                     / (split["gemm"] * 1e-3) / 1e12, 1)
        if split["select"] > 0:
            rec[f"select_gb_per_s_{tag}"] = round(M * Ng * 4 / (split["select"] * 1e-3) / 1e9, 1)

    # (b) centroid gallery
    Gc = torch.randn(1251, D, device=dev, generator=g)
    op = lambda: I.search(Q, Gc, 5)                         # noqa: E731
    op()
    rec["search_ms_b_M4874_Ng1251_k5"] = [round(time_events(op, args.iters * 20), 4) for _ in range(2)]

    # (d) enrolment
    spk = torch.randint(0, 5994, (Ng,), generator=torch.Generator().manual_seed(1)).numpy()
    spk[:5994] = np.arange(5994)
    op = lambda: I.enroll(G, spk)                           # noqa: E731
    op()
    rec["enroll_ms_d_U1092009_S5994"] = [round(time_events(op, args.iters * 2), 3) for _ in range(2)]
    rec["enroll_kernel_ms_d"] = kernel_split(op)

    # the selection alone, staged and not staged
    del G
    for cols in (16384, 65536):
        S = torch.randn(4096, cols, device=dev, generator=g)
        op = lambda S=S: EN.topk_indices(S, 10)             # noqa: E731
        op()
        ms = min(time_events(op, args.iters * 10) for _ in range(2))
        rec[f"select_alone_gb_per_s_4096x{cols}_k10"] = round(S.numel() * 4 / (ms * 1e-3) / 1e9, 1)
        del S
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
