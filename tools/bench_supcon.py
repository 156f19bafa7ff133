"""Supervised-contrastive loss: one JSON line with
  * microseconds per loss forward + backward at N = 512, 2048 and 8192 (two views of N / 2 utterances), D = 512,
    tau = 0.1, on the op (CUDA events around --iters back-to-back calls) and, for comparison, the same loss written as
    torch ops (oracle.supcon_oracle.loss_autograd: F.normalize, the Gram matrix, a masked logsumexp; fp32, TF32 off)
    on the same card;
  * utterances per second of supcon_step at 2 x 192 views, T = 160, fed by WaveBank.augmented_crops (RIR, noise and
    speed perturbation; the crops are made once, outside the timed window), beside batch_hard_step at N = 384
    (96 x 4) on the same crops, with FusedAdagrad (events around --steps steps after --warmup, alternated twice);
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_supcon.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402


def _views(dev, B, T):
    """Two augmented views of each of B synthetic utterances (8 s each), from a device WaveBank."""
    import numpy as np
    import torch

    from deepspeaker_pytorch_b200 import frontend as FR

    g = np.random.default_rng(0)
    speech = [np.round(g.normal(0, 0.1, 128000).clip(-1, 0.99) * 32768).astype(np.int16) for _ in range(B)]
    noise = [np.round(g.normal(0, 0.1, 64000).clip(-1, 0.99) * 32768).astype(np.int16) for _ in range(8)]
    rirs = [g.normal(size=lh) * np.exp(-np.arange(lh) / 800.0) for lh in (800, 4000, 8000)]
    sb, nb = FR.WaveBank.from_waveforms(speech, device=dev), FR.WaveBank.from_waveforms(noise, device=dev)
    rb = FR.RirBank.from_arrays(rirs, device=dev)
    utt = torch.arange(B).repeat(2)
    Ls = FR.segment_samples(T)
    plan = FR.augment_plan(2 * B, Ls, g, rb, 0.5, nb, [(range(8), (0.0, 15.0), (1, 2), 1.0)], 0.5,
                           speeds=(0.9, 1.0, 1.1))
    start = sb.random_starts(utt, Ls, g, plan)
    return sb.augmented_crops(utt, start, T, plan, rb, nb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from oracle import rescnn_oracle as O         # deterministic parameters only
    from oracle import supcon_oracle as S         # the torch-ops formulation the op is compared with

    assert torch.cuda.is_available(), "bench_supcon needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "supcon", **gpu_info()}
    D, tau = 512, 0.1
    crit = dsk.SupConLoss(tau)
    for N in (512, 2048, 8192):
        E = torch.randn(N, D, device=dev, generator=g)
        E = (10.0 * E / E.norm(dim=1, keepdim=True)).requires_grad_(True)
        labels = torch.arange(N // 2).repeat(2)             # CPU labels, as a loader yields them

        def op():
            E.grad = None
            crit(E, labels).backward()

        def torch_ops():
            E.grad = None
            S.loss_autograd(E, labels, tau).backward()

        for key, fn in (("op", op), ("torch_fp32", torch_ops)):
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            rec[f"fwd_bwd_us_{key}_N{N}"] = round(1e3 * time_events(fn, args.iters), 2)
        rec[f"tensor_gflop_N{N}"] = round(3 * 3 * 2 * N * N * D / 1e9, 3)   # three GEMMs, hi/lo x3
        del E

    B, T, C = 192, 160, 16
    x = _views(dev, B, T)
    lab_sc = torch.arange(B).repeat(2)
    lab_bh = torch.arange(2 * B) // 4
    sd = O.make_state_dict(0, num_classes=C)
    steps = {}
    for key in ("supcon_step", "batch_hard_step"):
        model = dsk.DeepSpeakerModel(512, C).to(dev).train()
        model.load_state_dict(sd)
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        if key == "supcon_step":
            steps[key] = lambda model=model, opt=opt: dsk.supcon_step(model, opt, x, lab_sc, temperature=tau)
        else:
            steps[key] = lambda model=model, opt=opt: dsk.batch_hard_step(model, opt, x, lab_bh, margin=0.5)
        for _ in range(args.warmup):
            steps[key]()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(2):                  # alternated, so both see the same card state
        for k, fn in steps.items():
            ms[k].append(time_events(fn, args.steps))
    for k, v in ms.items():
        rec[f"{k}_ms"] = [round(t, 3) for t in v]
        rec[f"{k}_utt_per_s"] = round(2 * B / (min(v) / 1e3), 1)
    rec["step_shape"] = {"N": 2 * B, "T": T, "optimizer": "FusedAdagrad", "supcon": f"2 x {B} views, tau {tau}",
                         "batch_hard": f"{2 * B // 4} x 4", "input": "augmented_crops: RIR, noise, speed"}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
