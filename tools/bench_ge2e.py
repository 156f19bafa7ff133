"""GE2E: one JSON line with
  * microseconds per loss forward + backward (embeddings, w and b) at (P, M, D) = (64, 10, 512), (256, 12, 512) and
    (1024, 4, 512), both methods, on the op (CUDA events around --iters back-to-back calls) and, for comparison, the same
    loss written as torch ops (oracle.ge2e_oracle.loss_autograd: F.normalize, one-hot matmuls, logsumexp / sigmoid;
    fp32, TF32 off) on the same card;
  * utterances per second of ge2e_step at N = 384 (64 speakers x 6), T = 160 with FusedAdagrad (softmax), beside
    aam_softmax_step (C = 1211) and batch_hard_step (96 x 4) at the same size (events around --steps steps after
    --warmup, alternated twice);
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_ge2e.py
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
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from oracle import ge2e_oracle as G          # the torch-ops formulation the op is compared with
    from oracle import rescnn_oracle as O        # deterministic parameters only

    assert torch.cuda.is_available(), "bench_ge2e needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "ge2e", **gpu_info()}
    D = 512
    for P, M in ((64, 10), (256, 12), (1024, 4)):
        N = P * M
        E = torch.randn(N, D, device=dev, generator=g)
        E = (10.0 * E / E.norm(dim=1, keepdim=True)).requires_grad_(True)
        labels = torch.arange(N) // M                       # CPU labels, as a loader yields them
        for method in ("softmax", "contrast"):
            crit = dsk.GE2ELoss(10.0, -5.0, method).to(dev)
            w = crit.w.detach().clone().requires_grad_(True)
            b = crit.b.detach().clone().requires_grad_(True)

            def op():
                E.grad = crit.w.grad = crit.b.grad = None
                crit(E, labels).backward()

            def torch_ops():
                E.grad = w.grad = b.grad = None
                G.loss_autograd(E, labels, w, b, method).backward()

            for key, fn in (("op", op), ("torch_fp32", torch_ops)):
                for _ in range(20):
                    fn()
                torch.cuda.synchronize()
                rec[f"fwd_bwd_us_{key}_{method}_P{P}_M{M}"] = round(1e3 * time_events(fn, args.iters), 2)
        rec[f"tensor_gflop_P{P}_M{M}"] = round(3 * 3 * 2 * N * P * D / 1e9, 3)   # three GEMMs, hi/lo x3

    Nst, T, C = 384, 160, 1211
    sd = O.make_state_dict(0, num_classes=C)
    x = torch.randn(Nst, 1, T, 64, device=dev, generator=g) * 3.0
    lab_ge2e = torch.arange(Nst) // 6
    lab_aam = torch.randint(0, C, (Nst,), generator=torch.Generator().manual_seed(1))
    lab_bh = torch.arange(Nst) // 4
    steps = {}
    for key in ("ge2e_step", "aam_softmax_step", "batch_hard_step"):
        model = dsk.DeepSpeakerModel(512, C).to(dev).train()
        model.load_state_dict(sd)
        if key == "ge2e_step":
            crit = dsk.GE2ELoss().to(dev)
            opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-3, lr_decay=1e-4)
            steps[key] = lambda model=model, opt=opt, crit=crit: dsk.ge2e_step(model, opt, x, lab_ge2e, loss=crit)
        else:
            opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
            if key == "aam_softmax_step":
                steps[key] = lambda model=model, opt=opt: dsk.aam_softmax_step(model, opt, x, lab_aam, margin=0.2,
                                                                               scale=30.0)
            else:
                steps[key] = lambda model=model, opt=opt: dsk.batch_hard_step(model, opt, x, lab_bh, margin=0.5)
        for _ in range(args.warmup):
            steps[key]()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(2):                  # alternated, so all see the same card state
        for k, fn in steps.items():
            ms[k].append(time_events(fn, args.steps))
    for k, v in ms.items():
        rec[f"{k}_ms"] = [round(t, 3) for t in v]
        rec[f"{k}_utt_per_s"] = round(Nst / (min(v) / 1e3), 1)
    rec["step_shape"] = {"N": Nst, "T": T, "optimizer": "FusedAdagrad", "ge2e": "64 x 6 softmax", "aam_C": C,
                         "batch_hard": "96 x 4"}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
