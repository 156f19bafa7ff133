"""AAM-softmax: one JSON line with
  * microseconds per loss forward + backward (embeddings and weight) at (N, C) = (384, 1211) and (1024, 5994), D = 512,
    on the op (CUDA events around --iters back-to-back calls) and, for comparison, the same loss written as torch ops
    (F.normalize, matmul, cross_entropy; fp32, TF32 off) on the same card;
  * utterances per second of aam_softmax_step at N = 384, T = 160, C = 1211 with FusedAdagrad, beside batch_hard_step
    (96 speakers x 4 utterances) at the same size (events around --steps steps after --warmup, alternated twice);
  * the sub-centre head with the inter-top-k penalty beside the plain head on speed-extended class counts: microseconds
    per loss forward + backward at (N, C) = (384, 3 x 1211) and (1024, 3 x 5994), D = 512, for K = 1 / topk = 0 and
    K = 3 / topk = 5 (m' = 0.1), on the op and as torch ops (fp32, TF32 off), and aam_softmax_step times at N = 384,
    T = 160, C = 3 x 1211 for both heads (events around --steps steps after --warmup, alternated twice);
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_aam_softmax.py
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
    import torch.nn.functional as F

    import deepspeaker_pytorch_b200 as dsk
    from oracle import aam_softmax_oracle as A   # the torch-ops formulation the op is compared with
    from oracle import subcentre_aam_oracle as SA
    from oracle import rescnn_oracle as O        # deterministic parameters only

    assert torch.cuda.is_available(), "bench_aam_softmax needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "aam_softmax", **gpu_info()}
    m, s, D = 0.2, 30.0, 512
    for N, C in ((384, 1211), (1024, 5994)):
        E = torch.randn(N, D, device=dev, generator=g)
        E = (10.0 * E / E.norm(dim=1, keepdim=True)).requires_grad_(True)
        W = (torch.randn(C, D, device=dev, generator=g) / D ** 0.5).requires_grad_(True)
        labels = torch.randint(0, C, (N,), device=dev, generator=g)
        crit = dsk.AAMSoftmaxLoss(W, m, s)

        def op():
            E.grad = W.grad = None
            crit.forward(E, labels).backward()

        def torch_ops():
            E.grad = W.grad = None
            A.loss_autograd(E, W, labels, m, s).backward()

        for key, fn in (("op", op), ("torch_fp32", torch_ops)):
            for _ in range(20):
                fn()
            torch.cuda.synchronize()
            rec[f"fwd_bwd_us_{key}_N{N}_C{C}"] = round(1e3 * time_events(fn, args.iters), 2)
        rec[f"tensor_gflop_N{N}_C{C}"] = round(3 * 3 * 2 * N * C * D / 1e9, 2)   # three GEMMs, hi/lo x3

    Nst, T, C = 384, 160, 1211
    sd = O.make_state_dict(0, num_classes=C)
    x = torch.randn(Nst, 1, T, 64, device=dev, generator=g) * 3.0
    lab_aam = torch.randint(0, C, (Nst,), generator=torch.Generator().manual_seed(1))   # CPU labels, as a loader yields them
    lab_bh = torch.arange(Nst) // 4
    steps = {}
    for key in ("aam_softmax_step", "batch_hard_step"):
        model = dsk.DeepSpeakerModel(512, C).to(dev).train()
        model.load_state_dict(sd)
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        if key == "aam_softmax_step":
            steps[key] = lambda model=model, opt=opt: dsk.aam_softmax_step(model, opt, x, lab_aam, margin=m, scale=s)
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
        rec[f"{k}_utt_per_s"] = round(Nst / (min(v) / 1e3), 1)
    rec["step_shape"] = {"N": Nst, "T": T, "C": C, "optimizer": "FusedAdagrad", "batch_hard": "96 x 4"}

    # sub-centre heads on speed-extended class counts (three speeds)
    tm = 0.1
    heads = {"K1_topk0": (1, 0), "K3_topk5": (3, 5)}
    for N, C in ((384, 3 * 1211), (1024, 3 * 5994)):
        E = torch.randn(N, D, device=dev, generator=g)
        E = (10.0 * E / E.norm(dim=1, keepdim=True)).requires_grad_(True)
        labels = torch.randint(0, C, (N,), device=dev, generator=g)
        for head, (K, topk) in heads.items():
            W = (torch.randn(C * K, D, device=dev, generator=g) / D ** 0.5).requires_grad_(True)
            crit = dsk.AAMSoftmaxLoss(W, m, s, subcentres=K, topk=topk, topk_margin=tm)

            def op(E=E, W=W, crit=crit, labels=labels):
                E.grad = W.grad = None
                crit.forward(E, labels).backward()

            def torch_ops(E=E, W=W, labels=labels, K=K, topk=topk):
                E.grad = W.grad = None
                SA.loss_autograd(E, W, labels, K, m, s, topk, tm).backward()

            for key, fn in (("op", op), ("torch_fp32", torch_ops)):
                for _ in range(20):
                    fn()
                torch.cuda.synchronize()
                rec[f"sc_fwd_bwd_us_{key}_{head}_N{N}_C{C}"] = round(1e3 * time_events(fn, args.iters), 2)
            del W, crit
    Csc = 3 * 1211
    sd = O.make_state_dict(0, num_classes=Csc)
    lab_sc = torch.randint(0, Csc, (Nst,), generator=torch.Generator().manual_seed(2))
    steps = {}
    for head, (K, topk) in heads.items():
        model = dsk.DeepSpeakerModel(512, Csc).to(dev).train()
        model.load_state_dict(sd)
        params = list(model.parameters())
        W = None
        if K > 1:
            W = torch.nn.Parameter(torch.randn(Csc * K, D, device=dev, generator=g) / D ** 0.5)
            params.append(W)
        opt = dsk.FusedAdagrad(params, lr=1e-3, lr_decay=1e-4)
        steps[head] = lambda model=model, opt=opt, W=W, K=K, topk=topk: dsk.aam_softmax_step(
            model, opt, x, lab_sc, margin=m, scale=s, weight=W, subcentres=K, topk=topk, topk_margin=tm)
        for _ in range(args.warmup):
            steps[head]()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(2):
        for k, fn in steps.items():
            ms[k].append(time_events(fn, args.steps))
    for k, v in ms.items():
        rec[f"sc_step_ms_{k}"] = [round(t, 3) for t in v]
    rec["sc_step_shape"] = {"N": Nst, "T": T, "C": Csc, "topk_margin": tm, "optimizer": "FusedAdagrad"}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
