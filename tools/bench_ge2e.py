"""GE2E: one JSON line with
  * microseconds per loss forward + backward (embeddings, w and b) at (P, M, D) = (64, 10, 512), (256, 12, 512) and
    (1024, 4, 512), both methods, on the op (CUDA events around --iters back-to-back calls) and, for comparison, the same
    loss written as torch ops (oracle.ge2e_oracle.loss_autograd: F.normalize, one-hot matmuls, logsumexp / sigmoid;
    fp32, TF32 off) on the same card;
  * utterances per second of ge2e_step at N = 384 (64 speakers x 6), T = 160 with FusedAdagrad (softmax), beside
    aam_softmax_step (C = 1211) and batch_hard_step (96 x 4) at the same size (events around --steps steps after
    --warmup, alternated twice);
  * microseconds for one rank's share of the global-batch op at R = 8 (ge2e_rows + ge2e_mean + ge2e_dcos_rows +
    ge2e_backward_rows for 384 of N = 3072 rows, P = 512, D = 512; the collectives' payloads taken as gathered) beside
    the whole op at N = 3072, both methods;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Under ``torchrun --nproc-per-node R``: ms per ge2e_step at 384 utterances per rank (64 x 6), T = 160, with across_ranks
False vs True (rank 0 prints the line).
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

    # one rank's share of the global-batch op at R = 8: the rows ops for 384 of N = 3072 rows (512 speakers x 6), P =
    # 512, forward + backward, beside the whole op at N = 3072 (what every rank would run on the gathered batch instead)
    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200.model import ge2e_batch, ge2e_csr_to

    N, rows, M = 3072, 384, 6
    E = torch.randn(N, D, device=dev, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    order, offsets, col, V = ge2e_batch(torch.arange(N) % (N // M))      # every speaker spans the ranks
    csr = ge2e_csr_to(order, offsets, col, dev)
    w, b, one = (torch.full((1,), v, device=dev) for v in (10.0, -5.0, 1.0))
    row0 = N - rows
    for method in ("softmax", "contrast"):
        Ec, _, cos, rec_all = EN.ge2e(E, csr, V, w, b, method)
        row_loss = EN.ge2e_rows(E, csr, V, w, b, method, 0, N)[3]
        dc_all, tdc_all, _, _ = EN.ge2e_dcos_rows(cos, rec_all, csr, V, w, b, method, 0, N, one)
        cos_r, rec_r = cos[row0:].contiguous(), rec_all[row0:].contiguous()

        def whole():
            Ec, _, c, r = EN.ge2e(E, csr, V, w, b, method)
            EN.ge2e_backward(Ec, csr, V, w, b, method, c, r, one)

        def share():     # the collectives' payloads are taken as already gathered
            EN.ge2e_rows(E, csr, V, w, b, method, row0, rows)
            EN.ge2e_mean(row_loss, V)
            EN.ge2e_dcos_rows(cos_r, rec_r, csr, V, w, b, method, row0, rows, one)
            EN.ge2e_backward_rows(E, csr, dc_all, tdc_all, row0, rows)

        for key, fn in ((f"whole_fwd_bwd_us_{method}_N3072", whole), (f"rows384_fwd_bwd_us_{method}_N3072", share)):
            for _ in range(20):   # the first call of each (re)builds the plan for its row range
                fn()
            torch.cuda.synchronize()
            rec[key] = round(1e3 * time_events(fn, args.iters), 2)
    rec["rows_shape"] = {"N": N, "P": N // M, "D": D, "rows": rows, "ranks": N // rows,
                         "tensor_gflop_whole": round(3 * 3 * 2 * N * (N // M) * D / 1e9, 2),
                         "tensor_gflop_rows": round(3 * 2 * (2 * rows + N) * (N // M) * D / 1e9, 2)}
    rec["data_parallel_step"] = "not measured in this run: run under torchrun --nproc-per-node R on R GPUs"

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


def main_distributed(args):
    """Under torchrun: ms per ge2e_step at n = 384 utterances per rank, T = 160, softmax, with the centroids of the rank's
    shard (across_ranks=False) vs of the global batch (across_ranks=True, including the label gather's host sync and the
    three GE2E all_gathers).  Rank r holds its own 64 speakers x 6 utterances (speakers 64 r .. 64 r + 63), so both arms
    run a full problem at every R: the shard arm 64 speakers x 6 per rank, the global arm P = 64 R speakers over
    N = 384 R rows (P = 512 at R = 8).  The costs depend on N, P, D and the speaker sizes, not on which rank holds a
    speaker's rows."""
    import torch
    import torch.distributed as dist

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200.model import ge2e_batch
    from oracle import rescnn_oracle as O  # deterministic parameters only

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        n, M, T = 384, 6, 160
        model = dsk.DeepSpeakerModel(512, 16).to(dev).train()
        model.load_state_dict(O.make_state_dict(0, num_classes=16))
        crit = dsk.GE2ELoss().to(dev)
        opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-3, lr_decay=1e-4)
        g = torch.Generator(device=dev).manual_seed(rank)
        x = torch.randn(n, 1, T, 64, device=dev, generator=g) * 3.0
        lab = torch.arange(world * n)[rank * n:(rank + 1) * n] // M
        glab = torch.arange(world * n) // M
        assert ge2e_batch(lab)[3] == n and ge2e_batch(glab)[3] == world * n, "every row must carry a loss term"
        rec = {"metric": "ge2e_step_data_parallel", "ranks": world, **gpu_info(),
               "shape": {"n_per_rank": n, "N": world * n, "speakers_per_rank": n // M, "P_global": world * n // M,
                         "utterances_per_speaker": M, "T": T}}
        for key, across in (("step_ms_shard_centroids", False), ("step_ms_across_ranks", True)):
            step = lambda: dsk.ge2e_step(model, opt, x, lab, loss=crit, across_ranks=across)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            dist.barrier()
            rec[key] = round(time_events(step, args.steps), 3)
        rec["across_ranks_overhead_ms"] = round(rec["step_ms_across_ranks"] - rec["step_ms_shard_centroids"], 3)
        if rank == 0:
            print(json.dumps(rec), flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        ap = argparse.ArgumentParser()
        ap.add_argument("--steps", type=int, default=20)
        ap.add_argument("--warmup", type=int, default=5)
        main_distributed(ap.parse_known_args()[0])
    else:
        main()
