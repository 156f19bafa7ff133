"""Batch-hard triplet loss: one JSON line with
  * microseconds per loss forward + backward at N = 1024, D = 512 (64 speakers x 16 utterances), on the tensor-core Gram
    path and on the exact CUDA-core path (CUDA events around --iters back-to-back calls), and per all-pairs top-8 query
    (dsk_allpairs_topk_tc) on the same batch;
  * utterances per second of batch_hard_step at N = 384 (96 x 4), T = 160, with FusedAdagrad (events around --steps
    steps after --warmup);
  * microseconds for one rank's share of the global-batch op (select_rows + bwd_rows, 384 anchor rows of N = 3072,
    i.e. R = 8) beside the whole-batch forward + backward at N = 3072;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Under ``torchrun --nproc-per-node R``: ms per batch_hard_step at 384 utterances per rank, T = 160, with across_ranks
False vs True (rank 0 prints the line).
Writes nothing but stdout.  Run: python tools/bench_batch_hard.py
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # the figures are still device timings; say that the card could not be named
        return {"gpu": None, "gpu_query_error": str(e)}


def time_events(fn, iters):
    import torch

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters   # ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200 import engine as EN

    assert torch.cuda.is_available(), "bench_batch_hard needs a GPU"
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    rec = {"metric": "batch_hard_triplet", **gpu_info()}

    N, D, K = 1024, 512, 16
    E = torch.randn(N, D, device=dev, generator=g)
    E = (10.0 * E / E.norm(dim=1, keepdim=True)).requires_grad_(True)
    labels = (torch.arange(N, device=dev) // K)
    for key, exact in (("loss_fwd_bwd_us_tensor_core", False), ("loss_fwd_bwd_us_exact", True)):
        crit = dsk.BatchHardTripletLoss(0.3, exact_cuda_cores=exact)

        def one():
            E.grad = None
            crit.forward(E, labels).backward()

        for _ in range(20):
            one()
        torch.cuda.synchronize()
        rec[key] = round(1e3 * time_events(one, args.iters), 2)
    rec["loss_shape"] = {"N": N, "D": D, "speakers": N // K, "utterances_per_speaker": K}
    Ed = E.detach()
    top8 = lambda: EN.allpairs_topk(Ed, labels, 8)   # noqa: E731
    for _ in range(20):
        top8()
    torch.cuda.synchronize()
    rec["allpairs_top8_us_N1024"] = round(1e3 * time_events(top8, args.iters), 2)

    from oracle import rescnn_oracle as O  # deterministic parameters only

    P, Ku, T = 96, 4, 160
    model = dsk.DeepSpeakerModel(512, 16).to(dev).train()
    model.load_state_dict(O.make_state_dict(0, num_classes=16))
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
    x = torch.randn(P * Ku, 1, T, 64, device=dev, generator=g) * 3.0
    lab = torch.arange(P * Ku) // Ku           # CPU labels, as a data loader yields them
    step = lambda: dsk.batch_hard_step(model, opt, x, lab, margin=0.5)
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    ms = time_events(step, args.steps)
    rec["step_ms"] = round(ms, 3)
    rec["step_utt_per_s"] = round(P * Ku / (ms / 1e3), 1)
    rec["step_shape"] = {"N": P * Ku, "speakers": P, "utterances_per_speaker": Ku, "T": T, "optimizer": "FusedAdagrad"}

    # one rank's share of the global-batch op: select_rows + bwd_rows for 384 of N = 3072 anchors (R = 8), beside the
    # whole-batch op at the same N (tensor-core path)
    N, rows = 3072, 384
    E = torch.randn(N, D, device=dev, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    labels = torch.arange(N, device=dev) // K
    one = torch.ones((), device=dev)
    _, _, *sel = EN.batch_hard_mine(E, labels, 0.3)
    row0 = N - rows

    def full():
        Ec, _, *s = EN.batch_hard_mine(E, labels, 0.3)
        EN.batch_hard_backward(Ec, *s, 0.3, one)

    def share():
        EN.batch_hard_select_rows(E, labels, row0, rows)
        EN.batch_hard_backward_rows(E, *sel, row0, rows, 0.3, one)

    for key, fn in (("full_fwd_bwd_us_N3072", full), ("rows384_select_bwd_us_N3072", share)):
        for _ in range(20):   # the first call of each (re)builds the Gram plan for its row range
            fn()
        torch.cuda.synchronize()
        rec[key] = round(1e3 * time_events(fn, args.iters), 2)
    rec["rows_shape"] = {"N": N, "D": D, "rows": rows, "gram_gflop_full": round(2 * N * N * D / 1e9, 2),
                         "gram_gflop_rows": round(2 * rows * N * D / 1e9, 2)}
    print(json.dumps(rec), flush=True)


def main_distributed(args):
    """Under torchrun: ms per batch_hard_step at n = 384 utterances per rank, T = 160, mining inside the rank's shard
    (across_ranks=False) vs over the global batch (across_ranks=True, including the label gather's host sync)."""
    import torch
    import torch.distributed as dist

    import deepspeaker_pytorch_b200 as dsk
    from oracle import rescnn_oracle as O  # deterministic parameters only

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        n, Ku, T = 384, 4, 160
        model = dsk.DeepSpeakerModel(512, 16).to(dev).train()
        model.load_state_dict(O.make_state_dict(0, num_classes=16))
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        g = torch.Generator(device=dev).manual_seed(rank)
        x = torch.randn(n, 1, T, 64, device=dev, generator=g) * 3.0
        lab = (torch.arange(world * n) % (world * n // Ku))[rank * n:(rank + 1) * n]   # speakers span the ranks
        rec = {"metric": "batch_hard_step_data_parallel", "ranks": world, **gpu_info(),
               "shape": {"n_per_rank": n, "N": world * n, "utterances_per_speaker": Ku, "T": T}}
        for key, across in (("step_ms_local_mining", False), ("step_ms_across_ranks", True)):
            step = lambda: dsk.batch_hard_step(model, opt, x, lab, margin=0.5, across_ranks=across)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            dist.barrier()
            rec[key] = round(time_events(step, args.steps), 3)
        rec["across_ranks_overhead_ms"] = round(rec["step_ms_across_ranks"] - rec["step_ms_local_mining"], 3)
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
