"""Synchronised BatchNorm: one JSON line with
  * ms per batch_hard_step at N = 384 (96 speakers x 4), T = 160, FusedAdagrad, with per-replica BatchNorm (the default)
    and with synchronised BatchNorm at one rank - the cost of the staged path without communication.  The two are
    timed alternately, --rounds times each, with CUDA events around --steps steps after --warmup;
  * the record bytes one rank sends per collective and per step, computed from the shapes;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Under ``torchrun --nproc-per-node R``: the same step at 384 utterances per rank, synchronised vs not (across_ranks=True
both), and the bytes each rank receives per step (rank 0 prints the line).
Writes nothing but stdout.  Run: python tools/bench_sync_bn.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_batch_hard import gpu_info, time_events  # noqa: E402

CHANNELS = [64] * 3 + [128] * 3 + [256] * 3 + [512] * 3


def record_bytes(n):
    """Bytes of this rank's records for n utterances: per forward exchange (12), per backward exchange (13)."""
    fwd = [n * 4 * (3 * c + 1) for c in CHANNELS]
    bwd = [n * 4] + [n * 8 * c for c in reversed(CHANNELS)]
    return {"forward_per_collective": fwd, "backward_per_collective": bwd, "forward_total": sum(fwd),
            "backward_total": sum(bwd)}


def _model(dev, sync, group=None):
    import deepspeaker_pytorch_b200 as dsk
    from oracle import rescnn_oracle as O  # deterministic parameters only

    m = dsk.DeepSpeakerModel(512, 16).to(dev).train()
    m.load_state_dict(O.make_state_dict(0, num_classes=16))
    if sync:
        m.sync_batchnorm(group)
    return m, dsk.FusedAdagrad(m.parameters(), lr=1e-3, lr_decay=1e-4)


def _timed(steps, args, rounds):
    """{key: [ms per step of each round]}, the configurations alternating round by round."""
    import torch

    out = {k: [] for k in steps}
    for k, fn in steps.items():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, fn in steps.items():
            out[k].append(round(time_events(fn, args.steps), 3))
    return out


def main(args):
    import torch

    import deepspeaker_pytorch_b200 as dsk

    assert torch.cuda.is_available(), "bench_sync_bn needs a GPU"
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    P, Ku, T = 96, 4, 160
    N = P * Ku
    x = torch.randn(N, 1, T, 64, device=dev, generator=g) * 3.0
    lab = torch.arange(N) // Ku
    steps = {}
    for key, sync in (("step_ms_per_replica_bn", False), ("step_ms_sync_bn_R1", True)):
        m, opt = _model(dev, sync)
        steps[key] = (lambda m=m, opt=opt: dsk.batch_hard_step(m, opt, x, lab, margin=0.5))
    times = _timed(steps, args, args.rounds)
    rec = {"metric": "sync_batchnorm_step", **gpu_info(),
           "shape": {"N": N, "speakers": P, "utterances_per_speaker": Ku, "T": T, "optimizer": "FusedAdagrad"},
           **{k: min(v) for k, v in times.items()}, "rounds_ms": times,
           "records_per_rank": record_bytes(N)}
    rec["sync_overhead_ms_R1"] = round(rec["step_ms_sync_bn_R1"] - rec["step_ms_per_replica_bn"], 3)
    print(json.dumps(rec), flush=True)


def main_distributed(args):
    """Under torchrun: ms per batch_hard_step(across_ranks=True) at n = 384 utterances per rank, T = 160, with
    per-replica vs synchronised BatchNorm."""
    import torch
    import torch.distributed as dist

    import deepspeaker_pytorch_b200 as dsk

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        n, Ku, T = 384, 4, 160
        g = torch.Generator(device=dev).manual_seed(rank)
        x = torch.randn(n, 1, T, 64, device=dev, generator=g) * 3.0
        lab = (torch.arange(world * n) % (world * n // Ku))[rank * n:(rank + 1) * n]   # speakers span the ranks
        steps = {}
        for key, sync in (("step_ms_per_replica_bn", False), ("step_ms_sync_bn", True)):
            m, opt = _model(dev, sync, dist.group.WORLD)
            steps[key] = (lambda m=m, opt=opt: dsk.batch_hard_step(m, opt, x, lab, margin=0.5, across_ranks=True))
        dist.barrier()
        times = _timed(steps, args, args.rounds)
        rb = record_bytes(n)
        rec = {"metric": "sync_batchnorm_step_data_parallel", "ranks": world, **gpu_info(),
               "shape": {"n_per_rank": n, "N": world * n, "utterances_per_speaker": Ku, "T": T},
               **{k: min(v) for k, v in times.items()}, "rounds_ms": times, "records_sent_per_rank": rb,
               "records_received_per_rank_per_step": world * (rb["forward_total"] + rb["backward_total"])}
        rec["sync_overhead_ms"] = round(rec["step_ms_sync_bn"] - rec["step_ms_per_replica_bn"], 3)
        if rank == 0:
            print(json.dumps(rec), flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_known_args()[0]
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        main_distributed(a)
    else:
        main(a)
