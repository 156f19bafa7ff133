"""Class-sharded AAM-softmax: one JSON line with
  * milliseconds per sharded loss forward + backward on one GPU at one emulated rank's share: N = 3072 gathered rows
    (n = 384 per rank), C = 3 x 5994 classes, K = 3, topk = 5, D = 512, rank 0's class range of class_shards(C, R) for
    R = 2, 4, 8 (the other ranks' exchanged records are stand-ins of the right size), beside the whole op at
    (384, C K) (CUDA events around --iters back-to-back calls);
  * the bytes of every collective per step, computed from shapes (not measured);
  * with >= 2 GPUs: sharded_aam_softmax_step vs aam_softmax_step (replicated weight) at n = 384 per rank, T = 160,
    alternated; otherwise recorded as not measured;
  * the card's name and power limit (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_sharded_aam.py
"""
import argparse
import json
import os
import socket
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_hard import gpu_info, time_events  # noqa: E402

C, K, TOPK, D, N_LOCAL, M, S, TM = 3 * 5994, 3, 5, 512, 384, 0.2, 30.0, 0.1


def collective_bytes(R, n=N_LOCAL):
    """Bytes each rank receives per step, from shapes.  The top-k keys, row maxima and partial-sum records are
    records of all N gathered rows on every rank, so each rank receives R of them; the all-reduce sizes are the
    gradient buckets (the triplet-path parameters of DeepSpeakerModel, plus the (C K, D) weight when replicated)."""
    import deepspeaker_pytorch_b200 as dsk
    from deepspeaker_pytorch_b200.parallel import path_parameters, shard_record_blocks

    N, nb = R * n, shard_record_blocks(C, R)
    bucket = 4 * sum(p.numel() for p in path_parameters(dsk.DeepSpeakerModel(D, 16)))
    return {"embeddings_all_gather": N * D * 4, "topk_keys_all_gather": R * N * TOPK * 8,
            "row_max_all_gather": R * N * 4, "partials_all_gather": R * N * (2 * nb + 2) * 4,
            "grad_rows_all_to_all": (R - 1) * n * D * 4, "labels_all_gather": N * 8, "network_all_reduce": bucket,
            "replicated_all_reduce": bucket + C * K * D * 4}


def shard_share(R, iters):
    """ms per forward + backward of rank 0's stages at R emulated ranks."""
    import torch

    from deepspeaker_pytorch_b200 import engine as EN
    from deepspeaker_pytorch_b200.parallel import class_shards, shard_record_blocks

    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(R)
    N = R * N_LOCAL
    c0, c1 = class_shards(C, R)[0]
    nb = shard_record_blocks(C, R)
    E = torch.randn(N, D, device=dev, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    W = torch.randn((c1 - c0) * K, D, device=dev, generator=g) / D ** 0.5
    y = torch.randint(0, C, (N,), device=dev, generator=g)
    gl = torch.ones((), device=dev)

    def step():
        cos, sub, keys = EN.aam_shard_cos(E, W, y, C, c0, c1, K, TOPK)
        top, thr, mloc = EN.aam_shard_merge(cos, y, keys.repeat(R, 1), R, C, c0, c1, TOPK, M, S, TM)
        m, rec = EN.aam_shard_partials(cos, y, thr, mloc.repeat(R), R, C, c0, c1, TOPK, nb, M, S, TM)
        loss, lse, row_loss, den = EN.aam_shard_finish(rec.repeat(R, 1), m, y, R, C, nb)
        gW, part = EN.aam_shard_backward(E, W, y, cos, sub, thr, m, den, C, c0, c1, M, S, K, TOPK, TM, gl)
        EN.aam_shard_backward_rows(E[:N_LOCAL].contiguous(), part[:N_LOCAL].repeat(R, 1), R)

    for _ in range(3):
        step()
    return time_events(step, iters)


def whole_op(iters):
    import torch

    from deepspeaker_pytorch_b200 import engine as EN

    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    E = torch.randn(N_LOCAL, D, device=dev, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    W = torch.randn(C * K, D, device=dev, generator=g) / D ** 0.5
    y = torch.randint(0, C, (N_LOCAL,), device=dev, generator=g)
    gl = torch.ones((), device=dev)

    def step():
        Ec, Wc, lab, loss, cos, lse, sub, top = EN.aam_softmax_sc(E, W, y, M, S, K, TOPK, TM)
        EN.aam_softmax_sc_backward(Ec, Wc, lab, cos, lse, sub, top, M, S, K, TOPK, TM, gl)

    for _ in range(3):
        step()
    return time_events(step, iters)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _step_worker(rank, world, port, steps, warmup, out):
    import torch
    import torch.distributed as dist

    import deepspeaker_pytorch_b200 as dsk
    from oracle import rescnn_oracle as O        # deterministic parameters only

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        sd = O.make_state_dict(0, num_classes=16)
        x = O.make_input(N_LOCAL, 160, seed=rank, scale=3.0).cuda()
        labels = torch.randint(0, C, (N_LOCAL,), generator=torch.Generator().manual_seed(rank))
        W0 = torch.randn(C * K, D, generator=torch.Generator().manual_seed(1)) / D ** 0.5
        rm = dsk.DeepSpeakerModel(512, 16).cuda().train()
        rm.load_state_dict(sd)
        Wr = torch.nn.Parameter(W0.cuda())
        ropt = dsk.FusedAdagrad(list(rm.parameters()) + [Wr], lr=1e-3, lr_decay=1e-4)
        sm = dsk.DeepSpeakerModel(512, 16).cuda().train()
        sm.load_state_dict(sd)
        head = dsk.ShardedAAMSoftmaxLoss(W0.cuda(), M, S, subcentres=K, topk=TOPK, topk_margin=TM,
                                         process_group=dist.group.WORLD)
        sopt = dsk.FusedAdagrad(list(sm.parameters()), lr=1e-3, lr_decay=1e-4)
        hopt = dsk.FusedAdagrad([head.weight], lr=1e-3, lr_decay=1e-4, process_group=dist.group.WORLD)
        kw = dict(margin=M, scale=S, weight=Wr, subcentres=K, topk=TOPK, topk_margin=TM)
        runs = {"replicated": lambda: dsk.aam_softmax_step(rm, ropt, x, labels, **kw),
                "sharded": lambda: dsk.sharded_aam_softmax_step(sm, sopt, x, labels, head=head, head_optimizer=hopt)}
        res = {k: [] for k in runs}
        for _ in range(2):                               # alternated twice
            for name, fn in runs.items():
                for _ in range(warmup):
                    fn()
                dist.barrier()
                res[name].append(time_events(fn, steps))
        out[rank] = res
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_sharded_aam needs a GPU"
    rec = {"metric": "sharded_aam_softmax", **gpu_info(), "C": C, "K": K, "topk": TOPK, "n_per_rank": N_LOCAL}
    rec["whole_op_384_ms"] = [round(whole_op(args.iters), 3) for _ in range(2)]
    for R in (2, 4, 8):
        rec[f"shard_share_R{R}_ms"] = [round(shard_share(R, args.iters), 3) for _ in range(2)]
        rec[f"collective_bytes_R{R}"] = collective_bytes(R)
    world = torch.cuda.device_count()
    if world >= 2:
        import torch.multiprocessing as mp

        mgr = mp.Manager()
        out = mgr.dict()
        mp.spawn(_step_worker, args=(world, _free_port(), args.steps, args.warmup, out), nprocs=world, join=True)
        rec[f"step_ms_R{world}"] = {k: [round(v, 3) for v in vals] for k, vals in out[0].items()}
    else:
        rec["step_ms"] = f"not measured: {world} GPU visible"
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
