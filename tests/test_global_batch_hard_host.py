"""GlobalBatchHardTripletLoss, host side (CPU, gloo, world size 2): the engine's three row-range ops are replaced in each
worker by stand-ins built from the batch-hard oracle (the full C selection, sliced to the rank's rows; the mean; the
fp64 loss, differentiated), so the plumbing is checked without a GPU: the rank offsets, the packing and unpacking of
the selection records, the global V, the loss over the union, the per-rank gradient rows and the collectives issued."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from deepspeaker_pytorch_b200.model import batch_hard_valid_count
from deepspeaker_pytorch_b200.parallel import (SELECTION_RECORD_BYTES, _pack_selection, _unpack_selection,
                                               gather_labels)
from oracle import batch_hard_oracle as BH

MARGIN = 6.0
COLLECTIVES = ("all_gather_into_tensor", "all_gather", "all_reduce", "broadcast", "reduce_scatter_tensor",
               "all_to_all_single", "barrier", "send", "recv")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _batch():
    g = torch.Generator().manual_seed(5)
    E = torch.randn(48, 32, generator=g)
    E = 10.0 * E / E.norm(dim=1, keepdim=True)
    labels = torch.arange(48) % 6              # every speaker spans both shards
    labels[47] = 99                            # a singleton: an invalid anchor on rank 1
    return E, labels


def _install_stand_ins(EN, log):
    def select_rows(E, labels, row0, rows, exact_cuda_cores=False):
        log["select"].append((int(row0), int(rows), E.shape[0]))
        _, pos, neg, d_ap, d_an, valid = BH.batch_hard_triplet(E.numpy(), labels.numpy(), MARGIN)
        sl = slice(row0, row0 + rows)
        return (E, torch.from_numpy(pos[sl].copy()), torch.from_numpy(neg[sl].copy()), torch.from_numpy(d_ap[sl].copy()),
                torch.from_numpy(d_an[sl].copy()), torch.from_numpy(valid[sl].copy()))

    def mean(d_ap, d_an, valid, margin):
        log["mean_in"] = [t.clone() for t in (d_ap, d_an, valid)]
        h = torch.clamp((margin + d_ap.double()) - d_an.double(), min=0.0) * valid.double()
        return (h.sum() / max(int(valid.sum()), 1)).float().reshape(1)

    def backward_rows(E, pos, neg, d_ap, d_an, valid, row0, rows, margin, grad_loss):
        with torch.enable_grad():                  # autograd runs a Function's backward with grad mode off
            E64 = E.double().requires_grad_(True)
            BH.batch_hard_loss(E64, pos, neg, valid, margin).backward()
        return E64.grad[row0:row0 + rows] * grad_loss.double()

    EN.batch_hard_select_rows = select_rows
    EN.batch_hard_mean = mean
    EN.batch_hard_backward_rows = backward_rows


def _count_collectives(counter):
    for name in COLLECTIVES:
        fn = getattr(dist, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            counter.append(_name)
            return _fn(*a, **k)

        setattr(dist, name, wrapped)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from deepspeaker_pytorch_b200 import engine as EN
        from deepspeaker_pytorch_b200.parallel import GlobalBatchHardTripletLoss

        log = {"select": []}
        _install_stand_ins(EN, log)
        calls = []
        _count_collectives(calls)
        E, labels = _batch()
        n = E.shape[0] // world
        local = E[rank * n:(rank + 1) * n].double().requires_grad_(True)
        glabels = gather_labels(labels[rank * n:(rank + 1) * n])
        n_labels = len(calls)
        loss = GlobalBatchHardTripletLoss(MARGIN).forward(local, glabels)
        fwd = calls[n_labels:]
        n_fwd = len(calls)
        loss.backward()
        bwd = calls[n_fwd:]
        out[rank] = dict(glabels=glabels.clone(), V=batch_hard_valid_count(glabels), select=log["select"],
                         mean_in=log["mean_in"], loss=loss.detach().clone(), grad=local.grad.clone(),
                         n_label_collectives=n_labels, fwd=fwd, bwd=bwd)
    finally:
        dist.destroy_process_group()


def test_global_loss_plumbing_against_the_oracle():
    world = 2
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    E, labels = _batch()
    N, n = E.shape[0], E.shape[0] // world
    oloss, opos, oneg, od_ap, od_an, ovalid = BH.batch_hard_triplet(E.numpy(), labels.numpy(), MARGIN)
    E64 = E.double().requires_grad_(True)
    BH.batch_hard_loss(E64, torch.from_numpy(opos), torch.from_numpy(oneg), torch.from_numpy(ovalid), MARGIN).backward()
    for r in range(world):
        o = out[r]
        assert torch.equal(o["glabels"], labels) and o["n_label_collectives"] == 1       # one gather, rank order
        assert o["V"] == int(ovalid.sum()) == N - 1                                       # the singleton is no anchor
        assert o["select"] == [(r * n, n, N)]                                             # this rank's rows, all N
        d_ap, d_an, valid = o["mean_in"]                                                  # unpacked: the whole batch
        assert np.array_equal(d_ap.numpy(), od_ap) and np.array_equal(d_an.numpy(), od_an)
        assert np.array_equal(valid.numpy(), ovalid) and valid.dtype == torch.bool
        assert o["loss"].dim() == 0 and abs(float(o["loss"]) - float(oloss)) <= 1e-6 * float(oloss)
        assert float(oloss) > 0
        assert torch.equal(o["grad"], E64.grad[r * n:(r + 1) * n])                        # this rank's fp64 rows
        assert o["fwd"] == ["all_gather_into_tensor"] * 2 and o["bwd"] == []
    assert torch.equal(out[0]["loss"], out[1]["loss"])


def test_selection_record_round_trip():
    g = torch.Generator().manual_seed(3)
    recs, fields = [], []
    for r in range(3):
        pos = torch.randint(-1, 100, (5,), generator=g)
        neg = torch.randint(-1, 100, (5,), generator=g)
        d_ap, d_an = torch.rand(5, generator=g), torch.rand(5, generator=g)
        d_an[r] = float("inf")
        valid = torch.rand(5, generator=g) > 0.3
        rec = _pack_selection(pos, neg, d_ap, d_an, valid)
        assert rec.dtype == torch.uint8 and rec.shape == (5 * SELECTION_RECORD_BYTES,) and SELECTION_RECORD_BYTES == 25
        recs.append(rec)
        fields.append((pos, neg, d_ap, d_an, valid))
    got = _unpack_selection(torch.stack(recs), 5)
    for k, t in enumerate(got):
        assert torch.equal(t, torch.cat([f[k] for f in fields]))
