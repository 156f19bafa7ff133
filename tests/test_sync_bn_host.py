"""Synchronised BatchNorm, host side (CPU, gloo, world size 2): the engine's stage generators are replaced by stand-ins
whose records are a numpy restatement of the per-utterance sums (include/dsk.h), so the driver - ``run_lockstep``
around ``parallel.gather_records`` - is checked without a GPU: records arrive in rank order, a forward issues exactly 12
collectives and a backward 13 (also for three forwards in lockstep), both ranks end with the same statistics, equal
to those of the whole batch, and the hard-triplet branch is refused on every rank before any collective."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from deepspeaker_pytorch_b200 import train as TR
from deepspeaker_pytorch_b200.parallel import gather_records

C = [4, 4, 4, 8, 8, 8, 8, 8, 8, 16, 16, 16]       # channels of the 12 stand-in layers
HW = [12, 12, 12, 6, 6, 6, 4, 4, 4, 2, 2, 2]      # pixels per utterance
N_LOCAL = 3
COLLECTIVES = ("all_gather_into_tensor", "all_gather", "all_reduce", "broadcast", "reduce_scatter_tensor",
               "all_to_all_single", "barrier", "send", "recv")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _raw(call, layer, u):
    """Utterance u's pixels (HW, C) of one layer: channel means near 100, far above their spread."""
    g = np.random.RandomState(10000 * call + 100 * layer + u)
    return (g.randn(HW[layer], C[layer]) * 2.0 + 100.0 + g.randn(C[layer]) * 5.0).astype(np.float32)


def fwd_record(x):
    """pivot (first pixel), sum (x - k), sum (x - k)^2 in fp32, the pixel count as int32 bits: 3C + 1 words."""
    k = x[0]
    d = x - k
    sd = np.zeros_like(k)
    ssd = np.zeros_like(k)
    for row in d:                                 # fp32, in pixel order
        sd = (sd + row).astype(np.float32)
        ssd = (ssd + row * row).astype(np.float32)
    return np.concatenate([k, sd, ssd, np.array([x.shape[0]], np.int32).view(np.float32)])


def records_of(call, layer, us):
    return torch.from_numpy(np.concatenate([fwd_record(_raw(call, layer, u)) for u in us]).view(np.uint8).copy())


def finalize(gathered, c):
    """The record finalize in double, in utterance order around record 0's pivot -> (mean, biased var)."""
    r = gathered.numpy().view(np.float32).reshape(-1, 3 * c + 1)
    K = r[0, :c].astype(np.float64)
    s1 = s2 = M = 0.0
    for row in r:
        dk = row[:c].astype(np.float64) - K
        sd, ssd = row[c:2 * c].astype(np.float64), row[2 * c:3 * c].astype(np.float64)
        n = float(row[3 * c:].view(np.int32)[0])
        s1 = s1 + sd + n * dk
        s2 = s2 + ssd + 2.0 * dk * sd + n * dk * dk
        M += n
    return K + s1 / M, s2 / M - (s1 / M) ** 2


def stand_in_forward(call, rank, log):
    stats = []
    for i in range(12):
        gathered = yield records_of(call, i, range(rank * N_LOCAL, (rank + 1) * N_LOCAL))
        log.append((call, i, gathered.clone()))
        stats.append(finalize(gathered, C[i]))
    return stats


def stand_in_backward(call, rank, log):
    sizes = [4] + [8 * C[i] for i in reversed(range(12))]      # the loss-scale maxima, then layers 11..0
    for st, size in enumerate(sizes):
        local = torch.full((N_LOCAL * size,), rank * 16 + st, dtype=torch.uint8)
        gathered = yield local
        log.append((call, st, gathered.clone()))
    return f"backward {call}"


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
        import deepspeaker_pytorch_b200 as dsk

        calls = []
        _count_collectives(calls)
        exchange = lambda local: gather_records(local, dist.group.WORLD)
        res = {}
        # branch B of train_step: refused before any collective (no GPU needed to reach the check)
        m = dsk.DeepSpeakerModel(512, 16).train().sync_batchnorm()
        x = torch.zeros(2, 1, 32, 64)
        try:
            dsk.train_step(m, None, x, x, x, torch.zeros(2), torch.ones(2), margin=0.1, epoch=1)
            res["refused"] = False
        except ValueError:
            res["refused"] = True
        res["collectives_before"] = list(calls)
        log = []
        (stats,) = TR.run_lockstep([stand_in_forward(0, rank, log)], exchange)
        res["fwd"], n0 = len(calls), len(calls)
        TR.run_lockstep([stand_in_backward(0, rank, log)], exchange)
        res["bwd"], n0 = len(calls) - n0, len(calls)
        trip = TR.run_lockstep([stand_in_forward(k, rank, log) for k in (1, 2, 3)], exchange)
        res["trip_fwd"], n0 = len(calls) - n0, len(calls)
        res["trip_bwd_out"] = TR.run_lockstep([stand_in_backward(k, rank, log) for k in (1, 2, 3)], exchange)
        res["trip_bwd"] = len(calls) - n0
        res["kinds"] = sorted(set(calls))
        res["stats"], res["trip_stats"], res["log"] = stats, trip, log
        out[rank] = res
    finally:
        dist.destroy_process_group()


def test_record_exchange_plumbing():
    world = 2
    port = _free_port()
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    N = world * N_LOCAL
    for r in range(world):
        o = out[r]
        assert o["refused"] and o["collectives_before"] == []
        assert o["fwd"] == 12 and o["bwd"] == 13 and o["trip_fwd"] == 12 and o["trip_bwd"] == 13
        assert o["kinds"] == ["all_gather_into_tensor"]
        assert o["trip_bwd_out"] == ["backward 1", "backward 2", "backward 3"]
        for call, i, gathered in o["log"][:12]:           # rank order: rank 0's utterances, then rank 1's
            assert torch.equal(gathered, records_of(call, i, range(N)))
    log0 = out[0]["log"]
    bwd = log0[12:25]
    for st, (call, s, gathered) in enumerate(bwd):
        assert s == st
        size = gathered.numel() // N
        expect = torch.cat([torch.full((N_LOCAL * size,), r * 16 + st, dtype=torch.uint8) for r in range(world)])
        assert torch.equal(gathered, expect)
    trip = log0[25:61]
    for k, (call, i, gathered) in enumerate(trip):       # three forwards in lockstep: each gets its own records
        assert (call, i) == (1 + k % 3, k // 3)
        assert torch.equal(gathered, records_of(call, i, range(N)))
    # identical statistics on both ranks, those of the whole batch
    flat = lambda s: [np.asarray(t) for layer in s for t in layer]
    assert all(np.array_equal(x, y) for x, y in zip(flat(out[0]["stats"]), flat(out[1]["stats"])))
    for a, b in zip(out[0]["trip_stats"], out[1]["trip_stats"]):
        assert all(np.array_equal(x, y) for x, y in zip(flat(a), flat(b)))
    for i, (mean, var) in enumerate(out[0]["stats"]):
        x = np.concatenate([_raw(0, i, u) for u in range(N)]).astype(np.float64)
        assert np.allclose(mean, x.mean(0), rtol=0, atol=1e-5 * x.std(0).max())
        assert np.allclose(var, x.var(0), rtol=1e-4)
