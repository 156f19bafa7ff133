"""Batch-hard mining over the global batch: the row-range ops are bit-identical to the whole-batch op on both distance
paths for every way of splitting the anchors, bad ranges are rejected, the across-ranks step at world size 1 is the
local step, and with >= 2 GPUs (NCCL) the across-ranks step reproduces the single-device loss and gradient."""
import os
import socket
import zlib

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as EN
from oracle import rescnn_oracle as O
from tests.test_gpu_batch_hard import _case, _hub_case, _norm10

pytestmark = pytest.mark.gpu

MARGIN = 0.3


def _global_case(name):
    if name == "1024x512_64x16_spread":            # relabelled so that every speaker spans every shard
        E, _ = _case("1024x512_64x16")
        return E, (torch.arange(1024) % 64).long(), MARGIN
    if name == "hub":
        E, labels = _hub_case()
        return E, labels, 12.0
    return (*_case(name), MARGIN)


CASES = ["1024x512_64x16_spread", "130_uneven_singletons", "D96_exact_path", "near_duplicates", "duplicated_rows", "hub"]


def _splits(N):
    """Contiguous anchor ranges: R = 1, 2, 4, 8 near-equal shards, and an uneven split with a one-row range and
    ranges that are not multiples of 128."""
    out = [[(N * r // R, N * (r + 1) // R - N * r // R) for r in range(R)] for R in (1, 2, 4, 8)]
    a = min(130, N - 2)
    out.append([(0, a), (a, 1), (a + 1, N - a - 1)])
    return out


def _rows_equal_full(E, labels, margin, exact, splits):
    """Each split is a list of consecutive ranges covering [lo, hi); the whole batch when lo = 0 and hi = N."""
    Ec, loss, *sel = EN.batch_hard_mine(E, labels, margin, exact)
    one = torch.ones((), device="cuda")
    gE = EN.batch_hard_backward(Ec, *sel, margin, one)
    for split in splits:
        lo, hi = split[0][0], split[-1][0] + split[-1][1]
        parts = [EN.batch_hard_select_rows(E, labels, r0, n, exact)[1:] for r0, n in split]
        cat = [torch.cat([p[k] for p in parts]) for k in range(5)]
        for a, b in zip(cat, sel):
            assert a.dtype == b.dtype and torch.equal(a, b[lo:hi]), split
        if (lo, hi) == (0, E.shape[0]):      # the concatenation is a whole-batch selection: the loss and the backward
            assert torch.equal(EN.batch_hard_mean(cat[2], cat[3], cat[4], margin), loss), split
            sel_all = cat
        else:
            sel_all = sel
        g = torch.cat([EN.batch_hard_backward_rows(Ec, *sel_all, r0, n, margin, one) for r0, n in split])
        assert torch.equal(g, gE[lo:hi]), split
    return sel


@pytest.mark.parametrize("exact", [False, True], ids=["tensor_core", "exact"])
@pytest.mark.parametrize("name", CASES)
def test_rows_ops_bit_identical_to_the_full_op(cuda_dev, name, exact):
    E, labels, margin = _global_case(name)
    E, labels = E.cuda(), labels.cuda()
    sel = _rows_equal_full(E, labels, margin, exact, _splits(E.shape[0]))
    assert bool(sel[4].any())


@pytest.mark.parametrize("exact", [False, True], ids=["tensor_core", "exact"])
def test_rows_ops_at_the_size_limit(cuda_dev, exact):
    N = 16384
    g = torch.Generator().manual_seed(zlib.crc32(b"16384"))
    E = _norm10(torch.randn(N, 512, generator=g)).cuda()
    labels = (torch.arange(N) % 1024).cuda()                   # 16 utterances per speaker, spread over the batch
    _rows_equal_full(E, labels, MARGIN, exact, [[(N - 2048, 2048)]])


def test_bad_row_ranges_are_rejected(cuda_dev):
    E = torch.randn(64, 64, device="cuda")
    labels = torch.arange(64, device="cuda") % 8
    _, _, *sel = EN.batch_hard_mine(E, labels, MARGIN)
    one = torch.ones((), device="cuda")
    for row0, rows in ((0, 0), (10, 0), (60, 5), (64, 1), (-1, 4)):      # empty, past N, negative start
        for exact in (False, True):
            with pytest.raises(RuntimeError):
                EN.batch_hard_select_rows(E, labels, row0, rows, exact)
        with pytest.raises(RuntimeError):
            EN.batch_hard_backward_rows(E, *sel, row0, rows, MARGIN, one)
    big = torch.zeros(16385, 8, device="cuda")                           # N > DSK_BATCH_HARD_MAX_N
    with pytest.raises(RuntimeError):
        EN.batch_hard_select_rows(big, torch.arange(16385) % 2, 0, 8, True)
    z = torch.zeros(16385, device="cuda")
    with pytest.raises(RuntimeError):
        EN.batch_hard_mean(z, z, z.bool(), MARGIN)


def _model(sd):
    m = dsk.DeepSpeakerModel(512, 16).cuda().train()
    m.load_state_dict(sd)
    return m


def test_across_ranks_step_at_world_size_one_is_the_local_step(cuda_dev):
    assert not (dist.is_available() and dist.is_initialized())
    sd = O.make_state_dict(0, num_classes=16)
    x = O.make_input(64, 32, seed=3, scale=3.0).cuda()
    labels = torch.arange(64) // 4
    outs, params = [], []
    for across in (False, True):
        model = _model(sd)
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        outs.append(dsk.batch_hard_step(model, opt, x, labels, margin=0.5, across_ranks=across))
        params.append([p.detach().clone() for p in model.parameters()])
    assert outs[0]["valid"] == outs[1]["valid"] == 64
    assert torch.equal(outs[0]["loss"], outs[1]["loss"])
    assert all(torch.equal(a, b) for a, b in zip(*params))


# ---- >= 2 GPUs, NCCL --------------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_LOCAL, T, K = 32, 32, 4


def _global_batch(world):
    N = world * N_LOCAL
    x = O.make_input(N, T, seed=7, scale=3.0)
    labels = torch.arange(N) % (N // K)                        # K utterances per speaker, one on each of K shards
    return x, labels


def _nccl_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from deepspeaker_pytorch_b200.parallel import shard

        model = _model(O.make_state_dict(0, num_classes=16))
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
        x, labels = _global_batch(world)
        seen = {}

        def hook(mod, inp, o):
            seen["emb"] = o.detach().clone()
            o.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

        h = model.register_forward_hook(hook)
        res = dsk.batch_hard_step(model, opt, shard(x, rank, world).cuda(), shard(labels, rank, world), margin=0.5,
                                  across_ranks=True)
        h.remove()
        torch.cuda.synchronize()
        raised = False
        try:                                                     # one speaker in the whole batch: global V = 0
            dsk.batch_hard_step(model, opt, shard(x, rank, world).cuda(), torch.zeros(N_LOCAL, dtype=torch.long),
                                margin=0.5, across_ranks=True)
        except ValueError:
            raised = True
        out[rank] = dict(loss=res["loss"].cpu(), valid=res["valid"], emb=seen["emb"].cpu(), grad=seen["grad"].cpu(),
                         params=[p.detach().cpu().clone() for p in model.parameters()], raised=raised,
                         collectives=opt.collectives)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_across_ranks_step_on_nccl(cuda_dev, world):
    visible = torch.cuda.device_count()
    if visible < world:
        pytest.skip(f"needs {world} GPUs, {visible} visible")
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_nccl_worker, args=(world, port, out), nprocs=world, join=True)
    res = [out[r] for r in range(world)]
    x, labels = _global_batch(world)
    N = world * N_LOCAL
    assert all(r["raised"] for r in res)
    assert all(r["valid"] == N for r in res) and all(r["collectives"] == 1 for r in res)
    # the loss: identical on every rank, bit-equal to the single-device op on the gathered embeddings
    E = torch.cat([r["emb"] for r in res]).cuda()
    Ec, loss, *sel = EN.batch_hard_mine(E, labels, 0.5)
    assert all(torch.equal(r["loss"], res[0]["loss"]) for r in res)
    assert torch.equal(res[0]["loss"].cuda(), loss.reshape(()))
    # the gradient entering each rank's network: R x the rank's rows of the single-device gE
    gE = EN.batch_hard_backward(Ec, *sel, 0.5, torch.ones((), device="cuda")).cpu()
    for r in range(world):
        assert torch.equal(res[r]["grad"], world * gE[r * N_LOCAL:(r + 1) * N_LOCAL])
    # parameters: identical across ranks, and those of a one-device emulation (per-shard BN forwards, full loss)
    for r in range(1, world):
        assert all(torch.equal(a, b) for a, b in zip(res[0]["params"], res[r]["params"]))
    model = _model(O.make_state_dict(0, num_classes=16))
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
    emb = torch.cat([model(x[r * N_LOCAL:(r + 1) * N_LOCAL].cuda()) for r in range(world)])
    opt.zero_grad()
    dsk.BatchHardTripletLoss(0.5).forward(emb, labels).backward()
    opt.step()
    worst, identical = 0.0, True
    for a, b in zip(res[0]["params"], model.parameters()):
        b = b.detach().cpu()
        identical &= torch.equal(a, b)
        worst = max(worst, float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)))
    print(f"\nR={world}: parameters vs the one-device emulation: worst rel-L2 {worst:.3e}, bit-identical {identical}")
    assert worst <= 1e-6
