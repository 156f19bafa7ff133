"""GE2E over the global batch: the row-range ops are bit-identical to the whole-batch op for every way of splitting the
rows (the w and b shares sum to the whole op's), bit-stable across repeats and other ops' calls, bad ranges are
rejected, the across-ranks step at world size 1 is the local step, and with >= 2 GPUs (NCCL) the across-ranks step
reproduces the single-device loss and gradient."""
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
from tests.test_gpu_ge2e import CASES, METHODS, _case, _csr, _hard_case, _scalar

pytestmark = pytest.mark.gpu


def _zero_case():
    """test_gpu_ge2e's zero-centroid case: a speaker of two opposite rows, and a zero row."""
    E, labels = _case([3] * 8, 64, "norm10", 5)
    E, labels = torch.cat([E, E[:1], -E[:1]]), torch.cat([labels, torch.tensor([1000, 1000])])
    E[5] = 0.0
    return E, labels


def _global_case(name):
    if name == "64x10x512_spread":                 # relabelled so that every speaker spans every shard
        E, _ = _case(*CASES["64x10x512"], "norm10", zlib.crc32(name.encode()))
        return E, torch.arange(640) % 64
    if name == "hard":
        return _hard_case()
    if name == "zero_centroid_zero_row":
        return _zero_case()
    if name == "3072x6x512":                       # P = 512: gC^'s 512-row K slices cut across the ranks' rows
        return _case([6] * 512, 512, "norm10", 7)
    if name.startswith("P"):                       # P = 127, 128, 129: the centroid tile's edge
        return _case([3] * int(name[1:]), 128, "arbitrary", int(name[1:]))
    return _case(*CASES[name], "norm10", zlib.crc32(name.encode()))


CASE_NAMES = ["64x10x512_spread", "ragged1000x192", "1024x4x512", "hard", "zero_centroid_zero_row", "3072x6x512",
              "P127", "P128", "P129"]


def _splits(N):
    """Contiguous row ranges: R = 1, 2, 4, 8 near-equal shards, and an uneven split with a one-row range and ranges
    that are not multiples of 128."""
    out = [[(N * r // R, N * (r + 1) // R - N * r // R) for r in range(R)] for R in (1, 2, 4, 8)]
    a = min(130, N - 2)
    out.append([(0, a), (a, 1), (a + 1, N - a - 1)])
    return out


def _whole(E, csr, V, w, b, method, g):
    Ec, loss, cos, rec = EN.ge2e(E, csr, V, w, b, method)
    return (Ec, loss, cos, rec) + tuple(EN.ge2e_backward(Ec, csr, V, w, b, method, cos, rec, g))


def _by_rows(E, csr, V, w, b, method, g, split):
    """The split's rows ops, as ranks would run them -> (cos, rec, row_loss, loss, dcos, tdc, gE, gw shares, gb
    shares), the per-range outputs concatenated in row order."""
    fwd = [EN.ge2e_rows(E, csr, V, w, b, method, r0, n)[1:] for r0, n in split]
    cos, rec, row_loss = (torch.cat([f[k] for f in fwd]) for k in range(3))
    loss = EN.ge2e_mean(row_loss, V)
    bwd = [EN.ge2e_dcos_rows(f[0], f[1], csr, V, w, b, method, r0, n, g) for f, (r0, n) in zip(fwd, split)]
    dcos, tdc = torch.cat([x[0] for x in bwd]), torch.cat([x[1] for x in bwd])
    gE = torch.cat([EN.ge2e_backward_rows(E, csr, dcos, tdc, r0, n) for r0, n in split])
    return cos, rec, row_loss, loss, dcos, tdc, gE, [x[2] for x in bwd], [x[3] for x in bwd]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", CASE_NAMES)
def test_rows_ops_bit_identical_to_the_whole_op(cuda_dev, name, method):
    E, labels = _global_case(name)
    E = E.cuda()
    csr, V = _csr(labels)
    w, b, g = _scalar(10.0), _scalar(-5.0), torch.ones((), device="cuda")
    Ec, loss, cos, rec, gE, gw, gb = _whole(E, csr, V, w, b, method, g)
    worst, identical = 0.0, True
    for split in _splits(E.shape[0]):
        c, r, _, l, _, _, gr, sw, sb = _by_rows(E, csr, V, w, b, method, g, split)
        assert torch.equal(c, cos) and torch.equal(r, rec), split
        assert torch.equal(l, loss), split
        assert torch.equal(gr, gE), split
        tw = sum(float(x) for x in sw)
        worst = max(worst, abs(tw - gw.item()) / max(abs(gw.item()), 1e-30))
        identical &= torch.equal(torch.stack(sw).sum(), gw) if len(split) > 1 else torch.equal(sw[0], gw)
        if method == "softmax":
            assert all(x.item() == 0.0 and not torch.signbit(x).item() for x in sb)
        else:
            tb = sum(float(x) for x in sb)
            worst = max(worst, abs(tb - gb.item()) / max(abs(gb.item()), 1e-30))
        if len(split) == 1:                       # the range (0, N) is the whole op, bit for bit
            assert torch.equal(sw[0], gw) and torch.equal(sb[0], gb)
    assert worst <= 1e-6, worst
    print(f"\n{name} {method}: summed w/b shares vs the whole op: worst rel {worst:.2e}, gw bit-identical {identical}")


def test_rows_ops_are_stable_across_repeats_and_other_ops(cuda_dev):
    E, labels = _global_case("3072x6x512")
    E = E.cuda()
    csr, V = _csr(labels)
    w, b, g = _scalar(10.0), _scalar(-5.0), torch.ones((), device="cuda")
    split = _splits(E.shape[0])[3]                                   # R = 8
    W = torch.randn(300, 512, generator=torch.Generator().manual_seed(3)).cuda()
    ya = torch.randint(0, 300, (E.shape[0],), generator=torch.Generator().manual_seed(4))
    first = _by_rows(E, csr, V, w, b, "contrast", g, split)
    whole = _whole(E, csr, V, w, b, "contrast", g)
    for k in range(2):
        Ec, Wc, lab, _, cos, lse = EN.aam_softmax(E, W, ya, 0.2, 30.0)
        EN.aam_softmax_backward(Ec, Wc, lab, cos, lse, 0.2, 30.0, g)
        EN.cohort_stats(E[:256], W, 50)
        again = _by_rows(E, csr, V, w, b, "contrast", g, split)
        for x, y in zip(first[:7], again[:7]):
            assert torch.equal(x, y)
        assert all(torch.equal(x, y) for x, y in zip(first[7] + first[8], again[7] + again[8]))
        w2 = _whole(E, csr, V, w, b, "contrast", g)
        assert all(torch.equal(x, y) for x, y in zip(whole, w2))


def test_bad_row_ranges_are_rejected(cuda_dev):
    E, labels = _case([4] * 16, 64, "norm10", 1)
    E = E.cuda()
    csr, V = _csr(labels)
    w, b, g = _scalar(10.0), _scalar(-5.0), torch.ones((), device="cuda")
    dcos, tdc = torch.zeros(64, 16, device="cuda"), torch.zeros(64, device="cuda")
    for row0, rows in ((0, 0), (10, 0), (60, 5), (64, 1), (-1, 4)):      # empty, past N, negative start
        with pytest.raises(RuntimeError):
            EN.ge2e_rows(E, csr, V, w, b, "softmax", row0, rows)
        cos, rec = torch.zeros(rows, 16, device="cuda"), torch.zeros(rows, device="cuda")   # the range's shapes
        with pytest.raises(RuntimeError):
            EN.ge2e_dcos_rows(cos, rec, csr, V, w, b, "softmax", row0, rows, g)
        with pytest.raises(RuntimeError):
            EN.ge2e_backward_rows(E, csr, dcos, tdc, row0, rows)
    _, _, cos, rec = EN.ge2e(E, csr, V, w, b, "softmax")
    with pytest.raises(RuntimeError):                                     # cos / rec not of the row range
        EN.ge2e_dcos_rows(cos, rec, csr, V, w, b, "softmax", 0, 32, g)
    with pytest.raises(RuntimeError):                                     # V > N
        EN.ge2e_mean(torch.zeros(64, device="cuda"), 65)
    with pytest.raises(RuntimeError):                                     # dcos not of the whole batch
        EN.ge2e_backward_rows(E, csr, dcos[:32], tdc[:32], 0, 32)


def _model(sd):
    m = dsk.DeepSpeakerModel(512, 16).cuda().train()
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("method", METHODS)
def test_across_ranks_step_at_world_size_one_is_the_local_step(cuda_dev, method):
    assert not (dist.is_available() and dist.is_initialized())
    sd = O.make_state_dict(0, num_classes=16)
    x = O.make_input(64, 32, seed=3, scale=3.0).cuda()
    labels = torch.arange(64) // 4
    outs, params = [], []
    for across in (False, True):
        model = _model(sd)
        crit = dsk.GE2ELoss(10.0, -5.0, method).cuda()
        opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-3, lr_decay=1e-4)
        outs.append(dsk.ge2e_step(model, opt, x, labels, loss=crit, across_ranks=across))
        params.append([p.detach().clone() for p in list(model.parameters()) + list(crit.parameters())])
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

        sd = O.make_state_dict(0, num_classes=16)
        model = _model(sd)
        crit = dsk.GE2ELoss(10.0, -5.0, "contrast").cuda()
        opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-3, lr_decay=1e-4)
        x, labels = _global_batch(world)
        xs, ls = shard(x, rank, world).cuda(), shard(labels, rank, world)
        seen = {}

        def hook(mod, inp, o):
            seen["emb"] = o.detach().clone()
            o.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

        h = model.register_forward_hook(hook)
        res = dsk.ge2e_step(model, opt, xs, ls, loss=crit, across_ranks=True)
        h.remove()
        torch.cuda.synchronize()
        raised = False
        try:                                                     # one speaker in the whole batch: global V = 0
            dsk.ge2e_step(model, opt, xs, torch.zeros(N_LOCAL, dtype=torch.long), loss=crit, across_ranks=True)
        except ValueError:
            raised = True
        params = [p.detach().cpu().clone() for p in list(model.parameters()) + list(crit.parameters())]
        smodel = _model(sd).sync_batchnorm()                     # synchronised BatchNorm over the ranks
        scrit = dsk.GE2ELoss(10.0, -5.0, "softmax").cuda()
        sopt = dsk.FusedAdagrad(list(smodel.parameters()) + list(scrit.parameters()), lr=1e-3, lr_decay=1e-4)
        sres = dsk.ge2e_step(smodel, sopt, xs, ls, loss=scrit, across_ranks=True)
        torch.cuda.synchronize()
        out[rank] = dict(loss=res["loss"].cpu(), valid=res["valid"], emb=seen["emb"].cpu(), grad=seen["grad"].cpu(),
                         params=params, raised=raised, collectives=opt.collectives, sync_loss=sres["loss"].cpu())
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
    # the loss: identical on every rank, bit-equal to GE2ELoss on the gathered embeddings
    E = torch.cat([r["emb"] for r in res]).cuda()
    crit = dsk.GE2ELoss(10.0, -5.0, "contrast").cuda()
    assert all(torch.equal(r["loss"], res[0]["loss"]) for r in res)
    assert torch.equal(res[0]["loss"].cuda(), crit(E, labels).detach())
    # the gradient entering each rank's network: R x the rank's rows of the single-device gE
    csr, V = _csr(labels)
    w, b = _scalar(10.0), _scalar(-5.0)
    Ec, _, cos, rec = EN.ge2e(E, csr, V, w, b, "contrast")
    gE, _, _ = EN.ge2e_backward(Ec, csr, V, w, b, "contrast", cos, rec, torch.ones((), device="cuda"))
    for r in range(world):
        assert torch.equal(res[r]["grad"], world * gE[r * N_LOCAL:(r + 1) * N_LOCAL].cpu())
    # parameters, w and b: identical across ranks, and those of a one-device emulation (per-shard BN, whole loss)
    for r in range(1, world):
        assert all(torch.equal(a, b) for a, b in zip(res[0]["params"], res[r]["params"]))
    model = _model(O.make_state_dict(0, num_classes=16))
    params = list(model.parameters()) + list(crit.parameters())
    opt = dsk.FusedAdagrad(params, lr=1e-3, lr_decay=1e-4)
    emb = torch.cat([model(x[r * N_LOCAL:(r + 1) * N_LOCAL].cuda()) for r in range(world)])
    opt.zero_grad()
    crit(emb, labels).backward()
    opt.step()
    worst = 0.0
    for a, b in zip(res[0]["params"], params):
        b = b.detach().cpu()
        worst = max(worst, float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)))
    print(f"\nR={world}: parameters, w, b vs the one-device emulation: worst rel-L2 {worst:.3e}")
    assert worst <= 1e-6
    # synchronised BatchNorm: the loss of the single-device synchronised step on the gathered batch
    smodel = _model(O.make_state_dict(0, num_classes=16)).sync_batchnorm()
    scrit = dsk.GE2ELoss(10.0, -5.0, "softmax").cuda()
    sopt = dsk.FusedAdagrad(list(smodel.parameters()) + list(scrit.parameters()), lr=1e-3, lr_decay=1e-4)
    sres = dsk.ge2e_step(smodel, sopt, x.cuda(), labels, loss=scrit)
    assert all(torch.equal(r["sync_loss"], sres["loss"].cpu()) for r in res)
