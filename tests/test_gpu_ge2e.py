"""GE2E on the GPU: cosines and loss against fp64 from the fp32 inputs, the backward against the explicit fp64 backward
with the engine's own cosines (and contrast argmax) pinned, the hard cases, determinism, plan isolation from the other
cosine ops, argument rejection, ``ge2e_step`` end to end and, with two GPUs, data parallelism on NCCL."""
import copy
import os
import socket
import zlib

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200.model import ge2e_batch
from oracle import ge2e_oracle as G
from oracle import rescnn_oracle as O

pytestmark = pytest.mark.gpu

METHODS = ["softmax", "contrast"]


def _labels(counts, seed):
    g = torch.Generator().manual_seed(seed)
    lab = torch.cat([torch.full((c,), 3 * k - 50, dtype=torch.int64) for k, c in enumerate(counts)])
    return lab[torch.randperm(lab.numel(), generator=g)]


def _case(counts, D, norms, seed):
    """Rows of speakers with counts[k] rows each (a shared speaker direction plus noise), shuffled."""
    g = torch.Generator().manual_seed(seed)
    labels = _labels(counts, seed)
    col, P, _ = G.speakers(labels)
    E = torch.randn(labels.numel(), D, generator=g) + 1.5 * torch.randn(P, D, generator=g)[col] / 1.0
    if norms == "norm10":                      # as the model emits them
        E = 10.0 * E / E.norm(dim=1, keepdim=True)
    else:                                      # arbitrary norms over four decades
        E = E * torch.exp(torch.empty(E.shape[0], 1).uniform_(-4.0, 5.0, generator=g))
    return E, labels


CASES = {
    "2x2x64": ([2, 2], 64),
    "64x10x512": ([10] * 64, 512),
    "1024x4x512": ([4] * 1024, 512),
    "ragged1000x192": (list(np.random.default_rng(3).integers(1, 18, 112)), 192),   # n_k 1..17, ~1000 rows
}


def _csr(labels):
    order, offsets, col, V = ge2e_batch(labels)
    return tuple(torch.from_numpy(a).cuda() for a in (order, offsets, col)), V


def _scalar(v):
    return torch.tensor([float(v)], device="cuda")


def _fwd(E, labels, w, b, method):
    csr, V = _csr(labels)
    Ec, loss, cos, rec = EN.ge2e(E.cuda(), csr, V, _scalar(w), _scalar(b), method)
    return Ec, csr, V, loss.reshape(()), cos, rec


def _bwd(Ec, csr, V, w, b, method, cos, rec, g=1.0):
    return EN.ge2e_backward(Ec, csr, V, _scalar(w), _scalar(b), method, cos, rec, torch.full((), float(g), device="cuda"))


def _row_rel(got, ref):
    """Per-row relative L2 error over rows with a nonzero reference gradient; a row below 1e-3 of the largest row's
    gradient is measured against that floor (as in the AAM-softmax test)."""
    err, den = (got.double().cpu() - ref).norm(dim=1), ref.norm(dim=1)
    nz = den > 0
    if not bool(nz.any()):
        return 0.0
    return float((err[nz] / torch.maximum(den[nz], 1e-3 * den.max())).max())


def _target_mask(labels):
    col, P, n = G.speakers(labels)
    tgt = torch.nn.functional.one_hot(col, P).bool()
    valid = n[col] >= 2
    return tgt & valid[:, None], valid


def _check_cos(cos, ref, labels, tol=1e-6):
    got = cos.double().cpu()
    tgt, _ = _target_mask(labels)
    d_nt = float((got - ref).abs()[~tgt].max())
    ulp = torch.from_numpy(np.spacing(np.abs(ref[tgt].numpy()).astype(np.float32)).astype(np.float64))
    d_t = (got[tgt] - ref[tgt]).abs()
    assert d_nt <= tol, d_nt
    assert bool((d_t <= ulp + 1e-12).all()), float((d_t - ulp).max())
    return d_nt, float(d_t.max())


@pytest.mark.parametrize("norms", ["norm10", "arbitrary"])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_vs_fp64(cuda_dev, name, norms):
    counts, D = CASES[name]
    E, labels = _case(counts, D, norms, zlib.crc32(f"{name}{norms}".encode()))
    for method in METHODS:
        for w in (10.0, 0.5, 1e-7):
            for b in (-5.0, 3.0):
                _, _, _, loss, cos, rec = _fwd(E, labels, w, b, method)
                oloss, ref_cos, _ = G.forward(E, labels, w, b, method)
                d_nt, d_t = _check_cos(cos, ref_cos, labels)
                dloss = abs(loss.item() - float(oloss))
                assert dloss <= 1e-5 * max(float(oloss), 1.0), (method, w, b, loss.item(), float(oloss))
        print(f"\n{name} {norms} {method}: max |dcos| non-target {d_nt:.2e}, target {d_t:.2e}, |dloss| {dloss:.2e}")


def _check_backward(E, labels, w, b, method, tol=1e-5, report=True):
    Ec, csr, V, loss, cos, rec = _fwd(E, labels, w, b, method)
    gE, gw, gb = _bwd(Ec, csr, V, w, b, method, cos, rec)
    am = rec.long().cpu() if method == "contrast" else None
    c = cos.cpu()
    rE, rw, rb = G.backward(E, labels, w, b, method, cos=c, argmax=am)
    assert bool(torch.isfinite(gE).all())
    eE = _row_rel(gE, rE)
    dS = G.score_grads(c, labels, w, b, method, argmax=am)
    ew = abs(gw.item() - rw) / max(abs(rw), float((dS * c.double()).abs().sum()) if w >= 1e-6 else 1.0, 1e-30)
    assert eE <= tol, (method, w, b, eE)
    assert ew <= 1e-6, (method, w, b, gw.item(), rw)
    if method == "softmax":
        assert gb.item() == 0.0 and not torch.signbit(gb).item()
    else:
        eb = abs(gb.item() - rb) / max(abs(rb), float(dS.abs().sum()))
        assert eb <= 1e-6, (method, w, b, gb.item(), rb)
    if report:
        fE, _, _ = G.backward(E, labels, w, b, method)       # fully fp64, reported only
        print(f"\n{method} w {w} b {b}: per-row rel-L2 gE {eE:.2e} (end to end fp64 {_row_rel(gE, fE):.2e}), "
              f"gw {ew:.2e}")
    return Ec, csr, V, loss, cos, rec, gE, gw, gb


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", list(CASES))
def test_backward_vs_fp64_with_cos_pinned(cuda_dev, name, method):
    counts, D = CASES[name]
    E, labels = _case(counts, D, "norm10", zlib.crc32(name.encode()))
    for w, b in ((10.0, -5.0), (0.5, 3.0), (1e-7, -5.0)):
        _check_backward(E, labels, w, b, method)


def _hard_case():
    """speaker 0: two near-duplicate rows (target cos -> 1); speakers 1 and 2: three identical rows each, close to the
    direction of speaker 3 (a contrast tie between columns 1 and 2 for speaker 3's rows); speakers 4 and 5: singletons;
    speakers 6..9: ordinary."""
    D = 128
    g = torch.Generator().manual_seed(17)
    u = torch.randn(D, generator=g)
    rows, labels = [10.0 * u / u.norm(), 10.0 * u / u.norm() + 1e-5 * torch.randn(D, generator=g)], [0, 0]
    v = torch.randn(D, generator=g)
    dup = [v + 0.1 * torch.randn(D, generator=g) for _ in range(3)]
    rows += dup + dup
    labels += [1, 1, 1, 2, 2, 2]
    rows += [v + 0.5 * torch.randn(D, generator=g) for _ in range(4)]
    labels += [3] * 4
    rows += [torch.randn(D, generator=g), torch.randn(D, generator=g)]
    labels += [4, 5]
    for k in range(6, 10):
        c = torch.randn(D, generator=g)
        rows += [c + 0.7 * torch.randn(D, generator=g) for _ in range(3)]
        labels += [k] * 3
    return torch.stack(rows), torch.tensor(labels)


@pytest.mark.parametrize("method", METHODS)
def test_hard_cases(cuda_dev, method):
    E, labels = _hard_case()
    Ec, csr, V, loss, cos, rec, gE, gw, gb = _check_backward(E, labels, 10.0, -5.0, method, report=False)
    assert V == E.shape[0] - 2
    oloss, ref_cos, _ = G.forward(E, labels, 10.0, -5.0, method)
    _check_cos(cos, ref_cos, labels)
    assert cos[0, 0].item() > 0.999999 and cos[1, 0].item() > 0.999999
    others = torch.tensor([0, 1] + list(range(8, E.shape[0])))
    assert torch.equal(cos[others, 1], cos[others, 2])             # identical speakers, identical columns
    if method == "contrast":
        assert bool((rec[8:12] == 1.0).all())                       # the tie goes to the lower column
    # singletons: no loss term, but a gradient through their centroid
    assert gE[12].abs().sum().item() > 0 and gE[13].abs().sum().item() > 0
    assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0)


@pytest.mark.parametrize("method", METHODS)
def test_zero_centroid_and_zero_row(cuda_dev, method):
    """A speaker whose two rows are opposite (a zero inclusive centroid: every other row's cosine to it is 0, and the
    gradient through it is finite) and a zero embedding row."""
    E, labels = _case([3] * 8, 64, "norm10", 5)
    E, labels = torch.cat([E, E[:1], -E[:1]]), torch.cat([labels, torch.tensor([1000, 1000])])
    E[5] = 0.0
    Ec, csr, V, loss, cos, rec, gE, gw, gb = _check_backward(E, labels, 10.0, -5.0, method, report=False)
    P = cos.shape[1]
    assert not bool(cos[:24, P - 1].any())
    assert bool(torch.isfinite(gE).all()) and not bool(cos[5].any())


def test_deterministic(cuda_dev):
    counts, D = CASES["ragged1000x192"]
    E, labels = _case(counts, D, "norm10", 9)
    for method in METHODS:
        runs = []
        for _ in range(2):
            Ec, csr, V, loss, cos, rec = _fwd(E, labels, 10.0, -5.0, method)
            runs.append((loss, cos, rec) + tuple(_bwd(Ec, csr, V, 10.0, -5.0, method, cos, rec)))
        for a, b in zip(*runs):
            assert torch.equal(a, b)


def test_plans_do_not_interfere(cuda_dev):
    """AAM-softmax, cohort statistics and all-pairs calls interleaved with GE2E calls of other shapes leave every op's
    outputs bit-identical to the isolated calls."""
    E1, l1 = _case([6] * 64, 512, "norm10", 1)
    E2, l2 = _case([4] * 100, 256, "norm10", 2)
    W = torch.randn(300, 512, generator=torch.Generator().manual_seed(3)).cuda()
    ya = torch.randint(0, 300, (E1.shape[0],), generator=torch.Generator().manual_seed(4))

    def ge2e_all(E, lab, method):
        Ec, csr, V, loss, cos, rec = _fwd(E, lab, 10.0, -5.0, method)
        return (loss, cos, rec) + tuple(_bwd(Ec, csr, V, 10.0, -5.0, method, cos, rec))

    def aam():
        Ec, Wc, lab, loss, cos, lse = EN.aam_softmax(E1.cuda(), W, ya, 0.2, 30.0)
        return (loss, cos, lse) + tuple(EN.aam_softmax_backward(Ec, Wc, lab, cos, lse, 0.2, 30.0,
                                                                torch.ones((), device="cuda")))

    cohort = lambda: EN.cohort_stats(E1.cuda(), W, 50)                                          # noqa: E731
    allpairs = lambda: EN.allpairs_topk(E1.cuda(), l1.cuda(), 5)                                # noqa: E731
    iso = [ge2e_all(E1, l1, "softmax"), aam(), cohort(), allpairs(), ge2e_all(E2, l2, "contrast")]
    mixed = [None] * 5
    mixed[4] = ge2e_all(E2, l2, "contrast")
    mixed[1] = aam()
    mixed[0] = ge2e_all(E1, l1, "softmax")
    mixed[2] = cohort()
    ge2e_all(E2, l2, "softmax")
    mixed[3] = allpairs()
    for a, b in zip(iso, mixed):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert torch.equal(ge2e_all(E1, l1, "softmax")[3], iso[0][3])


def test_bad_arguments_are_rejected(cuda_dev):
    E = torch.randn(8, 64, device="cuda")
    lab = torch.tensor([0, 0, 1, 1, 2, 2, 3, 3])
    crit = dsk.GE2ELoss().cuda()
    cases = [
        (torch.randn(8, 96, device="cuda"), lab, RuntimeError),          # D % 64 != 0
        (E, torch.zeros(8, dtype=torch.long), ValueError),                # P < 2
        (E, torch.arange(8), ValueError),                                 # V = 0
        (E, lab[:7], RuntimeError),                                       # labels mismatch
        (E.cpu(), lab, RuntimeError),                                     # CPU tensors
    ]
    for e, y, exc in cases:
        with pytest.raises(exc):
            crit.forward(e, y)
    with pytest.raises(ValueError):
        dsk.GE2ELoss(method="cosine")
    with pytest.raises(RuntimeError):                                     # the loss's scalars on another device
        dsk.GE2ELoss().forward(E, lab)
    csr, V = _csr(lab)
    with pytest.raises(ValueError):
        EN.ge2e(E, csr, V, _scalar(10.0), _scalar(-5.0), "angular")


def _model(sd):
    model = dsk.DeepSpeakerModel(512, 16).cuda().train()
    model.load_state_dict(sd)
    return model


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
@pytest.mark.parametrize("P,M,T", [(16, 4, 32), (64, 6, 160)])
def test_ge2e_step_end_to_end(cuda_dev, P, M, T, opt_kind, method):
    N = P * M
    sd = O.make_state_dict(0, num_classes=16)
    model = _model(sd)
    ref_model = copy.deepcopy(model)
    crit = dsk.GE2ELoss(10.0, -5.0, method).cuda()
    params = list(model.parameters()) + list(crit.parameters())
    opt = dsk.FusedAdagrad(params, lr=1e-2, lr_decay=1e-4) if opt_kind == "fused" else \
        torch.optim.Adagrad(params, lr=1e-2, lr_decay=1e-4)
    x = O.make_input(N, T, seed=N, scale=3.0)
    labels = _labels([M] * P, N)
    w0, b0 = crit.w.detach().clone(), crit.b.detach().clone()
    seen = {}

    def hook(mod, inp, out):
        seen["emb"] = out.detach().clone()
        out.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

    h = model.register_forward_hook(hook)
    out = dsk.ge2e_step(model, opt, x.cuda(), labels, loss=crit)
    h.remove()
    assert out["loss"].dim() == 0 and out["loss"].is_cuda and out["valid"] == N
    # the gradient entering the network's backward is the op's gE
    csr, V = _csr(labels)
    Ec, loss, cos, rec = EN.ge2e(seen["emb"], csr, V, w0.reshape(1), b0.reshape(1), method)
    gE, _, _ = EN.ge2e_backward(Ec, csr, V, w0.reshape(1), b0.reshape(1), method, cos, rec,
                                torch.ones((), device="cuda"))
    assert torch.equal(seen["grad"], gE) and torch.equal(loss.reshape(()), out["loss"])
    # against the oracle's fp32 train-mode forward and the fp64 GE2E
    with torch.no_grad():
        ref_emb = O.forward(sd, x, train=True)
    oloss, _, _ = G.forward(ref_emb, labels, 10.0, -5.0, method)
    assert abs(out["loss"].item() - float(oloss)) <= 1e-3, (out["loss"].item(), float(oloss))
    assert not torch.equal(crit.w.detach(), w0)
    if method == "softmax":
        assert torch.equal(crit.b.detach(), b0)
    else:
        assert not torch.equal(crit.b.detach(), b0)
    # running statistics: those of exactly one train-mode forward of the batch
    with torch.no_grad():
        ref_model(x.cuda())
    for (k, v), (_, r) in zip(model.state_dict().items(), ref_model.state_dict().items()):
        if "running" in k:
            assert torch.equal(v, r), k
    # a model with synchronised BatchNorm (one rank) runs the same step
    sync_model = _model(sd).sync_batchnorm()
    scrit = dsk.GE2ELoss(10.0, -5.0, method).cuda()
    sopt = dsk.FusedAdagrad(list(sync_model.parameters()) + list(scrit.parameters()), lr=1e-2, lr_decay=1e-4)
    sout = dsk.ge2e_step(sync_model, sopt, x.cuda(), labels, loss=scrit)
    assert abs(sout["loss"].item() - out["loss"].item()) <= 1e-3
    print(f"\nN={N} T={T} {opt_kind} {method}: loss {out['loss'].item():.6f} (oracle {float(oloss):.6f}, "
          f"sync BN {sout['loss'].item():.6f}), w {crit.w.item():.6f}, b {crit.b.item():.6f}")


# ---- >= 2 GPUs, NCCL --------------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_LOCAL, T_DP = 32, 32


def _dp_batch(world):
    """Speaker-whole shards with unequal V_r: rank r holds speakers of 4 rows, rank 1 also a singleton."""
    x = O.make_input(world * N_LOCAL, T_DP, seed=11, scale=3.0)
    labels = torch.arange(world * N_LOCAL) // 4
    labels[N_LOCAL + 3] = 10 ** 6                     # a singleton on rank 1 (its speaker keeps 3 rows)
    return x, labels


def _nccl_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        model = _model(O.make_state_dict(0, num_classes=16))
        crit = dsk.GE2ELoss(10.0, -5.0, "contrast").cuda()
        opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-2, lr_decay=1e-4)
        x, labels = _dp_batch(world)
        sl = slice(rank * N_LOCAL, (rank + 1) * N_LOCAL)
        seen = {}
        h = model.register_forward_hook(lambda mod, inp, o: seen.__setitem__("emb", o.detach().clone()))
        res = dsk.ge2e_step(model, opt, x[sl].cuda(), labels[sl], loss=crit)
        h.remove()
        torch.cuda.synchronize()
        out[rank] = dict(loss=res["loss"].cpu(), valid=res["valid"], emb=seen["emb"].cpu(),
                         params=[p.detach().cpu().clone() for p in list(model.parameters()) + list(crit.parameters())])
    finally:
        dist.destroy_process_group()


def test_data_parallel_on_nccl(cuda_dev):
    world = 2
    visible = torch.cuda.device_count()
    if visible < world:
        pytest.skip(f"needs {world} GPUs, {visible} visible")
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_nccl_worker, args=(world, port, out), nprocs=world, join=True)
    res = [out[r] for r in range(world)]
    x, labels = _dp_batch(world)
    crit = dsk.GE2ELoss(10.0, -5.0, "contrast").cuda()
    # each rank's loss is the op on its own shard
    for r in range(world):
        sl = slice(r * N_LOCAL, (r + 1) * N_LOCAL)
        assert torch.equal(res[r]["loss"].cuda(), crit(res[r]["emb"].cuda(), labels[sl]).detach())
    # parameters: a one-device emulation of the V_r-weighted mean of the ranks' gradients
    model = _model(O.make_state_dict(0, num_classes=16))
    params = list(model.parameters()) + list(crit.parameters())
    grads, Vs = [], []
    for r in range(world):
        sl = slice(r * N_LOCAL, (r + 1) * N_LOCAL)
        for p in params:
            p.grad = None
        crit(model(x[sl].cuda()), labels[sl]).backward()
        grads.append([p.grad.double().clone() for p in params])
        Vs.append(ge2e_batch(labels[sl])[3])
    assert [r["valid"] for r in res] == Vs and Vs[0] != Vs[1]
    opt = torch.optim.Adagrad(params, lr=1e-2, lr_decay=1e-4)
    for i, p in enumerate(params):
        p.grad = (sum(V * g[i] for V, g in zip(Vs, grads)) / sum(Vs)).float()
    opt.step()
    worst = 0.0
    for a, b in zip(res[0]["params"], params):
        b = b.detach().cpu()
        worst = max(worst, float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)))
    print(f"\nR={world}: parameters vs the one-device V_r-weighted emulation: worst rel-L2 {worst:.3e}")
    assert worst <= 1e-6
