"""The supervised-contrastive loss on the GPU: cosines, lse, row losses and the loss against fp64 from the fp32 inputs,
the backward against the explicit fp64 backward with the engine's cosines pinned, the hard cases, NaN containment,
determinism and plan isolation from the other cosine ops, bf16 and relabelling invariance, argument rejection,
``supcon_step`` end to end on augmented views and, with two GPUs, data parallelism on NCCL."""
import ctypes
import gc
import os
import socket
import zlib

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as FR
from deepspeaker_pytorch_b200.model import ge2e_batch, supcon_valid_count
from oracle import rescnn_oracle as O
from oracle import supcon_oracle as S

pytestmark = pytest.mark.gpu

TAUS = (0.05, 0.1, 0.5, 1.0)


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _embeddings(labels, D, norms, seed):
    """Rows clustered by label (a shared direction plus noise, so positives are close), norm 10 or spread over four
    decades of norm."""
    g = torch.Generator().manual_seed(seed)
    _, col = torch.unique(labels, return_inverse=True)
    E = 0.6 * torch.randn(labels.numel(), D, generator=g) + torch.randn(int(col.max()) + 1, D, generator=g)[col]
    if norms == "norm10":
        return 10.0 * E / E.norm(dim=1, keepdim=True)
    return E * torch.exp(torch.empty(E.shape[0], 1).uniform_(-4.6, 4.6, generator=g))


def _ragged(n_groups, seed):
    g = np.random.default_rng(seed)
    counts = g.integers(1, 18, n_groups)
    lab = np.repeat(np.arange(n_groups) * 7 - 300, counts)
    return torch.from_numpy(lab[g.permutation(lab.size)])


CASES = {   # name: (labels, D)
    "2x64": (lambda: torch.tensor([4, 4]), 64),
    "2x256views_512": (lambda: torch.arange(256).repeat(2), 512),
    "ragged1000x192": (lambda: _ragged(112, 3), 192),
    "4096x512": (lambda: torch.arange(2048).repeat(2), 512),
    "16384x256": (lambda: torch.arange(16384) // 8, 256),
}


def _fwd(E, labels, tau):
    V = supcon_valid_count(labels)
    Ec, lab, loss, cos, lse = EN.supcon(E.cuda(), labels, V, tau)
    return Ec, lab, V, loss.reshape(()), cos, lse


def _bwd(Ec, lab, V, tau, cos, lse, g=1.0):
    return EN.supcon_backward(Ec, lab, V, tau, cos, lse, torch.full((), float(g), device="cuda"))


def _row_rel(got, ref):
    """Per-row relative L2 error; a row below 1e-3 of the largest row's gradient is measured against that floor (as in
    the AAM-softmax and GE2E tests)."""
    err, den = (got.double() - ref.to(got.device)).norm(dim=1), ref.to(got.device).norm(dim=1)
    if float(den.max()) == 0.0:          # a zero gradient (N = 2, one label: each row's only other row is its positive)
        return float(err.max())
    return float((err / torch.maximum(den, 1e-3 * den.max())).max())


def _check(E, labels, tau, report=True):
    """The forward gates against fp64 from the fp32 inputs and the backward gate with the engine's cos pinned; returns
    the engine's outputs and the measured errors."""
    Ec, lab, V, loss, cos, lse = _fwd(E, labels, tau)
    gE = _bwd(Ec, lab, V, tau, cos, lse)
    Ed = Ec.double()
    oloss, ref_cos, ref_lse, ref_rows = S.forward(Ed, labels, tau)
    off = ~torch.eye(E.shape[0], dtype=torch.bool, device="cuda")
    eps = float((cos.double() - ref_cos).abs()[off].max())
    assert eps <= 1e-6, eps
    bound = lambda x: 2 * eps / tau + 1e-6 * x.abs().clamp_min(1.0)                     # noqa: E731
    # the engine's row losses reach the caller only through the loss; their lse part is checked directly and the rest
    # (the positives' mean of cos / tau) at the engine's cosines
    _, _, _, rows = S.forward(Ed, labels, tau, cos=cos.double())
    d_lse = (lse.double() - ref_lse).abs()
    assert bool((d_lse <= bound(ref_lse)).all()), float((d_lse - bound(ref_lse)).max())
    assert bool(((rows - ref_rows).abs() <= bound(ref_rows)).all())
    assert abs(loss.item() - float(oloss)) <= float(bound(oloss)), (loss.item(), float(oloss), eps)
    assert bool(torch.isfinite(gE).all())
    eg = _row_rel(gE, S.backward(Ed, labels, tau, cos=cos.double()))
    assert eg <= 1e-5, eg
    if report:
        efull = _row_rel(gE, S.backward(Ed, labels, tau))
        print(f"\nN={E.shape[0]} D={E.shape[1]} tau={tau}: max |dcos| {eps:.2e}, |dloss| "
              f"{abs(loss.item() - float(oloss)):.2e}, max |dlse| {float(d_lse.max()):.2e}, per-row rel-L2 gE "
              f"{eg:.2e} (fully fp64 {efull:.2e})")
    return Ec, lab, V, loss, cos, lse, gE


@pytest.mark.parametrize("norms", ["norm10", "decades"])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_and_backward_vs_fp64(cuda_dev, name, norms):
    make, D = CASES[name]
    labels = make()
    E = _embeddings(labels, D, norms, zlib.crc32(f"{name}{norms}".encode()))
    for tau in TAUS:
        _check(E, labels, tau)


def _singletons(labels, n, start=10 ** 6):
    return torch.cat([labels, torch.arange(start, start + n)])


def test_hard_cases(cuda_dev):
    D = 128
    g = torch.Generator().manual_seed(17)
    labels = torch.arange(48) // 3
    E = _embeddings(labels, D, "norm10", 5)
    # a near-duplicate positive pair (cos -> 1) at tau = 0.05
    E[1] = E[0] + 1e-5 * torch.randn(D, generator=g)
    *_, cos, _, _ = _check(E, labels, 0.05, report=False)
    assert cos[0, 1].item() > 0.999999
    # one label for the whole batch, and tau = 0.01 (logits reach 100)
    _check(E, torch.zeros(48, dtype=torch.long), 0.1, report=False)
    _, _, _, loss, cos, lse, _ = _check(E, labels, 0.01, report=False)
    assert lse.max().item() > 90.0 and torch.isfinite(loss)
    # singletons: no loss term, a gradient only through the other rows' terms
    lab_s = _singletons(labels, 5)
    E_s = torch.cat([E, torch.randn(5, D, generator=g)])
    _, _, V, _, _, _, gE = _check(E_s, lab_s, 0.1, report=False)
    assert V == 48 and bool((gE[48:].norm(dim=1) > 0).all())
    # a zero row (its cosines are 0; its gradient is divided by the 1e-12 floor, as F.normalize's)
    E_z = E.clone()
    E_z[7] = 0.0
    _, _, _, _, cos, _, gE = _check(E_z, labels, 0.1, report=False)
    assert not bool(cos[7].any()) and bool(torch.isfinite(gE).all())
    # all rows identical: every cosine ~1, the gradient's true value is 0 after the normalisation Jacobian
    E_i = E[:1].repeat(48, 1)
    Ec, lab, V, loss, cos, lse = _fwd(E_i, labels, 0.1)
    gE = _bwd(Ec, lab, V, 0.1, cos, lse)
    oloss, ref_cos, ref_lse, _ = S.forward(Ec.double(), labels, 0.1)
    eps = float((cos.double() - ref_cos).abs().max())
    assert eps <= 1e-6 and abs(loss.item() - float(oloss)) <= 2 * eps / 0.1 + 1e-6 * abs(float(oloss))
    dC = S.score_grads(cos.double(), labels, 0.1) / 0.1
    scale = (dC.abs().sum(1) + dC.abs().sum(0)) / Ec.double().norm(dim=1)       # |g^_i| / ||e_i|| bound
    assert bool((gE.double().norm(dim=1) <= 1e-5 * scale).all())


def test_nan_row_makes_the_loss_nan(cuda_dev):
    labels = torch.arange(32).repeat(2)
    E = _embeddings(labels, 64, "norm10", 1).cuda()
    E[5, 3] = float("nan")
    Ec, lab, V, loss, cos, lse = _fwd(E, labels, 0.1)               # returns DSK_OK (no exception)
    assert torch.isnan(loss) and bool(torch.isnan(lse).all())
    assert bool(torch.isnan(cos[5]).all()) and bool(torch.isnan(cos[:, 5]).all())
    E[5, 3] = float("inf")
    assert torch.isnan(_fwd(E, labels, 0.1)[3])


def _all(E, labels, tau):
    Ec, lab, V, loss, cos, lse = _fwd(E, labels, tau)
    return loss, cos, lse, _bwd(Ec, lab, V, tau, cos, lse)


def test_deterministic_and_plans_do_not_interfere(cuda_dev):
    """Two runs give the same bits; AAM-softmax, GE2E, cohort statistics and batch-hard calls between the forward and
    the backward leave every output bit-identical, theirs included."""
    labels = _ragged(112, 9)
    E = _embeddings(labels, 192, "norm10", 9)
    E1 = _embeddings(torch.arange(384) // 6, 512, "norm10", 1).cuda()
    l1 = torch.arange(384) // 6
    W = torch.randn(300, 512, generator=torch.Generator().manual_seed(3)).cuda()
    ya = torch.randint(0, 300, (384,), generator=torch.Generator().manual_seed(4))
    one = torch.ones((), device="cuda")

    def aam():
        Ec, Wc, lab, loss, cos, lse = EN.aam_softmax(E1, W, ya, 0.2, 30.0)
        return (loss, cos, lse) + tuple(EN.aam_softmax_backward(Ec, Wc, lab, cos, lse, 0.2, 30.0, one))

    def ge2e():
        order, offsets, col, V = ge2e_batch(l1)
        csr = tuple(torch.from_numpy(a).cuda() for a in (order, offsets, col))
        w, b = torch.tensor([10.0], device="cuda"), torch.tensor([-5.0], device="cuda")
        Ec, loss, cos, rec = EN.ge2e(E1, csr, V, w, b, "softmax")
        return (loss, cos, rec) + EN.ge2e_backward(Ec, csr, V, w, b, "softmax", cos, rec, one)

    def batch_hard():
        Ec, loss, pos, neg, d_ap, d_an, valid = EN.batch_hard_mine(E1, l1, 0.5)
        return (loss, pos, neg, d_ap, d_an, EN.batch_hard_backward(Ec, pos, neg, d_ap, d_an, valid, 0.5, one))

    cohort = lambda: EN.cohort_stats(E1, W, 50)                                                  # noqa: E731
    iso = _all(E, labels, 0.1)
    assert all(torch.equal(a, b) for a, b in zip(iso, _all(E, labels, 0.1)))
    others = [aam(), ge2e(), cohort(), batch_hard()]
    Ec, lab, V, loss, cos, lse = _fwd(E, labels, 0.1)
    mixed_others = [aam(), ge2e(), cohort(), batch_hard()]
    mixed = (loss, cos, lse, _bwd(Ec, lab, V, 0.1, cos, lse))
    for a, b in zip(iso, mixed):
        assert torch.equal(a, b)
    for a, b in zip(others, mixed_others):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_bf16_handle_and_relabelling_give_the_same_bits(cuda_dev):
    labels = torch.arange(64).repeat(3)
    E = _embeddings(labels, 256, "norm10", 2).cuda()
    ref = _all(E, labels, 0.1)
    h = ctypes.c_void_p()
    L.check(L.load().dsk_create(ctypes.byref(h), 0, L.DSK_BF16), "dsk_create")
    try:
        N, D = E.shape
        lab = labels.cuda()
        V = supcon_valid_count(labels)
        loss, lse = torch.empty(1, device="cuda"), torch.empty(N, device="cuda")
        cos, gE = torch.empty(N, N, device="cuda"), torch.empty_like(E)
        one = torch.ones(1, device="cuda")
        s = L.cur_stream()
        L.check(L.load().dsk_supcon(h, E.data_ptr(), lab.data_ptr(), N, D, V, 0.1, loss.data_ptr(), cos.data_ptr(),
                                    lse.data_ptr(), s), "dsk_supcon")
        L.check(L.load().dsk_supcon_bwd(h, E.data_ptr(), lab.data_ptr(), cos.data_ptr(), lse.data_ptr(), N, D, V, 0.1,
                                        one.data_ptr(), gE.data_ptr(), s), "dsk_supcon_bwd")
        for a, b in zip(ref, (loss.reshape(()), cos, lse, gE)):
            assert torch.equal(a, b)
    finally:
        torch.cuda.synchronize()
        L.load().dsk_destroy(h)
    relabelled = labels * -(2 ** 40) + 12345
    for a, b in zip(ref, _all(E, relabelled, 0.1)):
        assert torch.equal(a, b)


def test_bad_arguments_are_rejected_and_outputs_untouched(cuda_dev):
    lib = L.load()
    h = EN._allpairs_handle(torch.device("cuda:0"))
    s = L.cur_stream()

    def call(N, D, V, tau):
        E = torch.randn(N, D, device="cuda")
        lab = torch.arange(N, device="cuda") // 2
        loss, lse = torch.full((1,), 7.0, device="cuda"), torch.full((N,), 7.0, device="cuda")
        cos, gE = torch.full((N, N), 7.0, device="cuda"), torch.full((N, D), 7.0, device="cuda")
        one = torch.ones(1, device="cuda")
        rf = lib.dsk_supcon(h, E.data_ptr(), lab.data_ptr(), N, D, V, tau, loss.data_ptr(), cos.data_ptr(),
                            lse.data_ptr(), s)
        rb = lib.dsk_supcon_bwd(h, E.data_ptr(), lab.data_ptr(), cos.data_ptr(), lse.data_ptr(), N, D, V, tau,
                                one.data_ptr(), gE.data_ptr(), s)
        torch.cuda.synchronize()
        untouched = all(bool((t == 7.0).all()) for t in (loss, lse, cos, gE))
        del cos
        torch.cuda.empty_cache()
        return rf, rb, untouched

    for N, D, V, tau in [(1, 64, 1, 0.1), (L.DSK_SUPCON_MAX_N + 1, 64, 8, 0.1), (8, 96, 8, 0.1), (8, 64, 8, 0.0),
                         (8, 64, 8, -1.0), (8, 64, 8, float("nan")), (8, 64, 8, float("inf")), (8, 64, 0, 0.1)]:
        rf, rb, untouched = call(N, D, V, tau)
        assert rf == L.DSK_ERR_INVALID and rb == L.DSK_ERR_INVALID and untouched, (N, D, V, tau)
    crit = dsk.SupConLoss(0.1)
    E = torch.randn(8, 64, device="cuda")
    with pytest.raises(ValueError):
        crit(E, torch.arange(8))                                      # V = 0
    with pytest.raises(RuntimeError):
        crit(E, torch.arange(7) // 2)                                 # label count
    with pytest.raises(RuntimeError):
        crit(torch.randn(8, 96, device="cuda"), torch.arange(8) // 2)  # D % 64 != 0, from the C ABI


# ---- supcon_step on two augmented views of each utterance ----------------------------------------------------------
T_STEP = 32


def _banks():
    g = np.random.default_rng(40)
    t = np.arange(200000) / 16000.0
    speech = [np.round((0.3 * np.sin(2 * np.pi * (150 + 40 * k) * t[:n]) + g.normal(0, 0.05, n)).clip(-1, 0.99)
                       * 32768).astype(np.int16) for k, n in enumerate(g.integers(8000, 48000, 24))]
    noise = [np.round(g.normal(0, 0.1, n).clip(-1, 0.99) * 32768).astype(np.int16) for n in g.integers(4000, 40000, 6)]
    rirs = [g.normal(size=lh) * np.exp(-np.arange(lh) / 400.0) for lh in (1, 800, 3000)]
    return FR.WaveBank.from_waveforms(speech), FR.WaveBank.from_waveforms(noise), FR.RirBank.from_arrays(rirs)


def _views(sb, nb, rb, B, seed):
    """Two independently augmented views (RIR, noise, speed) of each of B utterances, labels arange(B).repeat(2)."""
    g = np.random.default_rng(seed)
    u = torch.from_numpy(g.choice(sb.num_utterances, B, replace=False))
    utt = torch.cat([u, u])
    Ls = FR.segment_samples(T_STEP)
    plan = FR.augment_plan(2 * B, Ls, g, rb, 0.7, nb, [(range(nb.num_utterances), (0.0, 15.0), (1, 2), 1.0)], 0.7,
                           speeds=(0.9, 1.0, 1.1))
    start = sb.random_starts(utt, Ls, g, plan)
    x = sb.augmented_crops(utt, start, T_STEP, plan, rb, nb)
    return x, torch.arange(B).repeat(2)


def _model(sd):
    model = dsk.DeepSpeakerModel(512, 16).cuda().train()
    model.load_state_dict(sd)
    return model


@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
def test_supcon_step_end_to_end(cuda_dev, opt_kind):
    sb, nb, rb = _banks()
    B, tau = 12, 0.1
    x, labels = _views(sb, nb, rb, B, 7)
    assert bool(torch.isfinite(x).all()) and not torch.equal(x[:B], x[B:])
    sd = O.make_state_dict(0, num_classes=16)

    def run():
        model = _model(sd)
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-2, lr_decay=1e-4) if opt_kind == "fused" else \
            torch.optim.Adagrad(model.parameters(), lr=1e-2, lr_decay=1e-4)
        seen = {}

        def hook(mod, inp, out):
            seen["emb"] = out.detach().clone()
            out.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

        h = model.register_forward_hook(hook)
        out = dsk.supcon_step(model, opt, x, labels, temperature=tau)
        h.remove()
        return model, out, seen

    model, out, seen = run()
    assert out["loss"].dim() == 0 and out["loss"].is_cuda and out["valid"] == 2 * B
    # the gradient entering the network's backward is the op's gE
    Ec, lab, V, loss, cos, lse = _fwd(seen["emb"], labels, tau)
    assert torch.equal(seen["grad"], _bwd(Ec, lab, V, tau, cos, lse)) and torch.equal(loss, out["loss"])
    # against the oracle's fp32 train-mode forward and the fp64 loss
    with torch.no_grad():
        ref_emb = O.forward(sd, x.cpu(), train=True)
    oloss = float(S.forward(ref_emb.double(), labels, tau)[0])
    assert abs(out["loss"].item() - oloss) <= 1e-3, (out["loss"].item(), oloss)
    # the same seeded step twice: the same bits
    model2, out2, _ = run()
    assert torch.equal(out["loss"], out2["loss"])
    for a, b in zip(model.parameters(), model2.parameters()):
        assert torch.equal(a, b)
    # a model with synchronised BatchNorm (one rank) runs the same step
    sync_model = _model(sd).sync_batchnorm()
    sopt = dsk.FusedAdagrad(sync_model.parameters(), lr=1e-2, lr_decay=1e-4)
    sout = dsk.supcon_step(sync_model, sopt, x, labels, temperature=tau)
    assert abs(sout["loss"].item() - out["loss"].item()) <= 1e-3
    print(f"\n{opt_kind}: loss {out['loss'].item():.6f} (oracle {oloss:.6f}, sync BN {sout['loss'].item():.6f})")


# ---- >= 2 GPUs, NCCL --------------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_LOCAL, T_DP = 32, 32


def _dp_batch(world):
    """Shards with unequal V_r: two views of 16 utterances per rank, rank 1's last view a singleton."""
    x = O.make_input(world * N_LOCAL, T_DP, seed=11, scale=3.0)
    labels = torch.cat([torch.arange(N_LOCAL // 2).repeat(2) + 100 * r for r in range(world)])
    labels[2 * N_LOCAL - 1] = 10 ** 6
    return x, labels


def _nccl_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        model = _model(O.make_state_dict(0, num_classes=16))
        opt = dsk.FusedAdagrad(model.parameters(), lr=1e-2, lr_decay=1e-4)
        x, labels = _dp_batch(world)
        sl = slice(rank * N_LOCAL, (rank + 1) * N_LOCAL)
        res = dsk.supcon_step(model, opt, x[sl].cuda(), labels[sl], temperature=0.1)
        torch.cuda.synchronize()
        out[rank] = dict(valid=res["valid"], params=[p.detach().cpu().clone() for p in model.parameters()])
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
    # parameters: a one-device emulation of the V_r-weighted mean of the ranks' gradients, per-shard BatchNorm
    model = _model(O.make_state_dict(0, num_classes=16))
    params = list(model.parameters())
    crit = dsk.SupConLoss(0.1)
    grads, Vs = [], []
    for r in range(world):
        sl = slice(r * N_LOCAL, (r + 1) * N_LOCAL)
        for p in params:
            p.grad = None
        crit(model(x[sl].cuda()), labels[sl]).backward()
        grads.append([p.grad.double().clone() for p in params])
        Vs.append(supcon_valid_count(labels[sl]))
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
