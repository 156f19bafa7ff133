"""AAM-softmax on the GPU: cosines and loss against fp64 from the fp32 inputs, the backward against the fp64 oracle with
the engine's own cosines pinned, the margin's branches, determinism, rows that do not depend on how the batch is split,
argument rejection and the training step end to end."""
import copy
import zlib

import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as EN
from oracle import aam_softmax_oracle as A
from oracle import rescnn_oracle as O

pytestmark = pytest.mark.gpu

SHAPES = [(384, 1211, 512), (1024, 5994, 512), (130, 1000, 192), (7, 3, 64)]


def _case(N, C, D, norms):
    g = torch.Generator().manual_seed(zlib.crc32(f"{N}x{C}x{D}{norms}".encode()))
    E = torch.randn(N, D, generator=g)
    if norms == "norm10":                      # as the model emits them
        E = 10.0 * E / E.norm(dim=1, keepdim=True)
    else:                                      # arbitrary norms over four decades
        E = E * torch.exp(torch.empty(N, 1).uniform_(-4.0, 5.0, generator=g))
    W = torch.randn(C, D, generator=g) * (1.0 / D ** 0.5)
    return E, W, torch.randint(0, C, (N,), generator=g)


def _fwd(E, W, labels, m, s):
    _, _, _, loss, cos, lse = EN.aam_softmax(E.cuda(), W.cuda(), labels.cuda(), m, s)
    return loss.reshape(()), cos, lse


def _bwd(E, W, labels, cos, lse, m, s, g=1.0):
    gl = torch.full((), float(g), device="cuda")
    return EN.aam_softmax_backward(E.cuda().contiguous(), W.cuda().contiguous(), labels.cuda(), cos, lse, m, s, gl)


def _row_rel(got, ref):
    """Per-row relative L2 error over rows with a nonzero reference gradient.  A row whose gradient is below 1e-3 of the
    largest row's is measured against that floor instead: rows on (or opposite) their class centre have a gradient of
    ~1e-13 of the others', the remainder of two opposite terms that fp32 cannot resolve."""
    err, den = (got.double().cpu() - ref).norm(dim=1), ref.norm(dim=1)
    nz = den > 0
    if not bool(nz.any()):
        return 0.0
    return float((err[nz] / torch.maximum(den[nz], 1e-3 * den.max())).max())


@pytest.mark.parametrize("norms", ["norm10", "arbitrary"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_forward_vs_fp64(cuda_dev, shape, norms):
    E, W, labels = _case(*shape, norms)
    ref_cos = None
    for m in (0.0, 0.2, 0.5):
        for s in (30.0, 64.0):
            loss, cos, lse = _fwd(E, W, labels, m, s)
            oloss, ref_cos, olse = A.forward(E, W, labels, m, s, cos=ref_cos)
            dcos = float((cos.double().cpu() - ref_cos).abs().max())
            dloss = abs(loss.item() - float(oloss))
            assert dcos <= 1e-6, (m, s, dcos)
            assert dloss <= 1e-5 * max(float(oloss), 1.0), (m, s, loss.item(), float(oloss))
    print(f"\n{shape} {norms}: max |dcos| {dcos:.2e}, |dloss| {dloss:.2e} (m 0.5, s 64)")


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_backward_vs_fp64_with_cos_pinned(cuda_dev, shape):
    E, W, labels = _case(*shape, "norm10")
    for m, s in ((0.0, 30.0), (0.2, 30.0), (0.5, 64.0)):
        loss, cos, lse = _fwd(E, W, labels, m, s)
        gE, gW = _bwd(E, W, labels, cos, lse, m, s)
        rE, rW = A.backward(E, W, labels, m, s, cos=cos.cpu())
        eE, eW = _row_rel(gE, rE), _row_rel(gW, rW)
        assert eE <= 1e-5 and eW <= 1e-5, (m, s, eE, eW)
        fE, fW = A.backward(E, W, labels, m, s)           # fully fp64, reported only
        print(f"\n{shape} m {m} s {s}: per-row rel-L2 with cos pinned gE {eE:.2e} gW {eW:.2e}; "
              f"end to end fp64 gE {_row_rel(gE, fE):.2e} gW {_row_rel(gW, fW):.2e}")


def _branch_case():
    """Rows past pi - m (cos - mm branch), a row equal to its class weight (sin = 0, cos = 1 exactly: a basis
    direction normalises without rounding), a row equal to the negated weight of its class, and a zero weight row."""
    N, C, D = 64, 100, 512
    E, W, labels = _case(N, C, D, "norm10")
    labels = labels.clone()
    wy = W[labels[:8]] / W[labels[:8]].norm(dim=1, keepdim=True)
    E[:8] = -10.0 * wy + 0.02 * torch.randn(8, D, generator=torch.Generator().manual_seed(5))
    u = torch.zeros(D)
    u[17] = 1.0
    W[40], labels[8], E[8] = 0.25 * u, 40, 10.0 * u               # on its class centre
    W[41], labels[9], E[9] = 0.25 * u, 41, -10.0 * u              # on the negated centre
    W[42], labels[10:12] = 0.0, 42                                 # a zero weight row, target of two rows
    return E, W, labels


@pytest.mark.parametrize("m,s", [(0.0, 30.0), (0.2, 30.0), (0.5, 64.0)])
def test_margin_branches(cuda_dev, m, s):
    E, W, labels = _branch_case()
    loss, cos, lse = _fwd(E, W, labels, m, s)
    oloss, ref_cos, _ = A.forward(E, W, labels, m, s)
    assert float((cos.double().cpu() - ref_cos).abs().max()) <= 1e-6
    assert abs(loss.item() - float(oloss)) <= 1e-5 * max(float(oloss), 1.0)
    c = cos.cpu()
    assert c[8, 40].item() == 1.0 and c[9, 41].item() == -1.0 and not bool(c[:, 42].any())
    if m > 0:
        assert bool((c[torch.arange(8), labels[:8]] < -torch.cos(torch.tensor(m))).all())
    gE, gW = _bwd(E, W, labels, cos, lse, m, s)
    assert bool(torch.isfinite(gE).all()) and bool(torch.isfinite(gW).all())
    rE, rW = A.backward(E, W, labels, m, s, cos=c)
    eE, eW = _row_rel(gE, rE), _row_rel(gW, rW)
    assert eE <= 1e-5 and eW <= 1e-5, (eE, eW)
    assert gW[42].abs().sum().item() > 0


def test_deterministic(cuda_dev):
    E, W, labels = _case(384, 1211, 512, "norm10")
    runs = []
    for _ in range(2):
        loss, cos, lse = _fwd(E, W, labels, 0.2, 30.0)
        gE, gW = _bwd(E, W, labels, cos, lse, 0.2, 30.0)
        runs.append((loss, cos, lse, gE, gW))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("split", [(192, 192), (96, 96, 96, 96), (1, 127, 256)], ids=["R2", "R4", "uneven"])
def test_rows_do_not_depend_on_the_split(cuda_dev, split):
    """Shards of one batch (as data-parallel ranks hold them): their cos rows, lse and gE rows are bit-identical to
    those rows of the whole batch when every shard's gradient is seeded with its row count (grad_loss / N = 1 on every
    shard); the shards' mean-loss weight gradients, weighted by n_r / N, sum to the whole batch's."""
    m, s = 0.2, 30.0
    E, W, labels = _case(384, 1211, 512, "norm10")
    N = E.shape[0]
    loss, cos, lse = _fwd(E, W, labels, m, s)
    gE, _ = _bwd(E, W, labels, cos, lse, m, s, g=N)
    _, gW = _bwd(E, W, labels, cos, lse, m, s, g=1.0)
    gW_sum, lo = torch.zeros_like(gW, dtype=torch.float64), 0
    for n in split:
        sl = slice(lo, lo + n)
        _, c_r, l_r = _fwd(E[sl], W, labels[sl], m, s)
        assert torch.equal(c_r, cos[sl]) and torch.equal(l_r, lse[sl])
        gE_r, _ = _bwd(E[sl], W, labels[sl], c_r, l_r, m, s, g=n)
        assert torch.equal(gE_r, gE[sl])
        _, gW_r = _bwd(E[sl], W, labels[sl], c_r, l_r, m, s, g=1.0)
        gW_sum += (n / N) * gW_r.double()
        lo += n
    rel = float((gW_sum - gW.double()).norm() / gW.double().norm())
    assert rel <= 1e-6, rel
    print(f"\nsplit {split}: sum_r (n_r/N) gW_r vs gW rel-L2 {rel:.2e}, bit-identical: {torch.equal(gW_sum.float(), gW)}")


def test_bad_arguments_are_rejected(cuda_dev):
    crit = lambda W: dsk.AAMSoftmaxLoss(W, 0.2, 30.0)  # noqa: E731
    E, W = torch.randn(8, 64, device="cuda"), torch.randn(10, 64, device="cuda")
    lab = torch.zeros(8, dtype=torch.long)
    cases = [
        (torch.randn(8, 96, device="cuda"), torch.randn(10, 96, device="cuda"), lab),   # D % 64 != 0
        (E, torch.randn(1, 64, device="cuda"), lab),                                    # C < 2
        (torch.randn(0, 64, device="cuda"), W, lab[:0]),                                # N = 0
        (E, torch.randn(10, 128, device="cuda"), lab),                                  # D mismatch
        (E, W, lab[:7]),                                                                # labels mismatch
        (E.cpu(), W.cpu(), lab),                                                        # CPU tensors
    ]
    for e, w, y in cases:
        with pytest.raises(RuntimeError):
            crit(w).forward(e, y)


@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
@pytest.mark.parametrize("N,T", [(64, 32), (384, 160)])
def test_aam_softmax_step_end_to_end(cuda_dev, N, T, opt_kind):
    C, m, s = 1211, 0.2, 30.0
    sd = O.make_state_dict(0, num_classes=C)
    model = dsk.DeepSpeakerModel(512, C).cuda().train()
    model.load_state_dict(sd)
    ref_model = copy.deepcopy(model)
    params = list(model.parameters())
    opt = dsk.FusedAdagrad(params, lr=1e-3, lr_decay=1e-4) if opt_kind == "fused" else \
        torch.optim.Adagrad(params, lr=1e-3, lr_decay=1e-4)
    x = O.make_input(N, T, seed=N, scale=3.0)
    labels = torch.randint(0, C, (N,), generator=torch.Generator().manual_seed(N))
    W0 = model.model.classifier.weight.detach().clone()
    b0 = model.model.classifier.bias.detach().clone()
    seen = {}

    def hook(mod, inp, out):
        seen["emb"] = out.detach().clone()
        out.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

    h = model.register_forward_hook(hook)
    out = dsk.aam_softmax_step(model, opt, x.cuda(), labels, margin=m, scale=s)
    h.remove()
    assert out["loss"].dim() == 0 and out["loss"].is_cuda
    # the gradient entering the network's backward is the op's gE
    Ec, Wc, lab, loss, cos, lse = EN.aam_softmax(seen["emb"], W0, labels, m, s)
    gE, _ = EN.aam_softmax_backward(Ec, Wc, lab, cos, lse, m, s, torch.ones((), device="cuda"))
    assert torch.equal(seen["grad"], gE) and torch.equal(loss.reshape(()), out["loss"])
    # against the oracle's fp32 train-mode forward and the fp64 loss
    with torch.no_grad():
        ref_emb = O.forward(sd, x, train=True)
    oloss, _, _ = A.forward(ref_emb, sd["model.classifier.weight"], labels, m, s)
    assert abs(out["loss"].item() - float(oloss)) <= 1e-3, (out["loss"].item(), float(oloss))
    assert not torch.equal(model.model.classifier.weight.detach(), W0)
    assert torch.equal(model.model.classifier.bias.detach(), b0)
    # running statistics: those of exactly one train-mode forward of the batch
    with torch.no_grad():
        ref_model(x.cuda())
    for (k, v), (_, r) in zip(model.state_dict().items(), ref_model.state_dict().items()):
        if "running" in k:
            assert torch.equal(v, r), k
    # a model with synchronised BatchNorm (one rank) runs the same step
    sync_model = dsk.DeepSpeakerModel(512, C).cuda().train()
    sync_model.load_state_dict(sd)
    sync_model.sync_batchnorm()
    sopt = dsk.FusedAdagrad(sync_model.parameters(), lr=1e-3, lr_decay=1e-4)
    sout = dsk.aam_softmax_step(sync_model, sopt, x.cuda(), labels, margin=m, scale=s)
    assert abs(sout["loss"].item() - out["loss"].item()) <= 1e-3
    print(f"\nN={N} T={T} {opt_kind}: loss {out['loss'].item():.6f} (oracle {float(oloss):.6f}, "
          f"sync BN {sout['loss'].item():.6f})")
