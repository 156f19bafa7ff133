"""Batch-hard triplet loss on the GPU: selection and loss bit-exact against the C oracle on both distance paths,
gradients against an fp64 restatement with the engine's selection pinned, deterministic backward, the training step
end to end and the data-parallel weighting by valid-anchor counts."""
import zlib

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as EN
from oracle import batch_hard_oracle as BH
from oracle import rescnn_oracle as O

pytestmark = pytest.mark.gpu


def _norm10(x):
    return 10.0 * x / x.norm(dim=1, keepdim=True)


def _case(name):
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    if name == "1024x512_64x16":
        return _norm10(torch.randn(1024, 512, generator=g)), (torch.arange(1024) // 16).long()
    if name == "130_uneven_singletons":
        sizes = [1, 7, 2, 1, 30, 5, 1, 40, 3, 1, 39]          # 4 singleton speakers: invalid anchors
        return _norm10(torch.randn(130, 512, generator=g)), torch.repeat_interleave(torch.arange(11), torch.tensor(sizes))
    if name == "2048_rows":
        return _norm10(torch.randn(2048, 512, generator=g)), (torch.arange(2048) % 128).long()
    if name == "D96_exact_path":
        return _norm10(torch.randn(200, 96, generator=g)), (torch.arange(200) % 25).long()
    if name == "near_duplicates":                               # gaps below the fp16 Gram error: exact fallback
        base = torch.randn(40, 512, generator=g)
        E = base.repeat_interleave(5, dim=0) + 1e-4 * torch.randn(200, 512, generator=g)
        return _norm10(E), (torch.arange(200) % 3).long()
    if name == "duplicated_rows":                               # exact ties on both sides
        base = _norm10(torch.randn(64, 512, generator=g))
        return torch.cat([base, base, base]), (torch.arange(192) % 48).long()
    raise KeyError(name)


CASES = ["1024x512_64x16", "130_uneven_singletons", "2048_rows", "D96_exact_path", "near_duplicates", "duplicated_rows"]


def _mine(E, labels, margin, exact=False):
    _, loss, pos, neg, d_ap, d_an, valid = EN.batch_hard_mine(E.cuda(), labels.cuda(), margin, exact)
    return [t.cpu().numpy() for t in (loss, pos, neg, d_ap, d_an, valid)]


@pytest.mark.parametrize("name", CASES)
def test_selection_and_loss_bit_exact_vs_oracle(cuda_dev, name):
    E, labels = _case(name)
    margin = 0.3
    loss, pos, neg, d_ap, d_an, valid = _mine(E, labels, margin)
    oloss, opos, oneg, od_ap, od_an, ovalid = BH.batch_hard_triplet(E.numpy(), labels.numpy(), margin)
    assert np.array_equal(valid, ovalid)
    assert np.array_equal(pos, opos) and np.array_equal(neg, oneg)
    assert np.array_equal(d_ap, od_ap) and np.array_equal(d_an, od_an)
    assert loss[0] == oloss or abs(loss[0] - oloss) <= 1e-6 * abs(oloss)
    # the tensor-core Gram path (default) and the exact CUDA-core path return the same bits
    for a, b in zip(_mine(E, labels, margin, exact=True), (loss, pos, neg, d_ap, d_an, valid)):
        assert np.array_equal(a, b)
    if name == "duplicated_rows":            # rows r, r+64, r+128 are one vector under three labels: the lower index
        assert (neg[:64] == np.arange(64) + 64).all()
    if name == "130_uneven_singletons":
        assert valid.sum() == 126


def test_bad_arguments_are_rejected(cuda_dev):
    crit = dsk.BatchHardTripletLoss(0.2)
    with pytest.raises(RuntimeError):
        crit.mine(torch.zeros(1, 64, device="cuda"), torch.zeros(1, dtype=torch.long))       # N < 2
    with pytest.raises(RuntimeError):                                                       # N > DSK_BATCH_HARD_MAX_N
        crit.mine(torch.zeros(16385, 8, device="cuda"), torch.arange(16385) % 2)


def _grad_vs_fp64(E, labels, margin, exact=False):
    Ed = E.cuda().requires_grad_(True)
    crit = dsk.BatchHardTripletLoss(margin, exact)
    loss = crit.forward(Ed, labels)
    assert loss.dim() == 0
    loss.backward()
    pos, neg, d_ap, d_an, valid = crit.mine(Ed, labels)
    E64 = E.double().requires_grad_(True)
    ref = BH.batch_hard_loss(E64, pos.cpu(), neg.cpu(), valid.cpu(), margin)
    ref.backward()
    g, r = Ed.grad.cpu().double(), E64.grad
    err, den = (g - r).norm(dim=1), r.norm(dim=1)
    assert bool((err <= 1e-5 * torch.maximum(den, 1e-3 * den.max())).all()), float((err / den.clamp_min(1e-30)).max())
    return loss, Ed.grad, (pos, neg, d_ap, d_an, valid)


@pytest.mark.parametrize("name", ["1024x512_64x16", "130_uneven_singletons", "D96_exact_path", "duplicated_rows"])
def test_gradient_vs_fp64_with_pinned_selection(cuda_dev, name):
    E, labels = _case(name)
    loss, g, _ = _grad_vs_fp64(E, labels, 0.3)
    assert loss.item() > 0 and g.abs().sum().item() > 0


def test_all_hinges_zero_and_no_valid_anchor(cuda_dev):
    g = torch.Generator().manual_seed(4)
    centers = _norm10(torch.randn(8, 512, generator=g))
    E = centers.repeat_interleave(4, dim=0) + 0.01 * torch.randn(32, 512, generator=g)
    labels = torch.arange(32) // 4
    loss, grad, _ = _grad_vs_fp64(E, labels, 0.1)                        # tight clusters: every hinge < 0
    assert loss.item() == 0.0 and not grad.any()
    for lab in (torch.zeros(32, dtype=torch.long), torch.arange(32)):   # one speaker / no speaker twice: V = 0
        Ed = E.cuda().requires_grad_(True)
        loss = dsk.BatchHardTripletLoss(0.1).forward(Ed, lab)
        loss.backward()
        assert loss.item() == 0.0 and not Ed.grad.any() and bool(torch.isfinite(Ed.grad).all())


def _hub_case():
    """Every anchor's nearest negative is one row: speakers sit on orthogonal directions at radius 10, the hub near the
    origin has a label of its own (a singleton, so not an anchor itself)."""
    g = torch.Generator().manual_seed(11)
    dirs = torch.eye(512)[:16] * 10.0
    E = dirs.repeat_interleave(8, dim=0) + 0.02 * torch.randn(128, 512, generator=g)
    E = torch.cat([E, 0.01 * torch.randn(1, 512, generator=g)])
    labels = torch.cat([torch.arange(128) // 8, torch.tensor([99])])
    return E, labels


def test_shared_negative_and_deterministic_backward(cuda_dev):
    E, labels = _hub_case()
    margin = 12.0                                               # d_ap ~ 0.6, d_an ~ 10: every hinge passes
    loss, grad, (pos, neg, d_ap, d_an, valid) = _grad_vs_fp64(E, labels, margin)
    assert bool((neg[:128] == 128).all()) and not bool(valid[128]) and grad[128].abs().sum().item() > 0
    oloss, opos, oneg, *_ = BH.batch_hard_triplet(E.numpy(), labels.numpy(), margin)
    assert np.array_equal(neg.cpu().numpy(), oneg) and np.array_equal(pos.cpu().numpy(), opos)
    Ec = E.cuda()
    one = torch.ones((), device="cuda")
    runs = [EN.batch_hard_backward(Ec, pos, neg, d_ap, d_an, valid, margin, one) for _ in range(2)]
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], grad)
    for name in ("1024x512_64x16", "duplicated_rows"):
        E2, lab2 = _case(name)
        _, _, *sel = EN.batch_hard_mine(E2.cuda(), lab2.cuda(), 0.3)
        a = EN.batch_hard_backward(E2.cuda(), *sel, 0.3, one)
        b = EN.batch_hard_backward(E2.cuda(), *sel, 0.3, one)
        assert torch.equal(a, b)


@pytest.mark.parametrize("P,K,T", [(16, 4, 32), (96, 4, 160)])
def test_batch_hard_step_end_to_end(cuda_dev, P, K, T):
    N, margin = P * K, 0.5
    sd = O.make_state_dict(0, num_classes=16)
    model = dsk.DeepSpeakerModel(512, 16).cuda().train()
    model.load_state_dict(sd)
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-3, lr_decay=1e-4)
    x = O.make_input(N, T, seed=P, scale=3.0)
    labels = torch.arange(N) // K                                          # CPU labels, as a loader yields them
    seen = {}

    def hook(mod, inp, out):
        seen["emb"] = out.detach().clone()
        out.register_hook(lambda gr: seen.__setitem__("grad", gr.detach().clone()))

    h = model.register_forward_hook(hook)
    out = dsk.batch_hard_step(model, opt, x.cuda(), labels, margin=margin)
    h.remove()
    assert out["valid"] == N and out["loss"].dim() == 0 and out["loss"].is_cuda
    # the gradient entering the network's backward is the op's gE
    Ec, loss, *sel = EN.batch_hard_mine(seen["emb"], labels, margin)
    gE = EN.batch_hard_backward(Ec, *sel, margin, torch.ones((), device="cuda"))
    assert torch.equal(seen["grad"], gE) and torch.equal(loss.reshape(()), out["loss"])
    # against the oracle's fp32 train forward + batch-hard loss (the loss is continuous in E)
    with torch.no_grad():
        ref_emb = O.forward(sd, x, train=True)
    oloss, opos, oneg, *_ = BH.batch_hard_triplet(ref_emb.numpy(), labels.numpy(), margin)
    got = out["loss"].item()
    assert abs(got - oloss) <= 1e-3 * abs(oloss), (got, oloss)
    pos, neg = sel[0].cpu().numpy(), sel[1].cpu().numpy()
    print(f"\nN={N} T={T}: loss {got:.6f} (oracle {oloss:.6f}); index agreement with the oracle forward: "
          f"positives {np.mean(pos == opos):.4f}, negatives {np.mean(neg == oneg):.4f}")


def test_data_parallel_weighting_by_valid_anchors(cuda_dev):
    """Two shards mined locally; sum_r V_r gE_r / sum_r V_r is the gradient of the mean over the union of valid
    anchors (what batch_hard_step's weighted allreduce computes across ranks)."""
    g = torch.Generator().manual_seed(21)
    E = _norm10(torch.randn(96, 512, generator=g))
    labels = torch.cat([torch.arange(64) // 4, 16 + torch.arange(32) // 2])   # different group sizes per shard
    labels[63] = 40                                                             # a singleton in shard 0
    margin, shards, grads, sels, Vs = 0.5, [(0, 64), (64, 96)], [], [], []
    for lo, hi in shards:
        Es = E[lo:hi].cuda().requires_grad_(True)
        crit = dsk.BatchHardTripletLoss(margin)
        crit.forward(Es, labels[lo:hi]).backward()
        grads.append(Es.grad.cpu().double())
        sels.append(crit.mine(Es, labels[lo:hi]))
        Vs.append(dsk.model.batch_hard_valid_count(labels[lo:hi]))
    assert Vs == [63, 32]
    combined = torch.cat([v * gr for v, gr in zip(Vs, grads)]) / sum(Vs)
    pos = torch.cat([s[0].cpu() + lo for s, (lo, _) in zip(sels, shards)])
    neg = torch.cat([s[1].cpu() + lo for s, (lo, _) in zip(sels, shards)])
    valid = torch.cat([s[4].cpu() for s in sels])
    E64 = E.double().requires_grad_(True)
    BH.batch_hard_loss(E64, pos, neg, valid, margin).backward()
    err, den = (combined - E64.grad).norm(dim=1), E64.grad.norm(dim=1)
    assert bool((err <= 1e-5 * torch.maximum(den, 1e-3 * den.max())).all())
