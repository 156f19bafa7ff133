"""PairwiseDistance / TripletMarginLoss / hard-triplet selection / all-pairs top-k: CUDA vs oracle + golden."""
import os

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import engine as E
from oracle import c_oracle as C
from tests.helpers import make_triplet_embeddings

pytestmark = pytest.mark.gpu


def test_distances_and_indices_bit_exact_vs_oracle(cuda_dev):
    for B, D, seed in ((64, 512, 5), (1, 512, 1), (37, 512, 2), (1000, 512, 3), (128, 256, 4), (5, 96, 6)):
        a, p, n = make_triplet_embeddings(B, D, seed)
        d_p = dsk.PairwiseDistance(2).forward(a.cuda(), p.cuda())
        d_n = dsk.PairwiseDistance(2).forward(a.cuda(), n.cuda())
        oloss, odp, odn = C.triplet_loss(a.numpy(), p.numpy(), n.numpy(), 0.1)
        assert np.array_equal(d_p.cpu().numpy(), odp) and np.array_equal(d_n.cpu().numpy(), odn)   # bit-exact
        idx, cnt = dsk.select_hard_triplets(d_p, d_n, 0.1)
        k = int(cnt.item())
        assert np.array_equal(idx[:k].cpu().numpy(), C.margin_select(odp, odn, 0.1))
        loss = dsk.TripletMarginLoss(0.1).forward(a.cuda(), p.cuda(), n.cuda())
        assert loss.dim() == 0 and abs(loss.item() - oloss) <= 1e-6 * max(1.0, abs(oloss))


def test_matches_reference_golden(cuda_dev, golden_dir):
    g = np.load(os.path.join(golden_dir, "triplet_loss.npz"))
    a, p, n = (t.cuda().requires_grad_(True) for t in make_triplet_embeddings())
    loss = dsk.TripletMarginLoss(0.1).forward(a, p, n)
    assert abs(loss.item() - float(g["loss"])) <= 1e-3 * float(g["loss"])
    loss.backward()
    for t, key in ((a, "ga"), (p, "gp"), (n, "gn")):
        ref = torch.from_numpy(g[key])
        assert ((t.grad.cpu() - ref).norm() / ref.norm()).item() < 1e-5
    d_p = dsk.PairwiseDistance(2).forward(a.detach(), p.detach())
    d_n = dsk.PairwiseDistance(2).forward(a.detach(), n.detach())
    assert np.allclose(d_p.cpu().numpy(), g["d_p"], rtol=1e-6) and np.allclose(d_n.cpu().numpy(), g["d_n"], rtol=1e-6)
    idx, cnt = dsk.select_hard_triplets(d_p, d_n, 0.1)
    assert np.array_equal(idx[: int(cnt.item())].cpu().numpy(), g["hard_idx"])
    # selected-subset loss, train_triplet.py:265-275, gathered on the device
    ga = E.gather_rows(a.detach(), idx, cnt)[: int(cnt.item())]
    gp = E.gather_rows(p.detach(), idx, cnt)[: int(cnt.item())]
    gn = E.gather_rows(n.detach(), idx, cnt)[: int(cnt.item())]
    sel = dsk.TripletMarginLoss(0.1).forward(ga, gp, gn)
    assert abs(sel.item() - float(g["selected_loss"])) <= 1e-5


def test_pairwise_distance_autograd(cuda_dev):
    a, p, _ = make_triplet_embeddings(9, 512, 8)
    x1, x2 = a.cuda().requires_grad_(True), p.cuda().requires_grad_(True)
    d = dsk.PairwiseDistance(2).forward(x1, x2)
    w = torch.arange(1, 10, device="cuda", dtype=torch.float32)
    (d * w).sum().backward()
    r1, r2 = a.clone().requires_grad_(True), p.clone().requires_grad_(True)
    from oracle import rescnn_oracle as O
    (O.pairwise_distance(r1, r2) * w.cpu()).sum().backward()
    assert torch.allclose(x1.grad.cpu(), r1.grad, rtol=1e-5, atol=1e-7)
    assert torch.allclose(x2.grad.cpu(), r2.grad, rtol=1e-5, atol=1e-7)


def test_selection_edge_cases(cuda_dev):
    d_p = torch.ones(70, device="cuda")
    idx, cnt = dsk.select_hard_triplets(d_p, d_p + 5.0, 0.1)
    assert int(cnt.item()) == 0                                   # empty: the reference skips the batch (:263-264)
    idx, cnt = dsk.select_hard_triplets(d_p, d_p, 0.1)
    assert int(cnt.item()) == 70 and torch.equal(idx.cpu(), torch.arange(70))
    d_n = d_p + torch.tensor(0.1, device="cuda")                  # exactly at the margin: strict '<' in fp32
    idx, cnt = dsk.select_hard_triplets(d_p, d_n, 0.1)
    exp = np.where((d_n.cpu().numpy() - d_p.cpu().numpy()) < np.float32(0.1))[0]
    assert np.array_equal(idx[: int(cnt.item())].cpu().numpy(), exp)
    big = torch.rand(5000, device="cuda")
    idx, cnt = dsk.select_hard_triplets(big, big.flip(0), 0.0)
    exp = np.where((big.flip(0).cpu().numpy() - big.cpu().numpy()) < np.float32(0.0))[0]
    assert np.array_equal(idx[: int(cnt.item())].cpu().numpy(), exp)


@pytest.mark.parametrize("N,k,groups", [(96, 5, 16), (1024, 8, 64), (130, 3, 7)])
def test_allpairs_topk_bit_exact_vs_oracle(cuda_dev, N, k, groups):
    """BASELINE config 4 (N=1024, k=8, 64 speakers x 16 utterances)."""
    g = torch.Generator().manual_seed(3)
    E_ = torch.randn(N, 512, generator=g)
    E_ = 10.0 * E_ / E_.norm(dim=1, keepdim=True)
    labels = (torch.arange(N) % groups).long()
    idx, val = dsk.allpairs_topk(E_.cuda(), labels.cuda(), k)                             # wgmma Gram + exact refinement
    oidx, oval = C.allpairs_topk(E_.numpy(), labels.numpy(), k)
    assert np.array_equal(idx.cpu().numpy(), oidx)
    assert np.array_equal(val.cpu().numpy(), oval)
    idx2, val2 = dsk.allpairs_topk(E_.cuda(), labels.cuda(), k, exact_cuda_cores=True)    # all-fp32 CUDA-core path
    assert torch.equal(idx2, idx) and torch.equal(val2, val)
    # properties: never the same speaker, ascending, symmetric distances
    assert bool((labels[idx.cpu()] != labels.view(-1, 1)).all())
    assert bool((val[:, 1:] >= val[:, :-1]).all())
    # Euclidean <-> cosine identity for norm-10 embeddings (SURVEY §0 fact 2)
    cos = (E_ @ E_.t()) / 100.0
    d_cos = torch.sqrt(torch.clamp(200.0 * (1 - cos), min=0) + 1e-4 / 512)
    assert torch.allclose(torch.gather(d_cos, 1, idx.cpu()), val.cpu(), atol=2e-3)


def test_allpairs_tc_path_near_duplicates_and_small_groups(cuda_dev):
    """Adversarial inputs for the candidate/refine scheme: near-duplicate rows (distance gaps below the fp16 Gram
    error -> the exact fallback must kick in), fewer valid columns than candidates, N not a multiple of 128."""
    g = torch.Generator().manual_seed(9)
    base = torch.randn(40, 512, generator=g)
    E_ = base.repeat_interleave(5, dim=0) + 1e-4 * torch.randn(200, 512, generator=g)     # clusters of near-duplicates
    E_ = 10.0 * E_ / E_.norm(dim=1, keepdim=True)
    labels = (torch.arange(200) % 3).long()
    for k in (1, 4, 8):
        idx, val = dsk.allpairs_topk(E_.cuda(), labels.cuda(), k)
        oidx, oval = C.allpairs_topk(E_.numpy(), labels.numpy(), k)
        assert np.array_equal(idx.cpu().numpy(), oidx) and np.array_equal(val.cpu().numpy(), oval)
    E2 = 10.0 * torch.nn.functional.normalize(torch.randn(20, 512, generator=g), dim=1)
    lab2 = torch.tensor([0] * 14 + [1] * 6)
    idx, val = dsk.allpairs_topk(E2.cuda(), lab2.cuda(), 5)                               # 6 valid columns for label 0
    oidx, oval = C.allpairs_topk(E2.numpy(), lab2.numpy(), 5)
    assert np.array_equal(idx.cpu().numpy(), oidx) and np.array_equal(val.cpu().numpy(), oval)
