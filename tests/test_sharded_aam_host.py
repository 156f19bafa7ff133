"""The class-sharded AAM-softmax without a GPU: ``class_shards``' boundaries, sizes and rejection; an fp64 restatement
of the staged decomposition (per-shard cosines and top-k candidates, the exact top-k merge, per-block partial sums
combined in global block order, and the backward's per-shard dcos, gW rows and gE partials added in rank order)
against ``oracle/subcentre_aam_oracle`` to 1e-12 at R = 1, 2, 3, 8, with ties across shards and a shard with fewer
candidates than topk; and argument rejection in the Python layer."""
import math

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import parallel as P
from oracle import aam_softmax_oracle as A
from oracle import subcentre_aam_oracle as S

M, SC, TM = 0.2, 30.0, 0.1


@pytest.mark.parametrize("C,R", [(128, 1), (1211, 1), (1211, 2), (1211, 4), (1211, 8), (3 * 5994, 8), (300, 2),
                                 (257, 2), (1024, 8), (1025, 8), (100000, 2), (53946 // 3, 3)])
def test_class_shards(C, R):
    sh = P.class_shards(C, R)
    assert len(sh) == R and sh[0][0] == 0 and sh[-1][1] == C
    sizes = [c1 - c0 for c0, c1 in sh]
    for (a0, a1), (b0, _) in zip(sh, sh[1:]):
        assert a1 == b0 and a1 % 128 == 0
    assert min(sizes) >= 128 and max(sizes) - min(sizes) <= 128, sizes
    assert P.shard_record_blocks(C, R) == max(-(-s // 128) for s in sizes)


@pytest.mark.parametrize("C,R", [(127, 1), (255, 2), (1023, 8), (0, 1), (300, 0), (300, -1)])
def test_class_shards_rejects(C, R):
    with pytest.raises(ValueError):
        P.class_shards(C, R)
    with pytest.raises(ValueError):
        P.class_shards(300, 2.0)


def _key(v, c):
    """The top-k order as a python sort key (smaller first): larger cosines first, ties to the lower class, NaN last."""
    return (1, 0.0, c) if math.isnan(v) else (0, -v + 0.0, c)


def staged(E, W, y, K, topk, ranges, margin=M, scale=SC, tm=TM, grad_loss=1.0):
    """fp64 restatement of the sharded op's stages over the class ranges -> (loss, cos, lse, top, gE, gW)."""
    y = torch.as_tensor(y, dtype=torch.int64)
    N, C = E.shape[0], W.shape[0] // K
    e, ne = A._normalize(E.double())
    w, nw = A._normalize(W.double())
    # stage 1: per shard class cosines, argmax and the local top-k candidates (global ids; None past the shard's)
    shard_cos, shard_sub, cands = [], [], []
    for c0, c1 in ranges:
        cr, sr = S.subcentre_max(e @ w[c0 * K:c1 * K].T, K)
        shard_cos.append(cr)
        shard_sub.append(sr)
        loc = []
        for i in range(N):
            cl = sorted((c0 + c for c in range(c1 - c0) if c0 + c != int(y[i])), key=lambda c: _key(float(cr[i, c - c0]), c))
            loc.append(cl[:topk] + [None] * (topk - len(cl[:topk])))
        cands.append(loc)
    cos = torch.cat(shard_cos, dim=1)
    # stage 2: the exact merge of the R topk candidates
    top = torch.zeros(N, topk, dtype=torch.int64)
    for i in range(N):
        allc = [c for loc in cands for c in loc[i] if c is not None]
        top[i] = torch.tensor(sorted(allc, key=lambda c: _key(float(cos[i, c]), c))[:topk], dtype=torch.int64)
    inT = torch.zeros(N, C, dtype=torch.bool)
    if topk:
        inT[torch.arange(N)[:, None], top] = True
    ar = torch.arange(N)

    def logits_of(c0, c1):
        cc = cos[:, c0:c1]
        lg = scale * cc.clone()
        t = inT[:, c0:c1]
        lg[t] = scale * S.psi(cc[t], tm)
        own = (y >= c0) & (y < c1)
        lg[ar[own], y[own] - c0] = scale * A.phi(cc[ar[own], y[own] - c0], margin)
        return lg, own
    # stage 2 / 3: local maxima, the global max, per-block partials; stage 4: sums in global block order
    m = torch.stack([logits_of(c0, c1)[0].max(dim=1).values for c0, c1 in ranges]).max(dim=0).values
    blocks, other, tl = [], [], torch.zeros(N, dtype=torch.float64)
    for c0, c1 in ranges:
        lg, own = logits_of(c0, c1)
        ex = torch.exp(lg - m[:, None])
        exo = ex.clone()
        exo[ar[own], y[own] - c0] = 0.0
        for b0 in range(0, c1 - c0, 128):
            blocks.append(ex[:, b0:b0 + 128].sum(1))
            other.append(exo[:, b0:b0 + 128].sum(1))
        tl[own] = lg[ar[own], y[own] - c0]
    Ssum, Sother = torch.stack(blocks).sum(0), torch.stack(other).sum(0)
    lse = m + torch.log(Ssum)
    loss = (lse - tl).sum() / N
    # backward: per shard dcos, gW rows, and gE partials added in rank order
    coef = grad_loss / N * scale / Ssum
    gE_hat = torch.zeros(N, e.shape[1], dtype=torch.float64)
    gWs = []
    for (c0, c1), sr in zip(ranges, shard_sub):
        lg, own = logits_of(c0, c1)
        cc = cos[:, c0:c1]
        d = torch.exp(lg - m[:, None]) * coef[:, None]
        t = inT[:, c0:c1]
        d[t] *= S.dpsi(cc[t], tm)
        ii, yy = ar[own], y[own] - c0
        d[ii, yy] = -Sother[own] * coef[own] * A.dphi(cc[ii, yy], margin)
        dx = torch.zeros(N, (c1 - c0) * K, dtype=torch.float64)
        dx[ar[:, None], torch.arange(c1 - c0)[None, :] * K + sr] = d
        wr = w[c0 * K:c1 * K]
        gw = dx.T @ e
        gWs.append((gw - wr * (wr * gw).sum(1, keepdim=True)) / nw[c0 * K:c1 * K])
        gE_hat = gE_hat + dx @ wr
    gE = (gE_hat - e * (e * gE_hat).sum(1, keepdim=True)) / ne
    return loss, cos, lse, top, gE, torch.cat(gWs)


def _case(N, C, K, D, seed):
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(N, D, generator=g, dtype=torch.float64)
    W = torch.randn(C * K, D, generator=g, dtype=torch.float64) / D ** 0.5
    return E, W, torch.randint(0, C, (N,), generator=g)


@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("K,topk", [(1, 0), (3, 5), (2, 64)])
def test_staged_decomposition_matches_the_oracle(R, K, topk):
    N, C, D = 12, 1100, 64
    E, W, y = _case(N, C, K, D, 7 * R + K)
    # ties across shards: class 1000's sub-centres copied onto classes 5 and 300, which land on other shards for R > 1;
    # rows 0-2 point at them, so the three tie for the top
    for c in (5, 300):
        W[c * K:(c + 1) * K] = W[1000 * K:1001 * K]
    E[:3] = 4.0 * W[1000 * K] + 0.01 * E[:3]
    y[:3] = torch.tensor([7, 600, 1099])
    ranges = P.class_shards(C, R)
    loss, cos, lse, top, gE, gW = staged(E, W, y, K, topk, ranges)
    oloss, ocos, olse, _, otop = S.forward(E, W, y, K, M, SC, topk, TM)
    oE, oW = S.backward(E, W, y, K, M, SC, topk, TM)
    assert torch.equal(cos, ocos) and torch.equal(top, otop)
    if topk:
        assert top[:3, :3].tolist() == [[5, 300, 1000]] * 3
    assert abs(float(loss) - float(oloss)) <= 1e-12 * max(1.0, abs(float(oloss)))
    assert float((lse - olse).abs().max()) <= 1e-12 * float(olse.abs().max())
    assert float((gE - oE).norm() / oE.norm()) <= 1e-12 and float((gW - oW).norm() / oW.norm()) <= 1e-12


def test_staged_with_a_shard_short_of_candidates():
    """A range the ABI accepts but class_shards never makes: 5 classes after a 128-class block, topk = 10 > 5."""
    N, C, K, D, topk = 6, 133, 2, 64, 10
    E, W, y = _case(N, C, K, D, 3)
    E[:2] = 3.0 * W[130 * K] + 0.05 * E[:2]                 # rows whose top classes sit on the short shard
    for ranges in ([(0, 128), (128, 133)], [(0, 133)]):
        loss, cos, lse, top, gE, gW = staged(E, W, y, K, topk, ranges)
        oloss, ocos, olse, _, otop = S.forward(E, W, y, K, M, SC, topk, TM)
        oE, oW = S.backward(E, W, y, K, M, SC, topk, TM)
        assert torch.equal(top, otop) and int(top[0, 0]) == 130
        assert abs(float(loss) - float(oloss)) <= 1e-12 * max(1.0, abs(float(oloss)))
        assert float((gE - oE).norm() / oE.norm()) <= 1e-12 and float((gW - oW).norm() / oW.norm()) <= 1e-12


def test_python_layer_rejects_bad_arguments():
    W = torch.randn(300 * 3, 64)
    good = dict(subcentres=3, topk=5, topk_margin=0.1)
    for w, kw in ((W, dict(good, subcentres=7)), (W, dict(good, topk=300)), (W, dict(good, topk_margin=-1.0)),
                  (W, dict(good, shard=(2, 2))), (W, dict(good, shard=(0, 3))), (torch.randn(900, 60), good),
                  (torch.randn(900), good), ((100000 * 2, 64), dict(subcentres=2, shard=(0, 2)))):
        with pytest.raises(ValueError):
            P.ShardedAAMSoftmaxLoss(w, 0.2, 30.0, device="cpu", **kw)
    for m, s in ((-0.1, 30.0), (0.2, 0.0), (math.nan, 30.0), (0.2, math.inf)):
        with pytest.raises(ValueError):
            P.ShardedAAMSoftmaxLoss(W, m, s, device="cpu", **good)
    head = P.ShardedAAMSoftmaxLoss(W, 0.2, 30.0, device="cpu", shard=(1, 2), **good)
    assert head.class_range == (128, 300) and tuple(head.weight.shape) == (172 * 3, 64)
    assert torch.equal(head.weight.detach(), W[128 * 3:])
    with pytest.raises(ValueError):
        head.load_full_weight(torch.randn(10, 64))
    head.load_full_weight(2 * W)
    assert torch.equal(head.weight.detach(), 2 * W[128 * 3:])
    seeded = [P.ShardedAAMSoftmaxLoss((900, 64), 0.2, 30.0, device="cpu", shard=(r, 2), seed=4, **good) for r in (0, 1)]
    full = torch.cat([h.weight.detach() for h in seeded])
    assert full.shape == (900, 64) and torch.equal(full, torch.randn(900, 64, generator=torch.Generator().manual_seed(4))
                                                    / 8.0)


def test_emulated_exchanges():
    R, n, D = 3, 2, 4
    parts = [torch.arange(R * n * D, dtype=torch.float32).reshape(R * n, D) + 100 * q for q in range(R)]
    got = P.emulated_all_to_all(parts)
    for r in range(R):
        assert torch.equal(got[r], torch.cat([parts[q][r * n:(r + 1) * n] for q in range(R)]))
    local = [torch.full((2, 3), float(q)) for q in range(R)]
    g = P.emulated_gather(local)
    assert len(g) == R and all(torch.equal(t, torch.tensor([0.0] * 6 + [1.0] * 6 + [2.0] * 6)) for t in g)
    assert np.array_equal(P.class_shards(1211, 4), [(0, 256), (256, 512), (512, 896), (896, 1211)])
