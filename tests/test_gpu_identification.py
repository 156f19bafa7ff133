"""Speaker identification on the GPU: the exact top-k selection bit for bit against the oracle on adversarial rows,
the gallery search bit for bit against the selection of dsk_cosine_matrix's cosines (ties across chunk boundaries
included), invariance to M, row position and interleaved ops, the search against fp64, the enrolment centroids, and
top-k accuracy end to end on synthetic speakers."""
import zlib

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import identification as I
from deepspeaker_pytorch_b200 import verification as V
from oracle import identification_oracle as O

pytestmark = pytest.mark.gpu

COS_GATE = 4e-6   # DESIGN.md section 2: the cosine gate of the scoring ops
SLICE = 65536     # dsk_cosine_matrix's column limit


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- 1. exact selection ---------------------------------------------------------------------------------------------
def _adversarial(rows, cols, seed):
    """Rows cycling through: random, quantised to 1/8, duplicated columns, all equal, signed zeros among small values,
    +-inf, NaN among values (and a row of NaN)."""
    rng = np.random.default_rng(seed)
    S = rng.standard_normal((rows, cols)).astype(np.float32) * 0.2
    for r in range(rows):
        kind = r % 8
        if kind == 1:
            S[r] = np.round(S[r] * 8) / 8
        elif kind == 2:
            h = cols // 2
            S[r, cols - h:] = S[r, :h]
        elif kind == 3:
            S[r] = np.float32(0.3125)
        elif kind == 4:
            S[r] = np.where(rng.random(cols) < 0.5, np.float32(-0.0), np.float32(0.0))
            S[r, :: max(cols // 7, 1)] = -0.25
            S[r, 1 :: max(cols // 5, 2)] = 0.5
        elif kind == 5:
            S[r, rng.integers(0, cols, 3)] = np.inf
            S[r, rng.integers(0, cols, 3)] = -np.inf
        elif kind == 6:
            S[r, rng.integers(0, cols, max(cols // 3, 1))] = np.nan
            S[r, rng.integers(0, cols, 2)] = -np.inf
        elif kind == 7 and r % 16 == 15:
            S[r] = np.nan
    return S


def _check_topk(St, k):
    idx, val = EN.topk_indices(St, k)
    ri, rv = O.topk_keys(St, k)
    assert torch.equal(idx, ri), k
    assert _bits_equal(val, rv), k


@pytest.mark.parametrize("cols", [1, 129, 16384, 16385, 65536])
def test_topk_indices_exact(cuda_dev, cols):
    rows = 32 if cols <= 16385 else 16
    S = _adversarial(rows, cols, seed=cols)
    St = torch.from_numpy(S).cuda()
    for k in sorted({k for k in (1, 2, 10, 1024, cols) if k <= min(cols, 1024)}):
        _check_topk(St, k)
    # the numpy lexsort definition itself on a few rows
    idx, _ = EN.topk_indices(St[:8], min(cols, 10))
    assert np.array_equal(idx.cpu().numpy(), O.topk(S[:8], min(cols, 10))[0])


def test_topk_indices_reads_a_strided_view(cuda_dev):
    S = torch.from_numpy(_adversarial(16, 1000, seed=1)).cuda()
    for k in (1, 10, 700):
        i_view, v_view = EN.topk_indices(S[:, 3:703], k)         # row stride 1000, unaligned rows
        i_full, v_full = EN.topk_indices(S[:, 3:703].contiguous(), k)
        assert torch.equal(i_view, i_full) and _bits_equal(v_view, v_full)
        _check_topk(S[:, 3:703].contiguous(), k)


# ---- 2. gallery search against the selection of dsk_cosine_matrix ---------------------------------------------------
def _gallery(M, Ng, D, seed):
    """Q (M, D), G (Ng, D) on the GPU.  Copies of gallery rows sit on both sides of every 16384-column boundary (so ties
    span chunks), a few queries are copies (scaled) of duplicated rows (ties at rank 1), and one gallery row is zero."""
    g = _gen("gallery", M, Ng, D, seed)
    G = torch.randn(Ng, D, generator=g)
    Q = torch.randn(M, D, generator=g) * 10.0
    for b in range(16384, Ng, 16384):
        G[b] = G[b - 1]
        if b + 2 < Ng:
            G[b + 2] = G[b - 3]
    if Ng > 16384:
        for i in range(0, M, 7):
            Q[i] = 3.0 * G[16383 + (i // 7 % 3) * (16384 if Ng > 3 * 16384 else 0)]
    elif Ng >= 4:
        G[Ng - 1] = G[1]
        Q[0] = G[1]
    if Ng > 6:
        G[5] = 0.0
    return Q.cuda(), G.cuda()


def _sliced_cosines(Q, G):
    """dsk_cosine_matrix of <= 65536-column slices, concatenated (a 1-column slice: the last of a 2-column one)."""
    if G.shape[0] == 1:
        return V.cosine_matrix(Q, torch.cat([G, G]))[:, :1]
    return torch.cat([V.cosine_matrix(Q, G[c:c + SLICE]) if G[c:c + SLICE].shape[0] > 1 else
                      V.cosine_matrix(Q, G[c - 1:c + 1])[:, 1:] for c in range(0, G.shape[0], SLICE)], dim=1)


SEARCH = [(1, 1), (130, 5), (5000, 16384), (130, 16385), (5000, 2 * 65536 + 77), (1, 300000), (130, 300000)]


@pytest.mark.parametrize("M,Ng", SEARCH, ids=lambda v: str(v))
def test_cosine_topk_is_topk_of_cosine_matrix(cuda_dev, M, Ng):
    Q, G = _gallery(M, Ng, 512, 0)
    S = _sliced_cosines(Q, G)
    for k in sorted({min(k, Ng) for k in (1, 10, 1024)}):
        idx, val = I.search(Q, G, k)
        ri, rv = O.topk_keys(S, k)
        bad = (idx != ri).any(dim=1) | (val.view(torch.int32) != rv.view(torch.int32)).any(dim=1)
        assert not bool(bad.any()), (k, int(bad.sum()), int(bad.nonzero()[0]))
    if Ng > 16384:   # the copied rows tie across chunks: the lower column wins
        i = I.search(Q[:1], G, 2)[0][0].tolist()
        assert i == [16383, 16384], i


def test_search_invariance(cuda_dev):
    """Repeat runs, rows sliced out of a larger M (other row chunks, other positions) and calls of the other plans in
    between give bit-identical results, and leave those ops' outputs unchanged."""
    Q, G = _gallery(5000, 70000, 512, 1)
    idx, val = I.search(Q, G, 10)
    for lo, hi in ((0, 1), (4095, 4097), (1000, 4500), (4999, 5000), (17, 17 + 130)):
        i2, v2 = I.search(Q[lo:hi], G, 10)
        assert torch.equal(i2, idx[lo:hi]) and _bits_equal(v2, val[lo:hi]), (lo, hi)
    g = _gen("interleave")
    Ea = torch.randn(384, 512, generator=g).cuda()
    W = (torch.randn(1211, 512, generator=g) / 512 ** 0.5).cuda()
    lab = torch.randint(0, 1211, (384,), generator=g).cuda()
    Ep = torch.randn(256, 512, generator=g).cuda()
    lab_p = torch.arange(256, device="cuda") // 4
    E, C = Q[:700], G[:5994]
    aam0 = EN.aam_softmax(Ea, W, lab, 0.2, 30.0)[3:]
    ap0 = EN.allpairs_topk(Ep, lab_p, 4)
    st0 = V.cohort_stats(E, C, 300)
    i1, v1 = I.search(Q, G, 10)
    st1 = V.cohort_stats(E, C, 300)
    aam1 = EN.aam_softmax(Ea, W, lab, 0.2, 30.0)[3:]
    i2, v2 = I.search(Q, G, 10)
    ap1 = EN.allpairs_topk(Ep, lab_p, 4)
    i3, v3 = I.search(Q, G, 10)
    for a, b in list(zip(aam0, aam1)) + list(zip(ap0, ap1)) + list(zip(st0, st1)):
        assert torch.equal(a, b)
    for i, v in ((i1, v1), (i2, v2), (i3, v3)):
        assert torch.equal(i, idx) and _bits_equal(v, val)


# ---- 3. against fp64 -------------------------------------------------------------------------------------------------
def _near_ties(cos64, k, eps):
    """Rows whose fp64 gap between ranks k and k + 1 is below 2 eps (there the fp32 top-k set may differ)."""
    top = torch.topk(cos64, min(k + 1, cos64.shape[1]), dim=1).values
    if top.shape[1] <= k:
        return torch.zeros(cos64.shape[0], dtype=torch.bool, device=cos64.device)
    return (top[:, k - 1] - top[:, k]) < 2 * eps


@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_search_vs_fp64(cuda_dev, kind):
    M, Ng, D, k = 1000, 2 * 65536 + 77, 512, 10
    g = _gen("fp64", kind)
    if kind == "random":
        G = torch.randn(Ng, D, generator=g)
        Q = torch.randn(M, D, generator=g)
    else:                              # utterances around 2000 speakers: cosines up to ~0.95, many close competitors
        C = torch.randn(2000, D, generator=g)
        C = C / C.norm(dim=1, keepdim=True)
        G = C[torch.randint(0, 2000, (Ng,), generator=g)] + (0.33 / D ** 0.5) * torch.randn(Ng, D, generator=g)
        Q = C[torch.randint(0, 2000, (M,), generator=g)] + (0.33 / D ** 0.5) * torch.randn(M, D, generator=g)
    Q, G = Q.cuda(), G.cuda()
    idx, val = I.search(Q, G, k)
    Qn, Gn = (X.double() / X.double().norm(dim=1, keepdim=True) for X in (Q, G))
    cos64 = Qn @ Gn.T
    eps = float((_sliced_cosines(Q, G).double() - cos64).abs().max())
    err = float((val.double() - torch.gather(cos64, 1, idx)).abs().max())
    ri = torch.topk(cos64, k, dim=1).indices
    same = (torch.sort(idx, 1).values == torch.sort(ri, 1).values).all(dim=1)
    near = _near_ties(cos64, k, eps)
    print(f"\n{kind}: eps {eps:.2e}, max |score - fp64| {err:.2e}; {int(near.sum())} near-tie rows of {M}, "
          f"{int((~same).sum())} rows with another top-{k} set")
    assert eps <= COS_GATE and err <= COS_GATE
    assert bool((same | near).all())


# ---- 4. enrolment centroids ------------------------------------------------------------------------------------------
def test_class_centroids_vs_fp64(cuda_dev):
    g = _gen("centroids")
    U, D = 20000, 320                               # D not a multiple of 256: a partial column block
    X = torch.randn(U, D, generator=g) * torch.exp(torch.empty(U, 1).uniform_(-3.0, 3.0, generator=g))
    X[7] = 0.0
    labels = torch.randint(0, 700, (U,), generator=g).numpy()
    cent, ids = I.enroll(X.cuda(), labels)
    ref, rids = O.centroids(X, labels)
    assert np.array_equal(ids, rids)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    err = np.abs(cent.cpu().double().numpy() - ref)
    print(f"\nmax |centroid - fp64| {err.max():.2e}, worst ratio to 1 ulp {(err / ulp).max():.3f}")
    assert (err <= ulp).all()
    # the raw ABI: an empty segment gives a zero row, an index out of range a NaN row; other rows keep their bits
    order = torch.arange(12, dtype=torch.int64)
    order[9] = U + 5
    offsets = torch.tensor([0, 4, 4, 8, 12], dtype=torch.int64)
    out = EN.class_centroids(X.cuda(), order, offsets)
    assert bool((out[1] == 0).all()) and bool(torch.isnan(out[3]).all())
    assert _bits_equal(out[0], EN.class_centroids(X.cuda(), order[:4], torch.tensor([0, 4]))[0])
    ref0, _ = O.centroids(X[:8], np.array([0] * 4 + [1] * 4))
    assert (np.abs(out[[0, 2]].cpu().double().numpy() - ref0) <= np.spacing(np.abs(ref0).astype(np.float32))).all()


# ---- 5. end to end on synthetic speakers -----------------------------------------------------------------------------
def _speakers(n_spk, per, D, seed, noise=(1.5, 5.0)):
    g = _gen("spk", n_spk, per, seed)
    centres = torch.randn(n_spk, D, generator=g)
    centres = centres / centres.norm(dim=1, keepdim=True)
    spk = torch.arange(n_spk).repeat_interleave(per)
    sigma = torch.empty(n_spk, 1).uniform_(*noise, generator=g)[spk] / D ** 0.5
    return (centres[spk] + sigma * torch.randn(n_spk * per, D, generator=g)) * 10.0, spk.numpy()


@pytest.mark.parametrize("gallery", ["centroids", "utterances"])
def test_end_to_end_synthetic_speakers(cuda_dev, gallery):
    """1251 speakers with per-speaker noise, 8 enrolment and 4 query utterances each.  The utterance gallery adds
    60 000 distractor utterances of 7 500 other speakers (70 008 rows, beyond one cosine_matrix slice)."""
    D, S, k = 512, 1251, 5
    X, spk = _speakers(S, 12, D, 0)
    enrol = np.tile(np.arange(12) < 8, S)
    Xe, le, Xq, lq = X[enrol], spk[enrol], X[~enrol].cuda(), spk[~enrol]
    if gallery == "centroids":
        Gd, gl = I.enroll(Xe.cuda(), le)
        G64, gl64 = O.centroids(Xe, le)
        assert np.array_equal(gl, gl64)
    else:
        Xd, ld = _speakers(7500, 8, D, 1)
        Gd = torch.cat([Xe, Xd]).cuda()
        gl = np.concatenate([le, ld + S])
        G64 = O.normalize(Gd)
    idx, score = I.search(Xq, Gd, k)
    acc = I.accuracy(idx, gl, lq, ks=(1, 5))
    cos64 = torch.from_numpy(O.normalize(Xq)).cuda() @ torch.from_numpy(G64 / np.maximum(
        np.linalg.norm(G64, axis=1, keepdims=True), 1e-12)).cuda().T
    ri = torch.topk(cos64, k, dim=1).indices.cpu().numpy()
    racc = O.accuracy(ri, gl, lq, ks=(1, 5))
    eps = float((score.double() - torch.gather(cos64, 1, idx)).abs().max())
    near = np.zeros(lq.size, dtype=bool)
    for kk in (1, 5):
        near |= _near_ties(cos64, kk, max(eps, COS_GATE)).cpu().numpy()
    ok = {kk: (gl[idx.cpu().numpy()[:, :kk]] == lq[:, None]).any(1) for kk in (1, 5)}
    rok = {kk: (gl[ri[:, :kk]] == lq[:, None]).any(1) for kk in (1, 5)}
    print(f"\n{gallery}: top-1 {acc[1]:.4f} (fp64 {racc[1]:.4f}), top-5 {acc[5]:.4f} (fp64 {racc[5]:.4f}); "
          f"{int(near.sum())} near-tie queries of {lq.size}, max |score - fp64| {eps:.2e}")
    assert eps <= COS_GATE
    for kk in (1, 5):
        assert ((ok[kk] == rok[kk]) | near).all()
        assert abs(acc[kk] - racc[kk]) <= near.sum() / lq.size
    assert 0.2 < acc[1] < 1.0


# ---- 6. rejection ----------------------------------------------------------------------------------------------------
def test_bad_inputs_are_rejected(cuda_dev):
    Q, G = torch.randn(8, 64).cuda(), torch.randn(10, 64).cuda()
    cases = [
        lambda: I.search(Q.cpu(), G, 3),
        lambda: I.search(Q, G, 11),                                          # Ng < k
        lambda: I.search(Q, G, 0),
        lambda: I.search(Q, torch.randn(2000, 64).cuda(), 1025),             # k > 1024
        lambda: I.search(torch.randn(8, 96).cuda(), torch.randn(10, 96).cuda(), 3),   # D % 64
        lambda: I.search(Q, torch.randn(10, 128).cuda(), 3),                 # D mismatch
        lambda: EN.topk_indices(torch.randn(4, 10).cuda(), 11),
        lambda: EN.topk_indices(torch.randn(4, 10).cuda().double(), 3),
        lambda: EN.topk_indices(torch.randn(4, 70000).cuda(), 3),            # cols > 65536
        lambda: I.enroll(Q, torch.arange(8).cuda()),                         # labels on the device
    ]
    for i, fn in enumerate(cases):
        with pytest.raises(RuntimeError):
            fn()
            pytest.fail(f"case {i} was accepted")
