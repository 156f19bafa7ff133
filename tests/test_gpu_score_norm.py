"""Cosine scoring and AS-norm on the GPU: the tensor-core cosines against fp64, the exact top-k statistics on adversarial
matrices, bit-identical composition / chunking / repeat runs, the cohort statistics and trial scores against the fp64
oracle with derived bounds, and EER / minDCF end to end on synthetic speakers."""
import math
import zlib

import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import verification as V
from oracle import score_norm_oracle as O

pytestmark = pytest.mark.gpu

SHAPES = [(4874, 5994, 512), (130, 1000, 192), (1, 2, 64)]
COS_GATE = 4e-6   # 22-bit operands (~2^-21) plus D/16 truncating K16 steps of the hi.hi part at <= 2^-23 of |cos| <= 1


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32("/".join(map(str, key)).encode()))


def _case(M, Nc, D, kind):
    """E (M, D), cohort (Nc, D) fp32 on the GPU.  norm10: rows as the model emits them; clustered: utterances are speaker
    centres plus noise and the cohort is the centres (cosines up to ~0.95); spread: norms over four decades, with a zero
    row in E (and in the cohort when Nc > 2)."""
    g = _gen(M, Nc, D, kind)
    if kind == "norm10":
        E = torch.randn(M, D, generator=g)
        E = 10.0 * E / E.norm(dim=1, keepdim=True)
        C = torch.randn(Nc, D, generator=g)
    elif kind == "clustered":
        C = torch.randn(Nc, D, generator=g)
        C = C / C.norm(dim=1, keepdim=True)
        spk = torch.randint(0, Nc, (M,), generator=g)
        E = 10.0 * (C[spk] + (0.33 / D ** 0.5) * torch.randn(M, D, generator=g))
    else:
        E = torch.randn(M, D, generator=g) * torch.exp(torch.empty(M, 1).uniform_(-4.0, 5.0, generator=g))
        C = torch.randn(Nc, D, generator=g) * torch.exp(torch.empty(Nc, 1).uniform_(-4.0, 5.0, generator=g))
        E[M // 2] = 0.0
        if Nc > 2:
            C[Nc - 1] = 0.0
    return E.cuda(), C.cuda()


def _cos_err(E, C):
    """The engine's cosines and their max |error| against fp64."""
    cos = V.cosine_matrix(E, C)
    return cos, float((cos.double() - O.cosine_matrix(E, C)).abs().max())


def _ulp(x):
    """fp32 spacing at |x| (x fp64), as fp64; inf / NaN stay as they are."""
    a = np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)
    return np.spacing(a).astype(np.float64)


def _bits_equal(*pairs):
    """Bit-identical float tensors (NaN payloads included)."""
    return all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in pairs)


def _within(got, ref, tol):
    """|got - ref| <= tol elementwise, with NaN == NaN and equal infinities accepted."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    same = (np.isnan(got) & np.isnan(ref)) | (np.isinf(ref) & (got == ref))
    with np.errstate(invalid="ignore"):
        err = np.where(same, 0.0, np.abs(got - ref))
        ok = same | (err <= tol)
    return bool(ok.all()), float(np.nanmax(err)) if got.size else 0.0


# ---- 1. cosine matrix against fp64 ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["norm10", "clustered", "spread"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_cosine_matrix_vs_fp64(cuda_dev, shape, kind):
    E, C = _case(*shape, kind)
    cos, err = _cos_err(E, C)
    assert cos.shape == shape[:2] and cos.dtype == torch.float32
    print(f"\n{shape} {kind}: max |dcos| {err:.3e} (max cos {float(cos.max()):.4f})")
    assert err <= COS_GATE, err
    if kind == "spread":
        assert not bool(cos[shape[0] // 2].any())


# ---- 2. exact top-k statistics -------------------------------------------------------------------------------------
def _np_topk(S, k):
    S = np.asarray(S, dtype=np.float64)
    top = -np.sort(-S, axis=1)[:, :k]
    with np.errstate(invalid="ignore"):
        mean = top.mean(axis=1)
        std = top.std(axis=1, ddof=1)
    nan = np.isnan(S).any(axis=1)
    mean[nan] = np.nan
    std[nan] = np.nan
    return mean, std


def _adversarial(rows, cols, seed):
    """Rows of kinds cycling through: random, quantised to 1/8 (massive ties), duplicated columns, all equal, signed
    zeros among small values, and +-inf."""
    rng = np.random.default_rng(seed)
    S = rng.standard_normal((rows, cols)).astype(np.float32) * 0.2
    for r in range(rows):
        kind = r % 6
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
            S[r, rng.integers(0, cols, 2)] = np.inf
            S[r, rng.integers(0, cols, 2)] = -np.inf
    return S


@pytest.mark.parametrize("cols", [2, 129, 5994, 65536])
def test_topk_mean_std_exact(cuda_dev, cols):
    rows = 24 if cols < 65536 else 12
    S = _adversarial(rows, cols, seed=cols)
    St = torch.from_numpy(S).cuda()
    for k in sorted({2, min(5, cols), min(300, cols), cols}):
        mean, std = EN.topk_mean_std(St, k)
        rm, rs = _np_topk(S, k)
        ok_m, dm = _within(mean.cpu().numpy(), rm, _ulp(rm))
        ok_s, ds = _within(std.cpu().numpy(), rs, _ulp(rs))
        assert ok_m and ok_s, (cols, k, dm, ds)
    eq = np.flatnonzero(np.arange(rows) % 6 == 3)               # all-equal rows: sigma exactly 0
    _, std = EN.topk_mean_std(St, cols)
    assert bool((std.cpu()[eq] == 0).all())
    # a NaN anywhere in a row gives NaN for both; the other rows keep their bits
    S2 = S.copy()
    S2[0, cols - 1] = np.nan
    S2[3, 0] = np.nan
    m2, s2 = EN.topk_mean_std(torch.from_numpy(S2).cuda(), 2)
    m1, s1 = EN.topk_mean_std(St, 2)
    m2, s2, m1, s1 = (t.cpu() for t in (m2, s2, m1, s1))
    assert all(bool(torch.isnan(t[[0, 3]]).all()) for t in (m2, s2))
    keep = [r for r in range(rows) if r not in (0, 3)]
    assert _bits_equal((m2[keep], m1[keep]), (s2[keep], s1[keep]))


def test_topk_mean_std_reads_a_strided_view(cuda_dev):
    S = torch.from_numpy(_adversarial(12, 1000, seed=1)).cuda()
    m_full, s_full = EN.topk_mean_std(S[:, :700].contiguous(), 50)
    m_view, s_view = EN.topk_mean_std(S[:, :700], 50)          # row stride 1000, unaligned rows
    assert _bits_equal((m_full, m_view), (s_full, s_view))


# ---- 3. composition and determinism --------------------------------------------------------------------------------
def _chunk_rows(M, Nc):
    Np = (Nc + 127) // 128 * 128
    cap = max(128, (256 << 20) // (Np * 4) // 128 * 128)
    return min(cap, (M + 127) // 128 * 128)


@pytest.mark.parametrize("M,Nc,k", [(4874, 5994, 300), (2500, 65536, 300), (600, 65536, 65536)])
def test_cohort_stats_is_topk_of_cosine_matrix(cuda_dev, M, Nc, k):
    E, C = _case(M, Nc, 512, "norm10")
    mean, std = V.cohort_stats(E, C, k)
    m2, s2 = EN.topk_mean_std(V.cosine_matrix(E, C), k)
    assert torch.equal(mean, m2) and torch.equal(std, s2)


@pytest.mark.parametrize("M,Nc", [(2500, 65536), (20000, 5994)])
def test_rows_do_not_depend_on_chunking(cuda_dev, M, Nc):
    """M = 2500 at Nc = 65536 spans three 1024-row chunks; M = 20000 at Nc = 5994 two 11136-row chunks.  Slices of E
    (other chunk sizes, other positions) give bit-identical rows."""
    assert -(-M // _chunk_rows(M, Nc)) >= 2
    E, C = _case(M, Nc, 512, "clustered")
    mean, std = V.cohort_stats(E, C, 300)
    cos = V.cosine_matrix(E, C) if Nc == 65536 else None
    for lo, hi in ((0, 1), (1000, 2100), (M - 1, M), (M - 130, M), (5, 5 + 1024 + 3)):
        m, s = V.cohort_stats(E[lo:hi], C, 300)
        assert torch.equal(m, mean[lo:hi]) and torch.equal(s, std[lo:hi]), (lo, hi)
        if cos is not None:
            assert torch.equal(V.cosine_matrix(E[lo:hi], C), cos[lo:hi]), (lo, hi)
    runs = [V.cohort_stats(E, C, 300) for _ in range(2)]
    assert torch.equal(runs[0][0], mean) and torch.equal(runs[1][1], std)


def test_other_ops_interleaved(cuda_dev):
    """The scoring plan has its own slot: AAM-softmax and all-pairs calls in between change neither its results nor
    theirs."""
    E, C = _case(4874, 5994, 512, "norm10")
    g = _gen("interleave")
    Ea = torch.randn(384, 512, generator=g).cuda()
    W = (torch.randn(1211, 512, generator=g) / 512 ** 0.5).cuda()
    lab = torch.randint(0, 1211, (384,), generator=g).cuda()
    Ep = torch.randn(256, 512, generator=g).cuda()
    lab_p = torch.arange(256, device="cuda") // 4
    aam0 = EN.aam_softmax(Ea, W, lab, 0.2, 30.0)[3:]
    ap0 = EN.allpairs_topk(Ep, lab_p, 4)
    ref = V.cohort_stats(E, C, 300)
    cos0 = V.cosine_matrix(E[:700], C)
    aam1 = EN.aam_softmax(Ea, W, lab, 0.2, 30.0)[3:]
    got = V.cohort_stats(E, C, 300)
    ap1 = EN.allpairs_topk(Ep, lab_p, 4)
    cos1 = V.cosine_matrix(E[:700], C)
    got2 = V.cohort_stats(E, C, 300)
    for a, b in zip(aam0, aam1):
        assert torch.equal(a, b)
    for a, b in zip(ap0, ap1):
        assert torch.equal(a, b)
    assert torch.equal(cos0, cos1)
    for r in (got, got2):
        assert torch.equal(r[0], ref[0]) and torch.equal(r[1], ref[1])


# ---- 4. cohort statistics against the fp64 oracle ------------------------------------------------------------------
def _stats_bounds(E, C, k):
    _, eps = _cos_err(E, C)
    mean, std = V.cohort_stats(E, C, k)
    rm, rs = O.cohort_stats(E, C, k)
    rm, rs = rm.cpu().numpy(), rs.cpu().numpy()
    dm = np.abs(mean.cpu().double().numpy() - rm)
    ds = np.abs(std.cpu().double().numpy() - rs)
    tol_m = eps + _ulp(rm)
    tol_s = eps * math.sqrt(k / (k - 1)) + _ulp(rs)
    return eps, mean, std, dm, ds, tol_m, tol_s


@pytest.mark.parametrize("kind,k", [("norm10", 300), ("norm10", 5994), ("clustered", 300), ("spread", 300)])
def test_cohort_stats_vs_fp64(cuda_dev, kind, k):
    E, C = _case(4874, 5994, 512, kind)
    eps, mean, std, dm, ds, tol_m, tol_s = _stats_bounds(E, C, k)
    print(f"\n{kind} k {k}: eps {eps:.2e}; max |dmu| {dm.max():.2e}, max |dsigma| {ds.max():.2e} "
          f"(worst ratio to bound {max((dm / tol_m).max(), (ds / tol_s).max()):.3f})")
    assert (dm <= tol_m).all() and (ds <= tol_s).all()


# ---- 5. trial scores -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [40000, 600000])
def test_score_trials(cuda_dev, T):
    U, D = 7000, 512
    X, C = _case(U, 2000, D, "spread")
    g = _gen("trials", T)
    trials = torch.randint(0, U, (T, 2), generator=g)
    trials[:20, 0] = torch.tensor([-1, U, 2 ** 40, -(2 ** 40), 0] * 4)  # out of range (and one valid pair per five)
    trials[20:40, 1] = torch.tensor([U, -1, 3, 2 ** 33] * 5)
    raw, normed = V.score_trials(X, trials.cuda())
    assert normed is None
    rr, _ = O.score_trials(X, trials.cuda())
    rr = rr.cpu().numpy()
    bad = ~((trials >= 0) & (trials < U)).all(dim=1).numpy()
    assert bad.sum() == 31 and np.isnan(raw.cpu().numpy()[bad]).all()
    ok, dr = _within(raw.cpu().numpy(), rr, 2.0 ** -24 + 0.5 * _ulp(rr))
    assert ok, dr
    mean, std = V.cohort_stats(X, C, 300)
    raw2, normed = EN.score_trials(X, trials, mean, std)
    assert _bits_equal((raw2, raw))
    _, rn = O.score_trials(X, trials.cuda(), mean, std)         # the oracle fed the engine's own statistics
    rn = rn.cpu().numpy()
    assert np.isnan(normed.cpu().numpy()[bad]).all()
    ok, dn = _within(normed.cpu().numpy(), rn, 2 * _ulp(rn))
    print(f"\nT {T}: max |draw| {dr:.2e}, max |dnormed| {dn:.2e}")
    assert ok, dn
    _, n2 = V.score_trials(X, trials, C, 300)
    assert _bits_equal((n2, normed))


def test_score_trials_sigma_zero_follows_ieee(cuda_dev):
    X = torch.randn(4, 64).cuda()
    trials = torch.tensor([[0, 1], [2, 3], [1, 1]])
    mean = torch.tensor([0.1, 0.2, 0.3, 0.4]).cuda()
    std = torch.tensor([0.0, 1.0, 0.5, 0.0]).cuda()
    raw, normed = EN.score_trials(X, trials, mean, std)
    _, rn = O.score_trials(X, trials, mean, std)
    got, ref = normed.cpu().numpy(), rn.cpu().numpy()
    assert np.isinf(got[0]) and np.isinf(got[1]) and got[2] == np.float32(ref[2])
    assert np.array_equal(np.sign(got[:2]), np.sign(ref[:2]))


# ---- 6. end to end on synthetic speakers ---------------------------------------------------------------------------
def test_end_to_end_synthetic_speakers(cuda_dev):
    """1000 test speakers with 8 utterances each (per-speaker noise levels, so the raw score scale varies by speaker),
    20 000 trials (half target), a cohort of 2000 other speakers' centres, AS-norm with k = 300."""
    D, S, per, k = 512, 1000, 8, 300
    g = _gen("e2e")
    centres = torch.randn(S + 2000, D, generator=g)
    centres = centres / centres.norm(dim=1, keepdim=True)
    spk = torch.arange(S).repeat_interleave(per)
    noise = torch.empty(S, 1).uniform_(0.6, 1.6, generator=g)[spk] / D ** 0.5
    X = (centres[spk] + noise * torch.randn(S * per, D, generator=g) + 0.3 * centres[S + 1999]).cuda()
    cohort = centres[S:].cuda()
    T = 20000
    e = torch.randint(0, S * per, (T,), generator=g)
    same = torch.rand(T, generator=g) < 0.5
    t_same = spk[e] * per + (e % per + torch.randint(1, per, (T,), generator=g)) % per
    t_diff = torch.randint(0, S * per, (T,), generator=g)
    t = torch.where(same, t_same, t_diff)
    trials = torch.stack([e, t], 1)
    targets = (spk[e] == spk[t]).numpy()

    raw, normed = V.score_trials(X, trials.cuda(), cohort, k)
    mean, std = V.cohort_stats(X, cohort, k)
    rm, rs = O.cohort_stats(X, cohort, k)
    rraw, rn = O.score_trials(X, trials.cuda(), rm, rs)           # the fp64 pipeline end to end
    eer, dcf = V.eer_min_dcf(normed, targets)
    reer, rdcf = V.eer_min_dcf(rn.cpu().numpy(), targets)
    eer_raw, _ = V.eer_min_dcf(raw, targets)
    print(f"\nEER {eer:.5f} (fp64 {reer:.5f}, raw cosine {eer_raw:.5f}), minDCF {dcf:.5f} (fp64 {rdcf:.5f})")
    assert abs(eer - reer) <= 1e-3 and abs(dcf - rdcf) <= 1e-3
    assert abs(eer - O.eer_min_dcf(normed.cpu().numpy(), targets)[0]) <= 1e-12
    # first-order propagation of the statistics' bounds (test 4) and of the raw score's into each normed score
    _, eps = _cos_err(X, cohort)
    mu, sd = mean.cpu().double().numpy(), std.cpu().double().numpy()
    bm = eps + _ulp(rm.cpu().numpy())
    bs = eps * math.sqrt(k / (k - 1)) + _ulp(rs.cpu().numpy())
    s = rraw.cpu().numpy()
    ei, ti = trials[:, 0].numpy(), trials[:, 1].numpy()
    bound = 0.5 * sum((2.0 ** -40 + bm[j]) / sd[j] + np.abs(s - mu[j]) * bs[j] / sd[j] ** 2 for j in (ei, ti))
    dn = np.abs(normed.cpu().double().numpy() - rn.cpu().numpy())
    worst = float((dn / (1.01 * bound + 2 * _ulp(rn.cpu().numpy()))).max())
    print(f"max |dnormed| {dn.max():.2e}, worst ratio to the propagated bound {worst:.3f}")
    assert worst <= 1.0


# ---- 7. rejection ------------------------------------------------------------------------------------------------
def test_bad_inputs_are_rejected(cuda_dev):
    E, C = torch.randn(8, 64).cuda(), torch.randn(10, 64).cuda()
    cases = [
        lambda: V.cosine_matrix(E.cpu(), C.cpu()),
        lambda: V.cohort_stats(E.cpu(), C, 5),
        lambda: V.score_trials(E.cpu(), torch.zeros(3, 2, dtype=torch.int64)),
        lambda: V.cosine_matrix(E, torch.randn(10, 128).cuda()),             # D mismatch
        lambda: V.cosine_matrix(torch.randn(8, 96).cuda(), torch.randn(10, 96).cuda()),   # D % 64
        lambda: V.cosine_matrix(E[0], C),                                    # 1-D
        lambda: V.cosine_matrix(E, C[:1]),                                   # Nc = 1
        lambda: V.cosine_matrix(E[:0], C),                                   # M = 0
        lambda: V.cohort_stats(E, C, 11),                                    # k > Nc
        lambda: V.cohort_stats(E, C, 1),                                     # k = 1
        lambda: V.cohort_stats(E, torch.randn(65537, 64).cuda(), 5),         # Nc > 65536
        lambda: V.score_trials(E, torch.zeros(3, 3, dtype=torch.int64)),     # trials not (T, 2)
        lambda: V.score_trials(E, torch.zeros(0, 2, dtype=torch.int64)),     # no trials
        lambda: EN.score_trials(E, torch.zeros(3, 2, dtype=torch.int64), torch.zeros(8).cuda(), None),
        lambda: EN.topk_mean_std(torch.randn(4, 10).cuda(), 11),
        lambda: EN.topk_mean_std(torch.randn(4, 10).cuda().double(), 3),
    ]
    for i, fn in enumerate(cases):
        with pytest.raises(RuntimeError):
            fn()
            pytest.fail(f"case {i} was accepted")
