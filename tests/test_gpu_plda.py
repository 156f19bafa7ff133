"""PLDA backend on the H100: the fp64 statistics (class sums, the tensor-core Gram) against numpy fp64 from the same fp32
inputs, the affine transform in every mode within 1 fp32 ulp of the oracle, LLR trials and matrices against the oracle
and each other, NaN containment, an end-to-end fit against the oracle fit, PLDA against cosine EER on anisotropic
data, and diarization with a PLDA affinity against scipy on the oracle's LLR matrix."""
import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import fcluster
from scipy.cluster.hierarchy import linkage as scipy_linkage
from scipy.spatial.distance import squareform

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as F
from deepspeaker_pytorch_b200 import plda as P
from deepspeaker_pytorch_b200 import verification as V
from oracle import plda_oracle as O
from oracle import rescnn_oracle as RO

pytestmark = pytest.mark.gpu


def _rel_fro(got, want):
    """Relative Frobenius error; an exactly zero reference (one row minus its own mean) must be matched exactly."""
    return np.linalg.norm(got - want) / max(np.linalg.norm(want), np.finfo(np.float64).tiny)


def _csr(lab):
    order = np.argsort(lab, kind="stable").astype(np.int64)
    _, counts = np.unique(lab, return_counts=True)
    return order, np.concatenate(([0], np.cumsum(counts))).astype(np.int64)


def _ulps(got, ref64):
    """|got - fp32(ref)| in units of fp32(ref)'s ulp (NaN where both are NaN counts as 0)."""
    r32 = ref64.astype(np.float32)
    g = got.astype(np.float64)
    sp = np.spacing(np.abs(r32)).astype(np.float64)
    u = np.abs(g - r32.astype(np.float64)) / sp
    return np.where(np.isnan(g) & np.isnan(r32), 0.0, u)


@pytest.mark.parametrize("D", [64, 200, 512])
@pytest.mark.parametrize("N", [1, 37, 4999, 70001])
def test_class_sums_and_gram_match_fp64(cuda_dev, N, D):
    rng = np.random.default_rng(N + D)
    X = (rng.normal(size=(N, D)) * rng.uniform(0.5, 3.0, D) + rng.normal(size=D)).astype(np.float32)
    lab = rng.integers(0, max(1, N // 7), N)
    order, offsets = _csr(lab)
    X64 = X.astype(np.float64)
    mu = X64.mean(axis=0)
    Xd = torch.from_numpy(X).cuda()
    mud = torch.from_numpy(mu).cuda()
    for m in (None, mu):
        Xc = X64 - (0 if m is None else m)
        sums = EN.class_sums_f64(Xd, torch.from_numpy(order).cuda(), torch.from_numpy(offsets).cuda(),
                                 None if m is None else mud).cpu().numpy()
        ref = np.stack([Xc[order[offsets[c]:offsets[c + 1]]].sum(axis=0) for c in range(offsets.size - 1)])
        G = EN.gram_f64(Xd, None if m is None else mud).cpu().numpy()
        Gref = Xc.T @ Xc
        es, eg = _rel_fro(sums, ref), _rel_fro(G, Gref)
        print(f"N {N} D {D} mu {m is not None}: class sums {es:.2e}, Gram {eg:.2e}")
        assert es < 1e-11 and eg < 1e-11


def test_gram_is_deterministic_and_exactly_symmetric(cuda_dev):
    rng = np.random.default_rng(5)
    X = torch.from_numpy(rng.normal(size=(100003, 200)).astype(np.float32)).cuda()
    mu = X.double().mean(dim=0)
    G1, G2 = EN.gram_f64(X, mu), EN.gram_f64(X, mu)
    assert torch.equal(G1, G2)
    assert torch.equal(G1, G1.T)


@pytest.mark.parametrize("mode", ["none", "length", "plda"])
@pytest.mark.parametrize("N,D,d", [(1, 64, 1), (1000, 512, 200), (777, 200, 200), (130, 96, 33)])
def test_affine_norm_within_one_ulp(cuda_dev, mode, N, D, d):
    rng = np.random.default_rng(N + D + d)
    X = (rng.normal(size=(N, D)) * 2 + 0.5).astype(np.float32)
    A = rng.normal(size=(d, D)) / np.sqrt(D)
    c = rng.normal(size=D) * 0.3
    psi = np.sort(rng.gamma(1.0, 2.0, d))[::-1].copy()
    counts = rng.integers(1, 6, N).astype(np.int32)
    Z = (X.astype(np.float64) - c) @ A.T
    if mode == "none":
        ref, kw = Z, {}
    elif mode == "length":
        ref, kw = O.length_norm(Z), {}
    else:
        dot = (Z * Z / (psi[None, :] + 1.0 / counts[:, None])).sum(axis=1)
        ref, kw = Z * np.sqrt(d / dot)[:, None], {"psi": torch.from_numpy(psi).cuda(), "counts": counts}
    Y = EN.affine_norm_f64(torch.from_numpy(X).cuda(), torch.from_numpy(A).cuda(), torch.from_numpy(c).cuda(), mode,
                           **kw).cpu().numpy()
    u = _ulps(Y, ref)
    print(f"{mode} N {N} D {D} d {d}: max {u.max():.2f} ulp")
    assert u.max() <= 1.0


def _scored_setup(seed, U=300, d=200):
    rng = np.random.default_rng(seed)
    psi = np.sort(rng.gamma(0.7, 4.0, d))[::-1].copy()
    Y = (rng.normal(size=(U, d)) * np.sqrt(psi + 1.0)).astype(np.float32)
    counts = rng.integers(1, 9, U).astype(np.int32)
    return rng, psi, Y, counts


def test_trial_llrs_match_the_oracle_and_are_independent(cuda_dev):
    rng, psi, Y, counts = _scored_setup(0)
    U = Y.shape[0]
    trials = rng.integers(0, U, size=(5000, 2))
    Yd, psid = torch.from_numpy(Y).cuda(), torch.from_numpy(psi).cuda()
    for cnt in (None, counts):
        got = EN.plda_score_trials(Yd, psid, trials, cnt).cpu().numpy().astype(np.float64)
        ref = O.score_trials(psi, Y, trials, cnt)
        err = np.abs(got - ref) / (4e-7 * np.abs(ref) + 1e-9)
        print(f"counts {cnt is not None}: max err / bound {err.max():.3f}, |llr| up to {np.abs(ref).max():.1f}")
        assert err.max() <= 1.0
    full = EN.plda_score_trials(Yd, psid, trials, counts)
    sub = EN.plda_score_trials(Yd, psid, trials[1234:1240], counts)
    rev = EN.plda_score_trials(Yd, psid, trials[::-1].copy(), counts)
    assert torch.equal(full[1234:1240], sub)
    assert torch.equal(full, rev.flip(0))


def test_score_matrix_agrees_with_trials_and_is_symmetric(cuda_dev):
    rng, psi, Y, _ = _scored_setup(1, U=333)
    Yd, psid = torch.from_numpy(Y).cuda(), torch.from_numpy(psi).cuda()
    Ya, Yb = Yd[:130], Yd[130:]
    S = EN.plda_score_matrix(Ya, Yb, psid).cpu().numpy().astype(np.float64)
    ii, jj = np.meshgrid(np.arange(130), np.arange(130, 333), indexing="ij")
    trials = np.stack([ii.ravel(), jj.ravel()], axis=1)
    T = EN.plda_score_trials(Yd, psid, trials).cpu().numpy().astype(np.float64).reshape(130, 203)
    err = np.abs(S - T) / (1e-6 * (1 + np.abs(T)))
    print(f"matrix vs trials: max err / bound {err.max():.3f}")
    assert err.max() <= 1.0
    ref = O.score_matrix(psi, Y[:20], Y[130:150])
    assert np.abs(S[:20, :20] - ref).max() <= 1e-6 * (1 + np.abs(ref)).max()
    Sq = EN.plda_score_matrix(Yd, Yd, psid).cpu().numpy().astype(np.float64)
    asym = np.abs(Sq - Sq.T) / (1e-6 * (1 + np.abs(Sq)))
    print(f"Ya = Yb: max asymmetry / bound {asym.max():.3f}")
    assert asym.max() <= 1.0


def test_nan_rows_and_bad_arguments_poison_only_their_outputs(cuda_dev):
    rng, psi, Y, counts = _scored_setup(2, U=200, d=72)
    psid = torch.from_numpy(psi).cuda()
    # the transform: a NaN input row gives a NaN output row, the others keep their bits
    X = rng.normal(size=(150, 96)).astype(np.float32)
    A = torch.from_numpy(rng.normal(size=(72, 96))).cuda()
    Xb = X.copy()
    Xb[17, 5] = np.nan
    for mode in ("none", "length", "plda"):
        kw = {"psi": psid} if mode == "plda" else {}
        a = EN.affine_norm_f64(torch.from_numpy(X).cuda(), A, None, mode, **kw)
        b = EN.affine_norm_f64(torch.from_numpy(Xb).cuda(), A, None, mode, **kw)
        assert torch.isnan(b[17]).all()
        keep = torch.arange(150, device=a.device) != 17
        assert torch.equal(a[keep], b[keep]), mode
    cnt0 = np.ones(150, np.int32)
    cnt0[3] = 0
    c = EN.affine_norm_f64(torch.from_numpy(X).cuda(), A, None, "plda", psi=psid, counts=cnt0)
    assert torch.isnan(c[3]).all() and torch.isfinite(c[torch.arange(150, device=c.device) != 3]).all()
    # class sums: only the class of the NaN row
    lab = np.arange(150) % 9
    order, offsets = _csr(lab)
    s = EN.class_sums_f64(torch.from_numpy(Xb).cuda(), order, offsets).cpu().numpy()
    bad = np.isnan(s).any(axis=1)
    assert bad.tolist() == [c_ == lab[17] for c_ in range(9)]
    assert np.isnan(s[lab[17], 5]) and np.isfinite(np.delete(s[lab[17]], 5)).all()
    order_bad = order.copy()
    order_bad[offsets[4]] = 150
    s2 = EN.class_sums_f64(torch.from_numpy(X).cuda(), order_bad, offsets).cpu().numpy()
    assert np.isnan(s2[4]).all() and np.isfinite(np.delete(s2, 4, axis=0)).all()
    # trials and matrix
    Yn = Y.copy()
    Yn[11, 40] = np.nan
    Yd, Ynd = torch.from_numpy(Y).cuda(), torch.from_numpy(Yn).cuda()
    trials = rng.integers(0, 200, size=(3000, 2))
    trials[:5] = [[11, 3], [4, 11], [200, 2], [-1, 5], [7, 7]]
    cnt = counts.copy()
    cnt[7] = 0
    clean = EN.plda_score_trials(Yd, psid, trials, cnt).cpu().numpy()
    dirty = EN.plda_score_trials(Ynd, psid, trials, cnt).cpu().numpy()
    hit = (trials == 11).any(axis=1) | (trials < 0).any(axis=1) | (trials >= 200).any(axis=1) | (trials[:, 0] == 7)
    assert np.isnan(dirty[hit]).all()
    assert np.array_equal(clean[~hit], dirty[~hit]) and np.isfinite(clean[~hit]).all()
    Sc = EN.plda_score_matrix(Yd[:90], Yd[90:], psid).cpu().numpy()
    Ya_n, Yb_n = Yd[:90].clone(), Yd[90:].clone()
    Ya_n[11, 40] = float("nan")
    Yb_n[23, 0] = float("nan")
    for Ya, Yb, row, col in ((Ya_n, Yd[90:], 11, None), (Yd[:90], Yb_n, None, 23)):
        Sd = EN.plda_score_matrix(Ya, Yb, psid).cpu().numpy()
        mask = np.zeros_like(Sd, dtype=bool)
        if row is not None:
            mask[row, :] = True
        else:
            mask[:, col] = True
        assert np.isnan(Sd[mask]).all()
        assert np.array_equal(Sd[~mask], Sc[~mask]) and np.isfinite(Sc).all()


def test_fit_end_to_end_matches_the_oracle_fit(cuda_dev):
    rng = np.random.default_rng(11)
    N, D, C = 20000, 512, 500
    lab = rng.permutation(np.arange(N) % C)
    centres = rng.normal(size=(C, D)) * np.linspace(0.2, 1.5, D)
    X = (centres[lab] + rng.normal(size=(N, D)) * np.linspace(1.2, 0.3, D) + 0.7).astype(np.float32)
    be = P.fit(torch.from_numpy(X).cuda(), lab, lda_dim=200, iters=10)
    ref = O.fit(X, lab, lda_dim=200, iters=10)
    rel = np.abs(be.psi.numpy() - ref["psi"]) / ref["psi"]
    print(f"fit: psi rel err {rel.max():.2e} (psi {ref['psi'][0]:.3f} .. {ref['psi'][-1]:.3e})")
    assert rel.max() < 1e-8
    sd = be.state_dict()
    assert set(sd) == {"mu", "lda", "plda_mean", "plda_transform", "psi"}
    assert all(v.dtype == torch.float64 and v.device.type == "cpu" for v in sd.values())
    # held-out speakers: enrolment means of 3 utterances against single test utterances
    Ch = 40
    hc = rng.normal(size=(Ch, D)) * np.linspace(0.2, 1.5, D)
    hl = np.repeat(np.arange(Ch), 4)
    Xh = (hc[hl] + rng.normal(size=(hl.size, D)) * np.linspace(1.2, 0.3, D) + 0.7).astype(np.float32)
    enr_rows = np.flatnonzero(np.arange(hl.size) % 4 != 3)
    tst_rows = np.flatnonzero(np.arange(hl.size) % 4 == 3)
    enr, counts, ids = P.enroll(torch.from_numpy(Xh[enr_rows]).cuda(), hl[enr_rows])
    assert counts.tolist() == [3] * Ch and ids.tolist() == list(range(Ch))
    Ye = be.transform(enr, counts)
    Yt = be.transform(torch.from_numpy(Xh[tst_rows]).cuda())
    Yall = torch.cat([Ye, Yt])
    cnt_all = torch.cat([counts, torch.ones(Ch, dtype=torch.int64)])
    ii, jj = np.meshgrid(np.arange(Ch), Ch + np.arange(Ch), indexing="ij")
    trials = np.stack([ii.ravel(), jj.ravel()], axis=1)
    got = be.score_trials(Yall, trials, cnt_all).cpu().numpy().astype(np.float64)
    enr_ref = np.stack([Xh[enr_rows][hl[enr_rows] == s].astype(np.float64).mean(axis=0) for s in range(Ch)])
    Ye_ref = O.transform(ref, enr_ref, np.full(Ch, 3))
    Yt_ref = O.transform(ref, Xh[tst_rows])
    want = np.array([O.llr(ref["psi"], Ye_ref[i], Yt_ref[j - Ch], 3) for i, j in trials])
    err = np.abs(got - want)
    print(f"held-out LLRs: max abs err {err.max():.2e}, |llr| up to {np.abs(want).max():.1f}; "
          f"target mean {want[ii.ravel() == jj.ravel() - Ch].mean():.1f}, non-target {want[ii.ravel() != jj.ravel() - Ch].mean():.1f}")
    assert err.max() < 1e-4
    be2 = P.PLDA.from_state_dict(sd)
    assert torch.equal(be2.transform(enr, counts), Ye)


def test_plda_beats_cosine_on_anisotropic_within_speaker_noise(cuda_dev):
    rng = np.random.default_rng(21)
    D = 128
    # speaker identity in every direction; the within-speaker noise is large in 12 nuisance directions (channel)
    nuis = np.linalg.qr(rng.normal(size=(D, 12)))[0]

    def draw(S, n):
        lab = np.repeat(np.arange(S), n)
        spk = rng.normal(size=(S, D))
        noise = rng.normal(size=(lab.size, D)) * 0.5 + (rng.normal(size=(lab.size, 12)) * 4.0) @ nuis.T
        return (spk[lab] + noise).astype(np.float32), lab

    Xtr, ltr = draw(400, 12)
    be = P.fit(torch.from_numpy(Xtr).cuda(), ltr, lda_dim=100)
    Xte, lte = draw(120, 6)
    ii, jj = np.triu_indices(lte.size, 1)
    trials = np.stack([ii, jj], axis=1)
    target = lte[ii] == lte[jj]
    Xd = torch.from_numpy(Xte).cuda()
    cos = EN.score_trials(Xd, trials)[0]
    llr = be.score_trials(be.transform(Xd), trials)
    eer_cos, _ = V.eer_min_dcf(cos, target)
    eer_plda, _ = V.eer_min_dcf(llr, target)
    print(f"EER: cosine {eer_cos:.4f}, PLDA {eer_plda:.4f}")
    # the margin: PLDA at most half the cosine EER
    assert eer_plda < 0.5 * eer_cos


def _model():
    sd = RO.make_state_dict(0, num_classes=16)
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(sd)
    return m.eval()


def _relabel(lab):
    lab = np.asarray(lab)
    _, first = np.unique(lab, return_index=True)
    order = np.argsort(first)
    out = np.empty_like(lab)
    for new, old in enumerate(np.unique(lab)[order]):
        out[lab == old] = new
    return out.astype(np.int32)


def test_diarize_with_plda_matches_scipy_on_oracle_llrs(cuda_dev):
    g = np.random.RandomState(8)
    lens = [3000, 100, 1777, 161, 2400]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [4, 0, 1, 2, 3]
    emb, _, _, wo = F.window_embeddings(model, bank, utt, 160, 40)
    # a backend fitted on perturbed copies of the windows, each recording a class
    lab = np.repeat(np.arange(len(utt)), np.diff(wo.numpy()))
    keep = np.isin(lab, np.flatnonzero(np.bincount(lab) >= 2))
    base = emb[torch.from_numpy(keep).cuda()]
    reps = [base + 0.05 * torch.randn(base.shape, generator=torch.Generator("cuda").manual_seed(s), device="cuda")
            for s in range(20)]
    be = P.fit(torch.cat(reps), np.tile(lab[keep], 20), lda_dim=2)
    # plda = None is exactly today's result
    ref0 = DZ.diarize(model, bank, utt, num_speakers=3)
    got0 = DZ.diarize(model, bank, utt, num_speakers=3, plda=None)
    for a, b in zip(ref0, got0):
        assert np.array_equal(a.frame_labels, b.frame_labels) and np.array_equal(a.Z, b.Z)
    # the oracle's LLRs of the transformed windows of the first recording, for a threshold between two merges
    a, b = int(wo[0]), int(wo[1])
    Y = be.transform(emb[a:b])
    S0 = O.score_matrix(be.psi.numpy(), Y.cpu().numpy(), Y.cpu().numpy())
    Z0 = scipy_linkage(squareform(S0.max() - S0, checks=False), "average")
    t = S0.max() - float(Z0[-6:-4, 2].mean())
    for kw in ({"num_speakers": 3}, {"threshold": t}):
        got = DZ.diarize(model, bank, utt, plda=be, **kw)
        for r in range(len(utt)):
            a, b = int(wo[r]), int(wo[r + 1])
            if b - a == 1:
                assert got[r].window_labels.tolist() == [0]
                continue
            Y = be.transform(emb[a:b]).cpu().numpy()
            S = O.score_matrix(be.psi.numpy(), Y, Y)
            # scipy refuses negative distances: shift 1 - S by a constant, which average linkage carries through
            Zs = scipy_linkage(squareform(S.max() - S, checks=False), "average")
            want = _relabel(fcluster(Zs, min(3, b - a), "maxclust") if "num_speakers" in kw
                            else fcluster(Zs, S.max() - t, "distance"))
            assert np.array_equal(got[r].window_labels, want), (kw, r)
        print(f"{kw}: speakers per recording {[int(x.window_labels.max()) + 1 for x in got]}")
    sp = torch.from_numpy(np.arange(sum(lens)) % 5 != 0)
    got_s = DZ.diarize(model, bank, utt, num_speakers=2, speech=sp, plda=be)
    assert len(got_s) == len(utt)
