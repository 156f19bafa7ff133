"""VBx on the H100: engine.vbx against the fp64 oracle (the full-matrix forward-backward) on the engine's own fp32
PLDA-space rows, bit-identical results alone, in a batch, in any order and on every call, a non-decreasing ELBO,
recovery of the speakers of the generative model, NaN containment, and diarize(plda=, vbx={}) end to end against a
host recomposition."""
import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as F
from deepspeaker_pytorch_b200 import plda as P
from oracle import rescnn_oracle as RO
from oracle import vbx_oracle as O

pytestmark = pytest.mark.gpu

DEFAULTS = dict(Fa=0.3, Fb=17.0, loop_p=0.99, init_smoothing=5.0)


def _generate(rng, K, W, d, phi, loop_p=0.99):
    """x_t = sqrt(phi) o y_{z_t} + N(0, I), y_k ~ N(0, I), z an HMM with self-loop probability loop_p."""
    Y = rng.normal(size=(K, d))
    z = np.empty(W, np.int64)
    z[0] = rng.integers(K)
    stay = rng.random(W) < loop_p
    jump = rng.integers(K, size=W)
    for t in range(1, W):
        z[t] = z[t - 1] if stay[t] else jump[t]
    return (np.sqrt(phi) * Y[z] + rng.normal(size=(W, d))).astype(np.float32), z


def _recording(rng, W, d, S, K=4):
    """A recording of W rows with initial labels over exactly S clusters (the true speaker split further)."""
    phi = np.sort(rng.gamma(2.0, 1.0, size=d))[::-1].copy()
    X, z = _generate(rng, min(K, S), W, d, phi)
    lab = (z * ((S + K - 1) // K) + rng.integers(0, (S + K - 1) // K, size=W)) % S
    lab[rng.permutation(W)[:min(S, W)]] = np.arange(min(S, W))          # every cluster present, the largest S - 1
    return X, lab.astype(np.int32), phi


def _run(X, offsets, labels, phi, max_iters=40, epsilon=1e-4, **kw):
    p = dict(DEFAULTS, **kw)
    out = EN.vbx(torch.from_numpy(X).cuda(), np.asarray(offsets, np.int64), torch.from_numpy(labels).cuda(), phi,
                 p["Fa"], p["Fb"], p["loop_p"], p["init_smoothing"], max_iters, epsilon)
    return [t.cpu().numpy() for t in out]


def _check(X, offsets, labels, phi, res, max_iters, epsilon, **kw):
    """Every recording against the oracle run for the engine's iteration count; -> the largest errors."""
    p = dict(DEFAULTS, **kw)
    gamma, pi, elbo, iters, lab = res
    worst = {"elbo_rel": 0.0, "gamma_abs": 0.0, "pi_abs": 0.0, "elbo_drop_rel": -np.inf, "label_diffs": 0}
    for r in range(len(offsets) - 1):
        a, b = offsets[r], offsets[r + 1]
        Sr = int(labels[a:b].max()) + 1
        n = int(iters[r])
        assert 1 <= n <= max_iters
        e = elbo[r]
        assert np.isfinite(e[:n]).all() and np.isnan(e[n:]).all()
        # the stop is consistent with the engine's own ELBO history
        gains = np.diff(e[:n])
        assert np.all(gains[:-1] >= epsilon) if n > 1 else True
        assert n == max_iters or (n >= 2 and gains[-1] < epsilon)
        if n > 1:
            worst["elbo_drop_rel"] = max(worst["elbo_drop_rel"], float((-gains / np.abs(e[1:n])).max()))
        o = O.vbx(X[a:b], phi, labels[a:b], p["Fa"], p["Fb"], p["loop_p"], p["init_smoothing"], n, -np.inf)
        assert o["iters"] == n
        worst["elbo_rel"] = max(worst["elbo_rel"], float((np.abs(e[:n] - o["elbo"]) / np.abs(o["elbo"])).max()))
        worst["gamma_abs"] = max(worst["gamma_abs"], float(np.abs(gamma[a:b, :Sr] - o["gamma"]).max()))
        worst["pi_abs"] = max(worst["pi_abs"], float(np.abs(pi[r, :Sr] - o["pi"]).max()))
        assert not gamma[a:b, Sr:].any() and not pi[r, Sr:].any()
        srt = np.sort(o["gamma"], axis=1)
        margin = srt[:, -1] - (srt[:, -2] if Sr > 1 else 0.0)
        sure = margin > 1e-6
        assert np.array_equal(lab[a:b][sure], o["labels"][sure]), r
        worst["label_diffs"] += int((lab[a:b] != o["labels"]).sum())
    assert worst["elbo_rel"] < 1e-10 and worst["gamma_abs"] < 1e-8 and worst["pi_abs"] < 1e-8, worst
    assert worst["elbo_drop_rel"] <= 1e-9, worst
    return worst


@pytest.mark.parametrize("W,d,S,max_iters", [(1, 1, 1, 40), (2, 128, 2, 40), (500, 128, 7, 40), (8997, 128, 40, 10),
                                             (32768, 200, 128, 3)])
def test_single_recording_matches_the_oracle(cuda_dev, W, d, S, max_iters):
    rng = np.random.default_rng(W + d + S)
    X, lab, phi = _recording(rng, W, d, S)
    res = _run(X, [0, W], lab, phi, max_iters)
    w = _check(X, [0, W], lab, phi, res, max_iters, 1e-4)
    print(f"W {W} d {d} S {S}: {int(res[3][0])} iterations, {w}")


def _batch(seed=13):
    rng = np.random.default_rng(seed)
    lens = [1, 3000, 2, 17, 640, 1500, 64, 65, 2999, 333, 1024, 7, 2048]
    Ss = [1, 33, 2, 5, 12, 20, 3, 8, 31, 1, 16, 7, 25]
    d = 96
    recs = [_recording(rng, n, d, s) for n, s in zip(lens, Ss)]
    phi = recs[0][2]
    X = np.concatenate([r[0] for r in recs])
    lab = np.concatenate([r[1] for r in recs])
    return X, lab, np.concatenate(([0], np.cumsum(lens))), phi


def test_batch_matches_the_oracle(cuda_dev):
    X, lab, off, phi = _batch()
    res = _run(X, off, lab, phi, 8)
    w = _check(X, off, lab, phi, res, 8, 1e-4)
    print(f"13 recordings: iterations {res[3].tolist()}, {w}")


@pytest.mark.parametrize("loop_p", [0.0, 0.5, 0.99, 1.0])
@pytest.mark.parametrize("init_smoothing", [0.0, 5.0])
def test_transition_and_smoothing_settings_match_the_oracle(cuda_dev, loop_p, init_smoothing):
    rng = np.random.default_rng(int(100 * loop_p) + int(init_smoothing))
    X1, l1, phi = _recording(rng, 600, 64, 10)
    X2, l2, _ = _recording(rng, 250, 64, 4)
    X, lab, off = np.concatenate([X1, X2]), np.concatenate([l1, l2]), [0, 600, 850]
    res = _run(X, off, lab, phi, 12, loop_p=loop_p, init_smoothing=init_smoothing)
    w = _check(X, off, lab, phi, res, 12, 1e-4, loop_p=loop_p, init_smoothing=init_smoothing)
    print(f"loop_p {loop_p} init_smoothing {init_smoothing}: iterations {res[3].tolist()}, {w}")


def _same(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


def test_results_are_bit_identical_alone_in_a_batch_and_in_any_order(cuda_dev):
    X, lab, off, phi = _batch()
    R = off.size - 1
    full = _run(X, off, lab, phi)
    assert _same(full, _run(X, off, lab, phi)), "two calls differ"
    rev = np.arange(R)[::-1]
    Xr = np.concatenate([X[off[r]:off[r + 1]] for r in rev])
    lr = np.concatenate([lab[off[r]:off[r + 1]] for r in rev])
    offr = np.concatenate(([0], np.cumsum(np.diff(off)[rev])))
    back = _run(Xr, offr, lr, phi)
    for i, r in enumerate(rev):
        a, b = off[r], off[r + 1]
        Sr = int(lab[a:b].max()) + 1
        alone = _run(X[a:b], [0, b - a], lab[a:b], phi)
        for other, rows, k in ((alone, slice(0, b - a), 0), (back, slice(offr[i], offr[i + 1]), i)):
            assert np.array_equal(other[0][rows, :Sr], full[0][a:b, :Sr]), r
            assert np.array_equal(other[1][k, :Sr], full[1][r, :Sr]), r
            assert np.array_equal(other[2][k], full[2][r], equal_nan=True), r
            assert other[3][k] == full[3][r] and np.array_equal(other[4][rows], full[4][a:b]), r
    print(f"iterations {full[3].tolist()}")


def test_nonfinite_rows_and_bad_labels_poison_only_their_recording(cuda_dev):
    X, lab, off, phi = _batch()
    clean = _run(X, off, lab, phi)
    Xb, lb = X.copy(), lab.copy()
    Xb[off[5] + 700, 3] = np.nan
    Xb[off[10] + 2, 0] = np.inf
    lb[off[8] + 1000] = -1                                             # a bad device-side initial label
    dirty = _run(Xb, off, lb, phi)
    for r in range(off.size - 1):
        a, b = off[r], off[r + 1]
        if r in (5, 8, 10):
            assert np.isnan(dirty[0][a:b]).all() and np.isnan(dirty[1][r]).all() and np.isnan(dirty[2][r]).all()
            assert dirty[3][r] == 0 and (dirty[4][a:b] == -1).all()
        else:
            Sr = int(lab[a:b].max()) + 1
            assert np.array_equal(dirty[0][a:b, :Sr], clean[0][a:b, :Sr]), r
            assert np.array_equal(dirty[1][r, :Sr], clean[1][r, :Sr]), r
            assert np.array_equal(dirty[2][r], clean[2][r], equal_nan=True), r
            assert dirty[3][r] == clean[3][r] and np.array_equal(dirty[4][a:b], clean[4][a:b]), r


def _speaker_embeddings(rng, C, n, D):
    centres = rng.normal(size=(C, D))
    lab = np.repeat(np.arange(C), n)
    return (centres[lab] + rng.normal(size=(C * n, D)) * np.linspace(0.5, 1.5, D)).astype(np.float32), lab


def test_recovers_the_speakers_of_the_generative_model(cuda_dev):
    rng = np.random.default_rng(2024)
    E, elab = _speaker_embeddings(rng, 300, 10, 128)
    be = P.fit(torch.from_numpy(E).cuda(), elab, lda_dim=64)          # cosine_matrix takes D a multiple of 64
    phi = be.psi.numpy()
    Ks, W = [3, 4, 5, 6], 1500
    Xs, zs, inits = [], [], []
    for K in Ks:
        X, z = _generate(rng, K, W, phi.size, phi)
        Xd = torch.from_numpy(X).cuda()
        _, init = EN.ahc(EN.cosine_matrix(Xd, Xd), "average", num_clusters=3 * K)
        Xs.append(X)
        zs.append(z)
        inits.append(init.cpu().numpy())
    off = np.arange(len(Ks) + 1) * W
    res = _run(np.concatenate(Xs), off, np.concatenate(inits), phi)
    for i, K in enumerate(Ks):
        got = res[4][off[i]:off[i + 1]]
        d_init = DZ.der(zs[i], inits[i]).der
        d_vbx = DZ.der(zs[i], got).der
        # a draw of 1 500 windows with about 15 turns can leave a speaker without windows (K = 5 at this seed draws 4):
        # VBx is to find the speakers that hold windows
        held = np.unique(zs[i]).size
        print(f"K {K} ({held} holding windows): psi {phi.min():.2f}..{phi.max():.2f}, {int(res[3][i])} iterations, "
              f"speakers {np.unique(got).size}, DER AHC at {3 * K} clusters {d_init:.4f}, VBx {d_vbx:.4f}")
        assert np.unique(got).size == held
        assert d_vbx < d_init


def _model():
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(RO.make_state_dict(0, num_classes=16))
    return m.eval()


def _backend(model, bank, utt, seed=0):
    """A PLDA fitted on perturbed copies of the windows, each recording of two or more windows a class."""
    emb, _, _, wo = F.window_embeddings(model, bank, utt, 160, 40)
    lab = np.repeat(np.arange(len(utt)), np.diff(wo.numpy()))
    keep = np.isin(lab, np.flatnonzero(np.bincount(lab) >= 2))
    base = emb[torch.from_numpy(keep).cuda()]
    reps = [base + 0.05 * torch.randn(base.shape, generator=torch.Generator("cuda").manual_seed(seed + s),
                                      device="cuda") for s in range(20)]
    return P.fit(torch.cat(reps), np.tile(lab[keep], 20), lda_dim=min(3, np.unique(lab[keep]).size - 1))


def _recompose(be, emb, spans, wls):
    """The host recomposition of diarize's VBx step: the engine's fp32 PLDA-space rows, the oracle's VBx for the
    engine's iteration count, renumbering.  -> (labels per recording, windows whose margin exceeds 1e-6)."""
    multi = [r for r, (a, b) in enumerate(spans) if b - a > 1]
    out, sure = [w.copy() for w in wls], [np.ones(w.size, bool) for w in wls]
    if not multi:
        return out, sure
    E = torch.cat([emb[spans[r][0]:spans[r][1]] for r in multi])
    off = np.concatenate(([0], np.cumsum([spans[r][1] - spans[r][0] for r in multi])))
    init = np.concatenate([wls[r] for r in multi])
    iters = DZ.vbx(be, E, off, init).iters.cpu().numpy()
    X = DZ._plda_space(be, E).cpu().numpy()
    for i, r in enumerate(multi):
        a, b = off[i], off[i + 1]
        o = O.vbx(X[a:b], be.psi.numpy(), init[a:b], max_iters=int(iters[i]), epsilon=-np.inf)
        srt = np.sort(o["gamma"], axis=1)
        sure[r] = srt[:, -1] - (srt[:, -2] if srt.shape[1] > 1 else 0.0) > 1e-6
        out[r] = DZ._renumber(o["labels"], [0, b - a])
    return out, sure


def test_diarize_with_vbx_matches_a_host_recomposition(cuda_dev):
    g = np.random.RandomState(8)
    lens = [3000, 100, 1777, 161, 2400, 8200]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [4, 0, 1, 2, 3, 5]
    be = _backend(model, bank, utt)
    emb, _, win_start, wo = F.window_embeddings(model, bank, utt, 160, 40)
    spans = [(int(wo[r]), int(wo[r + 1])) for r in range(len(utt))]
    ref0 = DZ.diarize(model, bank, utt, num_speakers=3, plda=be)
    got0 = DZ.diarize(model, bank, utt, num_speakers=3, plda=be, vbx=None)
    for a, b in zip(ref0, got0):
        assert np.array_equal(a.frame_labels, b.frame_labels) and np.array_equal(a.Z, b.Z)
        assert a.segments == b.segments and np.array_equal(a.window_labels, b.window_labels)
    Y = be.transform(emb[spans[0][0]:spans[0][1]])
    llr = be.score_matrix(Y, Y).cpu().numpy()
    t = float(np.quantile(llr[np.triu_indices(llr.shape[0], 1)], 0.1))
    for kw in ({"num_speakers": 6}, {"num_speakers": [8, 1, 4, 2, 12, 30]}, {"threshold": t}):
        ahc = DZ.diarize(model, bank, utt, plda=be, **kw)
        got = DZ.diarize(model, bank, utt, plda=be, vbx={}, **kw)
        want, sure = _recompose(be, emb, spans, [x.window_labels for x in ahc])
        for r, (a, b) in enumerate(spans):
            assert np.array_equal(got[r].Z, ahc[r].Z)
            assert np.array_equal(got[r].window_labels[sure[r]], want[r][sure[r]]), (kw, r)
            if sure[r].all():
                fl = DZ.frame_labels(win_start[a:b].numpy(), want[r], int(bank.lengths[utt[r]]), 160)
                assert np.array_equal(got[r].frame_labels, fl) and got[r].segments == DZ.segments(fl), (kw, r)
        print(f"{kw}: AHC speakers {[int(x.window_labels.max()) + 1 for x in ahc]}, VBx speakers "
              f"{[int(x.window_labels.max()) + 1 for x in got]}, uncertain windows {[int((~s).sum()) for s in sure]}")
    with pytest.raises(ValueError, match="129 initial clusters"):
        DZ.diarize(model, bank, [5], num_speakers=129, plda=be, vbx={})


def test_diarize_with_vbx_and_speech_masks_matches_a_host_recomposition(cuda_dev):
    g = np.random.RandomState(9)
    lens = [3000, 100, 1777, 2400]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [3, 0, 1, 2]
    be = _backend(model, bank, utt, seed=50)
    sp = np.zeros(sum(lens), bool)
    o = np.concatenate(([0], np.cumsum(lens)))
    sp[o[0]:o[0] + 1400] = True                          # bank row 0: two runs of speech
    sp[o[0] + 1600:o[1]] = True
    sp[o[1] + 20:o[1] + 90] = True                       # bank row 1: one short run, one window
    sp[o[3]:o[4]] = np.arange(lens[3]) % 900 < 700       # bank row 3: three runs; bank row 2 has no speech
    sp = torch.from_numpy(sp)
    ahc = DZ.diarize(model, bank, utt, num_speakers=5, speech=sp, plda=be)
    got = DZ.diarize(model, bank, utt, num_speakers=5, speech=sp, plda=be, vbx={})
    # the speech windows of each recording, in time order, as diarize cuts them
    u = np.asarray(utt)
    table, runs, run_off, kept = bank._run_table(sp, u, "diarize")
    rec, first, end = table[:, 0], table[:, 1], table[:, 2]
    rlen = end - first
    run_bank = F.FeatureBank(bank._gather(runs, run_off, rec.size, kept, u), np.concatenate(([0], np.cumsum(rlen))))
    emb, _, win_start, win_off = F.window_embeddings(model, run_bank, np.arange(rec.size), 160, 40)
    win_off = win_off.numpy()
    run_off_rec = np.searchsorted(rec, np.arange(len(utt) + 1))
    spans = [(int(win_off[run_off_rec[r]]), int(win_off[run_off_rec[r + 1]])) if run_off_rec[r] < run_off_rec[r + 1]
             else (0, 0) for r in range(len(utt))]
    want, sure = _recompose(be, emb, spans, [x.window_labels for x in ahc])
    assert got[3].window_labels.size == 0 and (got[3].frame_labels == -1).all() and got[3].segments == []
    assert got[2].window_labels.tolist() == [0]
    for r, (a, b) in enumerate(spans):
        assert np.array_equal(got[r].window_labels[sure[r]], want[r][sure[r]]), r
        if not sure[r].all() or b == a:
            continue
        fl = np.full(int(bank.lengths[utt[r]]), -1, np.int32)
        for i in range(run_off_rec[r], run_off_rec[r + 1]):
            w0, w1 = int(win_off[i]), int(win_off[i + 1])
            fl[first[i]:end[i]] = DZ.frame_labels(win_start[w0:w1].numpy(), want[r][w0 - a:w1 - a], int(rlen[i]), 160)
        assert np.array_equal(got[r].frame_labels, fl), r
        assert got[r].segments == [s for s in DZ.segments(fl) if s[2] >= 0], r
    print(f"speech: AHC speakers {[x.window_labels.size and int(x.window_labels.max()) + 1 for x in ahc]}, VBx "
          f"{[x.window_labels.size and int(x.window_labels.max()) + 1 for x in got]}")
