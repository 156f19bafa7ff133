"""Spectral clustering on the GPU: dsk_spectral_cluster's eigenvalues, NME selection and k-means partition against the
fp64 oracle (oracle/spectral_oracle.py, dense eigh), recovery of planted speakers, invariances, and diarize with
``spectral=`` against a host recomposition."""
import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import diarization as DZ
from deepspeaker_pytorch_b200 import engine as EN
from deepspeaker_pytorch_b200 import frontend as F
from oracle import ahc_oracle as O
from oracle import spectral_oracle as SO

pytestmark = pytest.mark.gpu


def _cos(N, seed, K=None, D=512, spread=0.6, sizes=None):
    """fp32 cosines of N unit rows: random, or K speakers (rows of a speaker around its centre; sizes optional)."""
    rng = np.random.default_rng(seed)
    if K is None:
        X = rng.standard_normal((N, D))
        lab = np.zeros(N, np.int64)
    else:
        C = rng.standard_normal((K, D))
        lab = np.repeat(np.arange(K), sizes) if sizes is not None else rng.integers(0, K, N)
        X = C[lab] + spread * rng.standard_normal((lab.size, D))
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return (X @ X.T).astype(np.float32), lab


def _run(S, pv, **kw):
    return EN.spectral_cluster(torch.from_numpy(S).cuda(), pv, **kw)


def _check_eigs(got, ref, subset=None):
    _, _, _, eig, lmax, ratio = got
    rows = range(len(ref.lambda_max)) if subset is None else subset
    for t in rows:
        lN = ref.lambda_max[t]
        assert np.max(np.abs(eig[t] - ref.eigenvalues[t])) <= 1e-9 * lN, t
        assert abs(lmax[t] - lN) <= 1e-9 * lN, t
        g = (ref.eigenvalues[t][ref.ks[t]] - ref.eigenvalues[t][ref.ks[t] - 1]) / lN
        if g >= 1e-4:
            assert abs(ratio[t] - ref.ratio[t]) <= 1e-6 * ref.ratio[t], t


@pytest.mark.parametrize("N", [2, 3, 9, 257, 2000])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_eigenvalues_match_the_oracle(cuda_dev, N, kind):
    S, _ = _cos(N, N, None if kind == "random" else 5)
    pv = SO.p_grid(N)
    _check_eigs(_run(S, pv), SO.spectral_cluster(S, pv))


def test_eigenvalues_at_one_hour(cuda_dev):
    """N = 8 997 (the one-hour recording of tools/bench_diarize.py).  Deviation from a whole-grid check: the oracle's
    dense eigh costs tens of seconds per level at this size, so the eigenvalues are compared at the first, middle and
    last levels of the default grid only; the call itself solves all 30 (every level must converge for it to
    return)."""
    N = 8997
    S, _ = _cos(N, 7, 5)
    pv = SO.p_grid(N)
    sub = [0, pv.size // 2, pv.size - 1]
    _check_eigs(_run(S, pv), SO.spectral_cluster(S, pv, subset=sub), sub)


def _tie_heavy():
    S, _ = _cos(300, 3, 4)
    S = np.round(S * 8) / 8
    S[10] = S[20]
    S[:, 10] = S[:, 20]
    return S.astype(np.float32)


def test_tie_heavy_inputs(cuda_dev):
    S = _tie_heavy()
    pv = SO.p_grid(300)
    _check_eigs(_run(S, pv), SO.spectral_cluster(S, pv))


def test_asymmetric_inputs(cuda_dev):
    rng = np.random.default_rng(11)
    A = (_tie_heavy() + 0.05 * rng.standard_normal((300, 300))).astype(np.float32)   # not symmetric, as LLRs
    pv = SO.p_grid(300)
    _check_eigs(_run(A, pv), SO.spectral_cluster(A, pv))


def _margins_hold(ref):
    r = np.sort(ref.ratio[np.isfinite(ref.ratio)])
    lam = ref.eigenvalues[ref.p_index]
    gaps = np.sort(np.diff(lam))[::-1]
    return (r.size < 2 or r[1] - r[0] > 1e-4 * r[0]) and (gaps.size < 2 or gaps[0] - gaps[1] > 1e-4 *
                                                           ref.lambda_max[ref.p_index])


def _same_partition(a, b):
    return np.array_equal(SO.renumber(a), SO.renumber(b))


@pytest.mark.parametrize("N,K,seed", [(257, 3, 1), (600, 5, 2), (2000, 4, 3)])
def test_selection_labels_and_embedding_match_the_oracle(cuda_dev, N, K, seed):
    S, _ = _cos(N, seed, K)
    pv = SO.p_grid(N)
    ref = SO.spectral_cluster(S, pv)
    assert _margins_hold(ref)
    lab, k, t, _, _, _, emb = _run(S, pv, return_embedding=True)
    assert (k, t) == (ref.k, ref.p_index)
    assert _same_partition(lab.cpu().numpy(), ref.labels)
    Y = emb[:, :k].cpu().numpy()
    Qa, _ = np.linalg.qr(Y)
    Qb, _ = np.linalg.qr(ref.embedding)
    s = np.linalg.svd(Qa.T @ Qb, compute_uv=False)
    assert np.sqrt(max(0.0, 1.0 - s.min() ** 2)) <= 1e-6
    for ns in (1, 2, 5, 8):
        ref_n = SO.spectral_cluster(S, pv, num_speakers=ns)
        lab_n, k_n, t_n, _, _, _ = _run(S, pv, num_speakers=ns)
        assert (k_n, t_n) == (ns, ref_n.p_index)
        lam = ref_n.eigenvalues[t_n]
        if lam[ns] - lam[ns - 1] >= 1e-4 * ref_n.lambda_max[t_n]:   # else the embedding is not defined
            assert _same_partition(lab_n.cpu().numpy(), ref_n.labels), ns


def test_recovers_planted_speakers(cuda_dev):
    for K in range(1, 9):
        rng = np.random.default_rng(100 + K)
        sizes = rng.integers(20, 120, K)
        S, lab = _cos(int(sizes.sum()), 100 + K, K, sizes=sizes, spread=0.5)
        res = DZ.spectral(torch.from_numpy(S).cuda())
        assert res.k == K, K
        assert _same_partition(res.labels.cpu().numpy(), lab), K


def test_invariances(cuda_dev):
    S, _ = _cos(700, 5, 4)
    S = (np.round(S * 4096) / 4096).astype(np.float32)   # so that 2 S + 3 is exact in fp32 and keeps every rank
    pv = SO.p_grid(700)
    St = torch.from_numpy(S).cuda()
    a = EN.spectral_cluster(St, pv)

    def same(x, y):
        assert torch.equal(x[0], y[0]) and x[1:3] == y[1:3]
        for u, v in zip(x[3:], y[3:]):
            assert np.array_equal(u, v)

    same(a, EN.spectral_cluster(St, pv))
    same(a, EN.spectral_cluster(2 * St + 3, pv))
    G = St.clone()
    G.fill_diagonal_(-1e30)
    same(a, EN.spectral_cluster(G, pv))
    big = torch.full((700, 777), float("nan"), device="cuda")
    big[:, :700] = St
    same(a, EN.spectral_cluster(big[:, :700], pv))
    E = torch.nn.functional.normalize(torch.randn(300, 512, device="cuda"), dim=1)
    EN.ahc(EN.cosine_matrix(E, E), num_clusters=3)
    EN.cosine_topk(E, E, 5)
    same(a, EN.spectral_cluster(St, pv))
    bad = St.clone()
    bad[3, 5] = float("nan")
    with pytest.raises(RuntimeError):
        EN.spectral_cluster(bad, pv)


def _model():
    from tests.test_gpu_diarization import _model as m
    return m()


def _cluster_host(E, k, plda):
    """The oracle's spectral clustering of the engine's affinity of one recording's windows E, as diarize takes it."""
    W = E.shape[0]
    if W == 1:
        return np.zeros(1, np.int32)
    if k is not None and k >= W:
        return np.arange(W, dtype=np.int32)
    if plda is None:
        S = EN.cosine_matrix(E, E).cpu().numpy()
    else:
        Y = plda.transform(E)
        S = plda.score_matrix(Y, Y).cpu().numpy()
    return SO.spectral_cluster(S, SO.p_grid(W), num_speakers=k).labels


def _host(model, bank, utt, ks, plda=None):
    """Without a speech mask: the engine's windows, the oracle's clustering, frame labels and segments."""
    emb, _, ws, wo = F.window_embeddings(model, bank, utt, 160, 40)
    out = []
    for r, u in enumerate(utt):
        a, b = int(wo[r]), int(wo[r + 1])
        fl = O.frame_labels_brute(ws[a:b].numpy(), _cluster_host(emb[a:b], ks[r], plda), int(bank.lengths[u]), 160)
        out.append((fl, O.segments_brute(fl)))
    return out


def _host_speech(model, bank, utt, speech, ks, plda=None):
    """With a speech mask: windows cut per run of speech as diarize cuts them, every window of a recording clustered
    together by the oracle, each run's frames labelled from its own windows, -1 elsewhere."""
    u = np.asarray(utt)
    table, runs, run_off, kept = bank._run_table(speech, u, "diarize")
    rec, first, end = table[:, 0], table[:, 1], table[:, 2]
    rlen = end - first
    run_bank = F.FeatureBank(bank._gather(runs, run_off, rec.size, kept, u), np.concatenate(([0], np.cumsum(rlen))))
    emb, _, win_start, win_off = F.window_embeddings(model, run_bank, np.arange(rec.size), 160, 40)
    win_off = win_off.numpy()
    run_off_rec = np.searchsorted(rec, np.arange(len(utt) + 1))
    out = []
    for r in range(len(utt)):
        r0, r1 = int(run_off_rec[r]), int(run_off_rec[r + 1])
        fl = np.full(int(bank.lengths[u[r]]), -1, np.int32)
        if r0 < r1:
            a, b = int(win_off[r0]), int(win_off[r1])
            wl = _cluster_host(emb[a:b], ks[r], plda)
            for i in range(r0, r1):
                w0, w1 = int(win_off[i]), int(win_off[i + 1])
                fl[first[i]:end[i]] = DZ.frame_labels(win_start[w0:w1].numpy(), wl[w0 - a:w1 - a], int(rlen[i]), 160)
        out.append((fl, [sg for sg in DZ.segments(fl) if sg[2] >= 0]))
    return out


def _compare(got, ref, what):
    for r, (res, (fl, segs)) in enumerate(zip(got, ref)):
        assert np.array_equal(res.frame_labels, fl), (what, r)
        assert res.segments == segs, (what, r)
        assert res.Z.shape == (0, 4)


def test_diarize_spectral_matches_a_host_recomposition(cuda_dev):
    from tests.test_gpu_vbx import _backend

    g = np.random.RandomState(8)
    lens = [3000, 100, 1777, 161, 2400]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [4, 0, 1, 2, 3]
    for ks in ([None] * 5, [3] * 5, [2, 1, 4, 3, 2]):
        got = DZ.diarize(model, bank, utt, T=160, hop=40, num_speakers=None if ks[0] is None else ks, spectral={})
        _compare(got, _host(model, bank, utt, ks), ("plain", ks))
    o = np.concatenate(([0], np.cumsum(lens)))
    sp = np.zeros(o[-1], bool)
    sp[o[4]:o[4] + 1400] = True                          # utt[0] (bank row 4): two runs of speech
    sp[o[4] + 1600:o[5]] = True
    sp[o[0] + 20:o[0] + 90] = True                       # utt[1] (bank row 0): one short run, one window
    sp[o[2]:o[3]] = np.arange(lens[2]) % 700 < 500       # utt[3] (bank row 2): three runs; bank row 1 has no speech
    sp[o[3]:o[4]] = True
    sp = torch.from_numpy(sp)
    for ks in ([None] * 5, [2] * 5):
        got = DZ.diarize(model, bank, utt, num_speakers=None if ks[0] is None else ks, spectral={}, speech=sp)
        _compare(got, _host_speech(model, bank, utt, sp, ks), ("speech", ks))
    be = _backend(model, bank, utt)
    for ks in ([None] * 5, [3] * 5):
        got = DZ.diarize(model, bank, utt, num_speakers=None if ks[0] is None else ks, spectral={}, plda=be)
        _compare(got, _host(model, bank, utt, ks, plda=be), ("plda", ks))
    got = DZ.diarize(model, bank, utt, num_speakers=2, spectral={}, speech=sp, plda=be)
    _compare(got, _host_speech(model, bank, utt, sp, [2] * 5, plda=be), ("speech plda", 2))
    plain = DZ.diarize(model, bank, utt, num_speakers=3)
    same = DZ.diarize(model, bank, utt, num_speakers=3, spectral=None)
    for x, y in zip(plain, same):
        assert np.array_equal(x.frame_labels, y.frame_labels) and np.array_equal(x.Z, y.Z)
        assert x.segments == y.segments and np.array_equal(x.window_labels, y.window_labels)
