"""Frame-energy VAD, runs and select, and speech-only diarization on the GPU: features bit-identical with and without
the VAD, energies and decisions independent of the batch, energies against the fp64 fbank oracle, decisions against the
oracle rule, a synthetic speech / silence layout, select and runs against numpy boolean indexing, and diarize with a
speech mask against a host recomposition."""
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
from oracle import ahc_oracle as AO
from oracle import fbank_oracle as FO
from oracle import rescnn_oracle as RO
from oracle import vad_oracle as VO

pytestmark = pytest.mark.gpu

FBANK_LENGTHS = [48000, 16000, 399, 400, 401, 560, 100003]      # tests/test_fbank.py


def synth(n, seed, sr=16000):
    g = np.random.RandomState(seed)
    t = np.arange(n) / sr
    x = 0.3 * np.sin(2 * np.pi * 440 * t) + 0.2 * np.sin(2 * np.pi * 2300 * t + 1.0) + 0.05 * g.randn(n)
    x *= np.linspace(0.2, 1.0, n)
    x[n // 3: n // 3 + n // 5] *= 1e-4                  # a quiet stretch, so both decisions occur
    return x.astype(np.float32)


def _batch(waves):
    return torch.from_numpy(np.concatenate(waves)).cuda(), [w.size for w in waves]


@pytest.mark.parametrize("sr", [16000, 8000])
def test_features_bit_identical_with_and_without_vad(cuda_dev, sr):
    waves = [synth(n, i, sr) for i, n in enumerate(FBANK_LENGTHS)]
    a, lens = _batch(waves)
    for log_scale in (True, False):
        for sub in (True, False):
            f0, o0 = F.mk_mfb_batch(a, lens, sr, log_scale, sub)
            f1, o1, e, s = F.mk_mfb_batch_vad(a, lens, sr, log_scale, sub)
            assert torch.equal(o0, o1) and torch.equal(f0, f1), (log_scale, sub)
            assert e.shape == s.shape == (f0.shape[0],) and e.dtype == torch.float32 and s.dtype == torch.bool
    bank = F.FeatureBank.from_waveforms(waves, sr, vad={})
    plain = F.FeatureBank.from_waveforms(waves, sr)
    assert torch.equal(bank.feats, plain.feats) and plain.speech is None
    assert torch.equal(bank.speech, F.mk_mfb_batch_vad(a, lens, sr)[3])
    small = F.FeatureBank.from_waveforms(waves, sr, chunk_samples=50000, vad={})   # several chunks
    assert torch.equal(small.feats, plain.feats) and torch.equal(small.speech, bank.speech)


def test_energies_and_decisions_do_not_depend_on_the_batch(cuda_dev):
    g = np.random.default_rng(0)
    lens = list(g.integers(1, 60000, 40)) + [1, 2, 399, 400, 401, 100003]
    waves = [synth(int(n), i) for i, n in enumerate(lens)]

    def per_utt(order):
        a, ls = _batch([waves[i] for i in order])
        _, off, e, s = F.mk_mfb_batch_vad(a, ls)
        off = off.numpy()
        return {u: (e[off[k]:off[k + 1]].cpu(), s[off[k]:off[k + 1]].cpu()) for k, u in enumerate(order)}

    ref = per_utt(list(range(len(waves))))
    for order in (list(g.permutation(len(waves))), list(g.permutation(len(waves)))[:17]):
        got = per_utt(order)
        for u in got:
            assert torch.equal(got[u][0], ref[u][0]) and torch.equal(got[u][1], ref[u][1]), u
    for u in (0, len(waves) - 1, len(waves) - 6):
        got = per_utt([u])
        assert torch.equal(got[u][0], ref[u][0]) and torch.equal(got[u][1], ref[u][1]), u


@pytest.mark.parametrize("sr", [16000, 8000])
def test_energies_and_decisions_against_the_oracle(cuda_dev, sr):
    waves = [synth(n, 10 + i, sr) for i, n in enumerate(FBANK_LENGTHS)]
    a, lens = _batch(waves)
    _, off, e, s = F.mk_mfb_batch_vad(a, lens, sr)
    off, e, s = off.numpy(), e.cpu().numpy(), s.cpu().numpy()
    worst, near, flagged = 0.0, 0, 0
    for u, w in enumerate(waves):
        eu, su = e[off[u]:off[u + 1]], s[off[u]:off[u + 1]]
        _, E64 = FO.fbank(w, samplerate=sr, nfilt=64)
        worst = max(worst, float(np.max(np.abs(eu - E64) / E64)))
        # the oracle rule fed the engine's own fp32 energies: equal except frames within 1e-12 max(1, |thr|) of thr
        s32, thr32, le32 = VO.decide(eu, [0, eu.size])
        tol = 1e-12 * max(1.0, abs(thr32[0]))
        close = np.abs(le32 - thr32[0]) <= tol
        n = eu.size
        win_close = np.array([close[max(0, f - 2):f + 3].any() for f in range(n)])
        assert np.all((s32 == su) | win_close), u
        near += int(close.sum())
        # the full fp64 oracle: each differing frame has a frame whose fp64 ln E is within 1e-4 of thr in its window
        s64, thr64, le64 = VO.decide(E64, [0, E64.size])
        c64 = np.abs(le64 - thr64[0]) <= 1e-4
        for f in np.flatnonzero(s64 != su):
            flagged += 1
            assert c64[max(0, f - 2):f + 3].any(), (u, f)
        assert 0 < su.sum() < n or n < 50, u          # the quiet stretch of synth() is dropped, the rest kept
    print(f"\n{sr} Hz: energy max rel err vs fp64 {worst:.3e}; frames within 1e-12 of thr {near}; "
          f"decisions differing from fp64 {flagged}")
    assert worst <= 1e-5


def _layout_audio(sr, seed):
    """Noise bursts of 0.2-3 s separated by near-silence (1e-5) and by exact zeros -> (audio, speech sample mask)."""
    g = np.random.default_rng(seed)
    parts, lab = [], []
    for k in range(14):
        n = int(g.uniform(0.2, 3.0) * sr)
        parts.append(0.1 * g.standard_normal(n))
        lab.append(np.ones(n, bool))
        m = int(g.uniform(0.3, 1.5) * sr)
        parts.append(np.zeros(m) if k % 3 == 2 else 1e-5 * g.standard_normal(m))
        lab.append(np.zeros(m, bool))
    return np.concatenate(parts).astype(np.float32), np.concatenate(lab)


@pytest.mark.parametrize("sr", [16000, 8000])
def test_synthetic_layout(cuda_dev, sr):
    flen, step = FO.round_half_up(0.025 * sr), FO.round_half_up(0.01 * sr)
    waves, labs = zip(*[_layout_audio(sr, s) for s in range(3)])
    zero = np.zeros(5 * sr, np.float32)
    a, lens = _batch(list(waves) + [zero])
    _, off, _, s = F.mk_mfb_batch_vad(a, lens, sr)
    off, s = off.numpy(), s.cpu().numpy()
    c = 2
    for u, lab in enumerate(labs):
        su = s[off[u]:off[u + 1]]
        n = su.size
        mid = np.minimum(np.arange(n) * step + flen // 2, lab.size - 1)
        want = lab[mid]
        edges = np.flatnonzero(np.diff(lab.astype(np.int8))) + 1             # sample boundaries
        fb = edges / step
        far = np.array([np.all(np.abs(f - fb) > c + 3) for f in range(n)])
        assert np.array_equal(su[far], want[far]), (sr, u, int(np.sum(su[far] != want[far])))
        print(f"\n{sr} Hz recording {u}: {n} frames, {int(far.sum())} away from boundaries, speech {su.mean():.3f}")
    assert not s[off[-2]:off[-1]].any()


# ---- select and runs ------------------------------------------------------------------------------------------------------
def _runs_numpy(mask, off, utt):
    out = []
    for j, u in enumerate(utt):
        m = np.asarray(mask[off[u]:off[u + 1]], np.int8)
        d = np.diff(np.concatenate(([0], m, [0])))
        a, b = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
        out.append(np.stack([np.full(a.size, j), a, b], 1))
    return np.concatenate(out).astype(np.int64)


def _check_select_and_runs(bank, feats_h, off, mask, utt):
    for m in (mask, torch.from_numpy(mask).cuda()):
        counts = np.add.reduceat(mask.astype(np.int64), off[:-1]) if mask.size else None
        if np.all(counts > 0):
            sel = bank.select(m)
            assert torch.equal(sel.feats.cpu(), torch.from_numpy(feats_h[mask]))
            assert np.array_equal(sel.lengths, counts)
        else:
            with pytest.raises(ValueError, match="without frames"):
                bank.select(m)
        want = _runs_numpy(mask, off, utt)
        if want.shape[0] == 0:
            with pytest.raises(ValueError):
                bank.runs(m, utt)
            continue
        rb, ru, rs = bank.runs(m, utt)
        assert np.array_equal(ru.numpy(), np.asarray(utt)[want[:, 0]])
        assert np.array_equal(rs.numpy(), want[:, 1])
        assert np.array_equal(rb.lengths, want[:, 2] - want[:, 1])
        rows = np.concatenate([np.arange(off[u] + a, off[u] + b) for u, a, b in
                               zip(np.asarray(utt)[want[:, 0]], want[:, 1], want[:, 2])])
        assert torch.equal(rb.feats.cpu(), torch.from_numpy(feats_h[rows]))


def test_select_and_runs_match_numpy(cuda_dev):
    g = np.random.default_rng(3)
    lens = np.concatenate(([1, 2, 3, 4096, 4097, 1], g.integers(1, 2000, 200)))
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    n = int(off[-1])
    feats_h = g.standard_normal((n, 64)).astype(np.float32)
    bank = F.FeatureBank(torch.from_numpy(feats_h).cuda(), off)
    strad = np.zeros(n, bool)
    for u in range(1, lens.size):
        strad[max(off[u] - 2, 0):off[u] + 2] = True                  # runs touching both sides of every boundary
    masks = {"empty": np.zeros(n, bool), "all": np.ones(n, bool), "alternating": np.arange(n) % 2 == 0,
             "straddling": strad, "random": g.random(n) < 0.6, "sparse": g.random(n) < 0.02}
    for name, mask in masks.items():
        for utt in (np.arange(lens.size), np.array([4, 0, 4, 3, 205])):
            _check_select_and_runs(bank, feats_h, off, mask, utt)
    sel = bank.select(torch.ones(n, dtype=torch.bool))
    assert torch.equal(sel.feats, bank.feats) and torch.equal(sel.offsets, bank.offsets)
    with pytest.raises(ValueError, match=r"\[3\]"):
        m = np.ones(n, bool)
        m[off[3]:off[4]] = False
        bank.select(m)
    with pytest.raises(ValueError):
        bank.select(np.ones(n - 1, bool))
    with pytest.raises(ValueError):
        bank.select(np.ones(n, np.float32))
    with pytest.raises(ValueError):
        bank.runs(np.ones(n, bool), [lens.size])


def test_select_and_runs_at_scale(cuda_dev):
    g = np.random.default_rng(4)
    lens = g.integers(1, 3000, 2100)
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    n = int(off[-1])
    assert n >= 3_000_000
    feats = torch.randn(n, 64, device=cuda_dev, generator=torch.Generator(device=cuda_dev).manual_seed(0))
    bank = F.FeatureBank(feats, off)
    # speech-like runs: a two-state chain, about 60 % kept
    flips = g.random(n) < np.where(np.arange(n) % 2 == 0, 0.02, 0.03)
    mask = (np.cumsum(flips) % 2 == 0)
    mask[off[:-1]] = True                                           # every utterance keeps a frame
    md = torch.from_numpy(mask).cuda()
    sel = bank.select(md)
    assert torch.equal(sel.feats, feats[md])
    assert np.array_equal(sel.lengths, np.add.reduceat(mask.astype(np.int64), off[:-1]))
    utt = g.permutation(lens.size)[:1500]
    rb, ru, rs = bank.runs(mask, utt)
    want = _runs_numpy(mask, off, utt)
    assert np.array_equal(ru.numpy(), utt[want[:, 0]]) and np.array_equal(rs.numpy(), want[:, 1])
    assert np.array_equal(rb.lengths, want[:, 2] - want[:, 1])
    rows = np.concatenate([np.arange(off[u] + a, off[u] + b) for u, a, b in zip(utt[want[:, 0]], want[:, 1], want[:, 2])])
    assert torch.equal(rb.feats, feats[torch.from_numpy(rows).cuda()])
    print(f"\n{n} frames, {want.shape[0]} runs in {utt.size} utterances")


# ---- diarize and embed with speech --------------------------------------------------------------------------------------
def _model():
    sd = RO.make_state_dict(0, num_classes=16)
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(sd)
    return m.eval()


def _relabel(lab):
    lab = np.asarray(lab)
    _, first = np.unique(lab, return_index=True)
    order = np.argsort(first)
    remap = np.empty(order.size, np.int64)
    remap[order] = np.arange(order.size)
    return remap[np.searchsorted(np.unique(lab), lab)].astype(np.int32)


def _host_diarize(model, feats_h, off, mask, utt, T, hop, k=None, t=None):
    """numpy-selected run bank -> window_embeddings -> scipy linkage + fcluster -> brute-force per-run labels."""
    runs = _runs_numpy(mask, off, utt)
    arrs = [feats_h[off[utt[j]] + a:off[utt[j]] + b] for j, a, b in runs]
    rb = F.FeatureBank.from_arrays(arrs)
    emb, _, ws, wo = F.window_embeddings(model, rb, np.arange(len(arrs)), T, hop)
    out = []
    for r, u in enumerate(utt):
        ri = np.flatnonzero(runs[:, 0] == r)
        n = int(off[u + 1] - off[u])
        if ri.size == 0:
            out.append((np.full(n, -1, np.int32), []))
            continue
        a, b = int(wo[ri[0]]), int(wo[ri[-1] + 1])
        if b - a == 1:
            wl = np.zeros(1, np.int32)
        else:
            E = emb[a:b]
            Zs = scipy_linkage(squareform(AO.distances(EN.cosine_matrix(E, E).cpu().numpy()), checks=False), "average")
            wl = _relabel(fcluster(Zs, min(k, b - a), "maxclust") if k is not None else fcluster(Zs, t, "distance"))
        run_ws = [ws[int(wo[i]):int(wo[i + 1])].numpy() for i in ri]
        run_wl = [wl[int(wo[i]) - a:int(wo[i + 1]) - a] for i in ri]
        fl = VO.frame_labels_runs_brute([(runs[i, 1], runs[i, 2]) for i in ri], run_ws, run_wl, n, T)
        segs = [sg for sg in AO.segments_brute(fl) if sg[2] >= 0]
        out.append((fl, segs))
    return out


def test_diarize_with_all_speech_equals_diarize(cuda_dev):
    g = np.random.RandomState(8)
    lens = [3000, 100, 1777, 161, 2400]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model()
    utt = [4, 0, 1, 2, 3]
    every = torch.ones(bank.feats.shape[0], dtype=torch.bool, device=cuda_dev)
    for kw in ({"num_speakers": 3}, {"threshold": 0.05}):
        a = DZ.diarize(model, bank, utt, **kw)
        b = DZ.diarize(model, bank, utt, speech=every, **kw)
        for x, y in zip(a, b):
            assert np.array_equal(x.Z, y.Z) and np.array_equal(x.window_labels, y.window_labels)
            assert np.array_equal(x.frame_labels, y.frame_labels) and x.segments == y.segments


def test_diarize_with_speech_matches_a_host_recomposition(cuda_dev):
    g = np.random.RandomState(9)
    lens = [3000, 700, 2500, 400, 1800]
    feats_h = [g.randn(n, 64).astype(np.float32) for n in lens]
    bank = F.FeatureBank.from_arrays(feats_h)
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    fh = np.concatenate(feats_h)
    rng = np.random.default_rng(1)
    mask = np.zeros(off[-1], bool)
    for u in (0, 2, 4):                         # runs of 20-900 frames (many shorter than T) with gaps
        f = 0
        while f < lens[u]:
            run, gap = int(rng.integers(20, 900)), int(rng.integers(5, 300))
            mask[off[u] + f:off[u] + min(f + run, lens[u])] = True
            f += run + gap
    mask[off[1] + 100:off[1] + 130] = True       # recording 1: one 30-frame run; recording 3: no speech
    model = _model()
    utt = np.array([0, 1, 2, 3, 4, 2])
    emb0 = F.window_embeddings(model, F.FeatureBank.from_arrays(
        [fh[off[0] + a:off[0] + b] for _, a, b in _runs_numpy(mask, off, [0])]), np.arange(
        len(_runs_numpy(mask, off, [0]))), 160, 40)[0]
    Zf, _ = EN.ahc(EN.cosine_matrix(emb0, emb0))
    t = float(Zf[-4:-2, 2].mean())
    for kw in ({"k": 3}, {"t": t}):
        got = DZ.diarize(model, bank, utt, T=160, hop=40, num_speakers=kw.get("k"), threshold=kw.get("t"),
                         speech=torch.from_numpy(mask).cuda())
        ref = _host_diarize(model, fh, off, mask, utt, 160, 40, **kw)
        for r, (res, (fl, segs)) in enumerate(zip(got, ref)):
            assert np.array_equal(res.frame_labels, fl), (kw, r)
            assert res.segments == segs, (kw, r)
            m = mask[off[utt[r]]:off[utt[r] + 1]]
            assert np.all((res.frame_labels >= 0) == m), (kw, r)
            for a, b, k in res.segments:
                assert k >= 0 and m[int(round(a / 0.01)):int(round(b / 0.01))].all()
        assert got[3].segments == [] and np.all(got[3].frame_labels == -1) and got[3].window_labels.size == 0
        assert "spk-1" not in DZ.to_rttm(got[0].segments, "rec0")
        print(f"\n{kw}: speakers per recording {[int(x.window_labels.max()) + 1 if x.window_labels.size else 0 for x in got]}")
    none = DZ.diarize(model, bank, [3], num_speakers=2, speech=np.zeros(off[-1], bool))
    assert none[0].segments == [] and np.all(none[0].frame_labels == -1)
    with pytest.raises(ValueError, match="hop"):
        big = F.FeatureBank.from_arrays([np.zeros((40000, 64))])
        DZ.diarize(model, big, [0], hop=1, num_speakers=2, speech=np.ones(40000, bool))


def test_embed_utterances_on_selected_speech(cuda_dev):
    g = np.random.RandomState(5)
    lens = [500, 161, 2000, 90]
    arrs = [g.randn(n, 64).astype(np.float32) for n in lens]
    bank = F.FeatureBank.from_arrays(arrs)
    mask = g.rand(sum(lens)) < 0.7
    off = np.concatenate(([0], np.cumsum(lens)))
    model = _model()
    utt = [2, 0, 3, 1]
    got = F.embed_utterances(model, bank.select(mask), utt)
    ref = F.embed_utterances(model, F.FeatureBank.from_arrays([a[mask[off[u]:off[u + 1]]] for u, a in enumerate(arrs)]), utt)
    assert torch.equal(got, ref)
