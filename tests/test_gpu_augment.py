"""Waveform augmentation on the GPU: segments against a numpy gather, reverberation and mixing against the fp64 oracle
(oracle/augment_oracle.py), augmented crops against the feature-bank path bit for bit, per-example independence, NaN
examples, host-memory banks, CUDA-graph capture, and the training steps fed from augmented crops.

Reverberation error bound.  The engine computes r = s * h (truncated to L) by uniformly partitioned overlap-save with
P = 1024 and fp32 complex FFTs of N = 2P points: output block k (samples [kP, (k+1)P)) is the last P samples of
IFFT(sum_{p <= k} X_{k-p} H_p), X_j = FFT(x_j), x_j = s[(j-1)P .. (j+1)P) (zero outside [0, L)), H_p = FFT(h_p zero-padded),
h_p = h[pP .. (p+1)P).  A radix-2 FFT computed in floating point with unit roundoff u and twiddles accurate to O(u)
satisfies ||fl(FFT x) - FFT x||_2 <= log2(N) eta ||FFT x||_2 with eta = O(u) (Higham, Accuracy and Stability of
Numerical Algorithms, Thm 24.2), and ||FFT x||_2 = sqrt(N) ||x||_2.  Each partition term passes through two forward
transforms, one product and (within the summed spectrum) one inverse transform, so its contribution to block k is an
error of order log2(N) u ||x_{k-p}||_2 ||h_p||_2 once the 1/N of the inverse and Parseval are applied, and the partition
sum adds the terms.  Hence the gates, for every output sample i of block k and for the block as a whole,
    |r_i - y_i| <= bound_k   and   ||r_k - y_k||_2 <= bound_k,   bound_k = log2(N) u sum_{p <= k} ||x_{k-p}||_2 ||h_p||_2,
y the fp64 convolution of the engine's own segment s and the RIR as stored (u = 2^-24, N = 2048).  The worst case over
all inputs carries a further factor ||h_p||_1 / ||h_p||_2 <= sqrt(P) (the error spectrum aligned with the peak of |H_p|);
the gates omit it, as rounding errors are not aligned with the spectrum, and a CPU fp32 emulation of the same algorithm
stays below 0.05 (per sample) and 0.2 (per block) of them.  They are still tight enough to catch a dropped partition, a
misaligned X/H pairing, a one-sample shift, a zeroed block or a wrong twiddle sign: tests/test_augment_host.py seeds each
of these into the emulation and checks that the gates fail.
"""
import gc

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import frontend as F
from oracle import augment_oracle as A
from oracle import fbank_oracle as FO
from oracle import rescnn_oracle as O

pytestmark = pytest.mark.gpu

T = 160
LS = 25840


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _pcm(n, seed, amp=0.3):
    g = np.random.default_rng(seed)
    t = np.arange(n) / 16000
    x = amp * np.sin(2 * np.pi * (200 + 50 * (seed % 7)) * t) * (1 + 0.5 * np.sin(2 * np.pi * 3 * t)) + g.normal(0, 0.05, n)
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """The banks are shared by the module's tests; when they are done, free them and every model the tests built (an
    Engine and its module reference each other, so only the cycle collector frees a model's train contexts) so later
    test modules get the device memory back."""
    yield
    _CACHE.clear()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _speech():
    if "speech" not in _CACHE:
        g = np.random.default_rng(10)
        lens = np.concatenate(([1, 100, 1023, LS - 1, LS, LS + 1], g.integers(16000, 160000, 120)))
        waves = [_pcm(n, i) for i, n in enumerate(lens)]
        waves[1][:3] = [-32768, 32767, 0]                    # the int16 extremes
        _CACHE["speech"] = (F.WaveBank.from_waveforms(waves), waves)
    return _CACHE["speech"]


def _noise():
    if "noise" not in _CACHE:
        g = np.random.default_rng(11)
        waves = [g.normal(0, 0.1 * (1 + i % 3), n).clip(-1, 32767 / 32768) for i, n in
                 enumerate(g.integers(4000, 200000, 30))]
        waves = [np.round(w * 32768).astype(np.int16) for w in waves]
        waves.append(np.zeros(30000, np.int16))              # a zero-energy source: gain 0
        _CACHE["noise"] = (F.WaveBank.from_waveforms(waves), waves)
    return _CACHE["noise"]


def _rir(lh, kind, seed):
    g = np.random.default_rng(seed)
    h = g.normal(size=lh)
    if kind == "decay":
        h *= np.exp(-np.arange(lh) / 800.0)
    return h


def _rirs():
    if "rirs" not in _CACHE:
        arrs = [_rir(lh, kind, i) for i, (lh, kind) in enumerate(
            [(lh, kind) for lh in (1, 2, 1023, 1024, 1025, 8000, 16000, 65536) for kind in ("flat", "decay")])]
        rb = F.RirBank.from_arrays(arrs)
        _CACHE["rirs"] = (rb, [rb.samples[rb.offsets[i]:rb.offsets[i + 1]].cpu().numpy() for i in range(rb.num_rirs)])
    return _CACHE["rirs"]


def _groups(nb):
    n = nb.num_utterances
    return [(range(0, 10), (0.0, 15.0), (1, 1), 1.0), (range(10, 20), (5.0, 15.0), (1, 1), 1.0),
            (range(20, n - 1), (13.0, 20.0), (3, 8), 1.0)]


def _case(B, seed, p_reverb=0.7, p_noise=0.8, L=LS):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    g = np.random.default_rng(seed)
    utt = g.integers(0, sb.num_utterances, B)
    start = sb.random_starts(utt, L, g)
    plan = F.augment_plan(B, L, g, rb, p_reverb, nb, _groups(nb), p_noise)
    return torch.from_numpy(utt), start, plan


# ---- 1. segments --------------------------------------------------------------------------------------------------------
def test_clean_segments_are_a_numpy_gather(cuda_dev):
    sb, waves = _speech()
    g = np.random.default_rng(1)
    B = 64
    utt = g.integers(0, sb.num_utterances, B)
    start = sb.random_starts(utt, LS, g).numpy()
    utt[:8] = [0, 1, 1, 2, 3, 4, 5, 5]
    start[:8] = [0, 0, 99, 1022, 0, LS - 1, 0, LS]       # short utterances wrap; starts near the end wrap
    for L in (LS, 1000, 1):
        got = sb.segments(torch.from_numpy(utt), torch.from_numpy(start), L).cpu().numpy()
        for b in range(B):
            w = waves[utt[b]]
            want = (w[(start[b] + np.arange(L)) % w.size].astype(np.float32) * np.float32(2.0 ** -15))
            assert np.array_equal(got[b].view(np.int32), want.view(np.int32)), (b, L)
    assert got.dtype == np.float32
    x = sb.segments(torch.tensor([1]), torch.tensor([0]), 3).cpu().numpy()[0]
    assert x.tolist() == [-1.0, 32767 / 32768, 0.0]


def test_an_utterance_past_sample_2_31(cuda_dev):
    w = _pcm(30000, 99)
    n0 = 2 ** 31 + 5
    samples = torch.zeros(n0 + w.size, dtype=torch.int16, device="cuda")
    samples[n0:] = torch.from_numpy(w).cuda()
    sb = F.WaveBank(samples, [0, 2 ** 30, n0, n0 + w.size])
    got = sb.segments(torch.tensor([2, 2]), torch.tensor([0, 29000]), LS).cpu().numpy()
    for b, s in enumerate((0, 29000)):
        want = w[(s + np.arange(LS)) % w.size].astype(np.float32) / np.float32(32768)
        assert np.array_equal(got[b], want)
    del samples, sb
    torch.cuda.empty_cache()


# ---- 2. reverberation ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [LS, 4096, 3000])
def test_reverb_within_the_fft_error_bound(cuda_dev, L):
    sb, _ = _speech()
    rb, hs = _rirs()
    R = rb.num_rirs
    g = np.random.default_rng(L)
    utt = torch.from_numpy(g.integers(6, sb.num_utterances, R))
    start = sb.random_starts(utt, L, g)
    s = sb.segments(utt, start, L).cpu().numpy()
    r = sb.segments(utt, start, L, {"rir_idx": torch.arange(R)}, rb).cpu().numpy()
    worst = (0.0, 0.0)
    for i in range(R):
        elem, blk = A.reverb_error_ratios(r[i], s[i], hs[i])
        assert elem <= 1.0 and blk <= 1.0, (L, hs[i].size, i, elem, blk)
        worst = (max(worst[0], elem), max(worst[1], blk))
    print(f"\nL = {L}: max err / bound per sample {worst[0]:.3f}, per block (L2) {worst[1]:.3f}")
    # rir_idx = -1 leaves the segment exactly
    r0 = sb.segments(utt, start, L, {"rir_idx": torch.full((R,), -1)}, rb).cpu().numpy()
    assert np.array_equal(r0.view(np.int32), s.view(np.int32))


# ---- 3. mixing -------------------------------------------------------------------------------------------------------
def test_mix_within_one_ulp_of_fp64(cuda_dev):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, nwaves = _noise()
    zero = nb.num_utterances - 1
    g = np.random.default_rng(5)
    B, M = 36, 8
    utt = torch.from_numpy(g.integers(6, sb.num_utterances, B))
    start = sb.random_starts(utt, LS, g)
    rir_idx = torch.from_numpy(np.where(np.arange(B) % 2 == 0, g.integers(0, rb.num_rirs, B), -1))
    q = g.integers(0, zero, (B, M))
    cnt = np.arange(B) % (M + 1)                               # M = 0 .. 8 sources
    q[np.arange(M)[None, :] >= cnt[:, None]] = -1
    q[10, 1] = zero                                            # a zero-energy source
    ns = np.zeros((B, M), np.int64)
    for b in range(B):
        for j in range(M):
            if q[b, j] >= 0:
                ns[b, j] = g.integers(0, nb.lengths[q[b, j]])
    snr = g.uniform(-5, 40, (B, M))
    snr[:, 0] = np.where(np.arange(B) % 3 == 0, -5.0, np.where(np.arange(B) % 3 == 1, 40.0, snr[:, 0]))
    plan = {"rir_idx": rir_idx, "noise_idx": torch.from_numpy(q), "noise_start": torch.from_numpy(ns),
            "snr_db": torch.from_numpy(snr)}
    r = sb.segments(utt, start, LS, {"rir_idx": rir_idx}, rb).cpu().numpy()     # the engine's r, pinned
    got = sb.segments(utt, start, LS, plan, rb, nb).cpu().numpy()
    worst = 0.0
    nbank, noff = np.concatenate(nwaves), np.concatenate(([0], np.cumsum([w.size for w in nwaves])))
    for b in range(B):
        srcs = [A.gather(nbank, noff, q[b, j], ns[b, j], LS) for j in range(M) if q[b, j] >= 0]
        want = A.mix(r[b].astype(np.float64), srcs, [snr[b, j] for j in range(M) if q[b, j] >= 0])
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        err = np.abs(got[b].astype(np.float64) - want)
        assert np.all(err <= ulp), (b, cnt[b], (err / ulp).max())
        worst = max(worst, (err / ulp).max())
        if cnt[b] == 0:
            assert np.array_equal(got[b].view(np.int32), r[b].view(np.int32))
    print(f"\nmix: max err {worst:.3f} fp32 ulp")


# ---- 4. features -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", [16000, 8000])
@pytest.mark.parametrize("log_scale,sub_mean", [(True, True), (True, False), (False, True), (False, False)])
def test_augmented_crops_are_the_feature_bank_crops_of_the_segments(cuda_dev, sr, log_scale, sub_mean):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    B = 48
    Ls = F.segment_samples(T, sr)
    utt, start, plan = _case(B, 7, L=Ls)
    tm, fm = F.spec_augment_masks(B, T, 2, 30, 2, 10, np.random.default_rng(8))
    got = sb.augmented_crops(utt, start, T, plan, rb, nb, tm, fm, sr, log_scale, sub_mean)
    seg = sb.segments(utt, start, Ls, plan, rb, nb)
    bank = F.FeatureBank(*F.mk_mfb_batch(seg.reshape(-1), [Ls] * B, sr, log_scale, sub_mean))
    want = bank.crops(torch.arange(B), torch.zeros(B, dtype=torch.int64), T, tm, fm)
    assert got.shape == (B, 1, T, 64) and _bits_equal(got, want)
    if sr == 16000 and log_scale and not sub_mean:
        # within the fbank gates of tests/test_fbank.py on the oracle's augmented audio
        sbh, waves = _speech()
        soff = np.concatenate(([0], np.cumsum([w.size for w in waves])))
        seg_np = seg.cpu().numpy()
        for b in range(0, B, 6):
            x = seg_np[b]
            ref_lin, _ = FO.fbank(x.astype(np.float64), samplerate=sr, nfilt=64)
            got_lin = sb.augmented_crops(utt[b:b + 1], start[b:b + 1], T, {k: v[b:b + 1] for k, v in plan.items()}, rb, nb,
                                         sample_rate=sr, use_logscale=False, subtract_mean=False)[0, 0].cpu().numpy()
            scale = np.maximum(ref_lin.max(axis=1, keepdims=True), 1e-12)
            assert (np.abs(got_lin - ref_lin) / scale).max() < 2e-5
            ref = FO.mk_mfb(x.astype(np.float64), sr)
            gm = sb.augmented_crops(utt[b:b + 1], start[b:b + 1], T, {k: v[b:b + 1] for k, v in plan.items()}, rb, nb,
                                    sample_rate=sr)[0, 0].cpu().numpy()
            loud = ref_lin > 1e-3 * scale
            assert np.abs(gm - ref)[loud].max() < 1e-2 and np.abs(gm - ref).max() < 0.5
            if plan["rir_idx"][b] < 0 and (plan["noise_idx"][b] < 0).all():
                assert np.array_equal(x, A.gather(np.concatenate(waves).astype(np.int16), soff, int(utt[b]),
                                                  int(start[b]), Ls).astype(np.float32))


# ---- 5. independence ---------------------------------------------------------------------------------------------------
def _sub(plan, idx):
    return {k: v[idx] for k, v in plan.items()}


def test_each_example_is_bit_identical_in_any_batch(cuda_dev):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    utt, start, plan = _case(384, 21)
    tm, fm = F.spec_augment_masks(384, T, 2, 30, 2, 10, np.random.default_rng(2))
    full = sb.augmented_crops(utt, start, T, plan, rb, nb, tm, fm)
    assert torch.isfinite(full).all()
    for B in (1, 7):
        for i in range(0, 384 - B + 1, 53):
            idx = torch.arange(i, i + B)
            part = sb.augmented_crops(utt[idx], start[idx], T, _sub(plan, idx), rb, nb, tm[idx], fm[idx])
            assert _bits_equal(part, full[idx]), (B, i)
    perm = torch.from_numpy(np.random.default_rng(3).permutation(384))
    permuted = sb.augmented_crops(utt[perm], start[perm], T, _sub(plan, perm), rb, nb, tm[perm], fm[perm])
    assert _bits_equal(permuted, full[perm])
    # repeated runs, with other ops' calls interleaved
    from deepspeaker_pytorch_b200 import engine, verification

    g = torch.Generator(device="cuda").manual_seed(0)
    E = torch.nn.functional.normalize(torch.randn(384, 512, device="cuda", generator=g), dim=1)
    W = torch.nn.functional.normalize(torch.randn(100, 512, device="cuda", generator=g), dim=1)
    lab = torch.arange(384, device="cuda") % 64
    ge2e = dsk.GE2ELoss(10.0, -5.0).cuda()
    for _ in range(3):
        engine.aam_softmax(E, W, lab % 100, 0.2, 30.0)
        ge2e(E, lab)
        verification.cohort_stats(E[:64], W, 50)
        assert _bits_equal(sb.augmented_crops(utt, start, T, plan, rb, nb, tm, fm), full)


def test_invalid_arguments_give_nan_examples(cuda_dev):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    B = 64
    utt, start, plan = _case(B, 31, p_reverb=0.5, p_noise=1.0)
    clean = sb.segments(utt.cuda(), start.cuda(), LS, {k: v.cuda() for k, v in plan.items()}, rb, nb)
    u, s = utt.clone(), start.clone()
    ri, ni, nst, snr = (plan[k].clone() for k in ("rir_idx", "noise_idx", "noise_start", "snr_db"))
    U, N = sb.num_utterances, nb.num_utterances
    u[0], u[1], u[2] = -1, U, 2 ** 40
    s[3], s[4] = -1, int(sb.lengths[int(u[4])])
    ri[5], ri[6] = rb.num_rirs, -2
    ni[7, 0], ni[8, 0] = N, -3
    nst[9, 0] = int(nb.lengths[int(ni[9, 0])])
    nst[10, 0] = -1
    snr[11, 0], snr[12, 0], snr[13, 0] = np.nan, np.inf, -np.inf
    bad = list(range(14))
    got = sb.segments(u.cuda(), s.cuda(), LS, {"rir_idx": ri.cuda(), "noise_idx": ni.cuda(), "noise_start": nst.cuda(),
                                               "snr_db": snr.cuda()}, rb, nb)
    assert torch.isnan(got[bad]).all()
    assert _bits_equal(got[14:], clean[14:])
    # a RIR longer than max_rir_len: a bank whose host-side limit is shorter than one of its RIRs
    short = F.RirBank(rb.samples, rb.offsets.cpu().numpy())
    short.max_len = 16000
    long_idx = int(np.nonzero(rb.lengths == 65536)[0][0])
    ri2 = torch.full((B,), 0, dtype=torch.int64)
    ri2[20] = long_idx
    got2 = sb.segments(utt.cuda(), start.cuda(), LS, {"rir_idx": ri2.cuda()}, short)
    ref2 = sb.segments(utt.cuda(), start.cuda(), LS, {"rir_idx": ri2.cuda()}, rb)
    assert torch.isnan(got2[20]).all()
    keep = [b for b in range(B) if b != 20]
    assert _bits_equal(got2[keep], ref2[keep])
    # CPU indices are checked on the host
    for kw in ({"utt": torch.tensor([U])}, {"start": torch.tensor([-1])}):
        with pytest.raises(ValueError):
            sb.segments(kw.get("utt", torch.tensor([3])), kw.get("start", torch.tensor([0])), LS)
    with pytest.raises(ValueError):
        sb.segments(utt, start, LS, {"rir_idx": ri}, rb)
    with pytest.raises(ValueError):
        sb.segments(utt, start, LS, {"noise_idx": ni, "noise_start": nst, "snr_db": snr}, None, nb)


# ---- 6. host-memory banks and graph capture ----------------------------------------------------------------------------
def test_pinned_host_banks_give_the_same_bits(cuda_dev):
    sb, waves = _speech()
    rb, hs = _rirs()
    nb, nwaves = _noise()
    sbh = F.WaveBank.from_waveforms(waves, pin=True)
    rbh = F.RirBank(rb.samples.cpu().pin_memory(), rb.offsets.cpu().numpy())
    nbh = F.WaveBank.from_waveforms(nwaves, pin=True)
    assert not sbh.samples.is_cuda and sbh.samples.is_pinned() and not rbh.samples.is_cuda
    utt, start, plan = _case(96, 41)
    dev = sb.augmented_crops(utt, start, T, plan, rb, nb)
    host = sbh.augmented_crops(utt, start, T, plan, rbh, nbh)
    assert _bits_equal(dev, host)
    with pytest.raises(ValueError):
        F.WaveBank(torch.from_numpy(np.concatenate(waves)), sbh.offsets.cpu().numpy())
    with pytest.raises(ValueError):
        F.RirBank(rb.samples.cpu(), rb.offsets.cpu().numpy())


def test_capture_in_a_cuda_graph(cuda_dev):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    utt, start, plan = _case(32, 51)     # small: memory allocated under capture stays in the graph memory pool
    tm, fm = F.spec_augment_masks(32, T, 2, 30, 2, 10, np.random.default_rng(9))
    args = [utt.cuda(), start.cuda(), T, {k: v.cuda() for k, v in plan.items()}, rb, nb, tm.cuda(), fm.cuda()]
    eager = sb.augmented_crops(*args)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        sb.augmented_crops(*args)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = sb.augmented_crops(*args)
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(out, eager)


# ---- 7. into the training steps ----------------------------------------------------------------------------------------
def _model():
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(O.make_state_dict(0, num_classes=16))
    return m.train()


def test_training_steps_from_augmented_crops(cuda_dev):
    sb, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    P, K = 32, 4
    g = np.random.default_rng(61)
    utt = np.repeat(g.choice(sb.num_utterances, P, replace=False), K)
    start = sb.random_starts(utt, LS, g)
    plan = F.augment_plan(P * K, LS, g, rb, 0.6, nb, _groups(nb), 0.8)
    tm, fm = F.spec_augment_masks(P * K, T, 2, 20, 2, 8, g)
    x = sb.augmented_crops(torch.from_numpy(utt), start, T, plan, rb, nb, tm, fm)
    labels = torch.from_numpy(np.repeat(np.arange(P), K))
    model = _model()
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-2, lr_decay=1e-4)
    out = dsk.batch_hard_step(model, opt, x, labels, margin=0.1)
    assert torch.isfinite(out["loss"]).all()
    model = _model()
    crit = dsk.GE2ELoss(10.0, -5.0).cuda()
    opt = dsk.FusedAdagrad(list(model.parameters()) + list(crit.parameters()), lr=1e-2, lr_decay=1e-4)
    out = dsk.ge2e_step(model, opt, x, labels, loss=crit)
    assert torch.isfinite(out["loss"]).all()
    del model, opt, crit, out
    gc.collect()
