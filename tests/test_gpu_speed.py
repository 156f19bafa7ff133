"""Speed perturbation on the GPU: the resampled segments against the fp64 oracle (oracle/speed_oracle.py) for every
factor and segment length, unit factors as the plain gather bit for bit, speed followed by reverb and noise, per-example
independence, NaN examples, host-memory banks, CUDA-graph capture and a classification step on speed-extended labels.

Parity gate, per sample: |y - y64| <= 1/2 ulp(y64) + 50 * 2^-53 * sum_d |h x| * 2^-15, y64 the fp64 sum of the
definition.  Every product h x of an fp32 tap and an int16 sample is exact in fp64, so the only roundings are the 49
additions and the final one to fp32; the engine adds in the definition's order, so it is also checked to be fp32(y64)
bit for bit.
"""
import gc
from fractions import Fraction

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import frontend as F
from oracle import augment_oracle as A
from oracle import rescnn_oracle as O
from oracle import speed_oracle as S

pytestmark = pytest.mark.gpu

T = 160
LS = 25840
FACTORS = (Fraction(1, 2), Fraction(9, 10), Fraction(19, 20), Fraction(11, 10), Fraction(2))


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
    yield
    _CACHE.clear()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _speech():
    if "speech" not in _CACHE:
        g = np.random.default_rng(20)
        lens = np.concatenate(([1, 3, 49, 100, 1023, LS - 1, LS, LS + 1], g.integers(16000, 160000, 40)))
        waves = [_pcm(n, i) for i, n in enumerate(lens)]
        waves[3][:3] = [-32768, 32767, 0]                    # the int16 extremes
        soff = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
        _CACHE["speech"] = (F.WaveBank.from_waveforms(waves), waves, np.concatenate(waves), soff)
    return _CACHE["speech"]


def _noise():
    if "noise" not in _CACHE:
        g = np.random.default_rng(21)
        waves = [np.round(g.normal(0, 0.1, n).clip(-1, 32767 / 32768) * 32768).astype(np.int16)
                 for n in g.integers(4000, 200000, 12)]
        _CACHE["noise"] = (F.WaveBank.from_waveforms(waves), waves)
    return _CACHE["noise"]


def _rirs():
    if "rirs" not in _CACHE:
        g = np.random.default_rng(22)
        arrs = [g.normal(size=lh) * np.exp(-np.arange(lh) / 800.0) for lh in (1, 1024, 1025, 8000, 16000)]
        rb = F.RirBank.from_arrays(arrs)
        _CACHE["rirs"] = (rb, [rb.samples[rb.offsets[i]:rb.offsets[i + 1]].cpu().numpy() for i in range(rb.num_rirs)])
    return _CACHE["rirs"]


def _dev(plan):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in plan.items()}


def _sub(plan, idx):
    return {k: (v[idx] if isinstance(v, torch.Tensor) else v) for k, v in plan.items()}


def _check_parity(got, bank, soff, utt, start, L_, alpha):
    """The gate of the module docstring and fp32(y64) bit for bit, per example; returns the worst err / gate."""
    worst = 0.0
    for b in range(len(utt)):
        u = int(utt[b])
        x = bank[soff[u]:soff[u + 1]]
        acc, mag = S.resample_sum(x, alpha, int(start[b]), L_)
        y64 = acc * 2.0 ** -15
        gate = 0.5 * np.spacing(np.abs(y64).astype(np.float32)).astype(np.float64) + 50 * 2.0 ** -53 * mag * 2.0 ** -15
        err = np.abs(got[b].astype(np.float64) - y64)
        assert np.all(err <= gate), (str(alpha), L_, b, u, int(start[b]), (err / gate).max())
        assert np.array_equal(got[b].view(np.int32), y64.astype(np.float32).view(np.int32)), (str(alpha), L_, b)
        worst = max(worst, float((err / gate).max()))
    return worst


# ---- 1. parity with the oracle -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("L_", [1, 1023, 1024, LS])
def test_speed_segments_match_the_oracle(cuda_dev, L_):
    sb, waves, bank, soff = _speech()
    U = sb.num_utterances
    g = np.random.default_rng(L_)
    utt = np.concatenate((np.arange(U), np.arange(8), g.integers(0, U, 8)))
    start = np.concatenate((np.zeros(U, np.int64), sb.lengths[:8] - 1, [g.integers(0, sb.lengths[u]) for u in utt[U + 8:]]))
    B = utt.size
    for k, alpha in enumerate(FACTORS):
        plan = {"speed_idx": torch.full((B,), k, dtype=torch.int64), "speeds": FACTORS}
        got = sb.segments(torch.from_numpy(utt), torch.from_numpy(start), L_, plan).cpu().numpy()
        worst = _check_parity(got, bank, soff, utt, start, L_, alpha)
        print(f"\nL = {L_}, alpha = {alpha}: max err / gate {worst:.3f}")


def test_speed_segments_match_the_oracle_past_3_2_20_samples(cuda_dev):
    sb, waves, bank, soff = _speech()
    L_ = 3 * 2 ** 20 + 5
    utt = np.array([10, 6, 20, 4, 30])
    start = np.array([0, LS - 1, 12345, 1022, 7])
    B = utt.size
    plan = {"speed_idx": torch.arange(B), "speeds": FACTORS}
    got = sb.segments(torch.from_numpy(utt), torch.from_numpy(start), L_, plan).cpu().numpy()
    for b, alpha in enumerate(FACTORS):
        _check_parity(got[b:b + 1], bank, soff, utt[b:b + 1], start[b:b + 1], L_, alpha)


def test_unit_factor_is_the_plain_gather_bit_for_bit(cuda_dev):
    sb, _, _, _ = _speech()
    B = 200
    g = np.random.default_rng(3)
    utt = torch.from_numpy(g.integers(0, sb.num_utterances, B))
    start = torch.from_numpy(np.array([g.integers(0, sb.lengths[u]) for u in utt.numpy()]))
    for L_ in (1, 1000, LS):
        plain = sb.segments(utt, start, L_)
        for speeds in ((1,), (Fraction(9, 10), 1, 2)):
            unit = speeds.index(1)
            for idx in (torch.full((B,), unit), torch.full((B,), -1)):
                got = sb.segments(utt.cuda(), start.cuda(), L_, {"speed_idx": idx.cuda(), "speeds": speeds})
                assert _bits_equal(got, plain), (L_, speeds)
        # mixed: the unit and -1 rows are the plain gather, the others the perturbed segments
        idx = torch.from_numpy(g.integers(-1, 3, B))
        speeds = (Fraction(9, 10), 1, 2)
        got = sb.segments(utt, start, L_, {"speed_idx": idx, "speeds": speeds})
        keep = (idx == -1) | (idx == 1)
        assert _bits_equal(got[keep], plain[keep])
        for k in (0, 2):
            rows = idx == k
            alone = sb.segments(utt[rows], start[rows], L_, {"speed_idx": torch.zeros(int(rows.sum()), dtype=torch.int64),
                                                             "speeds": (speeds[k],)})
            assert _bits_equal(got[rows], alone)


# ---- 2. speed, then reverb and noise -----------------------------------------------------------------------------------
def test_speed_then_reverb_and_noise_against_the_oracle(cuda_dev):
    sb, waves, bank, soff = _speech()
    rb, hs = _rirs()
    nb, nwaves = _noise()
    g = np.random.default_rng(7)
    B, M = 30, 3
    speeds = (Fraction(9, 10), 1, Fraction(11, 10))
    utt = torch.from_numpy(g.integers(8, sb.num_utterances, B))
    si = torch.from_numpy(g.integers(-1, 3, B))
    ri = torch.from_numpy(g.integers(0, rb.num_rirs, B))
    plan = {"speed_idx": si, "speeds": speeds}
    start = sb.random_starts(utt, LS, g, plan)
    q = g.integers(0, nb.num_utterances, (B, M))
    q[np.arange(M)[None, :] >= (np.arange(B) % (M + 1))[:, None]] = -1
    ns = np.where(q >= 0, [[g.integers(0, nb.lengths[max(v, 0)]) for v in row] for row in q], 0)
    snr = g.uniform(0, 20, (B, M))
    s = sb.segments(utt, start, LS, plan).cpu().numpy()
    r = sb.segments(utt, start, LS, dict(plan, rir_idx=ri), rb).cpu().numpy()
    full = dict(plan, rir_idx=ri, noise_idx=torch.from_numpy(q), noise_start=torch.from_numpy(ns),
                snr_db=torch.from_numpy(snr))
    got = sb.segments(utt, start, LS, full, rb, nb).cpu().numpy()
    nbank, noff = np.concatenate(nwaves), np.concatenate(([0], np.cumsum([w.size for w in nwaves])))
    worst = [0.0, 0.0, 0.0]
    for b in range(B):
        k = int(si[b])
        alpha = None if k < 0 else speeds[k]
        s64 = S.speed(bank, soff, int(utt[b]), int(start[b]), LS, alpha)
        assert np.array_equal(s[b], s64.astype(np.float32))
        elem, blk = A.reverb_error_ratios(r[b], s[b], hs[int(ri[b])])
        assert elem <= 1.0 and blk <= 1.0, (b, elem, blk)
        srcs = [A.gather(nbank, noff, q[b, j], ns[b, j], LS) for j in range(M) if q[b, j] >= 0]
        want = A.mix(r[b].astype(np.float64), srcs, [snr[b, j] for j in range(M) if q[b, j] >= 0])
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        err = np.abs(got[b].astype(np.float64) - want)
        assert np.all(err <= ulp), (b, (err / ulp).max())
        worst = [max(worst[0], elem), max(worst[1], blk), max(worst[2], (err / ulp).max())]
    # the oracle's composition agrees with the engine within the same bounds (speed, reverb, mix in fp64)
    b = int(np.nonzero(si.numpy() >= 0)[0][0])
    want = S.augment(bank, soff, int(utt[b]), int(start[b]), LS, speeds[int(si[b])], hs[int(ri[b])], nbank, noff,
                     q[b], ns[b], snr[b])
    assert np.abs(got[b] - want).max() <= 1e-4 * np.abs(want).max()
    print(f"\nreverb err / bound {worst[0]:.3f} per sample, {worst[1]:.3f} per block; mix {worst[2]:.3f} ulp")


# ---- 3. independence, NaN examples, host banks -------------------------------------------------------------------------
def _case(B, seed):
    sb, _, _, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    g = np.random.default_rng(seed)
    utt = g.integers(0, sb.num_utterances, B)
    plan = F.augment_plan(B, LS, g, rb, 0.5, nb, [(range(nb.num_utterances), (0.0, 15.0), (1, 3), 1.0)], 0.6,
                          speeds=(0.9, 1.0, 1.1))
    start = sb.random_starts(utt, LS, g, plan)
    return torch.from_numpy(utt), start, plan


def test_each_example_is_bit_identical_in_any_batch(cuda_dev):
    sb, _, _, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    utt, start, plan = _case(384, 31)
    tm, fm = F.spec_augment_masks(384, T, 2, 30, 2, 10, np.random.default_rng(2))
    full = sb.augmented_crops(utt, start, T, plan, rb, nb, tm, fm)
    assert torch.isfinite(full).all()
    for B in (1, 7):
        for i in range(0, 384 - B + 1, 53):
            idx = torch.arange(i, i + B)
            part = sb.augmented_crops(utt[idx], start[idx], T, _sub(plan, idx), rb, nb, tm[idx], fm[idx])
            assert _bits_equal(part, full[idx]), (B, i)
    perm = torch.from_numpy(np.random.default_rng(3).permutation(384))
    assert _bits_equal(sb.augmented_crops(utt[perm], start[perm], T, _sub(plan, perm), rb, nb, tm[perm], fm[perm]),
                       full[perm])
    from deepspeaker_pytorch_b200 import engine

    g = torch.Generator(device="cuda").manual_seed(0)
    E = torch.nn.functional.normalize(torch.randn(384, 512, device="cuda", generator=g), dim=1)
    W = torch.nn.functional.normalize(torch.randn(100, 512, device="cuda", generator=g), dim=1)
    other = dict(plan, speed_idx=torch.zeros(384, dtype=torch.int64), speeds=(2,))
    for _ in range(3):
        engine.aam_softmax(E, W, torch.arange(384, device="cuda") % 100, 0.2, 30.0)
        sb.segments(utt, start, 5000, other, rb, nb)                 # another factor table in between
        assert _bits_equal(sb.augmented_crops(utt, start, T, plan, rb, nb, tm, fm), full)


def test_bad_speed_index_or_table_row_gives_nan_examples(cuda_dev):
    sb, _, _, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    B = 48
    utt, start, plan = _case(B, 41)
    dplan = _dev(plan)
    clean = sb.segments(utt.cuda(), start.cuda(), LS, dplan, rb, nb)
    si = plan["speed_idx"].clone()
    si[0], si[1], si[2] = 3, -2, 2 ** 40
    got = sb.segments(utt.cuda(), start.cuda(), LS, dict(dplan, speed_idx=si.cuda()), rb, nb)
    assert torch.isnan(got[:3]).all()
    assert _bits_equal(got[3:], clean[3:])
    with pytest.raises(ValueError):                      # CPU indices are checked on the host
        sb.segments(utt, start, LS, dict(plan, speed_idx=si))
    # a table whose ratios are outside the limits: rows 0 (3/1) and 2 (18/20, not in lowest terms)
    speeds = (Fraction(9, 10), Fraction(1), Fraction(11, 10))
    ratio, taps = F._speed_table(torch.device("cuda", torch.cuda.current_device()), speeds)
    bad = ratio.clone()
    bad[0] = torch.tensor([3, 1], dtype=torch.int32)
    bad[2] = torch.tensor([18, 20], dtype=torch.int32)
    k = torch.from_numpy(np.arange(B) % 4 - 1).cuda()     # -1, 0, 1, 2
    u, s = utt.cuda(), start.cuda()

    def run(rt):
        out = torch.empty(B, LS, device="cuda")
        L.check(L.load().dsk_wave_augment_speed(sb.samples.data_ptr(), sb.offsets.data_ptr(), sb.num_utterances,
                                                u.data_ptr(), s.data_ptr(), B, LS, None, None, 0, 1, None, None, None,
                                                0, 0, None, None, None, rt.data_ptr(), taps.data_ptr(), 3, k.data_ptr(),
                                                out.data_ptr(), L.cur_stream()), "dsk_wave_augment_speed")
        return out

    good, worse = run(ratio), run(bad)
    nan_rows = (k == 0) | (k == 2)
    assert torch.isfinite(good).all() and torch.isnan(worse[nan_rows]).all()
    assert _bits_equal(worse[~nan_rows], good[~nan_rows])


def test_pinned_host_banks_give_the_same_bits(cuda_dev):
    sb, waves, _, _ = _speech()
    rb, _ = _rirs()
    nb, nwaves = _noise()
    sbh = F.WaveBank.from_waveforms(waves, pin=True)
    rbh = F.RirBank(rb.samples.cpu().pin_memory(), rb.offsets.cpu().numpy())
    nbh = F.WaveBank.from_waveforms(nwaves, pin=True)
    utt, start, plan = _case(96, 51)
    assert _bits_equal(sb.augmented_crops(utt, start, T, plan, rb, nb), sbh.augmented_crops(utt, start, T, plan, rbh, nbh))


# ---- 4. graph capture and training -------------------------------------------------------------------------------------
def test_capture_in_a_cuda_graph(cuda_dev):
    sb, _, _, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    utt, start, plan = _case(32, 61)
    tm, fm = F.spec_augment_masks(32, T, 2, 30, 2, 10, np.random.default_rng(9))
    args = [utt.cuda(), start.cuda(), T, _dev(plan), rb, nb, tm.cuda(), fm.cuda()]
    eager = sb.augmented_crops(*args)
    assert eager.shape == (32, 1, T, 64)
    seg = sb.segments(utt, start, LS, plan, rb, nb)
    bank = F.FeatureBank(*F.mk_mfb_batch(seg.reshape(-1), [LS] * 32))
    assert _bits_equal(eager, bank.crops(torch.arange(32), torch.zeros(32, dtype=torch.int64), T, tm, fm))
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


def test_aam_softmax_step_on_speed_extended_labels(cuda_dev):
    sb, _, _, _ = _speech()
    rb, _ = _rirs()
    nb, _ = _noise()
    C, K = 16, 4
    g = np.random.default_rng(71)
    utt = np.repeat(g.choice(sb.num_utterances, C, replace=False), K)
    plan = F.augment_plan(C * K, LS, g, rb, 0.5, nb, [(range(nb.num_utterances), (5.0, 15.0), (1, 1), 1.0)], 0.5,
                          speeds=(0.9, 1.0, 1.1))
    start = sb.random_starts(utt, LS, g, plan)
    tm, fm = F.spec_augment_masks(C * K, T, 2, 20, 2, 8, g)
    x = sb.augmented_crops(torch.from_numpy(utt), start, T, plan, rb, nb, tm, fm)
    labels = F.speed_labels(torch.from_numpy(np.repeat(np.arange(C), K)), plan, C)
    assert labels.min() >= 0 and labels.max() < 3 * C and (labels >= C).any()
    model = dsk.DeepSpeakerModel(512, 3 * C).cuda()
    model.load_state_dict(O.make_state_dict(0, num_classes=3 * C))
    model.train()
    opt = dsk.FusedAdagrad(model.parameters(), lr=1e-2, lr_decay=1e-4)
    out = dsk.aam_softmax_step(model, opt, x, labels, margin=0.2, scale=30.0)
    assert torch.isfinite(out["loss"]).all()
    del model, opt, out
    gc.collect()
