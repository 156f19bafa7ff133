"""Feature-bank front-end on the GPU: the batched log-fbank against the one-waveform call, bit for bit; crops against a
numpy gather; crops into the network and the training steps; utterance embeddings against an fp64 mean."""
import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import frontend as F
from oracle import rescnn_oracle as O
from tests.test_fbank import synth

pytestmark = pytest.mark.gpu

FIXED = [1, 399, 400, 401, 560, 16000, 48000, 100003]


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- 1. batched fbank ------------------------------------------------------------------------------------------------
_WAVES = {}


def _waves(sr):
    if sr not in _WAVES:
        lens = FIXED + np.random.RandomState(5).randint(8000, 200001, 300).tolist()
        lens = [max(1, n * sr // 16000) if n > 560 else n for n in lens]
        _WAVES[sr] = [synth(n, 1000 + i, sr) for i, n in enumerate(lens)]
    return _WAVES[sr]


@pytest.mark.parametrize("sr", [16000, 8000])
@pytest.mark.parametrize("log_scale,sub_mean", [(True, True), (True, False), (False, True), (False, False)])
def test_batch_rows_are_bit_identical_to_one_waveform_calls(cuda_dev, sr, log_scale, sub_mean):
    waves = _waves(sr)
    ref = [F.mk_mfb(torch.from_numpy(w).cuda(), sr, log_scale, sub_mean) for w in waves]
    for seed in (0, 1):
        perm = np.random.RandomState(seed).permutation(len(waves))
        audio = torch.from_numpy(np.concatenate([waves[i] for i in perm])).cuda()
        feats, off = F.mk_mfb_batch(audio, [waves[i].size for i in perm], sr, log_scale, sub_mean)
        assert off.dtype == torch.int64 and not off.is_cuda and int(off[-1]) == feats.shape[0]
        for j, i in enumerate(perm):
            assert _bits_equal(feats[off[j]:off[j + 1]], ref[i]), (sr, log_scale, sub_mean, seed, waves[i].size)


def test_an_utterance_past_sample_2_31(cuda_dev):
    x = synth(48003, 77)
    lens = [2 ** 30, 2 ** 30 + 10, x.size]
    audio = torch.empty(sum(lens), device="cuda", dtype=torch.float32)
    audio[:lens[0] + lens[1]].fill_(0.25)
    audio[lens[0] + lens[1]:].copy_(torch.from_numpy(x))
    feats, off = F.mk_mfb_batch(audio, lens)
    assert lens[0] + lens[1] > 2 ** 31 and int(off[3]) - int(off[2]) == F.mk_mfb(torch.from_numpy(x).cuda()).shape[0]
    assert _bits_equal(feats[off[2]:], F.mk_mfb(torch.from_numpy(x).cuda()))
    del audio, feats
    torch.cuda.empty_cache()


def test_batch_rejects_bad_input(cuda_dev):
    x = torch.from_numpy(synth(16000, 1)).cuda()
    with pytest.raises(ValueError):
        F.mk_mfb_batch(x, [8000, 0, 8000])
    with pytest.raises(ValueError):
        F.mk_mfb_batch(x, [8000, 7999])
    with pytest.raises(RuntimeError):
        F.mk_mfb_batch(x.cpu(), [16000])


def test_bank_from_waveforms_in_chunks(cuda_dev):
    waves = _waves(16000)[:40]
    bank = F.FeatureBank.from_waveforms(waves, 16000, chunk_samples=300000)
    assert bank.num_utterances == 40
    for i, w in enumerate(waves):
        o = bank.offsets.cpu()
        assert _bits_equal(bank.feats[o[i]:o[i + 1]], F.mk_mfb(torch.from_numpy(w).cuda()))
    arr = [np.random.RandomState(i).randn(50 + i, 64) for i in range(5)]      # read_MFB .npy features are float64
    b2 = F.FeatureBank.from_arrays(arr)
    assert np.array_equal(b2.feats.cpu().numpy(), np.concatenate(arr).astype(np.float32))
    assert b2.lengths.tolist() == [50, 51, 52, 53, 54]


# ---- 2. crops ---------------------------------------------------------------------------------------------------------
def _bank(U=1000, seed=0):
    g = np.random.RandomState(seed)
    lens = g.randint(50, 2001, U)
    lens[:4] = [50, 159, 160, 161]
    arrs = [g.randn(n, 64).astype(np.float32) for n in lens]
    return F.FeatureBank.from_arrays(arrs), arrs


def _np_crops(arrs, utt, start, T, tm=None, fm=None):
    out = np.empty((len(utt), 1, T, 64), np.float32)
    for b, (u, s) in enumerate(zip(utt, start)):
        if not (0 <= u < len(arrs)) or not (0 <= s < arrs[u].shape[0]):
            out[b] = np.nan
            continue
        a = arrs[u]
        out[b, 0] = a[(s + np.arange(T)) % a.shape[0]]
        for ms, mw in (tm[b] if tm is not None else []):
            out[b, 0, max(ms, 0):max(ms + mw, 0)] = 0
        for fs, fw in (fm[b] if fm is not None else []):
            out[b, 0, :, max(fs, 0):max(fs + fw, 0)] = 0
    return out


def _crop_case(bank, B=384, T=160, seed=1):
    g = np.random.default_rng(seed)
    lens = bank.lengths
    utt = g.integers(0, bank.num_utterances, B)
    start = bank.random_starts(utt, T, g).numpy()
    # wrapping (n < T), n = T, start = n - T, and starts near n that wrap
    utt[:4], start[:4] = [0, 1, 2, 3], [0, 0, 0, 1]
    utt[4], start[4] = 0, 49
    utt[5], start[5] = 1, 150
    big = np.nonzero(lens > 500)[0][:6]
    utt[6:12] = big
    start[6:12] = [lens[big[0]] - T, lens[big[1]] - 1, lens[big[2]] - 2, lens[big[3]] - 100, lens[big[4]] - T - 1, 0]
    tm, fm = F.spec_augment_masks(B, T, 2, 30, 2, 10, g)
    tm, fm = tm.numpy(), fm.numpy()
    tm[0] = [[10, 20], [20, 20]]       # overlapping
    tm[1] = [[0, 0], [5, 0]]           # width 0
    tm[2] = [[0, 7], [T - 9, 9]]       # at 0 and at T - w
    fm[0] = [[0, 5], [64 - 6, 6]]      # at 0 and 64 - w
    fm[1] = [[3, 0], [10, 12]]
    fm[2] = [[20, 10], [25, 10]]       # overlapping
    return utt, start, tm, fm


def test_crops_bit_exact_against_numpy(cuda_dev):
    bank, arrs = _bank()
    T = 160
    utt, start, tm, fm = _crop_case(bank)
    want = _np_crops(arrs, utt, start, T, tm, fm)
    for dev in ("cpu", "cuda"):
        got = bank.crops(torch.from_numpy(utt).to(dev), torch.from_numpy(start).to(dev), T,
                         torch.from_numpy(tm).to(dev), torch.from_numpy(fm).to(dev))
        assert got.shape == (384, 1, T, 64) and got.dtype == torch.float32
        assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
    plain = bank.crops(torch.from_numpy(utt), torch.from_numpy(start), T)
    assert np.array_equal(plain.cpu().numpy(), _np_crops(arrs, utt, start, T))
    # non-contiguous index and mask tensors
    U2 = torch.from_numpy(np.stack([utt, utt], 1)).cuda()[:, 1]
    S2 = torch.from_numpy(np.stack([start, start + 7], 1)).cuda()[:, 0]
    TM2 = torch.from_numpy(np.concatenate([tm, tm], 2)).cuda()[:, :, 2:]
    assert not U2.is_contiguous() and not S2.is_contiguous() and not TM2.is_contiguous()
    got = bank.crops(U2, S2, T, TM2, torch.from_numpy(fm).cuda())
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))


def test_invalid_indices_give_nan_crops_on_the_device(cuda_dev):
    bank, arrs = _bank()
    T, U = 160, bank.num_utterances
    utt, start, tm, fm = _crop_case(bank, seed=2)
    bad = {20: (-1, 0), 21: (U, 0), 22: (7, -1), 23: (7, int(bank.lengths[7])), 24: (2 ** 40, 0), 25: (7, 2 ** 40)}
    for b, (u, s) in bad.items():
        utt[b], start[b] = u, s
    got = bank.crops(torch.from_numpy(utt).cuda(), torch.from_numpy(start).cuda(), T,
                     torch.from_numpy(tm).cuda(), torch.from_numpy(fm).cuda()).cpu().numpy()
    want = _np_crops(arrs, utt, start, T, tm, fm)
    for b in bad:
        assert np.isnan(got[b]).all()
    ok = np.setdiff1d(np.arange(384), list(bad))
    assert np.array_equal(got[ok].view(np.int32), want[ok].view(np.int32))
    for b, (u, s) in bad.items():      # the host checks CPU indices
        with pytest.raises(ValueError):
            bank.crops(torch.tensor([3, u]), torch.tensor([0, s]), T)


# ---- 3. into the network ----------------------------------------------------------------------------------------------
def _torch_crops(bank, utt, start, T):
    u = torch.as_tensor(utt, dtype=torch.int64)
    s = torch.as_tensor(start, dtype=torch.int64)
    n = torch.from_numpy(bank.lengths)[u]
    rows = bank.offsets.cpu()[u][:, None] + (s[:, None] + torch.arange(T)) % n[:, None]
    return bank.feats[rows.cuda()].unsqueeze(1).contiguous()


def _model(train):
    sd = O.make_state_dict(0, num_classes=16)
    m = dsk.DeepSpeakerModel(512, 16).cuda()
    m.load_state_dict(sd)
    return m.train() if train else m.eval()


def test_crops_into_the_network_and_the_steps(cuda_dev):
    bank, _ = _bank(U=300, seed=3)
    T = 160
    P, K = 96, 4
    g = np.random.default_rng(4)
    utt = np.repeat(g.choice(bank.num_utterances, P, replace=False), K)
    start = bank.random_starts(utt, T, g)
    labels = torch.from_numpy(np.repeat(np.arange(P), K))
    xb = bank.crops(torch.from_numpy(utt), start, T)
    xt = _torch_crops(bank, utt, start, T)
    assert _bits_equal(xb, xt)
    m = _model(False)
    with torch.no_grad():
        assert _bits_equal(m(xb), m(_torch_crops(bank, utt, start, T)))
    for step in ("batch_hard", "ge2e"):
        res = []
        for x in (bank.crops(torch.from_numpy(utt), start, T), _torch_crops(bank, utt, start, T)):
            model = _model(True)
            if step == "batch_hard":
                opt = dsk.FusedAdagrad(model.parameters(), lr=1e-2, lr_decay=1e-4)
                out = dsk.batch_hard_step(model, opt, x, labels, margin=0.1)
                params = list(model.parameters())
            else:
                crit = dsk.GE2ELoss(10.0, -5.0).cuda()
                params = list(model.parameters()) + list(crit.parameters())
                opt = dsk.FusedAdagrad(params, lr=1e-2, lr_decay=1e-4)
                out = dsk.ge2e_step(model, opt, x, labels, loss=crit)
            res.append((out["loss"].clone(), [p.detach().clone() for p in params]))
        assert _bits_equal(res[0][0], res[1][0]), step
        assert all(_bits_equal(a, b) for a, b in zip(res[0][1], res[1][1])), step


# ---- 4. utterance embeddings ------------------------------------------------------------------------------------------
def _fp64_reference(model, bank, utt, T, hop, batch):
    wu, ws, wo = bank.windows(utt, T, hop)
    W = wu.numel()
    Bb = min(batch, W)
    nb = -(-W // Bb)
    pad = nb * Bb - W
    wu = torch.cat([wu, wu[-1:].expand(pad)])
    ws = torch.cat([ws, ws[-1:].expand(pad)])
    with torch.no_grad():
        e = torch.cat([model(_torch_crops(bank, wu[i * Bb:(i + 1) * Bb], ws[i * Bb:(i + 1) * Bb], T))
                       for i in range(nb)])[:W].double().cpu()
    e = e / e.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return torch.stack([e[wo[i]:wo[i + 1]].mean(0) for i in range(len(wo) - 1)]).numpy()


@pytest.mark.parametrize("case", ["mixed", "single", "short_only"])
def test_embed_utterances_against_an_fp64_mean(cuda_dev, case):
    g = np.random.RandomState(6)
    lens = {"mixed": np.concatenate(([40, 159, 160, 161, 241], g.randint(400, 2001, 40))),
            "single": np.array([1234]), "short_only": np.array([20, 100, 159])}[case]
    bank = F.FeatureBank.from_arrays([g.randn(n, 64) for n in lens])
    model = _model(False)
    utt = np.arange(bank.num_utterances)[::-1].copy()
    out = {}
    for batch in (7, 256):
        got = F.embed_utterances(model, bank, utt, T=160, hop=80, batch=batch)
        assert got.shape == (utt.size, 512) and got.is_cuda
        ref = _fp64_reference(model, bank, utt, 160, 80, batch)
        ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
        err = np.abs(got.cpu().double().numpy() - ref)
        assert (err <= ulp).all(), (batch, (err / ulp).max())
        out[batch] = got
    assert _bits_equal(out[7], out[256]), (f"{case}: batch 7 vs 256 differ, "
                                           f"max |diff| {(out[7] - out[256]).abs().max().item():.3e}")
    with pytest.raises(RuntimeError):
        F.embed_utterances(model.train(), bank, utt)
