"""Non-finite values through the network, the front-end and the losses: loud, and local where the reference is local.

The reference's clamps (Hardtanh(0, 20), torch.clamp(min=0) in TripletMarginLoss, numpy.maximum in mk_MFB) return NaN
for NaN.  So must the engine's:
- eval forward: a non-finite input element makes NaN exactly on its footprint in every activation
  (tests/test_nonfinite_host.py computes it), NaN in that utterance's embedding, and nothing in any other utterance
  (its activations and embedding keep their bits), with every pad still +0;
- a NaN running statistic makes every eval embedding NaN, as nn.BatchNorm2d in eval does;
- a train forward with one NaN crop spreads NaN over the batch through the batch statistics, as torch does, and
  leaves NaN in the running statistics exactly where the torch oracle's are; every training step's loss is NaN;
- mk_mfb: a NaN or inf sample makes NaN exactly where the fp64 oracle has it, the rest of the batch keeps its bits;
- augmented_crops of an invalid example: an all-NaN example;
- the triplet loss is non-finite when the reference's is; batch-hard gives a non-finite anchor NaN distances and a NaN
  loss, as oracle/batch_hard_oracle.c; AAM-softmax, GE2E and cross-entropy losses are NaN, the other rows unchanged;
- Adagrad steps NaN and inf gradients as torch does; embed_utterances and diarize keep a NaN window visible.
"""
import gc

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import frontend as F
from oracle import fbank_oracle as FO
from oracle import rescnn_oracle as O
from oracle import vad_oracle as V
from tests.test_fbank import synth
from tests.test_gpu_forward import _fresh_model
from tests.test_gpu_layer_parity import KNOBS, calibrated, read_eval_activations, unpack_eval_activations
from tests.test_nonfinite_host import check_nan_layer, nan_footprint, nonfinite_indicator

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


@pytest.fixture(autouse=True)
def _release_device_memory():
    """An Engine and its module reference each other, so only the cycle collector frees a model and its workspace: run
    it after each test and hand the allocator's cached blocks back."""
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _same_nan_and_bits(a, b):
    """Equal, with NaN compared as NaN (any payload)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and _bits_equal(torch.where(na, 0.0, a), torch.where(nb, 0.0, b))


# ---- eval forward, layer by layer ----------------------------------------------------------------------------
def _poisons(T):
    """(name, function poisoning one utterance (1, T, 64) in place)."""
    def at(t, f, v):
        def p(u):
            u[0, t, f] = v
        return p

    def whole(u):
        u.fill_(NAN)

    return [("whole NaN", whole), ("NaN frame 0", at(0, 21, NAN)), ("NaN frame T-1", at(T - 1, 40, NAN)),
            ("NaN bin 0", at(T // 3, 0, NAN)), ("NaN bin 63", at(2 * T // 3, 63, NAN)), ("+inf", at(T // 2, 30, INF)),
            ("-inf", at(T // 5, 9, -INF)), ("1e5", at(T - 3, 50, 1e5))]


def _forward_and_read(m, x, dt, planar_s2):
    side, cur = torch.cuda.Stream(), torch.cuda.current_stream()
    side.wait_stream(cur)
    with torch.no_grad(), torch.cuda.stream(side):
        emb = m(x).clone()
        bufs = read_eval_activations(m, x.shape[0], x.shape[2], dt, planar_s2)
    cur.wait_stream(side)
    torch.cuda.synchronize()
    return emb.cpu(), unpack_eval_activations(m._engine.lib, bufs, x.shape[0], x.shape[2])


def eval_nonfinite_case(dt, B, T, env):
    sd = calibrated(O.make_state_dict(4, 16), O.make_input(B, T, 301, 4.0).cuda())
    m = _fresh_model(sd, env, dt)
    planar_s2 = env.get("DSK_PLANAR_S2", "1") != "0"
    clean = O.make_input(B, T, 300, 4.0).cuda()
    emb0, acts0 = _forward_and_read(m, clean, dt, planar_s2)
    assert torch.isfinite(emb0).all()
    slots = [0, B // 2, B - 1]
    poisons = _poisons(T)
    for g in range(0, len(poisons), 3):
        group = poisons[g:g + 3]
        x = clean.clone()
        for slot, (_, poison) in zip(slots, group):
            poison(x[slot])
        tag = f"{dt} B={B} T={T} {'+'.join(f'{k}={v}' for k, v in env.items()) or 'default'} " \
              f"{[name for name, _ in group]}"
        emb, acts = _forward_and_read(m, x, dt, planar_s2)
        masks = nan_footprint(nonfinite_indicator(x.cpu(), fp16=dt == "fp16"))
        poisoned = nonfinite_indicator(x.cpu(), fp16=dt == "fp16").flatten(1).any(1)
        keep = torch.ones(B, dtype=torch.bool)
        keep[slots[:len(group)]] = False
        for i, ((img, pads), mask) in enumerate(zip(acts, masks)):
            check_nan_layer(f"{tag} activation {i}", img, pads, mask)
        assert torch.equal(torch.isnan(emb).all(1), poisoned) and torch.equal(torch.isnan(emb).any(1), poisoned), tag
        assert torch.isfinite(emb[~poisoned]).all(), tag
        assert _bits_equal(emb[keep], emb0[keep]), f"{tag}: an unpoisoned embedding changed"
        for i, ((img, _), (img0, _)) in enumerate(zip(acts, acts0)):
            assert _bits_equal(img[keep], img0[keep]), f"{tag}: activation {i} of an unpoisoned utterance changed"
        print(f"[{tag}] poisoned {poisoned.nonzero().flatten().tolist()}: footprints exact, others bit-identical")


@pytest.mark.parametrize("dt,B,T", [("fp16", 7, 160), ("fp16", 64, 160), ("bf16", 7, 160), ("bf16", 64, 160),
                                    ("fp16", 5, 800)])
def test_eval_nonfinite_footprints(cuda_dev, dt, B, T):
    eval_nonfinite_case(dt, B, T, {})


@pytest.mark.parametrize("env", KNOBS, ids=lambda e: "+".join(f"{k}={v}" for k, v in e.items()))
def test_eval_nonfinite_footprints_knobs(cuda_dev, env):
    eval_nonfinite_case("fp16", 64, 160, env)


def test_nan_crop_from_a_bad_cuda_index(cuda_dev):
    """A crop with an out-of-range CUDA index is NaN (FeatureBank.crops): its embedding is NaN, through the model and
    through EmbeddingPipeline, and the other crops' embeddings keep their bits."""
    feats = [torch.from_numpy(np.random.default_rng(i).normal(0, 3, (400 + 37 * i, 64)).astype(np.float32))
             for i in range(6)]
    bank = F.FeatureBank.from_arrays(feats, device=cuda_dev)
    B, T = 9, 160
    utt = torch.arange(B, device=cuda_dev) % 6
    start = torch.arange(B, device=cuda_dev) * 3
    bad = utt.clone()
    bad[0], bad[4], bad[B - 1] = -1, 6, 2 ** 40
    x_clean, x_bad = bank.crops(utt, start, T), bank.crops(bad, start, T)
    assert torch.isnan(x_bad[[0, 4, B - 1]]).all()
    m = _fresh_model(O.make_state_dict(4, 16), {}, "fp16")
    with torch.no_grad():
        e0, e1 = m(x_clean).cpu(), m(x_bad).cpu()
    keep = [b for b in range(B) if b not in (0, 4, B - 1)]
    assert torch.isnan(e1[[0, 4, B - 1]]).all() and torch.isfinite(e1[keep]).all()
    assert _bits_equal(e1[keep], e0[keep])
    pipe = dsk.EmbeddingPipeline(m, lanes=2)
    xh, out = x_bad.cpu().pin_memory(), torch.empty(B, 512).pin_memory()
    pipe.embed(xh, out)
    pipe.synchronize()
    assert torch.isnan(out[[0, 4, B - 1]]).all()
    assert _bits_equal(out[keep], e0[keep])


# ---- poisoned running statistics --------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("prefix", ["model.bn1", "model.layer2.0.bn1", "model.layer4.0.bn2"])
def test_nan_running_var_makes_every_embedding_nan(cuda_dev, dt, prefix):
    sd = O.make_state_dict(4, 16)
    sd[prefix + ".running_var"][3] = NAN
    m = _fresh_model(sd, {}, dt)
    x = O.make_input(16, 160, 5, 4.0)
    with torch.no_grad():
        emb = m(x.cuda()).cpu()
        ref = O.forward(sd, x)
    assert torch.isnan(ref).all()
    assert torch.isnan(emb).all(), f"{int(torch.isnan(emb).sum())} of {emb.numel()} elements NaN"


# ---- the train forward -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_train_forward_spreads_nan_through_the_batch_statistics(cuda_dev, dt):
    sd = O.make_state_dict(4, 16)
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).cuda().train()
    m.load_state_dict(sd)
    x = O.make_input(6, 64, 7, 3.0)
    x[2, 0, 10, 20] = NAN
    emb = m(x.cuda())
    torch.cuda.synchronize()
    stats = {}
    with torch.no_grad():
        ref = O.forward(sd, x, True, stats)
    assert torch.isnan(ref).all()
    assert torch.isnan(emb).all(), f"{int(torch.isnan(emb).sum())} of {emb.numel()} elements NaN"
    got = {k: v.cpu() for k, v in m.state_dict().items() if "running" in k}
    for k, v in got.items():
        # the oracle's stats_out holds the updated running statistics by state-dict key
        assert torch.equal(torch.isnan(v), torch.isnan(stats[k])), k


# ---- front-end ----------------------------------------------------------------------------------------------------
def _fbank_ref(x, sr, log_scale, sub_mean):
    fb, _ = FO.fbank(x.astype(np.float64), samplerate=sr, nfilt=64)
    if log_scale:
        fb = 20 * np.log10(np.maximum(fb, 1e-5))
    return fb - np.mean(fb, axis=0) if sub_mean else fb


@pytest.mark.parametrize("sr", [16000, 8000])
@pytest.mark.parametrize("log_scale,sub_mean", [(True, True), (True, False), (False, True), (False, False)])
def test_fbank_nan_and_inf_samples(cuda_dev, sr, log_scale, sub_mean):
    n = sr * 3 // 2
    waves = [synth(n + 101 * i, 40 + i, sr) for i in range(7)]
    bad = [w.copy() for w in waves]
    bad[0][n // 2] = np.nan
    bad[2][n // 3] = np.inf
    bad[3][0] = np.nan
    bad[5][-1] = np.nan
    bad[6][777] = -np.inf
    poisoned = [0, 2, 3, 5, 6]
    lens = [w.size for w in waves]
    clean, off = F.mk_mfb_batch(torch.from_numpy(np.concatenate(waves)).cuda(), lens, sr, log_scale, sub_mean)
    got, off2 = F.mk_mfb_batch(torch.from_numpy(np.concatenate(bad)).cuda(), lens, sr, log_scale, sub_mean)
    assert torch.equal(off, off2)
    clean, got = clean.cpu(), got.cpu()
    for u in range(len(waves)):
        g, c = got[off[u]:off[u + 1]], clean[off[u]:off[u + 1]]
        if u not in poisoned:
            assert _bits_equal(g, c), u
            continue
        with np.errstate(invalid="ignore"):
            ref = _fbank_ref(bad[u], sr, log_scale, sub_mean)
        want = torch.from_numpy(np.isnan(ref))
        assert torch.equal(torch.isnan(g), want), (u, int(torch.isnan(g).sum()), int(want.sum()))
        assert want.any()
        if sub_mean:
            assert want.all()
        else:   # the frames that do not cover the sample are those of the clean waveform
            fin = ~want.any(1)
            assert _bits_equal(g[fin], c[fin]), u
        one = F.mk_mfb(torch.from_numpy(bad[u]).cuda(), sr, log_scale, sub_mean).cpu()
        assert _same_nan_and_bits(one, g), u


def test_vad_on_a_nan_utterance_matches_the_oracle(cuda_dev):
    waves = [synth(24000 + 301 * i, 60 + i) for i in range(4)]
    waves[1][5000] = np.nan
    waves[3][0] = np.inf
    lens = [w.size for w in waves]
    feats, off, energy, speech = F.mk_mfb_batch_vad(torch.from_numpy(np.concatenate(waves)).cuda(), lens)
    e = energy.cpu().numpy()
    with np.errstate(invalid="ignore"):
        ref = V.decide(e, off.numpy())[0]
    assert np.array_equal(speech.cpu().numpy(), ref)
    f2, _ = F.mk_mfb_batch(torch.from_numpy(np.concatenate(waves)).cuda(), lens)
    assert _same_nan_and_bits(feats.cpu(), f2.cpu())


# ---- augmented_crops ----------------------------------------------------------------------------------------------
def test_augmented_crops_of_invalid_examples_are_nan(cuda_dev):
    from tests import test_gpu_augment as TA

    try:
        sb, _ = TA._speech()
        rb, _ = TA._rirs()
        nb, _ = TA._noise()
        B, T = 64, 160
        utt, start, plan = TA._case(B, 31, p_reverb=0.5, p_noise=1.0)
        cplan = {k: v.cuda() for k, v in plan.items()}
        clean = sb.augmented_crops(utt.cuda(), start.cuda(), T, cplan, rb, nb)
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
        got = sb.augmented_crops(u.cuda(), s.cuda(), T, {"rir_idx": ri.cuda(), "noise_idx": ni.cuda(),
                                                         "noise_start": nst.cuda(), "snr_db": snr.cuda()}, rb, nb)
        for b in range(14):
            assert torch.isnan(got[b]).all(), (b, int(torch.isnan(got[b]).sum()))
        assert _bits_equal(got[14:], clean[14:])
        # a RIR longer than the bank's max_rir_len
        short = F.RirBank(rb.samples, rb.offsets.cpu().numpy())
        short.max_len = 16000
        ri2 = torch.zeros(B, dtype=torch.int64)
        ri2[20] = int(np.nonzero(rb.lengths == 65536)[0][0])
        got2 = sb.augmented_crops(utt.cuda(), start.cuda(), T, {"rir_idx": ri2.cuda()}, short)
        ref2 = sb.augmented_crops(utt.cuda(), start.cuda(), T, {"rir_idx": ri2.cuda()}, rb)
        assert torch.isnan(got2[20]).all()
        keep = [b for b in range(B) if b != 20]
        assert _bits_equal(got2[keep], ref2[keep])
    finally:
        TA._CACHE.clear()


# ---- losses -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["a", "p", "n"])
@pytest.mark.parametrize("value", [NAN, INF, -INF])
def test_triplet_loss_of_a_nonfinite_row(cuda_dev, where, value):
    g = torch.Generator().manual_seed(3)
    a, p, n = (torch.nn.functional.normalize(torch.randn(33, 512, generator=g), dim=1) * 10 for _ in range(3))
    {"a": a, "p": p, "n": n}[where][17, 100] = value
    got = dsk.TripletMarginLoss(0.1).forward(a.cuda(), p.cuda(), n.cuda()).cpu()
    ref = O.triplet_margin_loss(a.double(), p.double(), n.double(), 0.1)
    if torch.isfinite(ref):   # an infinite negative: its hinge is clamp(-inf, min=0) = 0
        assert abs(float(got) - float(ref)) <= 1e-4 * max(1.0, abs(float(ref))), (float(got), float(ref))
    else:
        assert bool(torch.isnan(got)) == bool(torch.isnan(ref)) and (bool(torch.isnan(ref)) or float(got) == float(ref)), \
            (float(got), float(ref))


# ---- Adagrad --------------------------------------------------------------------------------------------------------
def test_adagrad_steps_nonfinite_gradients_as_torch(cuda_dev):
    gen = torch.Generator().manual_seed(9)
    shapes = [(64, 1, 5, 5), (7,), (513, 3), (1,)]
    init = [torch.randn(*sh, generator=gen) for sh in shapes]
    ours = [torch.nn.Parameter(t.to(cuda_dev)) for t in init]
    theirs = [torch.nn.Parameter(t.to(cuda_dev)) for t in init]
    fo = dsk.FusedAdagrad(ours, lr=0.1, lr_decay=1e-4, weight_decay=1e-3)
    to = torch.optim.Adagrad(theirs, lr=0.1, lr_decay=1e-4, weight_decay=1e-3, foreach=True)
    for it in range(3):
        fo.zero_grad()
        for i, (p, q) in enumerate(zip(ours, theirs)):
            S = torch.randn(p.shape, generator=gen).flatten()
            if it == 1:
                S[: min(3, S.numel())] = torch.tensor([NAN, INF, -INF])[: min(3, S.numel())]
            S = S.view(p.shape).to(cuda_dev)
            p.grad.copy_(S)
            q.grad = S.clone()
        fo.step()
        to.step()
        for i, (p, q) in enumerate(zip(ours, theirs)):
            assert _same_nan_and_bits(p.data, q.data), (it, i)
        for i, (p, o) in enumerate(zip(ours, fo.offsets)):
            assert _same_nan_and_bits(fo.flat_sum[o:o + p.numel()].view_as(p), to.state[theirs[i]]["sum"]), (it, i)


def _nonfinite_rows(case):
    g = torch.Generator().manual_seed(11)
    N, D = 96, 512
    E = torch.nn.functional.normalize(torch.randn(N, D, generator=g), dim=1) * 10
    labels = torch.arange(N) // 6
    for r, v in {"nan": [(0, NAN)], "inf": [(47, INF)], "-inf": [(95, -INF)],
                 "three": [(0, NAN), (40, INF), (95, NAN)]}[case]:
        E[r, 7] = v
    return E, labels


@pytest.mark.parametrize("case", ["nan", "inf", "-inf", "three"])
@pytest.mark.parametrize("exact", [False, True], ids=["gram", "exact"])
def test_batch_hard_nonfinite_anchor(cuda_dev, case, exact):
    from deepspeaker_pytorch_b200 import engine as EN
    from oracle import batch_hard_oracle as BH

    E, labels = _nonfinite_rows(case)
    margin = 0.3
    Ec, lc = E.cuda(), labels.cuda()
    _, loss, pos, neg, d_ap, d_an, valid = EN.batch_hard_mine(Ec, lc, margin, exact)
    oloss, opos, oneg, od_ap, od_an, ovalid = BH.batch_hard_triplet(E.numpy(), labels.numpy(), margin)
    bad = ~torch.isfinite(E).all(1)
    assert torch.isnan(loss).all() and np.isnan(oloss)
    assert torch.isnan(d_ap[bad.cuda()]).all() and torch.isnan(d_an[bad.cuda()]).all()
    assert valid[bad.cuda()].all()
    assert np.array_equal(valid.cpu().numpy(), ovalid)
    assert np.array_equal(pos.cpu().numpy(), opos) and np.array_equal(neg.cpu().numpy(), oneg)
    assert _same_nan_and_bits(d_ap.cpu(), torch.from_numpy(od_ap)) and _same_nan_and_bits(d_an.cpu(), torch.from_numpy(od_an))
    # the row-range ops give the whole op's bits
    parts = [EN.batch_hard_select_rows(Ec, lc, r0, n, exact)[1:] for r0, n in ((0, 33), (33, 40), (73, 23))]
    for k, whole in enumerate((pos, neg, d_ap, d_an, valid)):
        cat = torch.cat([p[k] for p in parts])
        assert (_same_nan_and_bits(cat.cpu(), whole.cpu()) if cat.dtype == torch.float32 else torch.equal(cat, whole)), k
    assert torch.isnan(EN.batch_hard_mean(d_ap, d_an, valid, margin)).all()
    # the backward reads no index of a non-finite anchor; the finite rows' gradients are finite or NaN, never a fault
    gE = EN.batch_hard_backward(Ec, pos, neg, d_ap, d_an, valid, margin, torch.ones(1, device="cuda"))
    torch.cuda.synchronize()
    assert gE.shape == E.shape


# ---- training steps with one bad CUDA crop index -------------------------------------------------------------------
def _crops(B, T, bad_slot=None):
    feats = [np.random.default_rng(i).normal(0, 3, (300 + 29 * i, 64)).astype(np.float32) for i in range(8)]
    bank = F.FeatureBank.from_arrays(feats, device="cuda")
    utt = torch.arange(B, device="cuda") % 8
    start = (torch.arange(B, device="cuda") * 7) % 300
    if bad_slot is not None:
        utt[bad_slot] = 8
    return bank.crops(utt, start, T)


def _oracle_running(sd, xs):
    cur = dict(sd)
    with torch.no_grad():
        for x in xs:
            st = {}
            O.forward(cur, x, True, st)
            cur.update(st)
    return cur


@pytest.mark.parametrize("opt_kind", ["fused", "torch"])
@pytest.mark.parametrize("step", ["batch_hard", "train_a", "train_p", "train_n", "train_b", "aam", "ge2e"])
def test_step_with_a_bad_crop_index(cuda_dev, step, opt_kind):
    T, B = 64, 16
    sd = O.make_state_dict(4, 16)
    m = dsk.DeepSpeakerModel(512, 16).cuda().train()
    m.load_state_dict(sd)
    crit = dsk.GE2ELoss(10.0, -5.0).cuda() if step == "ge2e" else None
    params = list(m.parameters()) + (list(crit.parameters()) if crit is not None else [])
    opt = (dsk.FusedAdagrad(params, lr=1e-2, lr_decay=1e-4) if opt_kind == "fused"
           else torch.optim.Adagrad(params, lr=1e-2, lr_decay=1e-4))
    labels = torch.arange(B) // 4
    if step.startswith("train"):
        which = {"train_a": 0, "train_p": 1, "train_n": 2, "train_b": 0}[step]
        xs = [_crops(B, T, 5 if k == which else None) for k in range(3)]
        lp, ln = torch.arange(B) % 16, (torch.arange(B) + 3) % 16
        out = dsk.train_step(m, opt, *xs, lp.cuda(), ln.cuda(), margin=0.1, epoch=1 if step == "train_b" else 3,
                             min_softmax_epoch=2)
        if step == "train_b":   # every distance NaN: d_n - d_p < margin selects nothing, as np.where does
            assert out is None
        ran = xs
    else:
        x = _crops(B, T, 9)
        if step == "batch_hard":
            out = dsk.batch_hard_step(m, opt, x, labels, margin=0.2)
        elif step == "aam":
            out = dsk.aam_softmax_step(m, opt, x, labels, margin=0.2, scale=30.0)
        else:
            out = dsk.ge2e_step(m, opt, x, labels, loss=crit)
        ran = [x]
    torch.cuda.synchronize()
    if out is not None:
        assert torch.isnan(out["loss"]).all(), float(out["loss"])
    ref = _oracle_running(sd, [x.cpu() for x in ran])
    for k, v in m.state_dict().items():
        if "running" in k:
            assert torch.equal(torch.isnan(v.cpu()), torch.isnan(ref[k])), k
    nan_params = [k for k, p in m.named_parameters() if torch.isnan(p).any()]
    print(f"[{step} {opt_kind}] parameters holding NaN after the step: {len(nan_params)} of "
          f"{len(list(m.parameters()))}")


@pytest.mark.parametrize("value", [NAN, INF])
def test_aam_ge2e_and_cross_entropy_of_a_nonfinite_row(cuda_dev, value):
    """The loss is not finite; AAM-softmax's cos / lse and cross-entropy's gradient rows of the other rows keep their
    bits (each row depends only on its own embedding or logits)."""
    from deepspeaker_pytorch_b200 import engine as EN

    g = torch.Generator().manual_seed(5)
    N, C, D = 48, 20, 512
    E = torch.randn(N, D, generator=g)
    W = torch.randn(C, D, generator=g)
    labels = torch.arange(N) % C
    bad = E.clone()
    bad[13, 40] = value
    keep = torch.arange(N) != 13
    *_, loss0, cos0, lse0 = EN.aam_softmax(E.cuda(), W.cuda(), labels.cuda(), 0.2, 30.0)
    *_, loss1, cos1, lse1 = EN.aam_softmax(bad.cuda(), W.cuda(), labels.cuda(), 0.2, 30.0)
    assert torch.isfinite(loss0).all() and torch.isnan(loss1).all()
    assert _bits_equal(cos1[keep.cuda()], cos0[keep.cuda()]) and _bits_equal(lse1[keep.cuda()], lse0[keep.cuda()])
    glabels = torch.arange(N) // 4   # 12 speakers x 4
    for method in ("softmax", "contrast"):
        crit = dsk.GE2ELoss(10.0, -5.0, method=method).cuda()
        assert torch.isfinite(crit(E.cuda(), glabels.cuda())).all()
        assert torch.isnan(crit(bad.cuda(), glabels.cuda())).all(), method
    if value != value:   # cross-entropy of a NaN logit row
        logits = torch.randn(N, C, generator=g) * 5
        lbad = logits.clone()
        lbad[13, 4] = value
        grads = []
        for lg in (logits, lbad):
            x = lg.cuda().requires_grad_(True)
            loss = dsk.CrossEntropyLoss()(x, labels.cuda())
            loss.backward()
            grads.append((loss.detach(), x.grad.cpu()))
        assert torch.isfinite(grads[0][0]).all() and torch.isnan(grads[1][0]).all()
        assert torch.isnan(grads[1][1][13]).all() and _bits_equal(grads[1][1][keep], grads[0][1][keep])


# ---- consumers ------------------------------------------------------------------------------------------------------
def test_embed_utterances_and_diarize_with_a_nan_frame(cuda_dev):
    feats = [np.random.default_rng(20 + i).normal(0, 3, (900 + 50 * i, 64)).astype(np.float32) for i in range(5)]
    m = _fresh_model(O.make_state_dict(4, 16), {}, "fp16")
    clean = F.FeatureBank.from_arrays(feats, device=cuda_dev)
    feats[2][333, 17] = np.nan
    bank = F.FeatureBank.from_arrays(feats, device=cuda_dev)
    utt = torch.arange(5)
    e0 = F.embed_utterances(m, clean, utt).cpu()
    e1 = F.embed_utterances(m, bank, utt).cpu()
    assert torch.isfinite(e0).all()
    assert torch.isnan(e1[2]).all()
    keep = [0, 1, 3, 4]
    assert torch.isfinite(e1[keep]).all() and _bits_equal(e1[keep], e0[keep])
    from deepspeaker_pytorch_b200 import diarization

    assert len(diarization.diarize(m, clean, [2], num_speakers=2)) == 1
    with pytest.raises(RuntimeError):
        diarization.diarize(m, bank, [2], num_speakers=2)
