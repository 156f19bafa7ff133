"""Where a non-finite input element goes in the eval forward: the NaN footprint of every activation.

A NaN input element reaches every output of a conv whose window covers it, in every channel (NaN * w is NaN, 0 * NaN
included), and the residual adds carry the block input's footprint on.  The engine treats +-inf the same way: conv1
splits x into 16-bit halves, x_lo = inf - inf is NaN.  `nan_footprint` computes the mask without any float arithmetic
on the poisoned values: the indicator taken through each conv as a conv with an all-ones kernel of the same size,
stride and padding, keeping the outputs > 0, ORed with the residual input's mask.  The reference model's clamps
(torch.clamp, Hardtanh) return NaN for NaN, so its activations are NaN exactly there.

`check_nan_layer` is the checker test_gpu_nonfinite.py applies to the engine's activations read back byte for byte.
This file checks the mask against torch's CPU conv2d chain in fp64 and fp32, the checker against an emulated layer
with seeded defects, and the batch-hard oracle's non-finite rule against a brute-force restatement.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import rescnn_oracle as O

CONV = O.conv_names()


def nan_footprint(ind):
    """ind (B, 1, T, 64) bool, the non-finite input elements -> the 12 activation masks, each (B, 1, H, W) bool (every
    channel of a layer has the same mask)."""
    masks = []
    prev = ind.double()
    for i, (_, _, k, stride) in enumerate(CONV):
        m = F.conv2d(prev, torch.ones(1, 1, k, k, dtype=torch.float64), None, stride, k // 2) > 0
        if i % 3 == 2:
            m = m | masks[i - 2]
        masks.append(m)
        prev = m.double()
    return masks


def nonfinite_indicator(x, fp16=False):
    """The input elements that make NaN: NaN and +-inf, and on fp16 operands also |x| >= 65520, which rounds to inf in
    conv1's hi half (x_lo = x - inf is then -inf, and x_hi * w + x_lo * w is NaN)."""
    ind = ~torch.isfinite(x)
    if fp16:
        ind = ind | (x.abs() >= 65520)
    return ind


def check_nan_layer(tag, img, pads, mask):
    """img (B, C, H, W) fp32, pads: the layout's pad values, mask (B, 1, H, W) bool.  NaN exactly on the mask in every
    channel; every pad +0.0 (a NaN or any non-zero bit pattern in a pad would be read by the neighbouring utterance's
    window)."""
    nan = torch.isnan(img)
    want = mask.expand_as(nan)
    if not torch.equal(nan, want):
        extra, missing = int((nan & ~want).sum()), int((~nan & want).sum())
        raise AssertionError(f"{tag}: NaN where the footprint has none: {extra}; footprint without NaN: {missing}")
    bad = pads.isnan() | (pads != 0) | torch.signbit(pads)
    assert not bool(bad.any()), f"{tag}: {int(bad.sum())} pad values are not +0"


# ---- the mask against torch's conv2d -----------------------------------------------------------------------------
def _poison(B, T, cases, seed=0):
    x = O.make_input(B, T, seed, 3.0)
    for b, (t, f, v) in cases.items():
        x[b, 0, t, f] = v
    return x


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("T", [16, 48])
def test_footprint_equals_torch_conv_nan_propagation(dtype, T):
    sd = {k: v.to(dtype) for k, v in O.make_state_dict(3, 16).items()}
    for wkey, _, _, _ in CONV:   # one all-zero output channel per conv: 0 * NaN is NaN, so it must not hide the footprint
        sd[wkey][5].zero_()
    B = 7
    # NaN only: the reference takes +-inf through conv1 as +-inf, and its clamp makes that finite
    cases = {0: (0, 0, float("nan")), 2: (T - 1, 63, float("nan")), 3: (T // 2, 17, float("nan")),
             5: (1, 40, float("nan")), 6: (T - 2, 0, float("nan"))}
    x = _poison(B, T, cases).to(dtype)
    x[4] = float("nan")
    taps = {}
    with torch.no_grad():
        emb = O.forward(sd, x, taps=taps)
    masks = nan_footprint(nonfinite_indicator(x))
    for i in range(12):
        C, H, W = taps[i].shape[1:]
        assert masks[i].shape == (B, 1, H, W)
        assert torch.equal(torch.isnan(taps[i]), masks[i].expand_as(taps[i])), f"layer {i}"
    assert masks[0][1].sum() == 0
    assert torch.equal(torch.isnan(emb).any(1), torch.tensor([b in cases or b == 4 for b in range(B)]))
    assert torch.equal(torch.isnan(emb).all(1), torch.isnan(emb).any(1))


def test_fp16_indicator_takes_values_past_the_fp16_range():
    x = torch.tensor([0.0, 65504.0, 65519.0, 65520.0, -65520.0, 1e5, float("inf"), float("nan")])
    assert nonfinite_indicator(x).tolist() == [False] * 6 + [True, True]
    assert nonfinite_indicator(x, fp16=True).tolist() == [False, False, False, True, True, True, True, True]
    assert torch.isinf(x[:6].half()).tolist() == [False, False, False, True, True, True]


# ---- the checker against an emulated layer -----------------------------------------------------------------------
def emulate_layer(a, w, s, b, pad_hw, defect=None):
    """A 3x3 s1 conv layer as the engine stores it: fp32 conv, affine, clamp to [0, 20], fp16 rounding; returns the
    image and the values in its zero-pad ring.  defect: 'clamp' (NaN -> 0, fminf(fmaxf(x, 0), 20)), 'pad' (the pad next
    to a NaN carries it), 'shift' (the output shifted down one row)."""
    y = F.conv2d(a, w, None, 1, 1) * s.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)
    y = torch.nan_to_num(y, nan=0.0).clamp(0, 20) if defect == "clamp" else y.clamp(0, 20)
    if defect == "shift":
        y = torch.cat([y[:, :, :1], y[:, :, :-1]], dim=2)
    y = y.half().float()
    pads = torch.zeros(y.shape[0], y.shape[1], pad_hw)
    if defect == "pad":
        pads[:, :, 0] = y[:, :, -1, 0]
    return y, pads


@pytest.mark.parametrize("defect", [None, "clamp", "pad", "shift"])
def test_checker_passes_the_nan_clamp_and_fails_seeded_defects(defect):
    g = torch.Generator().manual_seed(1)
    N, C, H, W = 3, 16, 8, 6
    a = torch.rand(N, C, H, W, generator=g) * 2
    a[1, 3, H - 1, 0] = float("nan")   # reaches the last row of utterance 1, next to its pad row
    w = torch.randn(C, C, 3, 3, generator=g) * 0.2
    s, b = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    ind = torch.isnan(a).any(1, keepdim=True)
    mask = F.conv2d(ind.double(), torch.ones(1, 1, 3, 3, dtype=torch.float64), None, 1, 1) > 0
    y, pads = emulate_layer(a, w, s, b, W, defect)
    if defect is None:
        check_nan_layer("nan clamp", y, pads, mask)
    else:
        with pytest.raises(AssertionError):
            check_nan_layer(defect, y, pads, mask)


# ---- the batch-hard oracle's non-finite rule -----------------------------------------------------------------------
def _batch_hard_brute(E, labels, margin):
    """numpy fp64 restatement: a NaN distance is never selected (an infinite one is, the lower index first among
    ties); an anchor whose row is not finite gets d_ap = d_an = NaN and is valid iff its label has another row and
    another label exists."""
    N, D = E.shape
    eps = 1e-4 / D
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.sqrt(((E[:, None, :].astype(np.float64) - E[None, :, :]) ** 2).sum(-1) + eps)
    out = []
    for i in range(N):
        same = [j for j in range(N) if labels[j] == labels[i] and j != i]
        other = [j for j in range(N) if labels[j] != labels[i]]
        ps = [j for j in same if not np.isnan(d[i, j])]
        ns = [j for j in other if not np.isnan(d[i, j])]
        p = max(ps, key=lambda j: (d[i, j], -j)) if ps else -1
        n = min(ns, key=lambda j: (d[i, j], j)) if ns else -1
        bad = not np.isfinite(E[i]).all()
        dap = np.nan if bad else (d[i, p] if p >= 0 else 0.0)
        dan = np.nan if bad else (d[i, n] if n >= 0 else np.inf)
        valid = bool(same if bad else p >= 0) and bool(other)
        out.append((p, n, dap, dan, valid))
    pos, neg, dap, dan, valid = (np.array(c) for c in zip(*out))
    h = margin + dap[valid] - dan[valid]
    with np.errstate(invalid="ignore"):
        loss = np.mean(np.where(np.isnan(h), h, np.maximum(h, 0))) if valid.any() else 0.0
    return loss, pos, neg, dap, dan, valid


@pytest.mark.parametrize("case", ["nan anchor", "inf anchor", "-inf element", "nan singleton", "two bad rows"])
def test_batch_hard_oracle_nonfinite_rule(case):
    from oracle import batch_hard_oracle as BH

    g = np.random.default_rng(7)
    N, D = 40, 24
    E = g.normal(size=(N, D)).astype(np.float32)
    labels = np.arange(N) // 4
    if case == "nan anchor":
        E[5, 3] = np.nan
    elif case == "inf anchor":
        E[17, 0] = np.inf
    elif case == "-inf element":
        E[39, 23] = -np.inf
    elif case == "nan singleton":
        labels[8] = 100
        E[8] = np.nan
    else:
        E[0, :] = np.nan
        E[22, 7] = np.inf
    loss, pos, neg, dap, dan, valid = BH.batch_hard_triplet(E, labels, 0.3)
    bloss, bpos, bneg, bdap, bdan, bvalid = _batch_hard_brute(E, labels, 0.3)
    assert np.array_equal(valid, bvalid)
    assert np.array_equal(pos, bpos) and np.array_equal(neg, bneg)
    for got, ref in ((dap, bdap), (dan, bdan)):
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        fin = ~np.isnan(ref)
        assert np.allclose(got[fin], ref[fin], rtol=1e-5)
    if case == "nan singleton":   # a row with no positive contributes nothing, finite or not
        assert not valid[8] and np.isfinite(loss)
    else:
        assert np.isnan(loss) and np.isnan(bloss)
