"""Every layer of the eval and train forwards against fp64, recomputed from that layer's own inputs.

The end-to-end gates (1e-3 on the embedding) leave room for an error of a few 1e-4 that stays inside one layer: one
tile, one 64-channel block, the image borders, the last tile.  Here the engine's own 16-bit activations are read back
after a production forward, each layer is recomputed in float64 from exactly what it consumed (16-bit activations,
weights rounded to the operand type like the kernels' to16), and EVERY element must lie within a worst-case bound
computed from magnitudes:

    ref   = clip(s * conv(a, w16) + b (+ r), 0, 20)          s, b: the folded eval BatchNorm, fp64 from the fp32 params
    A     = |s| * conv(|a|, |w16|)
    delta = (K + 8) 2^-23 A + 2^-22 (|b| + |mean*s| + |r|)  (+ operand term, conv1 only)
    bound = u (|ref| + delta) + 2^-25 + delta                 u = 2^-11 (fp16), 2^-8 (bf16)

K is the number of products summed.  2^-23 instead of 2^-24 allows for tensor-core accumulation that truncates; the +8
covers the fp32 folded scale; |mean*s| covers the fp32 bias beta - mean*s, whose error is relative to its terms, not to
its value; u (|ref| + delta) + 2^-25 is the 16-bit rounding of the stored output (2^-25: fp16 subnormals).  A wrong tap,
shift, tile, channel block or precision path fails at the element where it happens; the report says where violations
cluster (evenly spread errors just over the bound point at the accumulation model, clustered ones at a kernel bug).

The CPU self-test at the end runs the same checker on an emulated layer and on seeded defects, so it runs everywhere.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from oracle import rescnn_oracle as O
from tests.test_gpu_forward import _fresh_model
from tests.test_gpu_halo_conv import from_padded, from_planar
from tests.test_gpu_train_parity import read_saved_activations
from tests.train_plan import reduce_chain, stat_blocks

U = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}         # unit roundoff of the 16-bit storage
TD = {"fp16": torch.float16, "bf16": torch.bfloat16}
ACC = 2.0 ** -23                                     # per-product fp32 accumulation allowance (truncating adders)
TINY = 2.0 ** -25                                    # half the fp16 subnormal spacing
CONV = O.conv_names()


def rn16(t, dt):
    return t.to(TD[dt]).to(t.dtype)


def act_geometry(i, T):
    st = i // 3
    return 64 << st, T >> (st + 1), 64 >> (st + 1)   # C, H, W


# ---- the checker --------------------------------------------------------------------------------------------------
def locate(viol, ratio):
    """Where the violations of an (N,C,H,W) check sit: count, worst element, and how they cluster."""
    N, C, H, W = viol.shape
    idx = viol.nonzero()
    n, c, h, w = idx.unbind(1)
    worst = np.unravel_index(int(torch.where(viol, ratio, torch.zeros_like(ratio)).argmax()), viol.shape)
    on_border = lambda hh, ww: ((hh == 0) | (hh == H - 1) | (ww == 0) | (ww == W - 1)).double().mean().item()
    hh, ww = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    pos = (n * (H + 1) + h + 1) * (W + 1) + w + 1    # position in the zero-padded NHWC layout
    share = lambda t: torch.bincount(t).max().item() / t.numel()
    return (f"{idx.shape[0]} of {viol.numel()} elements over the bound, worst (n,c,h,w) = {tuple(int(v) for v in worst)} at "
            f"err/bound {ratio.max().item():.3g}; at image borders {on_border(h, w):.0%} (of all pixels "
            f"{on_border(hh, ww):.0%}); largest share in one 64-channel block {share(c // 64):.0%} of {(C + 63) // 64}, "
            f"one utterance {share(n):.0%} of {N}, one 128-position tile {share(pos // 128):.0%}")


def check(name, got, ref, bound, saturating=True):
    """Every element within its bound.  Prints the largest err/bound (and, for clipped outputs, the fraction of the
    reference strictly inside (0, 20)); returns (violation description or None, max err/bound, inside fraction).
    A NaN anywhere (got, ref or bound) is a violation with err/bound = inf."""
    ratio = torch.nan_to_num((got.double() - ref).abs() / bound, nan=float("inf"), posinf=float("inf"))
    worst = ratio.max().item()
    inside = ((ref > 0) & (ref < 20)).double().mean().item() if saturating else None
    viol = ~(ratio <= 1.0)
    print(f"  {name:<12} max err/bound {worst:.3f}" + (f"   inside (0,20) {inside:.2f}" if saturating else ""))
    msg = locate(viol.cpu(), ratio.cpu()) if bool(viol.any()) else None
    return msg, worst, inside


def assert_layer(name, got, ref, bound, saturating=True):
    msg, _, inside = check(name, got, ref, bound, saturating)
    assert msg is None, f"{name}: {msg}"
    if saturating:   # a check over a saturated layer would pass vacuously
        assert inside >= 0.2, f"{name}: only {inside:.1%} of the reference lies inside (0, 20)"


def conv_ref(a, w16, s, b, ms, r, stride, pad, u, extra=None, tiny=TINY):
    """Reference and bound of one conv + affine (+ residual) + clip layer (see the module docstring); s, b, ms per
    output channel (ms = mean * s).  s = 1, b = 0, u = 0 and no tiny give the fp32 raw output of a train-mode conv."""
    v = lambda t: t.view(1, -1, 1, 1)
    K = w16.shape[1] * w16.shape[2] * w16.shape[3]
    pre = F.conv2d(a, w16, None, stride, pad) * v(s) + v(b)
    A = F.conv2d(a.abs(), w16.abs(), None, stride, pad) * v(s.abs())
    side = v(b.abs() + ms.abs())
    if r is not None:
        pre = pre + r
        side = side + r.abs()
    delta = (K + 8) * ACC * A + 2.0 ** -22 * side
    if extra is not None:
        delta = delta + extra
    ref = pre.clamp(0, 20) if u else pre
    return ref, u * (ref.abs() + delta) + tiny + delta


def conv1_operand_term(x, w, s, u):
    """Error of conv1's hi/lo split (x = x_hi + x_lo, w = w_hi + w_lo, x_lo*w_lo dropped): 3u^2 conv(|x|,|w|) +
    2^-25 (conv(|x|, 1) + conv(1, |w|)) for subnormal lo halves, times |s| (csrc/conv1_umma.cuh)."""
    v = lambda t: t.view(1, -1, 1, 1)
    ones_w = torch.ones_like(w)
    ones_x = torch.ones_like(x)
    t = (3 * u * u * F.conv2d(x.abs(), w.abs(), None, 2, 2)
         + TINY * (F.conv2d(x.abs(), ones_w, None, 2, 2) + F.conv2d(ones_x, w.abs(), None, 2, 2)))
    return t * v(s.abs())


def rounding_fraction(got, ref, dt):
    """Among elements with 0 < ref < 20: the fraction whose stored value is not rn16(ref).  With conv1's lo halves the
    kernel is exact to ~1e-7 relative and the 16-bit rounding decides almost every element like fp64 does; without them
    about a quarter of the elements round the other way."""
    m = (ref > 0) & (ref < 20)
    return (got.double()[m] != rn16(ref[m], dt)).double().mean().item()


def tail_ref(act11, fc_w, fc_b):
    """emb = 10 * fc(mean over time of act11, column c*4+w) / L2, with a bound from the same accumulation model:
    delta_j on the fc output, propagated through the normalisation, plus the fp32 rounding of the result."""
    B, C, H4, W = act11.shape
    P = act11.mean(dim=2).reshape(B, C * W)
    Wd, bd = fc_w.double(), fc_b.double()
    y = P @ Wd.T + bd
    nrm = y.norm(dim=1, keepdim=True)
    emb = 10 * y / nrm
    delta = (C * W + H4 + 16) * ACC * (P.abs() @ Wd.abs().T) + 2.0 ** -22 * bd.abs()
    bound = 10 * (delta + y.abs() * delta.norm(dim=1, keepdim=True) / nrm) / nrm + 2.0 ** -20 * emb.abs() + 2.0 ** -30
    return emb, bound


def folded_bn(sd, prefix):
    g, be, rm, rv = (sd[prefix + k].double() for k in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / torch.sqrt(rv + O.BN_EPS)
    return s, be - rm * s, rm * s


def batch_stats(raw):
    """fp64 batch mean and biased variance per channel of an (N,C,H,W) tensor."""
    mean = raw.mean(dim=(0, 2, 3))
    var = (raw - mean.view(1, -1, 1, 1)).pow(2).mean(dim=(0, 2, 3))
    return mean, var


def stat_eps(mean, var, n):
    """Error of the engine's batch mean (relative to std) and variance (relative to var) per channel: fp32 chains of n
    additions (n 2^-24; stat_chains gives n per layer) of terms up to (mean^2 + var) in size.  The engine sums x itself
    while mean^2 <= 1024 var and x - pivot beyond that (bn_finalize_kernel; the synchronised records always sum around
    each utterance's first pixel), so mean^2 / var counts up to 1024."""
    return n * 2.0 ** -24 * (2 + (mean * mean / var.clamp_min(1e-300)).clamp(max=1024))


def running_stats_check(name, rm0, rv0, rm1, rv1, mean, var, M, n):
    """Running statistics after one train forward against the fp64 momentum update (unbiased variance); n: the length
    of the reductions' fp32 chains."""
    unb = var * M / max(M - 1, 1)
    eps = stat_eps(mean, var, n)
    em = 0.9 * rm0 + 0.1 * mean
    ev = 0.9 * rv0 + 0.1 * unb
    tm = 2.0 ** -22 * (rm0.abs() + mean.abs()) + 0.1 * eps * var.sqrt() + 1e-30
    tv = 2.0 ** -22 * (rv0.abs() + unb) + 0.1 * eps * unb + 1e-30
    r = max(((rm1 - em).abs() / tm).max().item(), ((rv1 - ev).abs() / tv).max().item())
    print(f"  {name:<12} running stats max err/bound {r:.3f} (chains of {n})")
    return r


def stat_chains(eng, tctx, B, T, sync):
    """Per layer, the longest fp32 chain of the BatchNorm reductions of the forward (and backward) `tctx` is bound to:
    the unsynchronised path's partial-block count gx as the library planned it (dsk_debug_backward_plan), or the
    synchronised path's per-utterance records."""
    out = []
    for i in range(12):
        C, H, W = act_geometry(i, T)
        v = (ctypes.c_int32 * 3)()
        L.check(eng.lib.dsk_debug_backward_plan(eng.handle, tctx, i, v), "dsk_debug_backward_plan")
        out.append(reduce_chain(B * H * W, H * W, v[2], sync))
    return out


# ---- eval chain ---------------------------------------------------------------------------------------------------
def calibrated(sd, x):
    """The state dict with each BatchNorm's running statistics set to the batch statistics of x (an oracle train-mode
    pass with momentum 1), so that no layer of the checked forward is saturated by random running statistics."""
    old = O.BN_MOMENTUM
    O.BN_MOMENTUM = 1.0
    try:
        st = {}
        with torch.no_grad():
            O.forward({k: v.to(x.device) for k, v in sd.items()}, x, True, st)
    finally:
        O.BN_MOMENTUM = old
    out = dict(sd)
    out.update({k: v.cpu() for k, v in st.items()})
    return out


def read_eval_activations(m, B, T, dt):
    """The 12 activation buffers of the handle's last eval forward, byte for byte (dsk_debug_read_eval_activation)."""
    eng = m._engine
    out = []
    for i in range(12):
        C, H, W = act_geometry(i, T)
        planar = i % 3 == 2 and i < 11
        if planar:
            npl = eng.lib.dsk_padded_positions(B, H // 2, W // 2)
            buf = torch.empty(4, npl // (W // 2 + 1), W // 2 + 1, C, dtype=TD[dt], device="cuda")
        else:
            npos = eng.lib.dsk_padded_positions(B, H, W)
            buf = torch.empty(npos // (W + 1), W + 1, C, dtype=TD[dt], device="cuda")
        flag = ctypes.c_int32(-1)
        L.check(eng.lib.dsk_debug_read_eval_activation(eng.handle, i, buf.data_ptr(), buf.numel() * 2, ctypes.byref(flag),
                                                       L.cur_stream()), "dsk_debug_read_eval_activation")
        out.append((buf, planar, flag))
    return out


def unpack_eval_activations(lib, bufs, B, T):
    """-> [(image (N,C,H,W) fp32 on the CPU, pad values)]; checks the layout flag the library returned."""
    out = []
    for i, (buf, planar, flag) in enumerate(bufs):
        assert flag.value == int(planar), (i, flag.value)
        C, H, W = act_geometry(i, T)
        if planar:
            out.append(from_planar(lib, buf, B, C, H, W))
        else:
            rows = (torch.arange(B).view(B, 1) * (H + 1) + torch.arange(H).view(1, H) + 1).flatten()
            out.append(from_padded(buf, rows, B, C, H, W))
    return out


def check_eval_chain(tag, sd, dt, x, acts, emb):
    """conv1 against the fp32 input, layers 1-11 from the engine's own act[i-1] (and act[i-2]), the pads, the tail."""
    u = U[dt]
    dev = x.device
    a = [img.to(dev).double() for img, _ in acts]
    print(f"[{tag}]")
    for i, (_, pads) in enumerate(acts):
        assert float(pads.abs().max()) == 0.0, f"{tag}: a pad position of activation {i} is not zero"
    s, b, ms = (t.to(dev) for t in folded_bn(sd, CONV[0][1]))
    xd, w0 = x.double(), sd[CONV[0][0]].to(dev).double()
    ref, bound = conv_ref(xd, w0, s, b, ms, None, 2, 2, u, extra=conv1_operand_term(xd, w0, s, u))
    assert_layer("conv 0", a[0], ref, bound)
    frac = rounding_fraction(a[0], ref, dt)
    print(f"  conv 0       stored != rn16(fp64): {frac:.2%}")
    if dt == "fp16":   # with bf16 halves the dropped x_lo*w_lo term is 2^-16: the fraction says less about the lo half
        assert frac <= 0.02, f"{tag}: conv1 rounds {frac:.1%} of its outputs away from rn16(fp64): is the lo half used?"
    for i in range(1, 12):
        wkey, prefix, k, stride = CONV[i]
        s, b, ms = (t.to(dev) for t in folded_bn(sd, prefix))
        w16 = rn16(sd[wkey].to(dev).double(), dt)
        r = a[i - 2] if i % 3 == 2 else None
        ref, bound = conv_ref(a[i - 1], w16, s, b, ms, r, stride, k // 2, u)
        assert_layer(f"conv {i}", a[i], ref, bound)
    eref, ebound = tail_ref(a[11], sd["model.fc.weight"].to(dev), sd["model.fc.bias"].to(dev))
    msg, _, _ = check("tail", emb.double().view(*eref.shape, 1, 1), eref.view(*eref.shape, 1, 1),
                      ebound.view(*eref.shape, 1, 1), saturating=False)
    assert msg is None, f"{tag} tail: {msg}"


def eval_case(dt, B, T, env, seed=300, shape_switch=False):
    sd0 = O.make_state_dict(4, 16)
    xs = [O.make_input(B, T, seed + j, 4.0).cuda() for j in range(3)]
    sd = calibrated(sd0, xs[2])
    m = _fresh_model(sd, env, dt)
    side, cur = torch.cuda.Stream(), torch.cuda.current_stream()
    side.wait_stream(cur)
    # three forwards back to back on one non-legacy stream: plain launches, graph capture, then a graph replay re-pointed
    # at a new input right behind another forward - the third is checked
    with torch.no_grad(), torch.cuda.stream(side):
        for x in xs:
            emb = m(x)
        bufs = read_eval_activations(m, B, T, dt)
    cur.wait_stream(side)
    torch.cuda.synchronize()
    tag = f"eval {dt} B={B} T={T} {' '.join(f'{k}={v}' for k, v in env.items()) or 'default'}"
    check_eval_chain(tag, sd, dt, xs[2], unpack_eval_activations(m._engine.lib, bufs, B, T), emb)
    if shape_switch:   # another shape re-zeroes the shared workspace for itself; coming back must leave every pad zero
        with torch.no_grad(), torch.cuda.stream(side):
            m(O.make_input(3, 32, seed + 7, 4.0).cuda())
            emb = m(xs[2])
            bufs = read_eval_activations(m, B, T, dt)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        for i, (_, pads) in enumerate(unpack_eval_activations(m._engine.lib, bufs, B, T)):
            assert float(pads.abs().max()) == 0.0, f"after a shape switch: a pad position of activation {i} is not zero"


EVAL_CASES = [("fp16", 64, 160), ("fp16", 64, 32), ("fp16", 1, 16), ("fp16", 33, 48), ("bf16", 64, 160)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,B,T", EVAL_CASES)
def test_eval_chain_layer_by_layer(cuda_dev, dt, B, T):
    eval_case(dt, B, T, {}, shape_switch=(dt, B, T) == ("fp16", 64, 160))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,B,T", EVAL_CASES + [("bf16", 33, 48)])
def test_eval_chain_layer_by_layer_kernel_by_kernel(cuda_dev, dt, B, T):
    """The same checks with the forward launched kernel by kernel (DSK_GRAPH=0) instead of as one CUDA graph."""
    eval_case(dt, B, T, {"DSK_GRAPH": "0"})


# ---- train chain --------------------------------------------------------------------------------------------------
def check_train_chain(tag, sd, dt, x, raw, y, emb, rm0, rv0, rm1, rv1, chains):
    """raw[0] against fp64 conv1 of x, raw[i] against fp64 conv(y[i-1], w16), y[i] against the clipped BatchNorm of the
    engine's raw[i] with fp64 batch statistics (+ y[i-2]), the running statistics, and the tail.  chains[i]: the length
    of layer i's BatchNorm reduction chains (stat_chains).  Each layer's fp64 tensors are dropped before the next."""
    u = U[dt]
    dev = x.device
    one = lambda C: torch.ones(C, dtype=torch.float64, device=dev)
    zero = lambda C: torch.zeros(C, dtype=torch.float64, device=dev)
    print(f"[{tag}]")
    worst_stats = 0.0
    for i in range(12):
        wkey, prefix, k, stride = CONV[i]
        rw, yy = raw[i].double(), y[i].double()
        C = rw.shape[1]
        w = sd[wkey].to(dev).double()
        a = x.double() if i == 0 else y[i - 1].double()
        ref, bound = conv_ref(a, w if i == 0 else rn16(w, dt), one(C), zero(C), zero(C), None, stride, k // 2, 0.0,
                              tiny=1e-30)
        del a
        assert_layer(f"raw {i}", rw, ref, bound, saturating=False)
        del ref, bound
        mean, var = batch_stats(rw)
        g, be = sd[prefix + ".weight"].to(dev).double(), sd[prefix + ".bias"].to(dev).double()
        v = lambda t: t.view(1, -1, 1, 1)
        sc = g / torch.sqrt(var + O.BN_EPS)
        xhat = (rw - v(mean)) / v(torch.sqrt(var + O.BN_EPS))
        pre = v(g) * xhat + v(be)
        side = (rw * v(sc)).abs() + v((mean * sc).abs() + be.abs())
        if i % 3 == 2:
            res = y[i - 2].double()
            pre = pre + res
            side = side + res.abs()
            del res
        ref = pre.clamp(0, 20)
        del pre
        # fp32 scale / shift and their fused multiply-add, then the batch statistics' own error
        delta = 2.0 ** -21 * side + v(stat_eps(mean, var, chains[i]) * g.abs()) * (1 + xhat.abs())
        del side, xhat
        assert_layer(f"y {i}", yy, ref, u * (ref.abs() + delta) + TINY + delta)
        del ref, delta, rw, yy
        M = raw[i].numel() // C
        worst_stats = max(worst_stats, running_stats_check(f"bn {i}", rm0[i].double(), rv0[i].double(), rm1[i].double(),
                                                           rv1[i].double(), mean, var, M, chains[i]))
    assert worst_stats <= 1.0, f"{tag}: running statistics off by {worst_stats:.3g} x their bound"
    eref, ebound = tail_ref(y[11].double(), sd["model.fc.weight"].to(dev), sd["model.fc.bias"].to(dev))
    msg, _, _ = check("tail", emb.detach().double().view(*eref.shape, 1, 1), eref.view(*eref.shape, 1, 1),
                      ebound.view(*eref.shape, 1, 1), saturating=False)
    assert msg is None, f"{tag} tail: {msg}"


def train_forward_and_check(tag, m, sd, dt, x, T):
    bns = [bn for _, bn in dsk.engine.conv_bn_modules(m)]
    rm0 = [bn.running_mean.detach().clone() for bn in bns]
    rv0 = [bn.running_var.detach().clone() for bn in bns]
    emb = m(x)
    raw = read_saved_activations(m, emb, T, which=0)
    y = read_saved_activations(m, emb, T, which=1)
    torch.cuda.synchronize()
    rm1 = [bn.running_mean.detach().clone() for bn in bns]
    rv1 = [bn.running_var.detach().clone() for bn in bns]
    chains = stat_chains(m._engine, emb.grad_fn.guard.tctx, x.shape[0], T, sync=False)
    check_train_chain(tag, sd, dt, x, raw, y, emb, rm0, rv0, rm1, rv1, chains)
    return emb


TRAIN_CASES = [("fp16", 128, 160), ("fp16", 6, 160), ("fp16", 5, 32), ("bf16", 16, 48)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,B,T", TRAIN_CASES)
def test_train_chain_layer_by_layer(cuda_dev, dt, B, T):
    sd = O.make_state_dict(6, 16)
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype=dt).to(cuda_dev)
    m.load_state_dict(sd)
    m.train()
    x = O.make_input(B, T, 400 + B, 3.0).cuda()
    train_forward_and_check(f"train {dt} B={B} T={T}", m, sd, dt, x, T)


@pytest.mark.gpu
def test_train_chain_after_rebinding_to_a_smaller_batch(cuda_dev):
    """A context sized for B=16 that served a forward and its backward is re-bound to B=7 (same T): its launch
    descriptors are rebuilt over the same buffers (ctx_bind)."""
    T = 48
    sd = O.make_state_dict(7, 16)
    m = dsk.DeepSpeakerModel(512, 16).to(cuda_dev)
    m.load_state_dict(sd)
    m.train()
    e = m(O.make_input(16, T, 500, 3.0).cuda())
    (e * torch.randn(e.shape, generator=torch.Generator().manual_seed(0)).cuda()).sum().backward()
    torch.cuda.synchronize()
    sd_now = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}   # running stats moved by the first call
    train_forward_and_check("train fp16 B=16 -> 7 T=48", m, sd_now, "fp16", O.make_input(7, T, 501, 3.0).cuda(), T)


# ---- CPU self-test of the checker ---------------------------------------------------------------------------------
def emulate_layer(a16, w16, s32, b32, r16, stride, pad, dt, defect=None):
    """An engine layer in fp32 arithmetic: im2col matmul of 16-bit operands, fp32 affine (+ residual), clip, rn16."""
    N, C, H, W = a16.shape
    if defect == "shift":
        a16 = torch.cat([a16[:, :, 1:], torch.zeros_like(a16[:, :, :1])], dim=2)
    if defect == "tap":
        w16 = w16.clone()
        w16[:, :, 0, 1] = 0
    k = w16.shape[2]
    cols = F.unfold(a16.float(), k, padding=pad, stride=stride)                    # (N, cin*k*k, P)
    acc = (w16.float().reshape(w16.shape[0], -1) @ cols)
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    out = acc.view(N, -1, Ho, Wo) * s32.view(1, -1, 1, 1) + b32.view(1, -1, 1, 1)
    if r16 is not None:
        out = out + r16.float()
    out = rn16(out.clamp(0, 20), dt).double()
    if defect == "last_tile":   # the last 128 positions of the padded output layout
        n, h, w = torch.meshgrid(torch.arange(N), torch.arange(Ho), torch.arange(Wo), indexing="ij")
        pos = (n * (Ho + 1) + h + 1) * (Wo + 1) + w + 1
        out = out * (pos < pos.max() - 127).unsqueeze(1)
    return out


def _layer_setup(dt, N=3, C=64, H=8, W=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    a16 = rn16(torch.randn(N, C, H, W, generator=g).abs() * 2, dt)
    w = torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    gam = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    beta = torch.randn(C, generator=g) * 0.1
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.empty(C).uniform_(0.5, 1.5, generator=g)
    r16 = rn16(torch.randn(N, C, H, W, generator=g).abs(), dt)
    s32 = gam / torch.sqrt(rv + 1e-5)
    b32 = beta - rm * s32
    sd = {"p.weight": gam, "p.bias": beta, "p.running_mean": rm, "p.running_var": rv}
    return a16, rn16(w, dt), s32, b32, r16, sd


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("defect", [None, "tap", "shift", "last_tile"])
def test_checker_passes_an_emulated_layer_and_fails_seeded_defects(dt, defect):
    a16, w16, s32, b32, r16, sd = _layer_setup(dt)
    s, b, ms = folded_bn(sd, "p")
    got = emulate_layer(a16, w16, s32, b32, r16, 1, 1, dt, defect)
    ref, bound = conv_ref(a16.double(), w16.double(), s, b, ms, r16.double(), 1, 1, U[dt])
    msg, worst, inside = check(f"{defect}", got, ref, bound)
    if defect is None:
        assert msg is None and inside >= 0.2, msg
    else:
        assert msg is not None, f"seeded defect {defect} passed (max err/bound {worst:.3g})"


def emulate_conv1(x, w, s32, b32, dt, lo=True):
    """conv1_umma_kernel's arithmetic: hi/lo 16-bit halves of x and w, x_hi*w_hi + x_lo*w_hi + x_hi*w_lo (without the
    lo halves: x_hi*w_hi only), fp32 affine, clip, rn16."""
    xh = rn16(x, dt)
    wh = rn16(w, dt)
    xl, wl = rn16(x - xh, dt), rn16(w - wh, dt)
    cv = lambda p, q: F.conv2d(p.double(), q.double(), None, 2, 2)
    acc = cv(xh, wh) + ((cv(xl, wh) + cv(xh, wl)) if lo else 0)
    out = acc.float() * s32.view(1, -1, 1, 1) + b32.view(1, -1, 1, 1)
    return rn16(out.clamp(0, 20), dt).double()


@pytest.mark.parametrize("lo", [True, False])
def test_checker_pins_the_conv1_lo_half(lo):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 1, 32, 64, generator=g) * 4
    w = torch.randn(64, 1, 5, 5, generator=g) * (2.0 / 25) ** 0.5
    gam, beta = torch.empty(64).uniform_(0.5, 1.5, generator=g), torch.randn(64, generator=g) * 0.1
    rm, rv = torch.randn(64, generator=g) * 0.1, torch.empty(64).uniform_(0.5, 1.5, generator=g)
    sd = {"p.weight": gam, "p.bias": beta, "p.running_mean": rm, "p.running_var": rv}
    s32 = gam / torch.sqrt(rv + 1e-5)
    got = emulate_conv1(x, w, s32, beta - rm * s32, "fp16", lo)
    s, b, ms = folded_bn(sd, "p")
    xd, wd = x.double(), w.double()
    ref, bound = conv_ref(xd, wd, s, b, ms, None, 2, 2, U["fp16"], extra=conv1_operand_term(xd, wd, s, U["fp16"]))
    msg, _, _ = check(f"conv1 lo={lo}", got, ref, bound)
    frac = rounding_fraction(got, ref, "fp16")
    print(f"  stored != rn16(fp64): {frac:.2%}")
    if lo:
        assert msg is None and frac <= 0.02, (msg, frac)
    else:
        assert frac > 0.02


def emulate_bn_stats(raw, pivot, gx=None, defect=None):
    """Batch mean / biased variance of an [M][C] fp32 tensor by bn_stats_partial_kernel + bn_finalize_kernel's
    summation order: per-thread fp32 chains over rows m = 32*bx + p + k*32*gx, a 32-term fp32 sum per block, the block
    partials added in fp64.  pivot=False: the plain sums E[x^2] - mean^2; pivot=True: sums of x - x[0].  gx: the
    partial blocks (default: the library's stat_blocks); defect "drop_block": the last block's partials are lost.
    -> (mean, var, the chains' length)."""
    M, C = raw.shape
    if gx is None:
        gx = stat_blocks(M, C)
    k = raw[0].astype(np.float32) if pivot else np.zeros(C, np.float32)
    n1 = -(-M // (32 * gx))
    pad = np.zeros((n1 * 32 * gx, C), np.float32)
    pad[:M] = raw - k
    valid = np.zeros((n1 * 32 * gx, 1), np.float32)
    valid[:M] = 1
    d = pad.reshape(n1, gx, 32, C)
    vmask = valid.reshape(n1, gx, 32, 1)
    s = np.zeros((gx, 32, C), np.float32)
    ss = np.zeros((gx, 32, C), np.float32)
    for i in range(n1):
        di = d[i] * vmask[i]
        s = (s + di).astype(np.float32)
        ss = (ss + di * di).astype(np.float32)     # fmaf: the square is exact enough here, one rounding per step
    bs = np.zeros((gx, C), np.float32)
    bss = np.zeros((gx, C), np.float32)
    for p in range(32):
        bs = (bs + s[:, p]).astype(np.float32)
        bss = (bss + ss[:, p]).astype(np.float32)
    if defect == "drop_block":
        bs, bss = bs[:-1], bss[:-1]
    S, SS = bs.astype(np.float64).sum(0), bss.astype(np.float64).sum(0)
    dm = S / M
    return k.astype(np.float64) + dm, SS / M - dm * dm, reduce_chain(M, 0, gx, False)


def emulate_record_stats(raw, N, defect=None):
    """The synchronised path's statistics of N utterances of HW = M / N rows each (bn_utt_record_kernel +
    bn_record_finalize_kernel): per utterance, fp32 sums of x - k_u (k_u its first row) by 32 lanes striding over the
    rows, a 5-level tree over the lanes; the records combined in fp64 around K = k_0.  defect "drop_record": the last
    utterance's record is lost.  -> (mean, var, the chains' length)."""
    M, C = raw.shape
    HW = M // N
    u = raw.reshape(N, HW, C)
    k = u[:, 0].astype(np.float32)                                  # (N, C)
    n1 = -(-HW // 32)
    pad = np.zeros((N, n1 * 32, C), np.float32)
    pad[:, :HW] = u - k[:, None]
    d = pad.reshape(N, n1, 32, C)                                   # lane p walks rows p, p + 32, ...
    s = np.zeros((N, 32, C), np.float32)
    ss = np.zeros((N, 32, C), np.float32)
    for i in range(n1):
        s = (s + d[:, i]).astype(np.float32)
        ss = (ss + d[:, i] * d[:, i]).astype(np.float32)
    half = 16
    while half:
        s = (s[:, :half] + s[:, half:2 * half]).astype(np.float32)
        ss = (ss[:, :half] + ss[:, half:2 * half]).astype(np.float32)
        half >>= 1
    keep = N - 1 if defect == "drop_record" else N
    sd, ssd = s[:keep, 0].astype(np.float64), ss[:keep, 0].astype(np.float64)
    dk = k[:keep].astype(np.float64) - k[0].astype(np.float64)
    S1 = (sd + HW * dk).sum(0)
    S2 = (ssd + 2 * dk * sd + HW * dk * dk).sum(0)
    Mk = keep * HW
    dm = S1 / Mk
    return k[0].astype(np.float64) + dm, S2 / Mk - dm * dm, reduce_chain(M, HW, 0, True)


# (how the statistics are summed, rows M, partial blocks gx or utterances N): the library's plan at 128 x 80 x 32 rows
# (chains of 50), and chains of 400 and more: the unsynchronised reductions when M / gx is large, the synchronised records
# of long utterances (2 x 12800 pixels)
STAT_SETUPS = {"plain M=327680": ("blocks", 128 * 80 * 32, None), "plain M=47104 gx=4": ("blocks", 47104, 4),
               "records N=2 HW=12800": ("records", 2 * 12800, 2)}


def _emulated_stats(setup, raw, pivot, defect=None):
    kind, _, arg = STAT_SETUPS[setup]
    if kind == "records":
        return emulate_record_stats(raw, arg, defect)
    return emulate_bn_stats(raw, pivot, arg, defect)


def _running_check(name, raw, mean_e, var_e, n):
    M, C = raw.shape
    r64 = torch.from_numpy(raw.astype(np.float64))
    mean, var = r64.mean(0), r64.var(0, unbiased=False)
    rm0, rv0 = torch.zeros(C, dtype=torch.float64), torch.ones(C, dtype=torch.float64)
    unb_e = torch.from_numpy(var_e) * M / (M - 1)
    rm1 = (0.9 * rm0 + 0.1 * torch.from_numpy(mean_e)).float().double()
    rv1 = (0.9 * rv0 + 0.1 * unb_e).float().double()
    return running_stats_check(name, rm0, rv0, rm1, rv1, mean, var, M, n)


@pytest.mark.parametrize("pivot", [True, False])
def test_checker_catches_unshifted_bn_statistics(pivot):
    """Batch variance at mean/std 1000 (M = 128*80*32 rows, the library's gx: chains of 50): from unshifted fp32 sums
    the running-variance check fails, from sums around a per-channel pivot it passes."""
    unshifted_case("plain M=327680", pivot)


@pytest.mark.parametrize("setup,pivot", [("plain M=47104 gx=4", True), ("plain M=47104 gx=4", False),
                                         ("records N=2 HW=12800", True)])
def test_checker_catches_unshifted_bn_statistics_at_long_chains(setup, pivot):
    """The same at chains of 400 and more (the synchronised records always sum around a pivot)."""
    assert unshifted_case(setup, pivot) >= 400


def unshifted_case(setup, pivot):
    g = np.random.RandomState(3)
    M, C = STAT_SETUPS[setup][1], 64
    raw = (g.standard_normal((M, C)) + 1000.0).astype(np.float32)
    mean_e, var_e, n = _emulated_stats(setup, raw, pivot)
    r = _running_check(f"pivot={pivot}", raw, mean_e, var_e, n)
    assert (r <= 1.0) == pivot, r
    return n


@pytest.mark.parametrize("setup", STAT_SETUPS)
@pytest.mark.parametrize("defect", [None, "drop"])
def test_checker_passes_long_bn_chains_and_catches_a_dropped_partial(setup, defect):
    """Channels of mean/std from 0 to 30 (the plain sums) summed in fp32 by the kernels' order, at chains of 50 to 405
    terms: within the n-dependent bound; with one partial block (synchronised: one utterance's record) lost, not."""
    g = np.random.RandomState(5)
    M, C = STAT_SETUPS[setup][1], 64
    raw = (g.standard_normal((M, C)) * np.linspace(0.5, 2, C) + np.linspace(0, 30, C)).astype(np.float32)
    kind = STAT_SETUPS[setup][0]
    d = None if defect is None else ("drop_record" if kind == "records" else "drop_block")
    mean_e, var_e, n = _emulated_stats(setup, raw, False, d)
    r = _running_check(f"{setup} defect={defect}", raw, mean_e, var_e, n)
    assert (r <= 1.0) == (defect is None), r
