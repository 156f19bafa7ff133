"""Every layer of the train backward against fp64, recomputed from that layer's own inputs.

The parameter-gradient gates of test_gpu_train_parity (4e-3 rel-L2 per tensor) leave room for a localised error: one
64x64 block of one tap of a weight gradient, a dropped K chunk, the last tile of a data gradient, one channel block of
dgamma; and errors build up through the layers, so a failure there cannot say which layer is wrong.  Here a production
backward runs with dsk_debug_set_backward_capture, which copies the gradients between layers out of the ping-pong
buffers the next layer overwrites, and every captured quantity is recomputed in float64 from exactly what the engine
consumed at that step: its own 16-bit gradients, its saved activations (dsk_train_ctx_read) and its loss scale S.  Every
element must lie within a worst-case bound computed from magnitudes (u = 2^-11 fp16, 2^-8 bf16, ACC = 2^-23 per fp32
accumulation step as in test_gpu_layer_parity, TINY = 2^-25 for fp16 subnormals):

  g_fc       10/|x| (g - xh (xh . g)), x the saved fc output: delta = (E + 16) ACC 10/|x| (|g| + |xh| sum|xh g|)
             (the fp32 norm and dot product are chains of E terms, a few more roundings on top).
  S          exact: 2^floor(log2(512 / max|g_fc|)) clamped to [2^-24, 2^40] (fp16, automatic), the value of
             dsk_set_loss_scale when set, 1 for bf16; {S, 1/S} are stored.
  fc grads   g_fc^T P with P the fp64 time mean of the engine's y_11: delta = (B + H4 + 16) ACC |g_fc|^T P (B products
             in fp32 plus the fp32 pooling of H4 rows, as tail_ref); the bias: (B + 2) ACC sum|g_fc|.
  dP         g_fc W_fc: delta = (E + 8) ACC |g_fc| |W_fc|.
  gy_11      dP S / H4 rounded once to 16 bit after an fp32 product: |err| <= (u + 2^-22) |ref| + TINY.
  G_i        a (gz - b - xhat d), gz = gy_i where the STORED y_i lies in (0, 20) (bn_bwd_reduce_kernel's rule), fp64
             batch statistics of raw_i, a = gamma rstd, b = sum gz / M, d = sum gz xhat / M.  The engine's fp32 mean /
             rstd are off by stat_eps (eps relative to std / var, from the forward's chains of the same n terms as
             below), so its xhat by dx = eps (1 + |xhat|) + 2^-22 |xhat|.  Its sums are fp32 chains of n terms (bn_bwd_reduce: ceil(M /
             32 gx) per thread + 32 in the block; synchronised path: ceil(HW / 32) per lane + a 5-level tree per
             utterance) added in fp64: db = (n + 2) 2^-24 sum|gz| / M, dd = ((n + 3) 2^-24 sum|gz xhat| + eps (sum|gz|
             + sum|gz xhat|) + 2^-22 sum|gz xhat|) / M.  delta = |a| (db + |xhat| dd + |d| dx + 2^-22 (|gz| + |b| +
             |xhat d|)) + |a| (eps + 2^-22) |gz - b - xhat d|; bound = u (|ref| + delta) + TINY + delta.
  gres_i     gz itself: bit-exact.
  dbeta      sum gz / S, delta = (n + 2) 2^-24 sum|gz| / S;  dgamma: sum gz xhat / S with M dd / S.
  gy_j       dgrad of layer j+1 from the engine's G_{j+1} and the 16-bit weight (+ gres_{j+2} when y_j is a skip
             input): the forward checker's form, delta = (K + 8) ACC A + 2^-22 |res|, K = 9 cout (stride 1) or
             {3,2} x {3,2} cout by the parity class of the input pixel (stride 2).
  dW_i       conv2d_weight(y_{i-1}, G_i) / S.  16-bit x 16-bit products are exact in fp32; the wgmma chain of a K
             split adds 8 K16 steps per 128-pixel chunk, each rounding by at most ACC of the running sum's magnitude
             <= A, then the ksplit slices are added in fp32: delta = (n + 2) ACC A with n = 8 per + ksplit (per =
             chunks per split; ksplit, per and the BatchNorm reductions' gx are the library's own plan, read with
             dsk_debug_backward_plan).  A long reduction with random signs makes that loose (A / |ref| ~
             sqrt(#pixels)), so each (tap, 64 cout, 64 cin) block is also held to a rel-L2 gate from the same chain
             under the probabilistic model of rounding errors (independent, mean zero, Higham & Mary 2019): rms error
             <= sqrt(n) ACC rms(A), gate = 2 sqrt(n) ACC ||A||_blk / ||ref||_blk.  It fails a block whose elements
             each stay inside their worst-case bound but together are further off than the accumulation can explain
             (the self-test seeds one at 0.8 of the bound), which the element check cannot see.
  dW_0       conv1_wgrad_partial (32 fmaf per lane + 8 warp partials in fp32) and fp64 sum_partials:
             delta = 44 2^-24 A.

Violations are reported with `locate` (where they cluster); a NaN or inf anywhere counts as one.  Every capture
buffer starts as NaN and must hold finite values after the backward, so a copy that never happens fails.  Each case
prints the largest err/bound of every check and the worst block rel-L2 with its gate, per layer.  The CPU self-test at
the end runs the same checks on a backward layer emulated in fp32 from 16-bit operands and on seeded defects, so it
runs everywhere.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from oracle import rescnn_oracle as O
from tests.test_gpu_layer_parity import (ACC, CONV, TD, TINY, U, act_geometry, batch_stats, calibrated, check,
                                         check_eval_chain, read_eval_activations, rn16, stat_eps,
                                         unpack_eval_activations)
from tests.train_plan import reduce_chain

U24 = 2.0 ** -24


# ---- the checker --------------------------------------------------------------------------------------------------
def as4d(t):
    return t.reshape(1, -1, 1, 1) if t.dim() == 1 else t.reshape(*t.shape[:2], 1, 1) if t.dim() == 2 else t


class Report:
    """Collects the per-element and per-block checks of one backward: prints every margin, asserts at the end (so a
    failing case still prints the whole table)."""

    def __init__(self, tag):
        self.tag, self.fails, self.worst = tag, [], {}
        print(f"[{tag}]")

    def elem(self, name, got, ref, bound):
        msg, worst, _ = check(name, as4d(got), as4d(ref), as4d(bound), saturating=False)
        self.worst[name] = worst
        if msg:
            self.fails.append(f"{name}: {msg}")

    def blocks(self, name, got, ref, A, n):
        rel, ratio = block_rel_l2(got, ref, A, n)
        ratio = torch.nan_to_num(ratio, nan=float("inf"), posinf=float("inf"))   # a NaN block fails
        worst = ratio.max().item()
        name = f"{name} blocks"
        self.worst[name] = worst
        print(f"  {name:<12} rel-L2 max {rel.max().item():.3g}, max rel-L2/gate {worst:.3f}")
        viol = ~(ratio <= 1.0)
        if bool(viol.any()):
            bad = viol.nonzero().tolist()
            self.fails.append(f"{name}: {len(bad)} of {ratio.numel()} (cout block, cin block, tap) blocks over the "
                              f"rel-L2 gate, first {bad[:4]}, worst rel-L2/gate {worst:.3g}")

    def exact(self, name, ok):
        print(f"  {name:<12} {'bit-exact' if ok else 'DIFFERS'}")
        if not ok:
            self.fails.append(f"{name}: not bit-exact")

    def assert_ok(self):
        assert not self.fails, f"{self.tag}:\n  " + "\n  ".join(self.fails)


def block_rel_l2(got, ref, A, n):
    """Per (64 cout, 64 cin, tap) block of a (cout, cin, k, k) weight gradient: rel-L2 and rel-L2 / gate with
    gate = 2 sqrt(n) ACC ||A|| / ||ref||."""
    co, ci, k, _ = ref.shape
    f = lambda t: t.reshape(co // 64, 64, ci // 64, 64, k * k).pow(2).sum(dim=(1, 3))
    e2, r2, a2 = f(got.double() - ref), f(ref), f(A)
    return (e2 / r2.clamp_min(1e-300)).sqrt(), e2.sqrt() / (2 * math.sqrt(n) * ACC * a2.sqrt() + 1e-30)


def bn_bwd_ref(gy, y, raw, gamma, nchain):
    """fp64 BatchNorm + clip backward of one layer from the engine's gy, stored y and raw (N,C,H,W), with the error
    model of the module docstring.  -> gz, G (times S), its delta, sum gz and sum gz xhat (times S) with their deltas."""
    v = lambda t: t.view(1, -1, 1, 1)
    dims = (0, 2, 3)
    gz = torch.where((y > 0) & (y < 20), gy, torch.zeros_like(gy))
    mean, var = batch_stats(raw)
    rstd = 1.0 / torch.sqrt(var + O.BN_EPS)
    xhat = (raw - v(mean)) * v(rstd)
    M = raw.numel() // raw.shape[1]
    s, ss = gz.sum(dims), (gz * xhat).sum(dims)
    sg, sgx = gz.abs().sum(dims), (gz * xhat).abs().sum(dims)
    a, b, d = gamma * rstd, s / M, ss / M
    inner = gz - v(b) - xhat * v(d)
    eps = stat_eps(mean, var, nchain)
    dx = v(eps) * (1 + xhat.abs()) + 2.0 ** -22 * xhat.abs()
    db = (nchain + 2) * U24 * sg / M
    dd = ((nchain + 3) * U24 * sgx + eps * (sg + sgx) + 2.0 ** -22 * sgx) / M
    delta = (v(a.abs()) * (v(db) + xhat.abs() * v(dd) + v(d.abs()) * dx
                           + 2.0 ** -22 * (gz.abs() + v(b.abs()) + (xhat * v(d)).abs()))
             + v(a.abs() * (eps + 2.0 ** -22)) * inner.abs())
    return gz, v(a) * inner, delta, (s, db * M), (ss, dd * M)


def dgrad_ref(G, w16, stride, shape, res, u):
    """fp64 data gradient of a conv (3x3 s1 p1 or 5x5 s2 p2) from G and the 16-bit weight, + res; (ref, bound)."""
    k = w16.shape[2]
    ref = conv2d_input(list(shape), w16, G, stride, k // 2)
    A = conv2d_input(list(shape), w16.abs(), G.abs(), stride, k // 2)
    cout = w16.shape[0]
    if stride == 1:
        K = 9 * cout
    else:   # input row parity 0 sees filter rows {0, 2, 4}, parity 1 rows {1, 3}; the same for columns
        par = lambda n: (3 - torch.arange(n) % 2).to(G.device, torch.float64)
        K = cout * par(shape[2]).view(-1, 1) * par(shape[3]).view(1, -1)
    delta = (K + 8) * ACC * A
    if res is not None:
        ref = ref + res
        delta = delta + 2.0 ** -22 * res.abs()
    return ref, u * (ref.abs() + delta) + TINY + delta


def check_wgrad(rep, name, got, a, G, S, stride, per, ksplit):
    k = got.shape[2]
    ref = conv2d_weight(a, got.shape, G, stride, k // 2) / S
    A = conv2d_weight(a.abs(), got.shape, G.abs(), stride, k // 2) / S
    n = 8 * per + ksplit
    rep.elem(name, got, ref, (n + 2) * ACC * A + 1e-30)
    rep.blocks(name, got, ref, A, n)


def check_bn(rep, i, gy, y, raw, gamma, nchain, G, dgamma, dbeta, S, u):
    gz, ref, delta, (s, ds), (ss, dss) = bn_bwd_ref(gy, y, raw, gamma, nchain)
    rep.elem(f"G {i}", G, ref, u * (ref.abs() + delta) + TINY + delta)
    rep.elem(f"dbeta {i}", dbeta, s / S, ds / S + 1e-30)
    rep.elem(f"dgamma {i}", dgamma, ss / S, dss / S + 1e-30)
    return gz


# ---- the engine's plans -------------------------------------------------------------------------------------------
def backward_plan(eng, tctx):
    """Per conv layer (ksplit, 128-pixel chunks per split, BatchNorm partial blocks gx) of the backward the context
    is bound to, as the library planned it (dsk_debug_backward_plan): the bounds follow the plan that runs."""
    out = []
    for i in range(12):
        v = (ctypes.c_int32 * 3)()
        L.check(eng.lib.dsk_debug_backward_plan(eng.handle, tctx, i, v), "dsk_debug_backward_plan")
        out.append(tuple(v))
    return out


def expected_scale(dt, fixed, g_fc):
    if fixed:
        return fixed
    if dt == "bf16":
        return 1.0
    m = g_fc.abs().max().item()
    if not (m > 0 and math.isfinite(m)):
        return 1.0
    f, e = math.frexp(m)                       # m = f 2^e, 0.5 <= f < 1: floor(log2(512 / m)) = 9 - e (+1 at f = 0.5)
    return min(max(2.0 ** (9 - e + (f == 0.5)), 2.0 ** -24), 2.0 ** 40)


# ---- GPU driver ---------------------------------------------------------------------------------------------------
def capture_buffers(B, T, E, dt, dev):
    """NaN-filled destinations of every capture entry (a copy that never happens shows up as NaN)."""
    cap, buf = L.DskBackwardCapture(), {"gy": [], "G": [], "gres": {}}
    nan = lambda shape, dtype: torch.full(shape, float("nan"), dtype=dtype, device=dev)
    for i in range(12):
        C, H, W = act_geometry(i, T)
        for key in ("gy", "G"):
            buf[key].append(nan((B, H, W, C), TD[dt]))
            getattr(cap, key)[i] = buf[key][i].data_ptr()
        if i % 3 == 2:
            buf["gres"][i] = nan((B, H, W, C), TD[dt])
            cap.gres[i] = buf["gres"][i].data_ptr()
    for key, shape in (("g_fc", (B, E)), ("fc_out", (B, E)), ("dP", (B, 2048)), ("loss_scale", (2,))):
        buf[key] = nan(shape, torch.float32)
        setattr(cap, key, buf[key].data_ptr())
    return cap, buf


def read_ctx(m, tctx, B, T, which):
    eng = m._engine
    out = []
    for i in range(12):
        C, H, W = act_geometry(i, T)
        t = torch.empty(B, C, H, W, device="cuda", dtype=torch.float32)
        L.check(eng.lib.dsk_train_ctx_read(eng.handle, tctx, which, i, t.data_ptr(), L.cur_stream()), "dsk_train_ctx_read")
        out.append(t)
    return out


def backward_case(tag, m, sd, dt, x, fixed_scale=None, sync=False):
    """Train forward, read raw / y, backward of (emb * w).sum() with the capture set, then every check.  The same
    backward without the capture must give bit-identical parameter gradients."""
    B, T, E = x.shape[0], x.shape[2], m.embedding_size
    dev = x.device
    eng = m._get_engine(dev)
    if fixed_scale:
        eng.set_loss_scale(fixed_scale)
    w = torch.randn(B, E, generator=torch.Generator().manual_seed(11)).to(dev)
    params = dict(m.named_parameters())
    grads_of = lambda: {k: p.grad.detach().clone() for k, p in params.items() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    (m(x) * w).sum().backward()
    plain = grads_of()
    m.zero_grad(set_to_none=True)
    emb = m(x)
    fn = emb.grad_fn
    tctx = fn.guards[0].tctx if sync else fn.guard.tctx
    raw, y = read_ctx(m, tctx, B, T, 0), read_ctx(m, tctx, B, T, 1)
    plan = backward_plan(eng, tctx)
    cap, buf = capture_buffers(B, T, E, dt, dev)
    L.check(eng.lib.dsk_debug_set_backward_capture(eng.handle, ctypes.byref(cap)), "dsk_debug_set_backward_capture")
    try:
        (emb * w).sum().backward()
    finally:
        L.check(eng.lib.dsk_debug_set_backward_capture(eng.handle, None), "dsk_debug_set_backward_capture")
    torch.cuda.synchronize()
    assert_captured(tag, buf)
    grads = grads_of()
    assert len(grads) == 38
    for k in grads:
        assert torch.equal(grads[k], plain[k]), f"{tag}: {k} differs with the capture on"
    check_backward(tag, sd, dt, x, raw, y, w, buf, grads, fixed_scale, sync, E, plan)


def assert_captured(tag, buf):
    """Every capture destination holds finite values only: each copy landed (the buffers start as NaN), and the
    engine wrote no NaN or inf, not even where a clip mask later drops the value."""
    items = ([(f"gy {i}", t) for i, t in enumerate(buf["gy"])] + [(f"G {i}", t) for i, t in enumerate(buf["G"])]
             + [(f"gres {i}", t) for i, t in buf["gres"].items()]
             + [(k, buf[k]) for k in ("g_fc", "fc_out", "dP", "loss_scale")])
    bad = [name for name, t in items if not bool(torch.isfinite(t).all())]
    assert not bad, f"{tag}: non-finite values (or a copy that never happened) in {', '.join(bad)}"


def check_backward(tag, sd, dt, x, raw, y, w, buf, grads, fixed_scale, sync, E, plan):
    u, dev = U[dt], x.device
    B, T = x.shape[0], x.shape[2]
    H4 = T // 16
    rep = Report(tag)
    nchw = lambda t: t.permute(0, 3, 1, 2).double()
    # tail: l2-norm backward, loss scale, fc, pooling
    fc_out, g = buf["fc_out"].double(), w.double()
    inv = 1.0 / torch.sqrt((fc_out * fc_out).sum(1, keepdim=True) + 1e-10)
    xh = fc_out * inv
    ref = 10 * inv * (g - xh * (xh * g).sum(1, keepdim=True))
    A = 10 * inv * (g.abs() + xh.abs() * (xh * g).abs().sum(1, keepdim=True))
    rep.elem("g_fc", buf["g_fc"], ref, (E + 16) * ACC * A + 1e-30)
    S = expected_scale(dt, fixed_scale, buf["g_fc"])
    ls = buf["loss_scale"].tolist()
    print(f"  S            {ls[0]:g} (expected {S:g})")
    assert ls == [S, 1.0 / S], f"{tag}: loss scale {ls}, expected [{S}, {1.0 / S}]"
    gf = buf["g_fc"].double()
    P = y[11].double().mean(dim=2).reshape(B, -1)                       # column c*4 + w, as fc.weight
    rep.elem("fc.weight", grads["model.fc.weight"], gf.T @ P, (B + H4 + 16) * ACC * (gf.abs().T @ P) + 1e-30)
    rep.elem("fc.bias", grads["model.fc.bias"], gf.sum(0), (B + 2) * ACC * gf.abs().sum(0) + 1e-30)
    Wfc = sd["model.fc.weight"].to(dev).double()
    dP = buf["dP"].view(B, 4, 512).transpose(1, 2).double()              # (B, c, w): engine column w*512 + c
    rep.elem("dP", dP.reshape(B, 2048), gf @ Wfc, (E + 8) * ACC * (gf.abs() @ Wfc.abs()) + 1e-30)
    ref = (dP * S / H4).unsqueeze(2).expand(B, 512, H4, 4)
    rep.elem("gy 11", nchw(buf["gy"][11]), ref, (u + 2.0 ** -22) * ref.abs() + TINY)
    # layers 11 .. 0
    for i in range(11, -1, -1):
        wkey, prefix, k, stride = CONV[i]
        C, H, W = act_geometry(i, T)
        ksplit, per, gx = plan[i]
        nchain = reduce_chain(B * H * W, H * W, gx, sync)
        # the bounds are first order in n 2^-24 (the n^2 2^-48 terms are dropped): n stays far below 2^14
        assert nchain * U24 <= 2.0 ** -10, f"layer {i}: reduction chains of {nchain} terms"
        yd = y[i].double()
        gz = check_bn(rep, i, nchw(buf["gy"][i]), yd, raw[i].double(), sd[prefix + ".weight"].to(dev).double(),
                      nchain, nchw(buf["G"][i]), grads[prefix + ".weight"], grads[prefix + ".bias"], S, u)
        if i % 3 == 2:
            keep = ((y[i] > 0) & (y[i] < 20)).permute(0, 2, 3, 1)
            gy16 = buf["gy"][i]
            rep.exact(f"gres {i}", torch.equal(torch.where(keep, gy16, torch.zeros_like(gy16)).view(torch.int16),
                                               buf["gres"][i].view(torch.int16)))
        del gz
        Gd = nchw(buf["G"][i])
        if i == 0:
            xd = x.double()
            ref = conv2d_weight(xd, (64, 1, 5, 5), Gd, 2, 2) / S
            A = conv2d_weight(xd.abs(), (64, 1, 5, 5), Gd.abs(), 2, 2) / S
            rep.elem("dW 0", grads[wkey], ref, 44 * U24 * A + 1e-30)
            continue
        w16 = rn16(sd[wkey].to(dev).double(), dt)
        assert ksplit >= 1 and per >= 1, f"layer {i}: weight-gradient plan {plan[i]}"
        check_wgrad(rep, f"dW {i}", grads[wkey], y[i - 1].double(), Gd, S, stride, per, ksplit)
        res = nchw(buf["gres"][i + 1]) if i % 3 == 1 else None          # y_{i-1} is the skip input of layer i+1
        ref, bound = dgrad_ref(Gd, w16, stride, y[i - 1].shape, res, u)
        rep.elem(f"gy {i - 1}", nchw(buf["gy"][i - 1]), ref, bound)
    rep.assert_ok()
    return rep


def train_model(E, dt, seed, dev):
    sd = O.make_state_dict(seed, 16, embedding_size=E)
    m = dsk.DeepSpeakerModel(E, 16, operand_dtype=dt).to(dev)
    m.load_state_dict(sd)
    return m.train(), sd


# the forward checker's train cases; B=2, T=16 (layer 11: 4 pixels per channel); B=33 (not a tile multiple)
CASES = [("fp16", 128, 160), ("fp16", 6, 160), ("fp16", 5, 32), ("bf16", 16, 48), ("fp16", 2, 16), ("fp16", 33, 48)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,B,T", CASES)
def test_backward_layer_by_layer(cuda_dev, dt, B, T):
    m, sd = train_model(512, dt, 6, cuda_dev)
    backward_case(f"backward {dt} B={B} T={T}", m, sd, dt, O.make_input(B, T, 400 + B, 3.0).cuda())


@pytest.mark.gpu
def test_backward_with_a_fixed_loss_scale_below_one(cuda_dev):
    m, sd = train_model(512, "fp16", 8, cuda_dev)
    backward_case("backward fp16 B=8 T=48 S=2^-4", m, sd, "fp16", O.make_input(8, 48, 410, 3.0).cuda(),
                  fixed_scale=2.0 ** -4)


@pytest.mark.gpu
def test_backward_after_rebinding_to_a_smaller_batch(cuda_dev):
    """A context sized for B=16 serves a forward and backward, then is re-bound to B=7 (ctx_bind)."""
    T = 48
    m, sd = train_model(512, "fp16", 7, cuda_dev)
    e = m(O.make_input(16, T, 500, 3.0).cuda())
    (e * torch.randn(e.shape, generator=torch.Generator().manual_seed(0)).cuda()).sum().backward()
    torch.cuda.synchronize()
    backward_case("backward fp16 B=16 -> 7 T=48", m, sd, "fp16", O.make_input(7, T, 501, 3.0).cuda())


@pytest.mark.gpu
def test_synchronised_batchnorm_backward_on_one_shard(cuda_dev):
    m, sd = train_model(512, "fp16", 9, cuda_dev)
    m.sync_batchnorm()
    backward_case("sync backward fp16 B=8 T=48", m, sd, "fp16", O.make_input(8, 48, 420, 3.0).cuda(), sync=True)


@pytest.mark.gpu
def test_backward_at_embedding_size_256(cuda_dev):
    m, sd = train_model(256, "fp16", 10, cuda_dev)
    backward_case("backward fp16 E=256 B=8 T=48", m, sd, "fp16", O.make_input(8, 48, 430, 3.0).cuda())


@pytest.mark.gpu
def test_eval_chain_at_embedding_size_128(cuda_dev):
    B, T = 16, 48
    x = O.make_input(B, T, 440, 4.0).cuda()
    sd = calibrated(O.make_state_dict(4, 16, embedding_size=128), x)
    m = dsk.DeepSpeakerModel(128, 16).to(cuda_dev)
    m.load_state_dict(sd)
    m.eval()
    with torch.no_grad():
        emb = m(x)
        bufs = read_eval_activations(m, B, T, "fp16")
    torch.cuda.synchronize()
    check_eval_chain(f"eval fp16 E=128 B={B} T={T}", sd, "fp16", x, unpack_eval_activations(m._engine.lib, bufs, B, T), emb)


# ---- CPU self-test of the checker ---------------------------------------------------------------------------------
def emulate_backward_layer(dt, defect=None, N=4, C=64, H=16, W=8, ksplit=4, S=8.0, seed=0):
    """One engine backward layer (3x3 s1, C -> C) in fp32 arithmetic from 16-bit operands: the train forward's stored
    y, the BatchNorm + clip backward with the engine's fp32 coefficients, the data gradient, and the weight gradient
    as 128-pixel chunks of K16 steps (each rounded once into an fp32 accumulator) in `ksplit` slices added in order.
    Every channel's largest xhat lands at pre = 19.9985, which the 16-bit storage rounds to 20 (clip closed).  The
    BatchNorm sums run as bn_bwd_reduce_kernel's fp32 chains with one partial block (M / 32 terms per thread, then the
    32 thread partials), so a tall layer (H = 400) makes chains of several hundred terms."""
    g = torch.Generator().manual_seed(seed)
    a16 = rn16(torch.randn(N, C, H, W, generator=g).abs() * 2, dt)
    w16 = rn16(torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5, dt)
    raw = F.conv2d(a16, w16, padding=1)
    gamma = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    mean, var = batch_stats(raw.double())
    rstd = 1.0 / torch.sqrt(var + O.BN_EPS)
    xmax = ((raw.double() - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1)).amax(dim=(0, 2, 3))
    beta = (19.9985 - gamma.double() * xmax).float()
    v = lambda t: t.view(1, -1, 1, 1)
    m32, r32 = mean.float(), rstd.float()
    sc = gamma * r32
    pre = raw * v(sc) + v(beta - m32 * sc)
    y16 = rn16(pre.clamp(0, 20), dt)
    gy16 = rn16(torch.randn(N, C, H, W, generator=g) * S, dt)
    # BatchNorm + clip backward (bn_bwd_reduce / finalize / apply)
    if defect == "clip_from_pre":
        pre64 = v(gamma.double()) * (raw.double() - v(mean)) * v(rstd) + v(beta.double())
        keep = (pre64 > 0) & (pre64 < 20)
    else:
        keep = (y16 > 0) & (y16 < 20)
    gz = torch.where(keep, gy16, torch.zeros_like(gy16))
    xh = (raw - v(m32)) * v(r32)
    M = N * H * W
    s, ss = chain_sums(gz, xh)
    G16 = rn16(v(gamma * r32) * (gz - v((s.double() / M).float()) - xh * v((ss.double() / M).float())), dt)
    dbeta = s if defect == "dbeta_unscaled" else s * (1.0 / S)
    dgamma = ss * (1.0 / S)
    # data gradient
    Gin, wd = G16, w16
    if defect == "shift":
        Gin = torch.cat([G16[:, :, :, 1:], torch.zeros_like(G16[:, :, :, :1])], dim=3)
    if defect == "tap":
        wd = w16.clone()
        wd[:, :, 0, 1] = 0
    gin = rn16(F.conv_transpose2d(Gin, wd, padding=1), dt)
    if defect == "last_tile":   # the last 128 pixels in (n, h, w) order
        gin = gin.permute(0, 2, 3, 1).reshape(M, C)
        gin[-128:] = 0
        gin = gin.view(N, H, W, C).permute(0, 3, 1, 2)
    # weight gradient: K16 steps of exact products (fp64 group sums), fp32 accumulation per slice, slices in order
    cols = F.unfold(a16.double(), 3, padding=1).view(N, C, 9, H * W).permute(0, 3, 1, 2).reshape(M, C * 9)
    Gm = G16.double().permute(0, 2, 3, 1).reshape(M, C)
    steps = torch.einsum("gpo,gpk->gok", Gm.view(M // 16, 16, C), cols.view(M // 16, 16, C * 9)).float()
    per = M // 128 // ksplit                              # 128-pixel chunks per slice
    dw = torch.zeros(C, C * 9)
    for sl in range(ksplit - (defect == "drop_slice")):
        acc = torch.zeros(C, C * 9)
        for st in range(sl * per * 8, (sl + 1) * per * 8):
            acc = acc + steps[st]
        dw = dw + acc
    dw = dw.view(C, C, 3, 3) * (1.0 / S)
    if defect == "block":
        dw[:, :, 1, 1] *= 1.01
    if defect == "block_within_bound":
        # every element of one (tap, 64 x 64) block off by 0.8 of its own worst-case bound, all in the same direction
        # (what a biased accumulation of that block looks like): each element passes, the block as a whole does not
        A = (Gm.abs().T @ cols.abs()).view(C, C, 3, 3) / S
        dw[:, :, 1, 1] += (0.8 * (8 * per + ksplit + 2) * ACC * A[:, :, 1, 1] * dw[:, :, 1, 1].sign()).float()
    if defect == "nan_element":
        gin[-1, -1, -1, -1] = float("nan")
    if defect == "missing_copy":   # what a capture entry whose copy never ran holds
        G16 = torch.full_like(G16, float("nan"))
    return dict(a16=a16, w16=w16, raw=raw, gamma=gamma, y16=y16, gy16=gy16, G16=G16, dbeta=dbeta, dgamma=dgamma,
                gin=gin, dw=dw, S=S, per=per, ksplit=ksplit, nchain=reduce_chain(M, H * W, 1, False))


def chain_sums(gz, xh):
    """sum gz and sum gz xhat per channel of (N,C,H,W) fp32 tensors in bn_bwd_reduce_kernel's order with one block:
    thread p adds rows p, p + 32, ... (NHWC row order) in fp32 (the second sum by fmaf: one rounding per step), then
    the 32 thread partials are added in order."""
    C = gz.shape[1]
    g = gz.permute(0, 2, 3, 1).reshape(-1, C)
    x = xh.permute(0, 2, 3, 1).reshape(-1, C)
    M = g.shape[0]
    pad = -(-M // 32) * 32 - M
    g = torch.cat([g, torch.zeros(pad, C)]).view(-1, 32, C)
    x = torch.cat([x, torch.zeros(pad, C)]).view(-1, 32, C)
    s, ss = torch.zeros(32, C), torch.zeros(32, C)
    for k in range(g.shape[0]):
        s = s + g[k]
        ss = (ss.double() + g[k].double() * x[k].double()).float()
    ts, tss = torch.zeros(C), torch.zeros(C)
    for p in range(32):
        ts, tss = ts + s[p], tss + ss[p]
    return ts, tss


# seeded defect -> the checks that must fail (None: any)
DEFECTS = {None: None, "tap": None, "shift": None, "last_tile": None, "drop_slice": None, "block": None,
           "clip_from_pre": None, "dbeta_unscaled": None, "block_within_bound": {"dW 1 blocks"},
           "nan_element": {"gy 0"}, "missing_copy": {"G 1", "dW 1", "dW 1 blocks", "gy 0"}}


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("defect", DEFECTS)
def test_checker_passes_an_emulated_backward_layer_and_fails_seeded_defects(dt, defect):
    check_emulated_layer(dt, defect, 16)


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("defect", DEFECTS)
def test_checker_at_bn_chains_of_several_hundred_terms(dt, defect):
    """The same emulated layer 400 pixels tall: BatchNorm chains of 432 terms, 25 chunks per weight-gradient split."""
    check_emulated_layer(dt, defect, 400)


def check_emulated_layer(dt, defect, H):
    e = emulate_backward_layer(dt, defect, H=H)
    print(f"  BatchNorm chains of {e['nchain']} terms")
    d = lambda t: t.double()
    rep = Report(f"emulated backward layer {dt}, defect {defect}")
    check_bn(rep, 1, d(e["gy16"]), d(e["y16"]), d(e["raw"]), d(e["gamma"]), e["nchain"], d(e["G16"]), e["dgamma"],
             e["dbeta"], e["S"], U[dt])
    check_wgrad(rep, "dW 1", e["dw"], d(e["a16"]), d(e["G16"]), e["S"], 1, e["per"], e["ksplit"])
    ref, bound = dgrad_ref(d(e["G16"]), d(e["w16"]), 1, e["a16"].shape, None, U[dt])
    rep.elem("gy 0", e["gin"], ref, bound)
    if defect is None:
        rep.assert_ok()
        assert float((e["y16"] == 20).double().mean()) > 0, "no element of the emulated layer is clipped at 20"
    else:
        assert rep.fails, f"seeded defect {defect} passed: {rep.worst}"
        caught = {f.split(":")[0] for f in rep.fails}
        print("  caught by: " + "; ".join(sorted(caught)))
        if DEFECTS[defect] is not None:
            assert caught == DEFECTS[defect], f"seeded defect {defect}: caught by {caught}, expected {DEFECTS[defect]}"


def test_a_capture_copy_that_never_happened_fails():
    """The capture destinations start as NaN; one that is never written (or an engine NaN / inf) must fail."""
    B, T, E = 2, 16, 64
    buf = {"gy": [], "G": [], "gres": {}}
    for i in range(12):
        C, H, W = act_geometry(i, T)
        buf["gy"].append(torch.zeros(B, H, W, C, dtype=torch.float16))
        buf["G"].append(torch.zeros(B, H, W, C, dtype=torch.float16))
        if i % 3 == 2:
            buf["gres"][i] = torch.zeros(B, H, W, C, dtype=torch.float16)
    for key, shape in (("g_fc", (B, E)), ("fc_out", (B, E)), ("dP", (B, 2048)), ("loss_scale", (2,))):
        buf[key] = torch.ones(shape)
    assert_captured("all written", buf)
    buf["G"][4] = torch.full_like(buf["G"][4], float("nan"))
    with pytest.raises(AssertionError, match="G 4"):
        assert_captured("G 4 never copied", buf)
    buf["G"][4].zero_()
    buf["gy"][7][0, 0, 0, 0] = float("inf")
    with pytest.raises(AssertionError, match="gy 7"):
        assert_captured("an inf in gy 7", buf)
