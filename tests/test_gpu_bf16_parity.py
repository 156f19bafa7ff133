"""The bf16 operand path (DSK_BF16, DeepSpeakerModel(operand_dtype="bf16")) held to the gates the fp16 path is held to.

Every tensor-core kernel has a bf16 instantiation, and a slip there (a 16-bit type or a pack / unpack for the wrong
format in one epilogue, a parity class of the 5x5 s2 backward, an edge of the 128-pixel tile or of a multi-wave grid
that only shows at B = 128) would pass a loose end-to-end gate.  So the bf16 path runs here at the fp16 path's shapes,
through the fp16 path's checkers:

- the standalone halo convs (3x3, 3x3 with a parity-planar output, 5x5 s2 from a parity-planar input, a tall image) and
  the implicit-GEMM conv (dsk_conv2d_nhwc) against fp64 from the bf16-rounded operands, every element within the
  per-element bound of test_gpu_layer_parity.conv_ref at u = 2^-8, every real pixel poisoned first and every pad
  position exactly 0 afterwards; a CPU self-test shows that bound fails a seeded defect of each kind;
- every layer of the train forward and backward (test_gpu_layer_parity, test_gpu_backward_layer_parity);
- the training step against the mask-pinned oracle rounding what the engine stores to bf16, and its bit reproducibility;
- the eval forward's batch invariance and EmbeddingPipeline, bit for bit.
"""
import ctypes

import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from oracle import rescnn_oracle as O
from tests.helpers import rel_l2
from tests.test_gpu_backward_layer_parity import backward_case, train_model
from tests.test_gpu_conv import SHAPES
from tests.test_gpu_forward import _fresh_model
from tests.test_gpu_forward_shapes import (POOL, _batch_calls, _check_activations, _env_id, _forward,
                                           _release_device_memory)  # noqa: F401  (_release_device_memory: autouse fixture)
from tests.test_gpu_halo_conv import from_padded, from_planar
from tests.test_gpu_layer_parity import (TINY, U, assert_layer, check, conv_ref, emulate_layer, read_eval_activations,
                                         rn16, train_forward_and_check, unpack_eval_activations)
from tests.test_gpu_train_parity import engine_step, make_model, oracle_step
from tests.test_halo_index_host import TALL_OP

BF = torch.bfloat16
UB = U["bf16"]


# ---- standalone convs: operands, layout, reference ---------------------------------------------------------------
def operands(seed, N, cin, cout, Hin, Win, k, stride):
    """fp32 input, weight, per-channel scale and bias, and residual of one conv (the fp16 conv tests' distributions)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, Hin, Win, generator=g) * 2.0
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (k * k * cin)) ** 0.5
    scale = torch.empty(cout).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(cout, generator=g) * 0.1
    res = torch.randn(N, cout, Hin // stride, Win // stride, generator=g) * 2.0
    return x, w, scale, bias, res


def affine_conv_ref(x16, w16, scale, bias, res16, stride, flags, u=UB):
    """fp64 reference and per-element bound of conv(x16, w16) * scale + bias (+ res16 if flags & 1) (clipped to
    [0, 20] if flags & 2): conv_ref's accumulation and rounding model, with the fp32 scale and bias passed as they
    are (no folded running mean).  Without the clip the bound is conv_ref's for the unclipped value."""
    s, b = scale.double(), bias.double()
    r = res16 if flags & 1 else None
    pad = w16.shape[2] // 2
    if flags & 2:
        return conv_ref(x16, w16, s, b, torch.zeros_like(s), r, stride, pad, u)
    pre, b0 = conv_ref(x16, w16, s, b, torch.zeros_like(s), r, stride, pad, 0.0)    # b0 = TINY + delta
    return pre, u * (pre.abs() + b0 - TINY) + b0


def real_rows(N, H):
    """Rows of the real pixels in the zero-padded NHWC layout (row n*(H+1)+h+1, csrc/conv3x3_halo.cuh)."""
    return (torch.arange(N).view(N, 1) * (H + 1) + torch.arange(H).view(1, H) + 1).flatten()


def padded_bf16(lib, t):
    """(N,C,H,W) fp32 -> zero-padded NHWC bf16 [rows][W+1][C] on the GPU."""
    N, C, H, W = t.shape
    buf = torch.zeros(lib.dsk_padded_positions(N, H, W) // (W + 1), W + 1, C, dtype=BF)
    buf[real_rows(N, H), 1:, :] = t.permute(0, 2, 3, 1).reshape(N * H, W, C).to(BF)
    return buf.cuda()


def planar_bf16(lib, t):
    """(N,C,H,W) fp32 -> parity-planar zero-padded bf16 [4 planes (h&1, w&1)][rows][W/2+1][C] on the GPU."""
    return torch.stack([padded_bf16(lib, t[:, :, ph::2, pw::2].contiguous()) for ph in (0, 1) for pw in (0, 1)])


def poisoned_output(lib, N, H, W, C, planes=0):
    """A zero-padded bf16 output buffer (`planes` = 4: parity-planar at half the resolution) whose every real pixel
    holds 7.0: the kernel must overwrite all of them and leave every pad 0."""
    if planes:
        H, W = H // 2, W // 2
    buf = torch.zeros(max(planes, 1), lib.dsk_padded_positions(N, H, W) // (W + 1), W + 1, C, dtype=BF, device="cuda")
    buf[:, real_rows(N, H).cuda(), 1:, :] = 7.0
    return buf if planes else buf[0]


def check_conv(name, got, pads, ref, bound, flags):
    assert float(pads.abs().max()) == 0.0, f"{name}: a pad position is not 0"
    assert_layer(name, got.to(ref.device), ref, bound, saturating=bool(flags & 2))


@pytest.fixture(scope="module")
def hb(cuda_dev):
    """A bf16 handle for the standalone conv entry points."""
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_BF16), "dsk_create")
    yield lib, h
    lib.dsk_destroy(h)


def run_conv3x3(lib, h, N, H, W, C, flags, out_planar, seed):
    x, w, scale, bias, res = operands(seed, N, C, C, H, W, 3, 1)
    d = lambda t: rn16(t, "bf16").double().cuda()
    ref, bound = affine_conv_ref(d(x), d(w), scale.cuda(), bias.cuda(), d(res), 1, flags)
    xp, rp = padded_bf16(lib, x), padded_bf16(lib, res)
    outp = poisoned_output(lib, N, H, W, C, planes=4 if out_planar else 0)
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()       # held: the library reads them after this line
    wp = torch.empty(C * C * 9, dtype=torch.int16, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), C, C, 3, s))
    L.check(lib.dsk_conv3x3_padded(h, xp.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), rp.data_ptr(),
                                   outp.data_ptr(), N, H, W, C, flags, 20.0, out_planar, s), "dsk_conv3x3_padded")
    torch.cuda.synchronize()
    got, pads = from_planar(lib, outp, N, C, H, W) if out_planar else from_padded(outp, real_rows(N, H), N, C, H, W)
    return got, pads, ref, bound


# ---- 1. the halo conv in bf16 -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C", [(80, 32, 64), (40, 16, 128), (20, 8, 256), (10, 4, 512), (16, 32, 64), (2, 4, 512)])
@pytest.mark.parametrize("N,flags", [(3, 2), (2, 3), (17, 0)])
def test_bf16_halo_conv_matches_fp64(hb, H, W, C, N, flags):
    """The cases of test_halo_conv_matches_conv2d on a bf16 handle."""
    lib, h = hb
    got, pads, ref, bound = run_conv3x3(lib, h, N, H, W, C, flags, 0, seed=N * 131 + C)
    check_conv(f"3x3 {N}x{C}x{H}x{W} flags {flags}", got, pads, ref, bound, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C", [(80, 32, 64), (40, 16, 128), (20, 8, 256), (4, 8, 256)])
@pytest.mark.parametrize("N", [3, 16])
def test_bf16_halo_conv_planar_output(hb, H, W, C, N):
    """The cases of test_halo_conv_planar_output (residual + clip, parity-planar output) on a bf16 handle."""
    lib, h = hb
    got, pads, ref, bound = run_conv3x3(lib, h, N, H, W, C, 3, 1, seed=N * 7 + C)
    check_conv(f"3x3 planar {N}x{C}x{H}x{W}", got, pads, ref, bound, 3)


@pytest.mark.gpu
def test_bf16_halo_conv_planar_output_tall(hb):
    """test_halo_conv_planar_output_tall's geometry (N = 2, H = 46 778: the last row of image 1 sits past the bound of
    the epilogue's old 32-bit reciprocal), W = 4."""
    lib, h = hb
    N, H = TALL_OP
    got, pads, ref, bound = run_conv3x3(lib, h, N, H, 4, 64, 3, 1, seed=4)
    check_conv(f"3x3 planar {N}x64x{H}x4", got, pads, ref, bound, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("Hout,Wout,cin,cout", [(40, 16, 64, 128), (20, 8, 128, 256), (10, 4, 256, 512), (2, 4, 256, 512),
                                                (8, 16, 64, 128)])
@pytest.mark.parametrize("N", [3, 17])
def test_bf16_conv5x5s2_planar_matches_fp64(hb, Hout, Wout, cin, cout, N):
    """The cases of test_conv5x5s2_planar_matches_conv2d (parity-planar input, clip) on a bf16 handle."""
    lib, h = hb
    x, w, scale, bias, _ = operands(N * 3 + cout, N, cin, cout, 2 * Hout, 2 * Wout, 5, 2)
    d = lambda t: rn16(t, "bf16").double().cuda()
    ref, bound = affine_conv_ref(d(x), d(w), scale.cuda(), bias.cuda(), None, 2, 2)
    xpl = planar_bf16(lib, x)
    outp = poisoned_output(lib, N, Hout, Wout, cout)
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()
    L.check(lib.dsk_conv5x5s2_planar(h, xpl.data_ptr(), wd.data_ptr(), sc.data_ptr(), bi.data_ptr(), outp.data_ptr(),
                                     N, Hout, Wout, cin, cout, 2, 20.0, L.cur_stream()), "dsk_conv5x5s2_planar")
    torch.cuda.synchronize()
    got, pads = from_padded(outp, real_rows(N, Hout), N, cout, Hout, Wout)
    check_conv(f"5x5s2 {N}x{cin}->{cout}x{Hout}x{Wout}", got, pads, ref, bound, 2)


# ---- 2. the implicit-GEMM conv in bf16 ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("B,flags", [(3, 0), (2, 3), (17, 2)])
def test_bf16_conv2d_nhwc_matches_fp64(hb, shape, B, flags):
    """Every shape and (B, flags) case of test_conv_fp16 on a bf16 handle: dense NHWC bf16 in and out."""
    lib, h = hb
    Hin, Win, cin, cout, k, stride = SHAPES[shape]
    x, w, scale, bias, res = operands(B, B, cin, cout, Hin, Win, k, stride)
    d = lambda t: rn16(t, "bf16").double().cuda()
    ref, bound = affine_conv_ref(d(x), d(w), scale.cuda(), bias.cuda(), d(res), stride, flags)
    Hout, Wout = Hin // stride, Win // stride
    s = L.cur_stream()
    xd, wd, rd, sc, bi = (t.cuda() for t in (x, w, res, scale, bias))
    i16 = lambda n: torch.empty(n, dtype=torch.int16, device="cuda")
    x16, r16, o16, wp = i16(x.numel()), i16(res.numel()), i16(res.numel()), i16(w.numel())
    out = torch.empty(B, cout, Hout, Wout, device="cuda")
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, xd.data_ptr(), x16.data_ptr(), B, cin, Hin, Win, s))
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, rd.data_ptr(), r16.data_ptr(), B, cout, Hout, Wout, s))
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), cout, cin, k, s))
    o16.fill_(int(torch.tensor(7.0, dtype=BF).view(torch.int16)))          # poison: every output must be written
    L.check(lib.dsk_conv2d_nhwc(h, x16.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), r16.data_ptr(),
                                o16.data_ptr(), B, Hin, Win, cin, cout, k, stride, flags, 20.0, s), "dsk_conv2d_nhwc")
    L.check(lib.dsk_nhwc16_to_nchw_f32(h, o16.data_ptr(), out.data_ptr(), B, cout, Hout, Wout, s))
    torch.cuda.synchronize()
    assert_layer(f"{shape} B={B} flags {flags}", out, ref, bound, saturating=bool(flags & 2))


# ---- 3. CPU self-test of the bound --------------------------------------------------------------------------------
def emulate_bf16_conv(defect=None, N=3, C=128, H=8, W=6, seed=0):
    """A bf16 halo / implicit-GEMM conv layer (3x3 s1, residual, clip) in fp32 from bf16 operands
    (test_gpu_layer_parity.emulate_layer), optionally with a seeded defect:
      tap       - one filter tap dropped;
      k_slice   - the last 64-channel K slice (input channels C-64 .. C-1, every tap) dropped;
      res_fp16  - the residual's bf16 bits read as fp16;
      out_fp16  - the output rounded to fp16 and its bits stored where bf16 is read."""
    g = torch.Generator().manual_seed(seed)
    x16 = rn16(torch.randn(N, C, H, W, generator=g) * 2.0, "bf16")
    w16 = rn16(torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5, "bf16")
    scale = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(C, generator=g) * 0.1
    r16 = rn16(torch.randn(N, C, H, W, generator=g) * 2.0, "bf16")
    ref, bound = affine_conv_ref(x16.double(), w16.double(), scale, bias, r16.double(), 1, 3)
    wk, rk = w16, r16
    if defect == "k_slice":
        wk = w16.clone()
        wk[:, C - 64:] = 0
    if defect == "res_fp16":
        rk = r16.to(BF).view(torch.float16).float()
    out_dt = "fp16" if defect == "out_fp16" else "bf16"
    got = emulate_layer(x16, wk, scale, bias, rk, 1, 1, out_dt, "tap" if defect == "tap" else None)
    if defect == "out_fp16":
        got = got.half().view(BF).double()
    return got, ref, bound


@pytest.mark.parametrize("defect", [None, "tap", "k_slice", "res_fp16", "out_fp16"])
def test_bf16_conv_bound_passes_the_emulation_and_fails_seeded_defects(defect):
    got, ref, bound = emulate_bf16_conv(defect)
    msg, worst, inside = check(f"{defect}", got, ref, bound)
    if defect is None:
        assert msg is None and inside >= 0.2, msg
    else:
        assert msg is not None, f"seeded defect {defect} passed (max err/bound {worst:.3g})"


# ---- 4. train forward, every layer --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(128, 160), (6, 160), (5, 32), (33, 48)])
def test_bf16_train_chain_layer_by_layer(cuda_dev, B, T):
    sd = O.make_state_dict(6, 16)
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype="bf16").to(cuda_dev)
    m.load_state_dict(sd)
    m.train()
    train_forward_and_check(f"train bf16 B={B} T={T}", m, sd, "bf16", O.make_input(B, T, 400 + B, 3.0).cuda(), T)


@pytest.mark.gpu
def test_bf16_train_chain_after_rebinding_to_a_smaller_batch(cuda_dev):
    """A bf16 context sized for B=16 that served a forward and its backward, re-bound to B=7 (same T)."""
    T = 48
    sd = O.make_state_dict(7, 16)
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype="bf16").to(cuda_dev)
    m.load_state_dict(sd)
    m.train()
    e = m(O.make_input(16, T, 500, 3.0).cuda())
    (e * torch.randn(e.shape, generator=torch.Generator().manual_seed(0)).cuda()).sum().backward()
    torch.cuda.synchronize()
    sd_now = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}   # running stats moved by the first call
    train_forward_and_check("train bf16 B=16 -> 7 T=48", m, sd_now, "bf16", O.make_input(7, T, 501, 3.0).cuda(), T)


# ---- 5. train backward, every layer -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(128, 160), (6, 160), (5, 32), (2, 16), (33, 48)])
def test_bf16_backward_layer_by_layer(cuda_dev, B, T):
    m, sd = train_model(512, "bf16", 6, cuda_dev)
    backward_case(f"backward bf16 B={B} T={T}", m, sd, "bf16", O.make_input(B, T, 400 + B, 3.0).cuda())


@pytest.mark.gpu
def test_bf16_backward_after_rebinding_to_a_smaller_batch(cuda_dev):
    T = 48
    m, sd = train_model(512, "bf16", 7, cuda_dev)
    e = m(O.make_input(16, T, 500, 3.0).cuda())
    (e * torch.randn(e.shape, generator=torch.Generator().manual_seed(0)).cuda()).sum().backward()
    torch.cuda.synchronize()
    backward_case("backward bf16 B=16 -> 7 T=48", m, sd, "bf16", O.make_input(7, T, 501, 3.0).cuda())


# ---- 6, 7. the training step --------------------------------------------------------------------------------------
# (B, T, max grad rel-L2 against the mask-pinned bf16-storage oracle, embedding rel): each bar within twice the value
# measured on an H100 80GB HBM3 (700 W): grad 1.75e-2 / 1.70e-2 / 1.58e-2, embedding 4.2e-3 / 6.8e-3 / 4.3e-3, loss
# 1.0e-3 / 2.2e-3 / 8.2e-4 relative; about 8 times the fp16 path's, as u_bf16 / u_fp16 = 8
STEP_CASES = [(6, 160, 3e-2, 7e-3), (16, 48, 3.2e-2, 1.2e-2), (128, 160, 3e-2, 8e-3)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,gtol,etol", STEP_CASES)
def test_bf16_step_matches_mask_pinned_oracle(cuda_dev, B, T, gtol, etol):
    """test_fp16_step_matches_mask_pinned_oracle with bf16 operands: the oracle rounds what the engine stores to bf16
    and differentiates through the engine's own clip masks.  It runs in fp64 on the GPU: in fp32 on the CPU it takes
    11 s at B = 128, and cuDNN's fp32 convolutions may run in TF32."""
    sd = O.make_state_dict(1, 16)
    m = make_model(sd, "bf16", cuda_dev)
    xs = [O.make_input(B, T, s, 3.0).cuda() for s in (20, 21, 22)]
    loss, outs, masks, grads = engine_step(m, xs, T)
    dev = lambda t: t.to(cuda_dev)
    oloss, ograds, oouts, own = oracle_step({k: dev(v) for k, v in sd.items()}, xs, 0.1,
                                            [{i: dev(t) for i, t in mk.items()} for mk in masks], torch.bfloat16, f64=True)
    cpu = lambda t: t.float().cpu()
    oloss, oouts = cpu(oloss), [cpu(o) for o in oouts]
    ograds = {k: cpu(g) for k, g in ograds.items() if g is not None}
    own = [{i: t.cpu() for i, t in mk.items()} for mk in own]
    flips = sum(int((masks[j][i] != own[j][i]).sum()) for j in range(3) for i in range(12))
    total = sum(masks[j][i].numel() for j in range(3) for i in range(12))
    erel = max(float(((outs[j] - oouts[j]).norm(dim=1) / oouts[j].norm(dim=1)).max()) for j in range(3))
    lrel = abs(loss.item() - oloss.item()) / max(abs(oloss.item()), 0.05)
    worst = max((rel_l2(grads[k], ograds[k]), k) for k in grads)
    print(f"bf16 B={B} T={T}: emb rel {erel:.2e}, loss {loss.item():.6f} vs {oloss.item():.6f} (rel {lrel:.2e}), "
          f"clip-mask flips {flips}/{total}, worst grad rel-L2 {worst[0]:.2e} ({worst[1]})")
    assert erel < etol
    assert lrel <= 8e-3
    assert len(grads) == 38
    for k in grads:
        assert rel_l2(grads[k], ograds[k]) < gtol, (k, rel_l2(grads[k], ograds[k]))


@pytest.mark.gpu
def test_bf16_gradients_are_bit_reproducible(cuda_dev):
    sd = O.make_state_dict(2, 16)
    xs = [O.make_input(8, 160, s, 3.0).cuda() for s in (1, 2, 3)]
    runs = []
    for _ in range(2):
        m = make_model(sd, "bf16", cuda_dev)
        loss, outs, _, grads = engine_step(m, xs, 160)
        runs.append((loss, outs, grads))
    assert torch.equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)
    assert len(runs[0][2]) == 38
    for k in runs[0][2]:
        assert torch.equal(runs[0][2][k], runs[1][2][k]), k


# ---- 8. eval batch invariance -------------------------------------------------------------------------------------
def _activations_bf16(m, B, T):
    bufs = read_eval_activations(m, B, T, "bf16")
    torch.cuda.synchronize()
    return unpack_eval_activations(m._engine.lib, bufs, B, T)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [16, 48, 160, 800])
@pytest.mark.parametrize("env", [{}, {"DSK_GRAPH": "0"}], ids=_env_id)
def test_bf16_eval_forward_is_batch_invariant(cuda_dev, env, T):
    """test_eval_forward_is_batch_invariant on a bf16 model: every embedding of the calls at B = 1, 7, 64, 256, 300 and
    a permuted 256 equals the batch of 300; utterances 0-6's slices of all 12 activations at B = 7 equal those at
    B = 300 (at T = 800: B = 64)."""
    sd = O.make_state_dict(4, 16)
    pool = O.make_input(POOL, T, 900 + T, 4.0).cuda()
    m = _fresh_model(sd, env, "bf16")
    big = 64 if T == 800 else POOL
    ref = _forward(m, pool)
    acts_big = _activations_bf16(m, POOL, T) if big == POOL else None
    for idx in _batch_calls(T):
        e = _forward(m, pool[idx.cuda()].contiguous())
        bad = (e != ref[idx.cuda()]).any(dim=1)
        assert not bool(bad.any()), (f"bf16 {_env_id(env)} T={T} B={idx.numel()}: {int(bad.sum())} embeddings differ "
                                     f"from the batch of {POOL}")
        if idx.numel() == big and big != POOL and bool((idx == torch.arange(big)).all()):
            acts_big = _activations_bf16(m, big, T)
        if idx.numel() == 7:
            acts_small = _activations_bf16(m, 7, T)
    _check_activations(f"bf16 {_env_id(env)} T={T} 7 vs {big}", acts_small, acts_big, slice(0, 7))


# ---- 9. EmbeddingPipeline -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 3])
def test_bf16_pipeline_matches_direct_forward(cuda_dev, lanes):
    """A bf16 model through EmbeddingPipeline: every lane runs plain, capturing and re-targeted graph launches, and the
    last batch is shorter (its shape re-zeroes the lane's workspace)."""
    m = dsk.DeepSpeakerModel(512, 16, operand_dtype="bf16").to(cuda_dev).eval()
    m.load_state_dict(O.make_state_dict(0, 16))
    pipe = dsk.EmbeddingPipeline(m, lanes=lanes)
    n = 4 * lanes + 3
    xs = [O.make_input(6 if i < n - 1 else 5, 48, seed=200 + i, scale=4.0) for i in range(n)]
    xh = [x.pin_memory() for x in xs]
    oh = [torch.empty(x.shape[0], 512).pin_memory() for x in xs]
    for i in range(n):
        pipe.embed(xh[i], oh[i])
    pipe.synchronize()
    with torch.no_grad():
        for i in range(n):
            assert torch.equal(oh[i], m(xs[i].cuda()).cpu()), i
