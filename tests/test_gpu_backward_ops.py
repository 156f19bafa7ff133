"""Backward building blocks through the C ABI vs torch autograd on the same (16-bit rounded) inputs:
wgmma data-gradient convs (3x3 s1, 5x5 s2 in four parity classes), the MN-major weight-gradient GEMM, and the
batch-statistics BatchNorm(+residual+clip) forward/backward kernels."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from deepspeaker_pytorch_b200 import _lib as L
from tests.test_gpu_conv import SHAPES

pytestmark = pytest.mark.gpu


TD = {"fp16": torch.float16, "bf16": torch.bfloat16}
U = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}    # unit roundoff of the 16-bit gradient / activation tensors


@pytest.fixture(scope="module", params=["fp16", "bf16"])
def hl(cuda_dev, request):
    """A handle of each operand type; the tests read its type as dt and round their inputs to it."""
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_BF16 if request.param == "bf16" else L.DSK_F16), "dsk_create")
    yield lib, h, request.param
    lib.dsk_destroy(h)


def to_nhwc16(lib, h, t):
    B, C, H, W = t.shape
    out = torch.empty(B * C * H * W, dtype=torch.int16, device="cuda")
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, t.cuda().contiguous().data_ptr(), out.data_ptr(), B, C, H, W, L.cur_stream()))
    return out


def from_nhwc16(lib, h, buf, B, C, H, W):
    out = torch.empty(B, C, H, W, device="cuda")
    L.check(lib.dsk_nhwc16_to_nchw_f32(h, buf.data_ptr(), out.data_ptr(), B, C, H, W, L.cur_stream()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("B", [3, 16])
def test_dgrad_and_wgrad_match_autograd(hl, shape, B):
    lib, h, dt = hl
    r16 = lambda t: t.to(TD[dt]).float()
    Hin, Win, cin, cout, k, stride = SHAPES[shape]
    g = torch.Generator().manual_seed(B)
    x = r16(torch.randn(B, cin, Hin, Win, generator=g) * 1.5)
    w = (torch.randn(cout, cin, k, k, generator=g) * (2.0 / (k * k * cin)) ** 0.5)
    Hout, Wout = Hin // stride, Win // stride
    gy = r16(torch.randn(B, cout, Hout, Wout, generator=g) * 0.5)
    res = r16(torch.randn(B, cin, Hin, Win, generator=g))
    xr = x.double().requires_grad_(True)
    wr = r16(w).double().requires_grad_(True)            # the engine multiplies with 16-bit-rounded weights
    F.conv2d(xr, wr, None, stride, k // 2).backward(gy.double())
    use_res = stride == 1
    ref_gin = xr.grad + (res.double() if use_res else 0)
    # wgrad is linear in (G, X): the reference with unrounded w is the same
    ref_dw = wr.grad
    s = L.cur_stream()
    G16, X16, R16 = to_nhwc16(lib, h, gy), to_nhwc16(lib, h, x), to_nhwc16(lib, h, res)
    gin16 = torch.zeros(B * cin * Hin * Win, dtype=torch.int16, device="cuda")
    wd = w.cuda()
    L.check(lib.dsk_conv2d_dgrad_nhwc(h, G16.data_ptr(), wd.data_ptr(), R16.data_ptr() if use_res else None, gin16.data_ptr(),
                                      B, Hin, Win, cin, cout, k, stride, s), "dgrad")
    gin = from_nhwc16(lib, h, gin16, B, cin, Hin, Win).double()
    tol = 2 * U[dt] * ref_gin.abs().clamp(min=1.0) + 2e-3   # 2^-10 (fp16), 2^-7 (bf16)
    assert bool(((gin - ref_gin).abs() <= tol).all()), float((gin - ref_gin).abs().max())
    dw = torch.empty(cout, cin, k, k, device="cuda")
    L.check(lib.dsk_conv2d_wgrad_nhwc(h, G16.data_ptr(), X16.data_ptr(), dw.data_ptr(), B, Hin, Win, cin, cout, k, stride,
                                      1.0, s), "wgrad")
    torch.cuda.synchronize()
    dwc = dw.cpu().double()
    rel = ((dwc - ref_dw).norm() / ref_dw.norm()).item()
    assert rel < 1e-5, rel                                 # exact 16-bit products, fp32 accumulation
    assert ((dwc - ref_dw).abs().max() / ref_dw.abs().max()).item() < 1e-4


# offset: 0 = channel means of order one; > 0 = raw = randn + offset[c], offsets log-spaced from 1 to `offset` (mean/std up
# to 1000: E[x^2] - mean^2 from plain fp32 sums would lose the variance there)
@pytest.mark.parametrize("M,C,with_res,offset", [(4 * 80 * 32, 64, False, 0), (3 * 40 * 16, 128, True, 0), (5 * 10 * 4 + 3, 512, True, 0),
                                                 (128 * 80 * 32, 64, False, 1000), (128 * 10 * 4, 512, True, 1000)])
def test_bn_act_train_forward_backward(hl, M, C, with_res, offset):
    lib, h, dt = hl
    r16 = lambda t: t.to(TD[dt]).float()
    g = torch.Generator().manual_seed(C)
    if offset:
        raw = torch.randn(M, C, generator=g) + torch.logspace(0, float(np.log10(offset)), C)[torch.randperm(C, generator=g)]
    else:
        raw = torch.randn(M, C, generator=g) * 3.0 + torch.randn(C, generator=g)
    gamma = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    beta = torch.randn(C, generator=g) * 0.5 + 1.0
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.empty(C).uniform_(0.5, 1.5, generator=g)
    res = r16(torch.randn(M, C, generator=g) * 2)
    gy = r16(torch.randn(M, C, generator=g))
    # torch reference (fp64), [M][C] treated as N x C for batch_norm
    rr = raw.double().requires_grad_(True)
    gm, bt = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rs = res.double().requires_grad_(True)
    rmr, rvr = rm.double().clone(), rv.double().clone()
    pre = F.batch_norm(rr, rmr, rvr, gm, bt, True, 0.1, 1e-5) + (rs if with_res else 0)
    yr = F.hardtanh(pre, 0.0, 20.0)                                  # Hardtanh(0, 20), model.py:36-39
    yr.backward(gy.double())
    dev = lambda t: t.cuda().contiguous()
    rawd, gd, bd, rmd, rvd = dev(raw), dev(gamma), dev(beta), dev(rm), dev(rv)
    res16, gy16 = dev(res.to(TD[dt])), dev(gy.to(TD[dt]))
    y16 = torch.empty(M, C, dtype=TD[dt], device="cuda")
    mean, rstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_bn_act_train_forward(h, rawd.data_ptr(), gd.data_ptr(), bd.data_ptr(), rmd.data_ptr(), rvd.data_ptr(),
                                         res16.data_ptr() if with_res else None, y16.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                         M, C, s), "bn fwd")
    torch.cuda.synchronize()
    assert torch.allclose(y16.float().cpu().double(), yr.detach(), rtol=2 * U[dt], atol=2e-3)
    assert torch.allclose(rmd.cpu().double(), rmr, rtol=1e-5, atol=1e-6) and torch.allclose(rvd.cpu().double(), rvr, rtol=1e-5, atol=1e-6)
    assert torch.allclose(mean.cpu().double(), raw.double().mean(0), rtol=1e-5, atol=1e-5)
    G16 = torch.empty(M, C, dtype=TD[dt], device="cuda")
    gres16 = torch.empty(M, C, dtype=TD[dt], device="cuda")
    dgam, dbet = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    L.check(lib.dsk_bn_act_train_backward(h, gy16.data_ptr(), y16.data_ptr(), rawd.data_ptr(), gd.data_ptr(), mean.data_ptr(),
                                          rstd.data_ptr(), G16.data_ptr(), gres16.data_ptr() if with_res else None,
                                          dgam.data_ptr(), dbet.data_ptr(), M, C, 1.0, s), "bn bwd")
    torch.cuda.synchronize()
    # elements whose pre-activation is within 16-bit rounding of the clip edges may take the other branch
    ew = 2e-2 if dt == "fp16" else 20 * 2 * U[dt]
    edge = ((pre.detach().abs() < ew) | ((pre.detach() - 20).abs() < ew))
    Gc, ref = G16.float().cpu().double(), rr.grad
    bad = ((Gc - ref).abs() > 4 * U[dt] * ref.abs().clamp(min=0.05) + 2e-3) & ~edge   # 2^-9 (fp16), 2^-6 (bf16)
    assert int(bad.sum()) == 0, int(bad.sum())
    assert ((Gc - ref).norm() / ref.norm()).item() < 1e-2
    assert ((dgam.cpu().double() - gm.grad).norm() / gm.grad.norm()).item() < 5e-3
    assert ((dbet.cpu().double() - bt.grad).norm() / bt.grad.norm()).item() < 5e-3
    if with_res:
        gr = gres16.float().cpu().double()
        assert int((((gr - rs.grad).abs() > 1e-3) & ~edge).sum()) == 0
