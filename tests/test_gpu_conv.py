"""wgmma implicit-GEMM conv (dsk_conv2d_nhwc) vs an fp64 CPU conv of the same 16-bit-rounded operands."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from deepspeaker_pytorch_b200 import _lib as L

pytestmark = pytest.mark.gpu

# (Hin, Win, cin, cout, k, stride): every tensor-core conv shape of the ResCNN at T=160 and T=32
SHAPES = {
    "l1_3x3": (80, 32, 64, 64, 3, 1), "l2_3x3": (40, 16, 128, 128, 3, 1), "l3_3x3": (20, 8, 256, 256, 3, 1),
    "l4_3x3": (10, 4, 512, 512, 3, 1), "conv2": (80, 32, 64, 128, 5, 2), "conv3": (40, 16, 128, 256, 5, 2),
    "conv4": (20, 8, 256, 512, 5, 2), "l1_3x3_T32": (16, 32, 64, 64, 3, 1), "conv4_T32": (4, 8, 256, 512, 5, 2),
    "l4_3x3_T32": (2, 4, 512, 512, 3, 1),
}


@pytest.fixture(scope="module")
def handles(cuda_dev):
    lib = L.load()
    hs = {}
    for name, op in (("fp16", L.DSK_F16), ("bf16", L.DSK_BF16)):
        h = ctypes.c_void_p()
        L.check(lib.dsk_create(ctypes.byref(h), 0, op), "dsk_create")
        hs[name] = h
    yield lib, hs
    for h in hs.values():
        lib.dsk_destroy(h)


def run_conv(lib, h, bf16, B, Hin, Win, cin, cout, k, stride, flags, seed):
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, Hin, Win, generator=g) * 2.0
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (k * k * cin)) ** 0.5
    scale = torch.empty(cout).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(cout, generator=g) * 0.1
    Hout, Wout = Hin // stride, Win // stride
    res = torch.randn(B, cout, Hout, Wout, generator=g) * 2.0
    ref = F.conv2d(x.to(dt).double(), w.to(dt).double(), None, stride, k // 2)
    ref = ref * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    if flags & 1:
        ref = ref + res.to(dt).double()
    if flags & 2:
        ref = ref.clamp(0, 20)
    s = L.cur_stream()
    xd, wd, rd, sc, bi = (t.cuda() for t in (x, w, res, scale, bias))
    i16 = lambda n: torch.empty(n, dtype=torch.int16, device="cuda")
    x16, r16, o16, wp = i16(x.numel()), i16(res.numel()), i16(res.numel()), i16(w.numel())
    out = torch.empty(B, cout, Hout, Wout, device="cuda")
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, xd.data_ptr(), x16.data_ptr(), B, cin, Hin, Win, s))
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, rd.data_ptr(), r16.data_ptr(), B, cout, Hout, Wout, s))
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), cout, cin, k, s))
    L.check(lib.dsk_conv2d_nhwc(h, x16.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), r16.data_ptr(),
                                o16.data_ptr(), B, Hin, Win, cin, cout, k, stride, flags, 20.0, s), "dsk_conv2d_nhwc")
    L.check(lib.dsk_nhwc16_to_nchw_f32(h, o16.data_ptr(), out.data_ptr(), B, cout, Hout, Wout, s))
    torch.cuda.synchronize()
    return out.cpu().double(), ref


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("B,flags", [(3, 0), (2, 3), (17, 2)])
def test_conv_fp16(handles, shape, B, flags):
    lib, hs = handles
    got, ref = run_conv(lib, hs["fp16"], False, B, *SHAPES[shape], flags, seed=B)
    # tolerance: one fp16 output rounding (2^-11 relative) + fp32 accumulation noise
    tol = 2.0 ** -10 * ref.abs().clamp(min=1.0) + 1e-3
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())


@pytest.mark.parametrize("shape", ["l2_3x3", "conv3", "l4_3x3"])
def test_conv_bf16(handles, shape):
    lib, hs = handles
    got, ref = run_conv(lib, hs["bf16"], True, 5, *SHAPES[shape], 3, seed=1)
    tol = 2.0 ** -7 * ref.abs().clamp(min=1.0) + 1e-3
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())


def test_conv_rejects_unsupported(handles):
    lib, hs = handles
    d = torch.zeros(1 << 16, dtype=torch.int16, device="cuda")
    args = lambda cin, cout, k, s: (hs["fp16"], d.data_ptr(), d.data_ptr(), None, None, None, d.data_ptr(), 1, 8, 8, cin,
                                    cout, k, s, 0, 20.0, None)
    assert lib.dsk_conv2d_nhwc(*args(64, 64, 7, 1)) < 0       # kernel size
    assert lib.dsk_conv2d_nhwc(*args(48, 64, 3, 1)) < 0       # cin not a multiple of 64
    assert lib.dsk_conv2d_nhwc(*args(64, 64, 3, 2)) < 0       # 3x3 stride 2 not on the path
    assert b"conv" in lib.dsk_last_error()
