"""conv3x3_halo_kernel (zero-padded NHWC layout, row-shifted wgmma descriptors, resident / 3-tap weight boxes) vs an
fp64 CPU conv of the same fp16-rounded operands; also checks that every pad position of the output stays zero."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from deepspeaker_pytorch_b200 import _lib as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["one_cta_per_sm"])
def hl(cuda_dev):
    """A handle for the halo kernel's one shape (384 threads, one CTA per SM, whole tiles; csrc/conv3x3_halo.cuh).
    The parameter names that shape in the test ids."""
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_F16), "dsk_create")
    yield lib, h
    lib.dsk_destroy(h)


def to_padded(lib, t):
    """(N,C,H,W) fp32 -> padded NHWC fp16 [positions][C] on the GPU."""
    N, C, H, W = t.shape
    npos = lib.dsk_padded_positions(N, H, W)
    buf = torch.zeros(npos // (W + 1), W + 1, C, dtype=torch.float16)
    rows = (torch.arange(N).view(N, 1) * (H + 1) + torch.arange(H).view(1, H) + 1).flatten()
    buf[rows, 1:, :] = t.permute(0, 2, 3, 1).reshape(N * H, W, C).half()
    return buf.cuda().contiguous(), rows


def from_padded(buf, rows, N, C, H, W):
    b = buf.cpu().float()
    img = b[rows, 1:, :].reshape(N, H, W, C).permute(0, 3, 1, 2)
    mask = torch.ones(b.shape[0], b.shape[1], dtype=torch.bool)
    mask[rows.unsqueeze(1), torch.arange(1, W + 1).unsqueeze(0)] = False
    return img, b[mask]          # image, pad values


@pytest.mark.parametrize("H,W,C", [(80, 32, 64), (40, 16, 128), (20, 8, 256), (10, 4, 512), (16, 32, 64), (2, 4, 512)])
@pytest.mark.parametrize("N,flags", [(3, 2), (2, 3), (17, 0)])
def test_halo_conv_matches_conv2d(hl, H, W, C, N, flags):
    lib, h = hl
    g = torch.Generator().manual_seed(N * 131 + C)
    x = torch.randn(N, C, H, W, generator=g) * 2.0
    w = torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    scale = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(C, generator=g) * 0.1
    res = torch.randn(N, C, H, W, generator=g) * 2.0
    ref = F.conv2d(x.half().double(), w.half().double(), None, 1, 1) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    if flags & 1:
        ref = ref + res.half().double()
    if flags & 2:
        ref = ref.clamp(0, 20)
    xp, rows = to_padded(lib, x)
    rp, _ = to_padded(lib, res)
    outp = torch.zeros_like(xp)              # pads start as zero (as in the engine's workspace) ...
    outp[rows.cuda(), 1:, :] = 7.0           # ... and every real pixel is poisoned: the kernel must overwrite all of them
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()
    wp = torch.empty(C * C * 9, dtype=torch.int16, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), C, C, 3, s))
    L.check(lib.dsk_conv3x3_padded(h, xp.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), rp.data_ptr(), outp.data_ptr(),
                                   N, H, W, C, flags, 20.0, 0, s), "dsk_conv3x3_padded")
    torch.cuda.synchronize()
    got, pads = from_padded(outp, rows, N, C, H, W)
    tol = 2.0 ** -10 * ref.abs().clamp(min=1.0) + 1e-3
    err = (got.double() - ref).abs()
    assert bool((err <= tol).all()), float(err.max())
    assert float(pads.abs().max()) == 0.0     # every pad position (left column, rows between images, slack) is still zero


def to_planar(lib, t):
    """(N,C,H,W) fp32 -> parity-planar padded fp16 [4][positions(N,H/2,W/2)][C] on the GPU."""
    planes = [to_padded(lib, t[:, :, ph::2, pw::2].contiguous())[0] for ph in (0, 1) for pw in (0, 1)]
    return torch.stack(planes).contiguous()


def from_planar(lib, buf, N, C, H, W):
    out = torch.zeros(N, C, H, W)
    pads = []
    for pl, (ph, pw) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        rows = (torch.arange(N).view(N, 1) * (H // 2 + 1) + torch.arange(H // 2).view(1, H // 2) + 1).flatten()
        img, pad = from_padded(buf[pl], rows, N, C, H // 2, W // 2)
        out[:, :, ph::2, pw::2] = img
        pads.append(pad)
    return out, torch.cat([p.flatten() for p in pads])


@pytest.mark.parametrize("H,W,C", [(80, 32, 64), (40, 16, 128), (20, 8, 256), (4, 8, 256)])
@pytest.mark.parametrize("N", [3, 16])
def test_halo_conv_planar_output(hl, H, W, C, N):
    """3x3 conv + residual + clip whose output is written parity-planar (the layout the next stage's 5x5 s2 conv reads)."""
    lib, h = hl
    g = torch.Generator().manual_seed(N * 7 + C)
    x = torch.randn(N, C, H, W, generator=g) * 2.0
    w = torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    scale = torch.empty(C).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(C, generator=g) * 0.1
    res = torch.randn(N, C, H, W, generator=g) * 2.0
    ref = (F.conv2d(x.half().double(), w.half().double(), None, 1, 1) * scale.double().view(1, -1, 1, 1)
           + bias.double().view(1, -1, 1, 1) + res.half().double()).clamp(0, 20)
    xp, _ = to_padded(lib, x)
    rp, _ = to_padded(lib, res)
    npl = lib.dsk_padded_positions(N, H // 2, W // 2)
    outp = torch.zeros(4, npl // (W // 2 + 1), W // 2 + 1, C, dtype=torch.float16, device="cuda")
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()
    wp = torch.empty(C * C * 9, dtype=torch.int16, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), C, C, 3, s))
    L.check(lib.dsk_conv3x3_padded(h, xp.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), rp.data_ptr(), outp.data_ptr(),
                                   N, H, W, C, 3, 20.0, 1, s), "dsk_conv3x3_padded planar")
    torch.cuda.synchronize()
    got, pads = from_planar(lib, outp, N, C, H, W)
    tol = 2.0 ** -10 * ref.abs().clamp(min=1.0) + 1e-3
    assert bool(((got.double() - ref).abs() <= tol).all()), float((got.double() - ref).abs().max())
    assert float(pads.abs().max()) == 0.0


@pytest.mark.parametrize("Hout,Wout,cin,cout", [(40, 16, 64, 128), (20, 8, 128, 256), (10, 4, 256, 512), (2, 4, 256, 512), (8, 16, 64, 128)])
@pytest.mark.parametrize("N", [3, 17])
def test_conv5x5s2_planar_matches_conv2d(hl, Hout, Wout, cin, cout, N):
    lib, h = hl
    g = torch.Generator().manual_seed(N * 3 + cout)
    x = torch.randn(N, cin, 2 * Hout, 2 * Wout, generator=g) * 2.0
    w = torch.randn(cout, cin, 5, 5, generator=g) * (2.0 / (25 * cin)) ** 0.5
    scale = torch.empty(cout).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(cout, generator=g) * 0.1
    ref = (F.conv2d(x.half().double(), w.half().double(), None, 2, 2) * scale.double().view(1, -1, 1, 1)
           + bias.double().view(1, -1, 1, 1)).clamp(0, 20)
    xpl = to_planar(lib, x)
    npos = lib.dsk_padded_positions(N, Hout, Wout)
    outp = torch.zeros(npos // (Wout + 1), Wout + 1, cout, dtype=torch.float16, device="cuda")
    rows = (torch.arange(N).view(N, 1) * (Hout + 1) + torch.arange(Hout).view(1, Hout) + 1).flatten()
    outp[rows.cuda(), 1:, :] = 7.0
    wd, sc, bi = w.cuda(), scale.cuda(), bias.cuda()
    L.check(lib.dsk_conv5x5s2_planar(h, xpl.data_ptr(), wd.data_ptr(), sc.data_ptr(), bi.data_ptr(), outp.data_ptr(), N, Hout, Wout,
                                     cin, cout, 2, 20.0, L.cur_stream()), "dsk_conv5x5s2_planar")
    torch.cuda.synchronize()
    got, pads = from_padded(outp, rows, N, cout, Hout, Wout)
    tol = 2.0 ** -10 * ref.abs().clamp(min=1.0) + 1e-3
    assert bool(((got.double() - ref).abs() <= tol).all()), float((got.double() - ref).abs().max())
    assert float(pads.abs().max()) == 0.0
