"""The halo conv's parity-planar output (staged in shared memory, copied out in 128-byte position rows) holds exactly the
values of its padded output (staged, TMA-stored): the same conv run both ways must agree bit for bit, pads included."""
import ctypes

import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L

pytestmark = pytest.mark.gpu

TD = {"fp16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module", params=["fp16", "bf16"])
def hd(cuda_dev, request):
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_BF16 if request.param == "bf16" else L.DSK_F16), "dsk_create")
    yield lib, h, request.param
    lib.dsk_destroy(h)


def to_padded(lib, t, dt):
    N, C, H, W = t.shape
    npos = lib.dsk_padded_positions(N, H, W)
    buf = torch.zeros(npos // (W + 1), W + 1, C, dtype=TD[dt])
    rows = (torch.arange(N).view(N, 1) * (H + 1) + torch.arange(H).view(1, H) + 1).flatten()
    buf[rows, 1:, :] = t.permute(0, 2, 3, 1).reshape(N * H, W, C).to(TD[dt])
    return buf.cuda().contiguous()


# batch 64 at the eval forward's block-final shapes, and small batches with a partial last tile
@pytest.mark.parametrize("N,H,W,C", [(64, 80, 32, 64), (64, 40, 16, 128), (64, 20, 8, 256), (3, 20, 8, 256), (5, 4, 8, 256)])
def test_planar_output_equals_padded_output(hd, N, H, W, C):
    lib, h, dt = hd
    g = torch.Generator().manual_seed(N + C + H)
    x = torch.randn(N, C, H, W, generator=g) * 2.0
    w = torch.randn(C, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    scale = torch.empty(C).uniform_(0.5, 1.5, generator=g).cuda()
    bias = (torch.randn(C, generator=g) * 0.1).cuda()
    xp = to_padded(lib, x, dt)
    rp = to_padded(lib, torch.randn(N, C, H, W, generator=g) * 2.0, dt)
    wp = torch.empty(C * C * 9, dtype=torch.int16, device="cuda")
    s = L.cur_stream()
    L.check(lib.dsk_pack_conv_weight(h, w.cuda().data_ptr(), wp.data_ptr(), C, C, 3, s))
    out = torch.zeros_like(xp)
    npl = lib.dsk_padded_positions(N, H // 2, W // 2)
    outp = torch.full((4, npl // (W // 2 + 1), W // 2 + 1, C), 0.0, dtype=TD[dt], device="cuda")
    for dst, planar in ((out, 0), (outp, 1)):
        L.check(lib.dsk_conv3x3_padded(h, xp.data_ptr(), wp.data_ptr(), scale.data_ptr(), bias.data_ptr(), rp.data_ptr(),
                                       dst.data_ptr(), N, H, W, C, 3, 20.0, planar, s), "dsk_conv3x3_padded")
    torch.cuda.synchronize()
    # the padded output rearranged into the four planes: pixel (n, h, w) -> plane (h & 1, w & 1) at (n, h >> 1, w >> 1)
    want = torch.zeros_like(outp)
    img = out[1:1 + N * (H + 1)].view(N, H + 1, W + 1, C)[:, :H, 1:]   # (N, H, W, C) real pixels
    H2, W2 = H // 2, W // 2
    for pl, (ph, pw) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        want[pl][1:1 + N * (H2 + 1)].view(N, H2 + 1, W2 + 1, C)[:, :H2, 1:].copy_(img[:, ph::2, pw::2])
    assert torch.equal(outp.view(torch.int16), want.view(torch.int16))
