"""GPU bring-up check of the wgmma conv kernel through the C ABI against a CPU fp64 conv of the
same 16-bit-rounded operands.  Usage: python tools/gpu_debug_conv.py <case> [bf16]
cases: s1..s4 (3x3 convs of stage 1..4), e2..e4 (5x5 s2 entry convs), all."""
import ctypes
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepspeaker_pytorch_b200 import _lib as L  # noqa: E402


def run_case(h, lib, name, B, Hin, Win, cin, cout, k, stride, flags, bf16, seed=0):
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, Hin, Win, generator=g) * 2.0
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (k * k * cin)) ** 0.5
    scale = torch.empty(cout).uniform_(0.5, 1.5, generator=g)
    bias = torch.randn(cout, generator=g) * 0.1
    Hout, Wout = Hin // stride, Win // stride
    res = torch.randn(B, cout, Hout, Wout, generator=g) * 2.0
    xq, wq, rq = x.to(dt).double(), w.to(dt).double(), res.to(dt).double()
    ref = F.conv2d(xq, wq, None, stride, k // 2) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    if flags & 1:
        ref = ref + rq
    if flags & 2:
        ref = ref.clamp(0, 20)
    dev = "cuda"
    s = L.cur_stream()
    xd, wd, rd = x.to(dev), w.to(dev), res.to(dev)
    sc, bi = scale.to(dev), bias.to(dev)
    x16 = torch.empty(B * Hin * Win * cin, dtype=torch.int16, device=dev)
    r16 = torch.empty(B * Hout * Wout * cout, dtype=torch.int16, device=dev)
    o16 = torch.zeros(B * Hout * Wout * cout, dtype=torch.int16, device=dev)
    wp = torch.empty(cout * cin * k * k, dtype=torch.int16, device=dev)
    out = torch.empty(B, cout, Hout, Wout, device=dev)
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, xd.data_ptr(), x16.data_ptr(), B, cin, Hin, Win, s))
    L.check(lib.dsk_nchw_f32_to_nhwc16(h, rd.data_ptr(), r16.data_ptr(), B, cout, Hout, Wout, s))
    L.check(lib.dsk_pack_conv_weight(h, wd.data_ptr(), wp.data_ptr(), cout, cin, k, s))
    L.check(lib.dsk_conv2d_nhwc(h, x16.data_ptr(), wp.data_ptr(), sc.data_ptr(), bi.data_ptr(), r16.data_ptr(),
                                o16.data_ptr(), B, Hin, Win, cin, cout, k, stride, flags, 20.0, s), "conv")
    L.check(lib.dsk_nhwc16_to_nchw_f32(h, o16.data_ptr(), out.data_ptr(), B, cout, Hout, Wout, s))
    torch.cuda.synchronize()
    got = out.cpu().double()
    err = (got - ref).abs()
    tol = (2.0 ** -7 if bf16 else 2.0 ** -10) * ref.abs().clamp(min=1.0) + 1e-3
    bad = (err > tol)
    nbad = int(bad.sum())
    print(f"[{name}] B={B} {cin}->{cout} k{k}s{stride} {Hin}x{Win} flags={flags} {'bf16' if bf16 else 'f16'}: "
          f"max_err={err.max():.3e} mean_err={err.mean():.3e} ref_absmax={ref.abs().max():.2f} bad={nbad}/{err.numel()}",
          flush=True)
    if nbad:
        ix = bad.nonzero()[:8]
        for i in ix:
            i = tuple(int(v) for v in i)
            print("   bad at (n,c,h,w)=", i, "got", float(got[i]), "ref", float(ref[i]))
        # error structure: which n / c / h / w have errors
        for d, nm in enumerate("nchw"):
            dims = [k_ for k_ in range(4) if k_ != d]
            print("   bad count by", nm, bad.sum(dim=dims).tolist()[:40])
    return nbad == 0


CASES = {
    # name: (Hin, Win, cin, cout, k, stride)
    "s1": (80, 32, 64, 64, 3, 1),
    "s2": (40, 16, 128, 128, 3, 1),
    "s3": (20, 8, 256, 256, 3, 1),
    "s4": (10, 4, 512, 512, 3, 1),
    "e2": (80, 32, 64, 128, 5, 2),
    "e3": (40, 16, 128, 256, 5, 2),
    "e4": (20, 8, 256, 512, 5, 2),
}


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    bf16 = len(sys.argv) > 2 and sys.argv[2] == "bf16"
    lib = L.load()
    h = ctypes.c_void_p()
    L.check(lib.dsk_create(ctypes.byref(h), 0, L.DSK_BF16 if bf16 else L.DSK_F16), "create")
    names = list(CASES) if which == "all" else [which]
    ok = True
    for nm in names:
        Hin, Win, cin, cout, k, st = CASES[nm]
        for B, flags in ((3, 0), (2, 3), (17, 2)):
            ok &= run_case(h, lib, nm, B, Hin, Win, cin, cout, k, st, flags, bf16)
    print("ALL OK" if ok else "FAILED")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
