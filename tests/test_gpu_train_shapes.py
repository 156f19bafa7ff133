"""Every layer of the train forward and backward against fp64 at the shapes that put the train convs in every regime
their plans reach for B <= 256 utterances of up to 1600 frames.

The layer checkers (test_gpu_layer_parity.train_forward_and_check, test_gpu_backward_layer_parity.backward_case) run
unchanged; what is new is where.  The train convs tile each layer's output grid with a 128-pixel box (wt, hb, nb)
chosen from (B, H), the weight gradient splits its K chunks over slices, and the BatchNorm reductions run gx partial
blocks (tests/train_plan.py restates all three).  The cases below reach every box shape, boxes taller than the image,
boxes ragged in h, in n and in both, weight-gradient splits that get no chunk or fewer than the others, BatchNorm grids
at their cap and reduction chains longer than 64 terms; tests/test_train_tiles_host.py fails if a case is removed or a
regime goes unreached.  Before the checkers run, each case asserts that the library planned what the restatement says
(dsk_debug_train_tiles, dsk_debug_backward_plan), so the regimes claimed are the regimes run.  Each case prints every
layer's largest err/bound, its wall time and its peak memory.
"""
import ctypes
import time

import pytest
import torch

from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200.engine import conv_bn_modules
from oracle import rescnn_oracle as O
from tests import train_plan as P
from tests.test_gpu_backward_layer_parity import backward_case, read_ctx, train_model
from tests.test_gpu_layer_parity import check_train_chain, stat_chains, train_forward_and_check

pytestmark = pytest.mark.gpu

# (B, T): all fp16 unless listed again for bf16 or the synchronised path.  The fp16 cases reach every regime; the bf16
# cases every box shape the earlier bf16 checker cases never built; the synchronised case chains longer than 64 terms.
FP16_SHAPES = [(9, 272), (3, 80), (17, 16), (64, 800), (1, 16), (2, 16), (5, 16)]
BF16_SHAPES = [(9, 272), (3, 80), (128, 400)]
SYNC_SHAPES = [(16, 400)]


def assert_plan(eng, tctx, B, T):
    """The tiles, weight-gradient split and BatchNorm grid the library bound `tctx` to, layer by layer, against
    tests/train_plan.py."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    for i in range(12):
        tiles, plan = (ctypes.c_int32 * 6)(), (ctypes.c_int32 * 3)()
        L.check(eng.lib.dsk_debug_train_tiles(eng.handle, tctx, i, tiles), "dsk_debug_train_tiles")
        L.check(eng.lib.dsk_debug_backward_plan(eng.handle, tctx, i, plan), "dsk_debug_backward_plan")
        C, H, W = P.out_geometry(i, T)
        gx = P.stat_blocks(B * H * W, C)
        if i == 0:
            want_tiles, want_plan = (0,) * 6, (0, 0, gx)
        else:
            p = P.layer_plan(i, B, T, sms)
            want_tiles, want_plan = p["tile"] * 2, (p["ksplit"], p["per"], gx)
        assert tuple(tiles) == want_tiles, f"layer {i}: library tiles {tuple(tiles)}, restated {want_tiles}"
        assert tuple(plan) == want_plan, f"layer {i}: library plan {tuple(plan)}, restated {want_plan}"


def plan_of_a_forward(m, x, sync):
    """One train forward to bind a context, then its plan checked; the context goes back to the pool."""
    B, T = x.shape[0], x.shape[2]
    emb = m(x)
    fn = emb.grad_fn
    assert_plan(m._engine, fn.guards[0].tctx if sync else fn.guard.tctx, B, T)
    del emb, fn
    torch.cuda.synchronize()


class Measured:
    """Wall time and peak memory of one case: the PyTorch allocator's peak (the checkers' fp64 tensors) and the device
    memory in use at the end (the engine's train contexts included)."""

    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        print(f"[{self.tag}] {time.perf_counter() - self.t0:.1f} s, PyTorch peak "
              f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB, device in use at the end "
              f"{(total - free) / 2 ** 30:.2f} GiB ({torch.cuda.get_device_name()})")


@pytest.mark.parametrize("dt,B,T", [("fp16", B, T) for B, T in FP16_SHAPES] + [("bf16", B, T) for B, T in BF16_SHAPES])
def test_train_forward_and_backward_at_every_tile_regime(cuda_dev, dt, B, T):
    tag = f"{dt} B={B} T={T}"
    print(f"\n{tag}: " + ", ".join(f"stage {s} {r}" for s, r in sorted(P.case_regimes(B, T))))
    with Measured(tag):
        m, sd = train_model(512, dt, 6, cuda_dev)
        x = O.make_input(B, T, 400 + B, 3.0).cuda()
        plan_of_a_forward(m, x, sync=False)
        train_forward_and_check(f"train {tag}", m, sd, dt, x, T)
        backward_case(f"backward {tag}", m, sd, dt, x)


@pytest.mark.parametrize("B,T", SYNC_SHAPES)
def test_synchronised_train_forward_and_backward_on_one_shard(cuda_dev, B, T):
    dt = "fp16"
    tag = f"sync {dt} B={B} T={T}"
    print(f"\n{tag}: " + ", ".join(f"stage {s} {r}" for s, r in sorted(P.case_regimes(B, T, sync=True))))
    with Measured(tag):
        m, sd = train_model(512, dt, 9, cuda_dev)
        m.sync_batchnorm()
        x = O.make_input(B, T, 420, 3.0).cuda()
        plan_of_a_forward(m, x, sync=True)
        bns = [bn for _, bn in conv_bn_modules(m)]
        rm0 = [bn.running_mean.detach().clone() for bn in bns]
        rv0 = [bn.running_var.detach().clone() for bn in bns]
        emb = m(x)
        tctx = emb.grad_fn.guards[0].tctx
        raw, y = read_ctx(m, tctx, B, T, 0), read_ctx(m, tctx, B, T, 1)
        torch.cuda.synchronize()
        rm1 = [bn.running_mean.detach().clone() for bn in bns]
        rv1 = [bn.running_var.detach().clone() for bn in bns]
        check_train_chain(f"sync train {tag}", sd, dt, x, raw, y, emb, rm0, rv0, rm1, rv1,
                          stat_chains(m._engine, tctx, B, T, sync=True))
        del emb, raw, y
        backward_case(f"sync backward {tag}", m, sd, dt, x, sync=True)

