"""Eval-forward halo convs: one JSON line with, for fp16 and bf16 operands, the batch-64 eval forward at T = 160
(bench.py's headline workload, one forward in flight):
  * the CUDA-event time of each of the 11 tensor-core conv launches (dsk_set_profiling(1): an event after every
    launch), averaged over --forwards forwards after --warmup, and the conv chain timed back to back between two
    events (dsk_set_profiling(2));
  * per launch, from the shapes and the tile schedule build_halo uses (128-position tiles, 64-channel chunks, 3-tap
    weight boxes): computed and useful FLOP, weight bytes streamed from L2, halo-tile and residual bytes, achieved
    TFLOP/s and achieved L2 -> shared-memory read GB/s;
  * the card's name, power limit and SM clock (read-only nvidia-smi query in the same run).
Writes nothing but stdout.  Run: python tools/bench_halo.py
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_model  # noqa: E402
from tools.bench_batch_hard import gpu_info  # noqa: E402

TILE = 128  # padded positions per tile (HaloSmem<N>::kTileRows)


def conv_layers(T):
    """The 11 halo-conv launches of the eval forward: (index, H, W, cin, cout, taps, residual) at the OUTPUT geometry."""
    out = []
    for i in range(1, 12):
        st = i // 3
        H, W, C = T >> (st + 1), 64 >> (st + 1), 64 << st
        k = i % 3
        if k == 0:
            out.append((i, H, W, C // 2, C, 25, False))  # parity-planar 5x5 s2 stage entry
        else:
            out.append((i, H, W, C, C, 9, k == 2))      # 3x3, the block's second conv adds the residual
    return out


def launch_traffic(B, H, W, cin, cout, taps, residual, num_sms=132):
    """Tiles, FLOP and L2 read bytes of one launch, restating build_halo's schedule (dsk_api.cu)."""
    q_end = B * (H + 1) * (W + 1)
    tiles_m = (q_end - (W + 1) + TILE - 1) // TILE
    n_tile = 64 if cout == 64 else 128
    tiles_c = cout // n_tile
    chunks = cin // 64
    planes = 4 if taps == 25 else 1
    num_tiles = tiles_m * tiles_c
    grid = min(num_tiles, num_sms)
    resident = chunks == 1 and tiles_c == 1 and taps == 9 and n_tile == 64
    tap_bytes = n_tile * 64 * 2
    # a resident CTA loads its channel tile's 9 taps once; otherwise every (tile, chunk) streams all taps again
    weight = grid * taps * tap_bytes if resident else num_tiles * chunks * taps * tap_bytes
    halo = num_tiles * chunks * planes * (TILE + 2 * W + 4) * 128
    res = num_tiles * TILE * n_tile * 2 if residual else 0
    return {"tiles_m": tiles_m, "tiles_c": tiles_c, "waves": round(num_tiles / num_sms, 2), "weights_resident": resident,
            "flop_computed": 2 * num_tiles * TILE * n_tile * cin * taps, "flop_useful": 2 * B * H * W * cout * cin * taps,
            "weight_bytes": weight, "halo_bytes": halo, "residual_bytes": res}


def sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        clk, pw = (s.strip() for s in out.split(","))
        return {"sm_clock_after": clk, "power_draw_after": pw}
    except Exception as e:
        return {"sm_clock_query_error": str(e)}


def measure(dtype, B, T, forwards, warmup):
    import torch

    from deepspeaker_pytorch_b200 import _lib as L

    dev = torch.device("cuda:0")
    model = make_model(dtype, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    xs = [torch.randn(B, 1, T, 64, device=dev, generator=g) for _ in range(8)]
    buf = (ctypes.c_float * 32)()
    n = ctypes.c_int32(0)
    with torch.no_grad():
        for i in range(warmup):
            model(xs[i % len(xs)])
        torch.cuda.synchronize()
        eng = model._engine

        def profile(level):
            L.check(eng.lib.dsk_set_profiling(eng.handle, level))
            acc = None
            for i in range(forwards):
                model(xs[i % len(xs)])
                L.check(eng.lib.dsk_get_launch_times(eng.handle, buf, 32, ctypes.byref(n)))
                v = [buf[j] for j in range(n.value)]
                acc = v if acc is None else [a + b for a, b in zip(acc, v)]
            L.check(eng.lib.dsk_set_profiling(eng.handle, 0))
            return [a / forwards for a in acc]

        sec = profile(2)      # conv1 | the 11 halo convs back to back | tail
        per = profile(1)      # conv1, convs 1..11, pool, fc, l2norm
    launches = []
    for (i, H, W, cin, cout, taps, res) in conv_layers(T):
        t = launch_traffic(B, H, W, cin, cout, taps, res)
        ms = per[i]
        l2 = t["weight_bytes"] + t["halo_bytes"] + t["residual_bytes"]
        launches.append({"conv": i, "out_hw": [H, W], "cin": cin, "cout": cout, "taps": taps, **t, "ms": round(ms, 5),
                         "tflops": round(t["flop_computed"] / (ms * 1e-3) / 1e12, 1),
                         "l2_read_gbs": round(l2 / (ms * 1e-3) / 1e9, 1)})
    return {"conv_chain_ms": round(sec[1], 4), "sum_of_launch_ms": round(sum(per[1:12]), 4), "launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=160)
    ap.add_argument("--forwards", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dtypes", default="fp16,bf16")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_halo needs a GPU"
    rec = {"metric": "eval_halo_conv_launches", **gpu_info(), "batch": args.batch, "frames": args.frames,
           "forwards": args.forwards}
    for dt in args.dtypes.split(","):
        rec[dt] = measure(dt, args.batch, args.frames, args.forwards, args.warmup)
    rec.update(sm_clock())
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
