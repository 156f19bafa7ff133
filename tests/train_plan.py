"""The train convs' plans restated from the host code of csrc/dsk_api.cu, and the regimes they put a layer in.

For conv layer i (1..11) of a train forward at batch B and T frames, ctx_bind builds the forward conv, its data-gradient
convs and the weight-gradient GEMM over the layer's output grid B x H x W, each tiled by the 128-pixel box (wt, hb, nb)
of choose_tile; the weight gradient splits its 128-pixel K chunks over `ksplit` slices of `per` chunks each; the
BatchNorm reductions of the unsynchronised path run gx = stat_blocks(M, C) blocks of 32 threads per 64 channels.
dsk_debug_train_tiles and dsk_debug_backward_plan report what the library chose, so a GPU test can hold this
restatement to it; tests/test_train_tiles_host.py holds the GPU cases to every regime it finds reachable.
"""
from itertools import product

STAT_BLOCKS_MAX = 592      # kStatBlocksMax: BatchNorm partial blocks per 64 channels at most
H100_SMS = 132             # SMs of the H100 SXM, what the weight-gradient K split is planned for
MAX_B, MAX_T = 256, 1600   # the training shapes enumerated: B <= 256 utterances of T <= 1600 frames (16 s)


def layer_cfg(i):
    """(cin, cout, ksize, stride) of conv layer i (dsk_api.cu layer_cfg)."""
    ch = (64, 128, 256, 512)
    st = i // 3
    if i % 3 == 0:
        return (1 if st == 0 else ch[st - 1]), ch[st], 5, 2
    return ch[st], ch[st], 3, 1


def out_geometry(i, T):
    """(C, H, W) of conv layer i's output (act_shape)."""
    st = i // 3
    return 64 << st, T >> (st + 1), 64 >> (st + 1)


def stage(i):
    """1..4: the resolution stage of conv layer i's output (W = 32, 16, 8, 4)."""
    return i // 3 + 1


def choose_tile(B, H, W, total=128):
    """(wt, hb, nb), wt hb nb = total: the full width, then the power-of-two split of the rows over h and n that pads
    the grid least (ties to the taller box)."""
    wt = min(W, total)
    rows = total // wt
    best, hb, nb = None, 1, rows
    h = rows
    while h >= 1:
        n = rows // h
        padded = -(-H // h) * h * (-(-B // n) * n)
        if best is None or padded < best:
            best, hb, nb = padded, h, n
        h >>= 1
    return wt, hb, nb


def wgrad_split(B, H, W, cin, cout, taps, num_sms=H100_SMS):
    """(ksplit, per, chunks) of the weight-gradient GEMM (build_wgrad): >= 2 work items per SM, at least 4 chunks per
    split; split k takes chunks [k per, min((k + 1) per, chunks))."""
    wt, hb, nb = choose_tile(B, H, W)
    chunks = -(-W // wt) * -(-H // hb) * -(-B // nb)
    swapped = cout == 64
    n_tile = 64 if swapped else (128 if cin >= 128 else 64)
    items0 = (taps + 1) // 2 if swapped else taps * (cout // 128) * (cin // n_tile)
    ksplit = max(1, min(-(-2 * num_sms // items0), max(chunks // 4, 1)))
    return ksplit, -(-chunks // ksplit), chunks


def stat_blocks(M, C):
    return max(1, min(STAT_BLOCKS_MAX // (C // 64), -(-M // 32)))


def reduce_chain(M, HW, gx, sync):
    """Longest fp32 chain of the BatchNorm reductions of one layer (forward statistics and backward sums): gx blocks
    of 32 threads striding over the M rows, then 32 thread partials per block; the synchronised path sums each
    utterance's HW pixels over 32 lanes, then a 5-level tree."""
    if sync:
        return -(-HW // 32) + 5
    return -(-M // (32 * gx)) + 32


def layer_plan(i, B, T, num_sms=H100_SMS):
    """Everything the library plans for conv layer i >= 1 at (B, T): tile, weight-gradient split, BatchNorm grid."""
    cin, cout, k, _ = layer_cfg(i)
    C, H, W = out_geometry(i, T)
    ksplit, per, chunks = wgrad_split(B, H, W, cin, cout, k * k, num_sms)
    M = B * H * W
    return dict(tile=choose_tile(B, H, W), ksplit=ksplit, per=per, chunks=chunks, gx=stat_blocks(M, C), M=M, HW=H * W,
                C=C, H=H, W=W)


def regimes(i, B, T, sync=False, num_sms=H100_SMS):
    """The regimes conv layer i >= 1 runs in at (B, T), as (stage, name) pairs:
      tile hbxnb                the box shape (wt is always the full width)
      box taller than the image hb > H: the rows past the image come from TMA's out-of-bounds fill only
      ragged h / n / h and n    the last box row (utterance) block runs past H (B)
      empty K split             a weight-gradient slice that gets no chunk (it stores zeros)
      uneven K split            the last non-empty slice gets fewer chunks than the others
      BN grid at its cap        more rows than gx = kStatBlocksMax / (C / 64) blocks of 32 cover in one pass
      plain chain > 64          unsynchronised BatchNorm reductions whose fp32 chains are longer than 64 terms
      sync chain > 64           the same for the per-utterance records of synchronised BatchNorm
    The two chain regimes are counted once for the whole forward (stage 0): a longer chain is the same kernel looping
    more often, and what it tests is the checkers' n-dependent bound.  Per stage they would need B T > 303104 (stage 4),
    a forward too large to check in fp64 on a shared GPU; the stage-dependent part, a BatchNorm grid at its cap (gx
    blocks striding over the rows more than once), is counted per stage."""
    p = layer_plan(i, B, T, num_sms)
    _, hb, nb = p["tile"]
    s = stage(i)
    out = {(s, f"tile {hb}x{nb}")}
    rh, rn = p["H"] % hb != 0, B % nb != 0
    if hb > p["H"]:
        out.add((s, "box taller than the image"))
    if rh or rn:
        out.add((s, "ragged h and n" if rh and rn else "ragged h" if rh else "ragged n"))
    ksplit, per, chunks = p["ksplit"], p["per"], p["chunks"]
    if (ksplit - 1) * per >= chunks:
        out.add((s, "empty K split"))
    elif chunks % per:
        out.add((s, "uneven K split"))
    if sync:
        if reduce_chain(p["M"], p["HW"], p["gx"], True) > 64:
            out.add((0, "sync chain > 64"))
    else:
        if -(-p["M"] // 32) > STAT_BLOCKS_MAX // (p["C"] // 64):
            out.add((s, "BN grid at its cap"))
        if reduce_chain(p["M"], p["HW"], p["gx"], False) > 64:
            out.add((0, "plain chain > 64"))
    return out


def case_regimes(B, T, sync=False, num_sms=H100_SMS):
    return set().union(*(regimes(i, B, T, sync, num_sms) for i in range(1, 12)))


def reachable(sync, num_sms=H100_SMS):
    """Every regime some B <= MAX_B, T <= MAX_T (a multiple of 16) reaches, with the first (B, T) that does."""
    seen = {}
    for B, T in product(range(1, MAX_B + 1), range(16, MAX_T + 1, 16)):
        for r in case_regimes(B, T, sync, num_sms):
            seen.setdefault(r, (B, T))
    return seen
