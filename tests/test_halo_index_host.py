"""conv3x3_halo_kernel's epilogue index arithmetic, emulated exactly on the CPU.

For every padded position q of a tile the epilogue computes the row R = q / (W+1), the column q - R (W+1), the image
R / (H+1), whether q is a pad ("junk"), and for a parity-planar output the destination plane and position.  Both
divisions are multiplications by a rounded-up reciprocal (csrc/conv3x3_halo.cuh, is_junk / planar_dst).  Here that
arithmetic is restated in numpy, bit for bit, and checked against integer division over every row of every eval
layer's geometry (at each row's first, second and last column), up to the largest batch whose eval workspace fits in
80 GiB.  Whether a row maps right depends only on its index, not on the batch, so the largest batch covers all smaller
ones.

The 32-bit reciprocal the kernel used before, floor(2^32/d) + 1, is exact only for q < 2^32/d.  Its emulation must
fail at the long-utterance geometries below; the GPU tests (test_gpu_forward_shapes.py) take their shapes from the same
code, so they keep crossing that bound.
"""
import numpy as np
import pytest

GIB = 1 << 30
MEM = 80 * GIB
I32 = 1 << 31
EMB, FC_SPLIT = 512, 16          # embedding width, dsk::kFcSplit
SLOTS = 2 * 132                  # CTAs of one halo launch at most (two per SM on the 132-SM H100)
TS = (16, 160, 800, 2000, 8000, 24000, 48000)
# frames T -> smallest batch whose eval forward the 32-bit reciprocal gets wrong, and the first wrong (image, row)
OLD_FAILS = {48000: (16, (15, 23999)), 24000: (34, (33, 11999)), 14400: (138, (137, 7199)), 32000: (53, (52, 15999))}
TALL_OP = (2, 46778)             # dsk_conv3x3_padded with a planar output: (N, H) whose last row the old formula misplaces


# ---- the layout (dsk_api.cu: padded_positions, act_shape, get_plan, build_halo) -------------------------------------
def padded_positions(N, H, W):
    return (1 + N * (H + 1) + (128 + W + 3 + W) // (W + 1) + 2) * (W + 1)


def act_shape(i, T):
    st = i // 3
    return T >> (st + 1), 64 >> (st + 1), 64 << st      # H, W, C


def planar_act(i):
    return i % 3 == 2 and i < 11                          # convs 2, 5, 8 write a parity-planar output (the default)


def eval_workspace(B, T):
    """Bytes of the eval forward's workspace at (B, T): the 12 activations, each rounded up to 1 KiB, then the pooled
    features, the fc output and its K-slice partials."""
    total = 0
    for i in range(12):
        H, W, C = act_shape(i, T)
        b = 4 * padded_positions(B, H // 2, W // 2) * C * 2 if planar_act(i) else padded_positions(B, H, W) * C * 2
        total += -(-b // 1024) * 1024
    return total + B * 2048 * 4 + B * EMB * 4 + FC_SPLIT * B * EMB * 4


def max_batch(T, mem=MEM):
    lo, hi = 1, 1
    while eval_workspace(hi, T) <= mem:
        hi *= 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if eval_workspace(mid, T) <= mem else (lo, mid)
    return lo


def halo_stages(T):
    """Output geometry of the halo convs of each stage of the eval forward: (stage, H, W, C, parity-planar output).
    Every halo conv of a stage (the 3x3 convs, and from stage 1 on the 5x5 s2 stage entry) tiles that geometry; the
    stage's last conv writes the next stage's input parity-planar (stages 0-2)."""
    return [(st, T >> (st + 1), 64 >> (st + 1), 64 << st, st < 3) for st in range(4)]


# ---- the kernel's arithmetic ----------------------------------------------------------------------------------------
def magic(d, bits):
    return (1 << bits) // d + 1


def umulhi32(x, m):
    """__umulhi(x, m) for uint64 arrays x < 2^32 and m < 2^32."""
    return (x * np.uint64(m)) >> np.uint64(32)


def umul64hi(x, m):
    """__umul64hi(x, m) for uint64 arrays x < 2^32 and m < 2^64: the high word of x * (mh 2^32 + ml)."""
    mh, ml = np.uint64(m >> 32), np.uint64(m & 0xFFFFFFFF)
    return (x * mh + ((x * ml) >> np.uint64(32))) >> np.uint64(32)


def div(x, d, formula):
    if formula == "old":
        return umulhi32(x, magic(d, 32))
    return umul64hi(x, magic(d, 64))


def epilogue(q, N, H, W, formula):
    """is_junk and planar_dst of positions q (int64): (junk, plane, position in the plane) as the kernel computes them."""
    pitch = W + 1
    R = div(q.astype(np.uint64), pitch, formula).astype(np.int64)
    cc = q - R * pitch
    img = div(R.astype(np.uint64), H + 1, formula).astype(np.int64)
    junk = (cc == 0) | (R - img * (H + 1) == 0) | (R >= N * (H + 1) + 1)
    hh, ww = R - 1 - img * (H + 1), cc - 1
    q2 = (img * (H // 2 + 1) + (hh >> 1) + 1) * (W // 2 + 1) + (ww >> 1) + 1
    plane = (hh & 1) * 2 + (ww & 1)
    return junk, plane, q2


def exact(q, N, H, W):
    """The same three results from integer division."""
    R, cc = q // (W + 1), q % (W + 1)
    n, hp = R // (H + 1), R % (H + 1)
    junk = (cc == 0) | (hp == 0) | (R >= N * (H + 1) + 1)
    h, w = hp - 1, cc - 1
    q2 = (n * (H // 2 + 1) + h // 2 + 1) * (W // 2 + 1) + w // 2 + 1
    return junk, (h % 2) * 2 + w % 2, q2


def tile_rows(N, H, W):
    """Every row index the tiles of a launch cover: 128-position tiles from q = W+1 to the last real position."""
    q_end = N * (H + 1) * (W + 1)
    tiles = -(-(q_end - (W + 1)) // 128)
    q_last = W + 1 + tiles * 128 - 1
    return np.arange(0, q_last // (W + 1) + 1, dtype=np.int64), tiles, q_last


def wrong_rows(N, H, W, planar, formula):
    """(image, h) of the real rows where the kernel's junk flag or planar destination differs from integer division,
    checked at the first, second and last column of every row the launch covers (a rounded-up reciprocal errs first at
    the last column, q mod (W+1) = W; its row division at the last row of an image, R mod (H+1) = H)."""
    R, _, _ = tile_rows(N, H, W)
    bad = np.zeros(R.shape, bool)
    for c in (0, 1, W):
        q = R * (W + 1) + c
        q = q[q >= W + 1]
        jk, pl, q2 = epilogue(q, N, H, W, formula)
        ej, epl, eq2 = exact(q, N, H, W)
        diff = jk != ej
        if planar:
            diff |= ~ej & ((pl != epl) | (q2 != eq2))
        bad[q // (W + 1)] |= diff
    rows = R[bad]
    return [(int(r // (H + 1)), int(r % (H + 1) - 1)) for r in rows]


def under_old_bound(N, H, W):
    """Every dividend of the launch below 2^32/d, where floor(2^32/d) + 1 is exact: the rows need no emulation."""
    R, _, q_last = tile_rows(N, H, W)
    return q_last * (W + 1) < 1 << 32 and int(R[-1]) * (H + 1) < 1 << 32


def first_failing_batch(T, formula="old", limit=None):
    """(smallest batch at which a halo conv of the eval forward at T frames maps a row wrong, that (image, h)), or None
    up to `limit` images (default: the largest batch that fits in 80 GiB)."""
    limit = limit or max_batch(T)
    best = None
    for st, H, W, C, planar in halo_stages(T):
        if formula == "old" and under_old_bound(limit, H, W):
            continue
        w = wrong_rows(limit, H, W, planar, formula)
        if w and (best is None or w[0][0] < best[1][0]):
            best = (w[0][0] + 1, w[0])
    return best


# ---- tests ------------------------------------------------------------------------------------------------------------
def test_umul64hi_emulation_matches_exact_integers():
    g = np.random.RandomState(0)
    x = np.concatenate([g.randint(0, 1 << 32, 4000, dtype=np.uint64), np.array([0, 1, (1 << 32) - 1], np.uint64)])
    for d in (2, 5, 17, 33, 35, 81, 24001, 46779, (1 << 20) + 1):
        m = magic(d, 64)
        got = umul64hi(x, m)
        assert [int(a) for a in got] == [(int(b) * m) >> 64 for b in x], d
        assert np.array_equal(got, x // np.uint64(d)), d


def test_workspace_model():
    """130 MiB at 64 x 160; under 10 GiB for each long-utterance GPU test."""
    assert eval_workspace(64, 160) == 136416256
    assert eval_workspace(16, 48000) < 9 * GIB and eval_workspace(34, 24000) < 10 * GIB


@pytest.mark.parametrize("T", sorted(set(TS) | set(OLD_FAILS)))
def test_epilogue_indices_exact_up_to_80_gib(T):
    B = max_batch(T)
    for st, H, W, C, planar in halo_stages(T):
        assert not wrong_rows(B, H, W, planar, "new"), (T, B, st)
    print(f"T={T}: every halo conv exact up to B={B} ({eval_workspace(B, T) / GIB:.1f} GiB)")


@pytest.mark.parametrize("T", sorted(OLD_FAILS))
def test_old_reciprocal_fails_where_expected(T):
    """Self-check: the 32-bit reciprocal misplaces the last row of image B-1 of conv 2 (stage 0) at these batches."""
    assert first_failing_batch(T) == OLD_FAILS[T]
    B = OLD_FAILS[T][0]
    assert first_failing_batch(T, limit=B - 1) is None
    assert first_failing_batch(T, "new") is None


def test_old_reciprocal_exact_at_serving_shapes():
    """Every T <= 8000 at B <= 256 and every T <= 2000 at B <= 1024 was exact before the fix: outputs there keep their
    bits."""
    for T in range(16, 8001, 16):
        assert first_failing_batch(T, limit=256) is None, T
    for T in range(16, 2001, 16):
        assert first_failing_batch(T, limit=1024) is None, T


@pytest.mark.parametrize("W", [4, 8])
def test_tall_op_geometry(W):
    """dsk_conv3x3_padded with a planar output at (N, H) = TALL_OP: the old formula misplaces exactly the last row of
    image 1; one image, or two at H - 2, stay under the bound."""
    N, H = TALL_OP
    assert wrong_rows(N, H, W, True, "old") == [(1, H - 1)]
    assert wrong_rows(N - 1, H, W, True, "old") == []
    assert wrong_rows(N, H - 2, W, True, "old") == []
    assert wrong_rows(N, H, W, True, "new") == []
    assert padded_positions(N, H, W) * 64 * 2 < 128 * (1 << 20)     # cheap: one input buffer of 64 channels


@pytest.mark.parametrize("T", sorted(set(TS) | {16 * k for k in (3, 7, 10, 50, 125, 333, 1000, 5000)}))
def test_32_bit_position_arithmetic_fits(T):
    """The kernel's other 32-bit position arithmetic at the largest batch that fits in 80 GiB (every term grows with
    the batch): the tile index, q0 + row, the halo box row box_plane * plane_positions + q0 - (W+2) of a 5x5 input,
    and n * (H2+1) in planar_dst."""
    B = max_batch(T)
    for st, H, W, C, planar in halo_stages(T):
        _, tiles, q_last = tile_rows(B, H, W)
        npos = padded_positions(B, H, W)
        assert 2 * tiles * (C // 64) + SLOTS < I32, (T, B, st)  # 64-position, 64-channel tiles: the most a layer has
        assert q_last < npos < I32, (T, B, st)                  # q0 + row, and the 3x3 halo box rows
        if st > 0:                                              # the 5x5 s2 stage entry reads four input planes
            assert 4 * npos < I32, (T, B, st)                   # (build_halo rejects a launch past this)
            assert 3 * npos + q_last - (W + 2) < I32, (T, B, st)
        if planar:
            assert B * (H // 2 + 1) + H // 2 + 1 < I32, (T, B, st)
            assert 4 * padded_positions(B, H // 2, W // 2) < I32, (T, B, st)
