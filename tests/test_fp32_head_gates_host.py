"""CPU self-test of the gates of tests/test_gpu_fp32_head_ops.py: an fp32 numpy emulation of each kernel passes its
gate, and the same emulation with a seeded defect fails it.  No GPU involved."""
import numpy as np
import pytest

from tests import test_gpu_fp32_head_ops as G

f32, f64 = np.float32, np.float64


def _fma(a, b, c):
    """fmaf(a, b, c) elementwise: the product of two fp32 values is exact in double."""
    return (a.astype(f64) * b.astype(f64) + c.astype(f64)).astype(f32)


def _gemm(a, b, drop_tail):
    """sgemm_strided_kernel: C = A (M,K) B (K,N), one fmaf chain per output in ascending k from 0.  drop_tail: the
    defect of a K loop that skips the last, partial 16-deep slice."""
    K = a.shape[1]
    kk = K // 16 * 16 if drop_tail else K
    acc = np.zeros((a.shape[0], b.shape[1]), f32)
    for k in range(kk):
        acc = _fma(a[:, k:k + 1], b[k:k + 1, :], acc)
    return acc


def linear_emulate(x, w, b, gy, drop_tail=False, swap_gw=False):
    y = _gemm(x, w.T, drop_tail)
    if b is not None:
        y = (y + b).astype(f32)
    gx = _gemm(gy, w, drop_tail)
    # swapped operands: the (K, N) product x^T gy written into the (N, K) buffer
    gw = _gemm(x.T, gy, drop_tail).reshape(w.shape) if swap_gw else _gemm(gy.T, x, drop_tail)
    gb = np.zeros(w.shape[0], f32)
    for i in range(gy.shape[0]):
        gb = (gb + gy[i]).astype(f32)
    return y, gx, gw, gb


@pytest.mark.parametrize("M,N,K", [(65, 5, 17), (63, 30, 15), (1, 1, 1), (20, 7, 33)])
def test_linear_gate_passes_the_emulation_and_fails_the_defects(M, N, K):
    x, w, b, gy = (t.numpy() for t in G._linear_inputs(M, N, K, M + N + K))
    r = G.linear_gate(x, w, b, gy, *linear_emulate(x, w, b, gy))
    assert max(r.values()) <= 1.0, r
    if K % 16:
        assert G.linear_gate(x, w, b, gy, *linear_emulate(x, w, b, gy, drop_tail=True))["y"] > 1.0
    if N * K > 1:
        assert G.linear_gate(x, w, b, gy, *linear_emulate(x, w, b, gy, swap_gw=True))["gw"] > 1.0


def ce_emulate(x, labels, gl, no_max=False, finite_invalid_grad=False):
    """ce_rows_kernel / mean_rows_kernel / ce_bwd_kernel in fp32 (numpy's own summation order)."""
    M, C = x.shape
    valid = (labels >= 0) & (labels < C)
    y = np.where(valid, labels, 0)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        m = np.zeros((M, 1), f32) if no_max else x.max(1, keepdims=True)
        s = np.exp((x - m).astype(f32)).astype(f32).sum(1, dtype=f32)
        lse = (m[:, 0] + np.log(s).astype(f32)).astype(f32)
        rows = np.where(valid, (lse - x[np.arange(M), y]).astype(f32), f32(np.nan)).astype(f32)
        loss = f32(rows.sum(dtype=f32) / f32(M))
        g = f32(f32(gl) / f32(M))
        p = np.exp((x - lse[:, None]).astype(f32)).astype(f32)
        onehot = np.zeros_like(p)
        onehot[np.arange(M), y] = 1.0
        d = ((p - onehot).astype(f32) * g).astype(f32)
    if not finite_invalid_grad:
        d[~valid] = np.nan
    return lse, rows, float(loss), d


def test_ce_gate_passes_the_emulation_and_fails_the_defects():
    for scale, C, M in ((1.0, 1211, 64), (30.0, 1211, 65), (3e4, 2, 33), (1e3, 1, 3)):
        x, labels = G.ce_case(scale, C, M, 1)
        r = G.ce_gate(x, labels, 2.5, *ce_emulate(x, labels, 2.5))
        assert max(r.values()) <= 1.0, (scale, C, M, r)
        if scale >= 30:   # without the max subtraction exp overflows from |x| > 88.7 on
            r = G.ce_gate(x, labels, 2.5, *ce_emulate(x, labels, 2.5, no_max=True))
            assert r["lse"] > 1.0, (scale, r)
    x, labels = G.ce_case(30.0, 1211, 65, 2)
    labels[3], labels[60] = -1, 1211
    assert max(G.ce_gate(x, labels, 1.0, *ce_emulate(x, labels, 1.0)).values()) <= 1.0
    assert G.ce_gate(x, labels, 1.0, *ce_emulate(x, labels, 1.0, finite_invalid_grad=True))["grad"] > 1.0


def adagrad_emulate(p, s, S, step, hp, d, recip=False):
    """One adagrad_flat_kernel step in fp32 on the summed gradient S: g = S / d (recip: the defect S * fp32(1/d))."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        g = (S * f32(1.0 / f32(d))).astype(f32) if recip else (S / f32(d)).astype(f32)
        if hp["weight_decay"]:
            g = _fma(p, np.full_like(p, f32(hp["weight_decay"])), g)
        s = _fma(g, g, s)
        std = (np.sqrt(s).astype(f32) + f32(hp["eps"])).astype(f32)
        minus_clr = f32(-hp["lr"] / (1.0 + (step - 1) * hp["lr_decay"]))
        p = (p + ((g * minus_clr).astype(f32) / std).astype(f32)).astype(f32)
    return p, s


@pytest.mark.parametrize("d,differs", [(3, True), (37, True), (7, True), (2, False), (8, False), (1, False)])
def test_adagrad_reciprocal_defect_is_visible(d, differs):
    """The GPU test compares bits with torch stepping on S / d.  A kernel that multiplies by fp32(1/d) instead differs
    in a large share of elements for d = 3, 7, 37 (so those tests catch it) and in none for powers of two."""
    rng = np.random.default_rng(d)
    n = 100000
    p0, S = rng.standard_normal(n).astype(f32), rng.standard_normal(n).astype(f32)
    s0 = np.zeros(n, f32)
    hp = dict(G.HP_BASE, weight_decay=1e-3)
    pa, sa = adagrad_emulate(p0, s0, S, 1, hp, d)
    pb, sb = adagrad_emulate(p0, s0, S, 1, hp, d, recip=True)
    n_diff = int(((pa.view(np.int32) != pb.view(np.int32)) | (sa.view(np.int32) != sb.view(np.int32))).sum())
    assert (n_diff > n // 20) if differs else n_diff == 0, n_diff


def test_adagrad_zero_weight_defect_is_visible():
    """sum_k = 0 with S = 0: the quotient by max(0, 1e-30) is 0, the reciprocal of 0 makes 0 * inf = NaN."""
    p0, S, s0 = np.ones(8, f32), np.zeros(8, f32), np.zeros(8, f32)
    assert np.isfinite(adagrad_emulate(p0, s0, S, 1, G.HP_BASE, max(0.0, 1e-30))[0]).all()
    assert np.isnan(adagrad_emulate(p0, s0, S, 1, G.HP_BASE, 0.0, recip=True)[0]).all()


def triplet_bwd_emulate(a, p, n, d_p, d_n, gl, margin, strict=False):
    """triplet_loss_bwd_kernel in fp32; strict: the defect of a hinge test with > instead of >=."""
    pre = ((f32(margin) + d_p) - d_n).astype(f32)
    act = (pre > 0 if strict else pre >= 0).astype(f32)[:, None]
    g = (act * f32(gl) / f32(a.shape[0])).astype(f32)
    up = ((g * (a - p).astype(f32)).astype(f32) / d_p[:, None]).astype(f32)
    un = ((-g * (a - n).astype(f32)).astype(f32) / d_n[:, None]).astype(f32)
    return (up + un).astype(f32), -up, -un


def test_triplet_gates_pass_the_emulation_and_fail_a_strict_hinge():
    a, p, n, d_p, d_n, margin = G.hinge_edge_case()
    r = G.triplet_bwd_gate(a, p, n, d_p, d_n, 2.0, margin, *triplet_bwd_emulate(a, p, n, d_p, d_n, 2.0, margin))
    assert max(r.values()) <= 1.0, r
    r = G.triplet_bwd_gate(a, p, n, d_p, d_n, 2.0, margin,
                           *triplet_bwd_emulate(a, p, n, d_p, d_n, 2.0, margin, strict=True))
    assert r["ga"] > 1.0 and r["gp"] > 1.0
    # distances: the fp32 squared differences summed in fp32, + fp32 eps, sqrt
    x1, x2 = (t.numpy() for t in G._triplet_inputs(300, 513, 0)[:2])
    diff = (x1 - x2).astype(f32)
    dist = np.sqrt(((diff * diff).astype(f32).sum(1, dtype=f32) + f32(1e-4 / 513)).astype(f32)).astype(f32)
    assert G.distance_gate(x1, x2, dist) <= 1.0
    assert G.distance_gate(x1, x2, (dist * f32(1 + 2.0 ** -10)).astype(f32)) > 1.0
    pre = ((f32(0.5) + dist) - dist[::-1]).astype(f32)
    loss = f32(np.maximum(pre, 0).sum(dtype=f32) / f32(dist.size))
    assert G.triplet_loss_gate(dist, dist[::-1].copy(), 0.5, loss) <= 1.0


def test_threshold_reference_is_np_less():
    d, same, th = G._threshold_case(2049, 257, "random", 0)
    tp, fp = G.threshold_reference(d, same, th)
    below = np.less(d.astype(f64)[None, :], th[:, None])
    assert np.array_equal(tp, (below & same).sum(1)) and np.array_equal(fp, (below & ~same).sum(1))
