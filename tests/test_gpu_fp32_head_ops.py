"""The small fp32 kernels every training step runs, against fp64 (or bit for bit against numpy / torch):

  a. ``LinearFn`` / ``dsk_linear_*`` (``sgemm_strided_kernel``, ``colsum_kernel``)
  b. ``dsk_cross_entropy(_bwd)`` (``ce_rows_kernel``, ``mean_rows_kernel``, ``ce_bwd_kernel``)
  c. ``dsk_adagrad_step`` / ``FusedAdagrad`` (``adagrad_flat_kernel``) vs ``torch.optim.Adagrad`` (CUDA, foreach)
  d. ``dsk_pairwise_distance``, ``dsk_triplet_loss`` and their backwards
  e. ``select_hard_triplets``, ``gather_rows``, ``threshold_counts`` vs numpy

Every gate is a bound derived from the kernel's operation order, with u = 2^-24 and gamma(n) = n u / (1 - n u) (the
bound on n successive roundings of non-negative terms, or of a chain whose error is measured against the sum of the
terms' magnitudes).  The gate functions take numpy arrays and return {name: max err / bound}; a structural failure (a
NaN that should not be there, a finite value that should be NaN) counts as inf.  ``tests/test_fp32_head_gates_host.py``
runs them on CPU fp32 emulations of the kernels and on emulations with seeded defects, which they must reject.
"""
import math

import numpy as np
import pytest
import torch

import deepspeaker_pytorch_b200 as dsk
from deepspeaker_pytorch_b200 import _lib as L
from deepspeaker_pytorch_b200 import engine, head, verification

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -148        # 2 ulp of the smallest fp32 subnormal: expf's absolute error where it underflows
f32, f64 = np.float32, np.float64


def gamma(n):
    return n * U / (1.0 - n * U)


def _ratio(err, bound):
    """max err / bound elementwise; err > 0 where bound == 0 (or err NaN) is inf."""
    err = np.asarray(err, f64)
    bound = np.broadcast_to(np.asarray(bound, f64), err.shape)
    bad = np.isnan(err) | ((bound <= 0) & (err > 0))
    r = np.divide(err, bound, out=np.zeros_like(err), where=bound > 0)
    r[bad] = np.inf
    return float(r.max()) if r.size else 0.0


def _report(name, ratios):
    print(f"{name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v <= 1.0, (name, k, v)


# ---- a. linear -----------------------------------------------------------------------------------------------------
def linear_gate(x, w, b, gy, y, gx, gw, gb):
    """y = x w^T + b: each output is ONE fmaf chain in ascending k from 0 (K roundings), then the bias add:
         |dy_ij| <= gamma(K + 1) (sum_k |x_ik| |w_jk| + |b_j|).
    gx = gy w (chain length N), gw = gy^T x (chain length M, the transposed-stride loader), gb = column sums of gy
    (M sequential adds from 0): the same form with their own chain lengths."""
    x64, w64, gy64 = x.astype(f64), w.astype(f64), gy.astype(f64)
    M, K = x.shape
    N = w.shape[0]
    out = {}
    ref = x64 @ w64.T
    mag = np.abs(x64) @ np.abs(w64).T
    if b is not None:
        ref = ref + b.astype(f64)
        mag = mag + np.abs(b.astype(f64))
    out["y"] = _ratio(np.abs(y - ref), gamma(K + 1) * mag)
    if gx is not None:
        out["gx"] = _ratio(np.abs(gx - gy64 @ w64), gamma(N) * (np.abs(gy64) @ np.abs(w64)))
    if gw is not None:
        if gw.shape != (N, K):
            return dict(out, gw=np.inf)
        out["gw"] = _ratio(np.abs(gw - gy64.T @ x64), gamma(M) * (np.abs(gy64).T @ np.abs(x64)))
    if gb is not None:
        out["gb"] = _ratio(np.abs(gb - gy64.sum(0)), gamma(M) * np.abs(gy64).sum(0))
    return out


def _linear_inputs(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    gy = torch.randn(M, N, generator=g)
    return x, w, b, gy


# every edge value of M in {1, 63, 64, 65, 1536}, N in {1, 5, 1211, 5994}, K in {1, 15, 16, 17, 96, 512, 513}
LINEAR_CASES = [(1, 1, 1, True), (63, 5, 15, False), (64, 1211, 16, True), (65, 5994, 17, False),
                (1536, 1211, 512, True), (1, 5994, 513, False), (65, 1, 96, True), (64, 5, 513, True),
                (1536, 1, 17, False), (63, 1211, 1, False), (1536, 5, 96, True), (65, 1211, 513, False),
                (1, 5, 16, False), (64, 5994, 15, True)]


@pytest.mark.parametrize("M,N,K,bias", LINEAR_CASES)
def test_linear_within_fp64_bound(cuda_dev, M, N, K, bias):
    x, w, b, gy = _linear_inputs(M, N, K, 100 + M + N + K)
    xc, wc = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    bc = b.cuda().requires_grad_(True) if bias else None
    y = head.LinearFn.apply(xc, wc, bc)
    y.backward(gy.cuda())
    r = linear_gate(x.numpy(), w.numpy(), b.numpy() if bias else None, gy.numpy(), y.detach().cpu().numpy(),
                    xc.grad.cpu().numpy(), wc.grad.cpu().numpy(), bc.grad.cpu().numpy() if bias else None)
    _report(f"linear M={M} N={N} K={K} bias={bias}", r)
    # only the gradients asked for are written (NULL output pointers): gw alone gives the same bits
    wc2 = w.cuda().requires_grad_(True)
    head.LinearFn.apply(x.cuda(), wc2, None).backward(gy.cuda())
    assert torch.equal(wc2.grad, wc.grad)


def test_linear_rows_are_independent_and_deterministic(cuda_dev):
    """Row i of y does not depend on the other rows of the batch (the tile it lands in, the rows beside it), and two
    runs give identical bits."""
    M, N, K = 1536, 1211, 513
    x, w, b, _ = _linear_inputs(M, N, K, 7)
    xc, wc, bc = x.cuda(), w.cuda(), b.cuda()
    y = head.LinearFn.apply(xc, wc, bc)
    assert torch.equal(y, head.LinearFn.apply(xc, wc, bc))
    for i in (0, 1, 63, 64, 65, 777, 1535):
        assert torch.equal(head.LinearFn.apply(xc[i:i + 1].clone(), wc, bc)[0], y[i]), i
    assert torch.equal(head.LinearFn.apply(xc[100:300].clone(), wc, bc), y[100:300])


# ---- b. cross-entropy -----------------------------------------------------------------------------------------------
def ce_gate(logits, labels, gl, lse, rows, loss, d):
    """Per row (one block of 256 threads): m = max_j x_j (exact); t_j = x_j - m (|dt_j| <= u |x_j - m|);
    e_j = expf(t_j) (2 ulp: relative 4u, absolute 2^-148 where it underflows); s = sum_j e_j over ceil(C/256)
    thread-strided adds, 5 shuffle levels and 8 warp partials (n_s = ceil(C/256) + 13 roundings of non-negative terms);
    lse = m + logf(s) (1 ulp, then one add).  So with p_j = exp(x_j - m) in fp64:
        |ds| <= sum_j p_j ((1 + 4u) exp(u |x_j - m|) - 1) + C 2^-148 + gamma(n_s) sum_j p_j (1 + that),
        |dlse| <= -log(1 - |ds|/s) + 2u |log s| (1 + u) + u |lse|,     |drow| <= |dlse| (1 + u) + u |lse - x_y|.
    The mean (1024 threads: ceil(M/1024) strided adds, 5 shuffles, 32 partials, then / M) is within
        sum_i |drow_i| / M + gamma(ceil(M/1024) + 38) sum_i (|row_i| + |drow_i|) / M.
    The gradient (x_j - lse_hat rounded, expf, - [j == y], * fp32(gl / M)) per element:
        |dd| <= |g| ((1 + u)^3 |p^ - p| + ((1 + u)^3 - 1) |p - [j == y]|) + 2^-149   (the product's rounding where
                                                                                     it underflows is absolute),
        |p^ - p| <= p ((1 + 4u) exp(|dlse| + u (|x_j - lse| + |dlse|)) - 1) + 2^-148.
    A label outside [0, C): that row's loss, the mean and the whole gradient row are NaN."""
    x = logits.astype(f64)
    M, C = x.shape
    valid = (labels >= 0) & (labels < C)
    fin = np.isfinite(x)
    m = x.max(1, keepdims=True)
    t = np.where(fin, x - m, -np.inf)
    p = np.exp(t)
    s = p.sum(1)
    eta = np.where(fin, (1 + 4 * U) * np.exp(U * np.abs(np.where(fin, t, 0.0))) - 1, 0.0)
    n_s = -(-C // 256) + 13
    ds = (p * eta).sum(1) + C * TINY + gamma(n_s) * (p * (1 + eta)).sum(1)
    ref_lse = m[:, 0] + np.log(s)
    dlse = -np.log1p(-ds / s) + 2 * U * np.abs(np.log(s)) * (1 + U) + U * np.abs(ref_lse)
    out = {"lse": _ratio(np.abs(lse - ref_lse), dlse)}
    y = np.where(valid, labels, 0)
    xy = x[np.arange(M), y]
    ref_row = ref_lse - xy
    drow = dlse * (1 + U) + U * np.abs(ref_row)
    out["row_loss"] = _ratio(np.where(valid, np.abs(rows - ref_row), 0.0), drow)
    if not np.isnan(rows[~valid]).all():
        out["row_loss"] = np.inf
    if valid.all():
        nm = -(-M // 1024) + 38
        bound = drow.sum() / M + gamma(nm) * (np.abs(ref_row) + drow).sum() / M
        out["loss"] = _ratio(abs(float(loss) - ref_row.mean()), bound)
    else:
        out["loss"] = 0.0 if np.isnan(loss) else np.inf
    g = float(f32(gl) / f32(M))
    onehot = np.zeros_like(x)
    onehot[np.arange(M), y] = 1.0
    ref_p = np.where(fin, np.exp(np.where(fin, x - ref_lse[:, None], 0.0)), 0.0)
    arg = dlse[:, None] + U * (np.abs(np.where(fin, x - ref_lse[:, None], 0.0)) + dlse[:, None])
    dp = np.where(fin, ref_p * ((1 + 4 * U) * np.exp(arg) - 1), 0.0) + TINY
    c3 = (1 + U) ** 3
    bound = abs(g) * (c3 * dp + (c3 - 1) * np.abs(ref_p - onehot)) + 2.0 ** -149
    err = np.abs(d - (ref_p - onehot) * g)
    out["grad"] = _ratio(np.where(valid[:, None], err, 0.0), bound)
    if not np.isnan(d[~valid]).all():
        out["grad"] = np.inf
    return out


def _ce_run(logits, labels, gl):
    """The two ABI calls CrossEntropyFn makes; returns (lse, row_loss, loss, dlogits) as numpy."""
    lg = torch.from_numpy(logits).cuda()
    lab = torch.from_numpy(labels).cuda()
    M, C = logits.shape
    loss = torch.empty(1, device="cuda")
    lse = torch.empty(M, device="cuda")
    rows = torch.empty(M, device="cuda")
    g = torch.tensor([gl], dtype=torch.float32, device="cuda")
    d = torch.empty_like(lg)
    lib = L.load()
    L.check(lib.dsk_cross_entropy(lg.data_ptr(), lab.data_ptr(), M, C, loss.data_ptr(), lse.data_ptr(),
                                  rows.data_ptr(), L.cur_stream()), "dsk_cross_entropy")
    L.check(lib.dsk_cross_entropy_bwd(lg.data_ptr(), lab.data_ptr(), lse.data_ptr(), g.data_ptr(), M, C,
                                      d.data_ptr(), L.cur_stream()), "dsk_cross_entropy_bwd")
    return lse.cpu().numpy(), rows.cpu().numpy(), float(loss.item()), d.cpu().numpy()


def ce_case(scale, C, M, seed):
    """Logits scale * randn, labels uniform with row 0 at 0 and the last row at C - 1; for C >= 2 row M // 2 has every
    non-label column at -inf."""
    rng = np.random.default_rng(seed)
    x = (scale * rng.standard_normal((M, C))).astype(f32)
    labels = rng.integers(0, C, M).astype(np.int64)
    labels[0], labels[-1] = 0, C - 1
    if C >= 2 and M >= 3:
        i = M // 2
        keep = x[i, labels[i]]
        x[i, :] = -np.inf
        x[i, labels[i]] = keep
    return x, labels


# scales {1, 30, 1e3, 3e4} x C {1, 2, 1211, 5994, 20000} x M {1, 1023, 1024, 1025, 3000}, sampled with every edge value
CE_CASES = [(1.0, 1, 1), (1.0, 5994, 1024), (30.0, 2, 3000), (30.0, 1211, 1025), (1e3, 20000, 1023),
            (3e4, 1211, 1024), (3e4, 20000, 1), (1e3, 5994, 1), (3e4, 2, 1025), (30.0, 1, 1023), (1.0, 20000, 3)]


@pytest.mark.parametrize("scale,C,M", CE_CASES)
def test_cross_entropy_within_fp64_bound(cuda_dev, scale, C, M):
    x, labels = ce_case(scale, C, M, int(scale) + C + M)
    gl = 2.5
    lse, rows, loss, d = _ce_run(x, labels, gl)
    _report(f"cross-entropy scale={scale} C={C} M={M}", ce_gate(x, labels, gl, lse, rows, loss, d))
    if C >= 2 and M >= 3:   # the -inf row: loss exactly 0, gradient exactly 0
        i = M // 2
        assert rows[i] == 0.0 and not d[i].any()


@pytest.mark.parametrize("C,M", [(1211, 1025), (5, 4)])
def test_cross_entropy_invalid_labels_are_nan_rows(cuda_dev, C, M):
    """Labels -1 and C: that row's loss and its whole gradient row are NaN and the mean is NaN; every other row's lse,
    loss and gradient are bit-identical to the run with those labels replaced by valid ones (same M, same g / M)."""
    x, labels = ce_case(30.0, C, M, 5)
    bad = labels.copy()
    bad[1], bad[-2] = -1, C
    lse_b, rows_b, loss_b, d_b = _ce_run(x, bad, 1.0)
    lse_g, rows_g, loss_g, d_g = _ce_run(x, labels, 1.0)
    inv = np.zeros(M, bool)
    inv[[1, M - 2]] = True
    _report(f"cross-entropy invalid labels C={C} M={M}", ce_gate(x, bad, 1.0, lse_b, rows_b, loss_b, d_b))
    assert np.isnan(loss_b) and np.isnan(rows_b[inv]).all() and np.isnan(d_b[inv]).all()
    assert np.array_equal(lse_b, lse_g)
    assert np.array_equal(rows_b[~inv], rows_g[~inv]) and np.array_equal(d_b[~inv], d_g[~inv])
    # through the autograd Function as train_step uses it
    lg = torch.from_numpy(x).cuda().requires_grad_(True)
    dsk.CrossEntropyLoss()(lg, torch.from_numpy(bad).cuda()).backward()
    assert torch.isnan(lg.grad[torch.from_numpy(inv).cuda()]).all()
    assert np.array_equal(lg.grad.cpu().numpy()[~inv], d_g[~inv])


# ---- c. fused Adagrad -----------------------------------------------------------------------------------------------
LENGTHS = (1, 2, 3, 5, 4 * 1024 + 3, 4 * (1 << 20) + 3)   # the scalar tail alone, vector + tail, grid-stride + tail


def _adagrad_call(p, s, g, step, hp, div=1.0, denom=None):
    """What FusedAdagrad.step passes to dsk_adagrad_step."""
    L.check(L.load().dsk_adagrad_step(p.data_ptr(), g.data_ptr(), s.data_ptr(), p.numel(), float(hp["lr"]),
                                      float(hp["lr_decay"]), float(hp["weight_decay"]), float(hp["eps"]), int(step),
                                      float(div), L.ptr(denom), L.cur_stream()), "dsk_adagrad_step")


def _hard_gradient(n, gen, scale=1.0):
    """randn with zeros, subnormals and values near +-1e30 sprinkled in."""
    g = torch.randn(n, generator=gen) * scale
    if n >= 5:
        k = max(1, n // 16)
        pos = torch.randperm(n, generator=gen)[:3 * k]
        g[pos[:k]] = 0.0
        g[pos[k:2 * k]] = torch.randn(k, generator=gen).sign() * 1e-40
        g[pos[2 * k:]] = torch.randn(k, generator=gen) * 1e30
    elif n >= 3:
        g[0], g[1] = 0.0, 3e-41
    return g


HP_BASE = dict(lr=0.1, lr_decay=1e-4, weight_decay=0.0, eps=1e-10, initial_accumulator_value=0.0)


def _run_adagrad_vs_torch(dev, divisor, weighted, hp, steps, seed, start_step=0, lengths=LENGTHS):
    """For each length: our buffers stepped by dsk_adagrad_step on the summed gradient S, torch.optim.Adagrad (CUDA,
    foreach) stepped on S.div(d) with d a CUDA tensor (GradBucket's true division; ATen would turn a CPU-scalar divisor
    into a product with its reciprocal).  Weighted: d = divisor.clamp_min(1e-30), divisor the device scalar sum_k.
    Returns the number of elements whose parameter or sum bits differ, over all steps and lengths."""
    gen = torch.Generator().manual_seed(seed)
    d_t = torch.tensor(float(divisor), dtype=torch.float32, device=dev)
    if weighted:
        d_t = d_t.clamp_min(1e-30)
    denom = torch.tensor([float(divisor)], dtype=torch.float32, device=dev)
    differ = 0
    for n in lengths:
        p0 = torch.randn(n, generator=gen).to(dev)
        s0 = torch.full((n,), float(hp["initial_accumulator_value"]), device=dev)
        if start_step:
            s0 = s0 + torch.rand(n, generator=gen).to(dev) * 10.0
        q = torch.nn.Parameter(p0.clone())
        opt = torch.optim.Adagrad([q], lr=hp["lr"], lr_decay=hp["lr_decay"], weight_decay=hp["weight_decay"],
                                  eps=hp["eps"], initial_accumulator_value=hp["initial_accumulator_value"], foreach=True)
        opt.state[q]["sum"].copy_(s0)
        opt.state[q]["step"].fill_(float(start_step))
        p, s = p0.clone(), s0.clone()
        for it in range(steps):
            S = (torch.zeros(n) if divisor == 0 else _hard_gradient(n, gen, 10.0 ** -(it % 3))).to(dev)
            q.grad = S.div(d_t)
            opt.step()
            _adagrad_call(p, s, S, start_step + it + 1, hp, div=1.0 if weighted else divisor,
                          denom=denom if weighted else None)
            differ += int(((p.view(torch.int32) != q.detach().view(torch.int32))
                           | (s.view(torch.int32) != opt.state[q]["sum"].view(torch.int32))).sum())
        if divisor == 0:
            assert torch.isfinite(p).all() and torch.isfinite(s).all()
    return differ


@pytest.mark.parametrize("R", range(1, 9))
def test_adagrad_unweighted_divides_by_world(cuda_dev, R):
    """g = S / R (the sum-allreduce's mean over R ranks) before the step: bit-identical to torch on S.div(R)."""
    assert _run_adagrad_vs_torch(cuda_dev, R, False, HP_BASE, 5, R) == 0


@pytest.mark.parametrize("sum_k", [1, 3, 37, 3072, 0])
def test_adagrad_weighted_divides_by_sum_k(cuda_dev, sum_k):
    """g = S / max(sum_k, 1e-30), S = sum_r k_r g_r: bit-identical to GradBucket.allreduce_weighted_mean + torch.
    sum_k = 0 (every rank selected nothing: S = 0) leaves the parameters finite and equal to that reference."""
    assert _run_adagrad_vs_torch(cuda_dev, sum_k, True, HP_BASE, 5, 50 + sum_k) == 0


@pytest.mark.parametrize("name,hp,steps,start,div,weighted", [
    ("weight decay", dict(HP_BASE, weight_decay=1e-3), 5, 0, 3, True),
    ("weight decay unweighted", dict(HP_BASE, weight_decay=1e-3), 5, 0, 7, False),
    ("initial accumulator", dict(HP_BASE, initial_accumulator_value=0.1), 5, 0, 37, True),
    ("eps 1e-6", dict(HP_BASE, eps=1e-6), 5, 0, 5, False),
    ("300 steps", HP_BASE, 300, 0, 3, True),
    ("state at step 1e5", dict(HP_BASE, lr=0.07, weight_decay=1e-3), 3, 100000, 6, False),
])
def test_adagrad_hyper_parameters(cuda_dev, name, hp, steps, start, div, weighted):
    lengths = LENGTHS[:5] if steps > 10 else LENGTHS
    assert _run_adagrad_vs_torch(cuda_dev, div, weighted, hp, steps, len(name), start, lengths) == 0, name


@pytest.mark.parametrize("sum_k", [3.0, 37.0, 0.0])
def test_fused_adagrad_weighted_step_matches_torch(cuda_dev, sum_k):
    """Through the class, in one process: allreduce(weight=k) stores k beside the gradients and returns without a
    collective; step() divides by max(k, 1e-30).  Same bits as torch stepping on grad.div(k.clamp_min(1e-30))."""
    gen = torch.Generator().manual_seed(int(sum_k))
    shapes = [(64, 1, 5, 5), (7,), (513, 3), (1211, 512), (1,), (2,)]
    init = [torch.randn(*sh, generator=gen) for sh in shapes]
    ours = [torch.nn.Parameter(t.to(cuda_dev)) for t in init]
    theirs = [torch.nn.Parameter(t.to(cuda_dev)) for t in init]
    fo = dsk.FusedAdagrad(ours, lr=0.1, lr_decay=1e-4, weight_decay=1e-3)
    to = torch.optim.Adagrad(theirs, lr=0.1, lr_decay=1e-4, weight_decay=1e-3, foreach=True)
    k = torch.tensor(sum_k, device=cuda_dev)
    for it in range(4):
        fo.zero_grad()
        for p, q in zip(ours, theirs):
            S = (torch.zeros(p.shape) if sum_k == 0 else _hard_gradient(p.numel(), gen).reshape(p.shape)).to(cuda_dev)
            p.grad.copy_(S)
            q.grad = S.div(k.clamp_min(1e-30))
        assert fo.allreduce(weight=k) is None and fo.collectives == 0
        fo.step()
        to.step()
        for i, (p, q) in enumerate(zip(ours, theirs)):
            assert torch.equal(p.data, q.data), (it, i)
            assert torch.isfinite(p.data).all() or sum_k != 0
        for i, (p, o) in enumerate(zip(ours, fo.offsets)):
            assert torch.equal(fo.flat_sum[o:o + p.numel()].view_as(p), to.state[theirs[i]]["sum"]), (it, i)


# ---- d. triplet loss and distance ---------------------------------------------------------------------------------
def distance_gate(x1, x2, d):
    """sqrt(sum_j (x1_j - x2_j)^2 + fp32(1e-4 / D)): the difference rounded (2u on its square), a per-lane fmaf chain
    of ceil(D/32) terms, 5 butterfly adds, the eps add, a correctly rounded sqrt.  Relative to the fp64 value:
        |dd| / d <= (ceil(D/32) + 7) u     (the sum's relative error, not halved by the sqrt, plus the sqrt's u)."""
    D = x1.shape[1]
    eps = f64(f32(1e-4 / D))
    ref = np.sqrt(((x1.astype(f64) - x2.astype(f64)) ** 2).sum(1) + eps)
    return _ratio(np.abs(d - ref), (-(-D // 32) + 7) * U * ref)


def distance_bwd_gate(x1, x2, dist, go, g1, g2):
    """g1 = go * (x1 - x2) / dist with the engine's dist pinned: three roundings, gamma(3) relative; g2 = -g1."""
    ref = go.astype(f64)[:, None] * (x1.astype(f64) - x2.astype(f64)) / dist.astype(f64)[:, None]
    return {"g1": _ratio(np.abs(g1 - ref), gamma(3) * np.abs(ref)),
            "g2": 0.0 if np.array_equal(g2, -g1) else np.inf}


def hinge_mask(d_p, d_n, margin):
    """The engine's active rows: (margin + d_p) - d_n >= 0 in fp32 (torch.clamp(min=0) passes the gradient at 0)."""
    return ((f32(margin) + d_p.astype(f32)) - d_n.astype(f32)) >= 0


def triplet_bwd_gate(a, p, n, d_p, d_n, gl, margin, ga, gp, gn):
    """With the engine's d_p, d_n and hinge mask pinned: g = fp32(gl / B) on active rows; up = g (a - p) / d_p and
    un = -g (a - n) / d_n (difference, product, quotient: 3 roundings, plus g's); ga = up + un (one more):
        |dga| <= gamma(5) (|up| + |un|),   |dgp| <= gamma(4) |up|,   |dgn| <= gamma(4) |un|."""
    B = a.shape[0]
    act = hinge_mask(d_p, d_n, margin).astype(f64)[:, None]
    g = act * float(gl) / B
    up = g * (a.astype(f64) - p.astype(f64)) / d_p.astype(f64)[:, None]
    un = -g * (a.astype(f64) - n.astype(f64)) / d_n.astype(f64)[:, None]
    return {"ga": _ratio(np.abs(ga - (up + un)), gamma(5) * (np.abs(up) + np.abs(un))),
            "gp": _ratio(np.abs(gp + up), gamma(4) * np.abs(up)),
            "gn": _ratio(np.abs(gn + un), gamma(4) * np.abs(un))}


def triplet_loss_gate(d_p, d_n, margin, loss):
    """mean_i max((margin + d_p) - d_n, 0) from the engine's distances: 2 roundings per hinge term, ceil(B/1024)
    strided adds and a 10-level tree over 1024 threads, then / B."""
    B = d_p.size
    pre = f64(margin) + d_p.astype(f64) - d_n.astype(f64)
    h = np.maximum(pre, 0.0)
    e = U * np.abs(f64(margin) + d_p.astype(f64)) * (1 + U) + U * (np.abs(pre) + U * np.abs(f64(margin) + d_p))
    bound = e.sum() / B + gamma(-(-B // 1024) + 10) * (h + e).sum() / B + U * (h.mean() + e.sum() / B)
    return _ratio(abs(float(loss) - h.mean()), bound)


def _triplet_inputs(B, D, seed):
    g = torch.Generator().manual_seed(seed)
    a, p, n = (torch.randn(B, D, generator=g) for _ in range(3))
    p[1::7] = a[1::7]                                 # rows with a = p: d_p = sqrt(eps)
    n[::11] = a[::11] + 1e-3 * torch.randn(len(range(0, B, 11)), D, generator=g)   # active hinges, row 0 among them
    return a, p, n


@pytest.mark.parametrize("B,D", [(1, 96), (1023, 513), (1024, 512), (1025, 96), (5000, 513), (1024, 96), (1, 513)])
def test_triplet_loss_and_distance_within_fp64_bound(cuda_dev, B, D):
    a, p, n = _triplet_inputs(B, D, B + D)
    ac, pc, nc = a.cuda(), p.cuda(), n.cuda()
    lib = L.load()
    dist = torch.empty(B, device="cuda")
    L.check(lib.dsk_pairwise_distance(ac.data_ptr(), pc.data_ptr(), B, D, dist.data_ptr(), L.cur_stream()))
    go = torch.randn(B, generator=torch.Generator().manual_seed(1)).cuda()
    g1, g2 = torch.empty_like(ac), torch.empty_like(ac)
    L.check(lib.dsk_pairwise_distance_bwd(ac.data_ptr(), pc.data_ptr(), dist.data_ptr(), go.data_ptr(), B, D,
                                          g1.data_ptr(), g2.data_ptr(), L.cur_stream()))
    margin = 0.5
    loss, d_p, d_n = torch.empty(1, device="cuda"), torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    L.check(lib.dsk_triplet_loss(ac.data_ptr(), pc.data_ptr(), nc.data_ptr(), B, D, margin, loss.data_ptr(),
                                 d_p.data_ptr(), d_n.data_ptr(), L.cur_stream()))
    gl = torch.tensor([1.5], device="cuda")
    ga, gp, gn = (torch.empty_like(ac) for _ in range(3))
    L.check(lib.dsk_triplet_loss_bwd(ac.data_ptr(), pc.data_ptr(), nc.data_ptr(), d_p.data_ptr(), d_n.data_ptr(),
                                     gl.data_ptr(), B, D, margin, ga.data_ptr(), gp.data_ptr(), gn.data_ptr(),
                                     L.cur_stream()))
    A, P, N = a.numpy(), p.numpy(), n.numpy()
    dn_, dp_, dist_ = d_n.cpu().numpy(), d_p.cpu().numpy(), dist.cpu().numpy()
    r = {"dist": distance_gate(A, P, dist_), "d_n": distance_gate(A, N, dn_)}
    r.update(distance_bwd_gate(A, P, dist_, go.cpu().numpy(), g1.cpu().numpy(), g2.cpu().numpy()))
    r["loss"] = triplet_loss_gate(dp_, dn_, margin, loss.item())
    r.update(triplet_bwd_gate(A, P, N, dp_, dn_, 1.5, margin, ga.cpu().numpy(), gp.cpu().numpy(), gn.cpu().numpy()))
    _report(f"triplet B={B} D={D}", r)
    assert np.array_equal(dp_, dist_)              # the same row reduction in both kernels
    assert hinge_mask(dp_, dn_, margin).any()
    # the autograd Functions return the same bits as the ABI calls
    assert torch.equal(engine.PairwiseDistanceFn.apply(ac, pc), dist)
    assert torch.equal(engine.TripletLossFn.apply(ac, pc, nc, margin).reshape(1), loss)


def hinge_edge_case(B=64, D=96, seed=3):
    """d_p, d_n crafted so that (margin + d_p) - d_n is exactly 0 in fp32 on every even row, and -1 ulp of d_n (an
    inactive row) or positive on the odd rows."""
    rng = np.random.default_rng(seed)
    a, p, n = (rng.standard_normal((B, D)).astype(f32) for _ in range(3))
    margin = f32(0.5)
    d_p = (1.0 + rng.random(B)).astype(f32)
    d_n = (margin + d_p).astype(f32)                      # (margin + d_p) - d_n == 0 exactly
    d_n[1::4] = np.nextafter(d_n[1::4], f32(np.inf))      # inactive by one ulp
    d_n[3::4] = d_n[3::4] - f32(0.25)                     # active
    assert (((margin + d_p) - d_n)[0::2] == 0).all()
    return a, p, n, d_p, d_n, float(margin)


def test_triplet_backward_passes_the_gradient_at_the_hinge(cuda_dev):
    a, p, n, d_p, d_n, margin = hinge_edge_case()
    B, D = a.shape
    t = [torch.from_numpy(v).cuda() for v in (a, p, n, d_p, d_n)]
    gl = torch.tensor([2.0], device="cuda")
    ga, gp, gn = (torch.empty_like(t[0]) for _ in range(3))
    L.check(L.load().dsk_triplet_loss_bwd(*[v.data_ptr() for v in t], gl.data_ptr(), B, D, margin, ga.data_ptr(),
                                          gp.data_ptr(), gn.data_ptr(), L.cur_stream()))
    ga, gp, gn = ga.cpu().numpy(), gp.cpu().numpy(), gn.cpu().numpy()
    _report("triplet hinge edge", triplet_bwd_gate(a, p, n, d_p, d_n, 2.0, margin, ga, gp, gn))
    assert (np.abs(ga[0::2]).max(1) > 0).all() and not ga[1::4].any()
    # the mask is torch's own rule: clamp(min=0) passes the gradient where its input is exactly 0
    pre = torch.from_numpy((f32(margin) + d_p) - d_n).requires_grad_(True)
    torch.clamp(pre, min=0.0).sum().backward()
    assert np.array_equal(pre.grad.numpy() != 0, hinge_mask(d_p, d_n, margin))


# ---- e. selection, gather, threshold sweep --------------------------------------------------------------------------
def select_reference(d_p, d_n, margin):
    """np.where(d_n - d_p < margin) in fp32 (NaN compares False)."""
    with np.errstate(invalid="ignore"):
        return np.nonzero((d_n.astype(f32) - d_p.astype(f32)) < f32(margin))[0]


def _selection_case(B, seed, margin):
    rng = np.random.default_rng(seed)
    d_p = rng.random(B).astype(f32)
    d_n = (d_p + rng.standard_normal(B).astype(f32) * f32(0.3)).astype(f32)
    if B >= 16:
        k = B // 16
        pos = rng.permutation(B)
        d_n[pos[:k]] = (d_p[pos[:k]] + f32(margin)).astype(f32)             # near or at the margin
        d_p[pos[k:2 * k]], d_n[pos[k:2 * k]] = 0.0, f32(margin)            # exactly at the margin: not selected
        d_n[pos[2 * k:3 * k]] = np.nan
        d_p[pos[3 * k:4 * k]] = rng.choice([np.inf, -np.inf, np.nan], k)
        d_n[pos[4 * k:5 * k]] = rng.choice([np.inf, -np.inf], k)
        d_p[pos[5 * k:6 * k]] = d_n[pos[5 * k:6 * k]]                        # equal distances
    return d_p, d_n


@pytest.mark.parametrize("B", [1, 1023, 1024, 1025, 100000])
@pytest.mark.parametrize("margin", [0.0, 0.1])
def test_select_hard_triplets_is_numpy_exact(cuda_dev, B, margin):
    d_p, d_n = _selection_case(B, B, margin)
    idx, cnt = dsk.select_hard_triplets(torch.from_numpy(d_p).cuda(), torch.from_numpy(d_n).cuda(), margin)
    k = int(cnt.item())
    ref = select_reference(d_p, d_n, margin)
    assert k == ref.size and np.array_equal(idx[:k].cpu().numpy(), ref)


@pytest.mark.parametrize("rows,count", [(5, 0), (37, 1), (37, 37), (300, 123)])
def test_gather_rows_is_exact(cuda_dev, rows, count):
    """Rows of 160 x 64 floats (one utterance's fbank): out[j] = src[idx[j]] for j < count, zeros after."""
    rng = np.random.default_rng(rows + count)
    src = rng.standard_normal((rows, 1, 160, 64)).astype(f32)
    src[0, 0, 0, :4] = [np.nan, np.inf, -0.0, 1e-40]
    idx = rng.integers(0, rows, rows).astype(np.int64)
    out = engine.gather_rows(torch.from_numpy(src).cuda(), torch.from_numpy(idx).cuda(),
                             torch.tensor([count], dtype=torch.int32).cuda()).cpu().numpy()
    ref = np.zeros_like(src)
    ref[:count] = src[idx[:count]]
    assert out.view(np.int32).tobytes() == ref.view(np.int32).tobytes()


def threshold_reference(d, same, th):
    """tp[t] = #{same & float64(d) < t}, fp[t] = #{!same & float64(d) < t} (np.less), by sorted search."""
    out = []
    for sel in (same, ~same):
        v = np.sort(d[sel].astype(f64))
        v = v[~np.isnan(v)]
        c = np.searchsorted(v, th, side="left").astype(np.int64)
        c[np.isnan(th)] = 0
        out.append(c)
    return out


def _threshold_case(P, nT, labels, seed):
    rng = np.random.default_rng(seed)
    d = (rng.random(P) * 30).astype(f32)
    d[P - P // 10:] = d[:P // 10]                                    # duplicated distances
    if P >= 8:
        d[:8] = [np.nan, np.inf, -np.inf, -0.0, 0.0, f32(0.1), f32(0.1), 29.999]
    th = np.arange(nT, dtype=f64) * (30.0 / nT)
    if nT >= 8:
        th[:8] = [np.nan, np.inf, -np.inf, 0.0, -0.0, f64(f32(0.1)), 0.1, f64(d[-1])]
        th[8:8 + min(nT - 8, 64)] = d[rng.integers(0, P, min(nT - 8, 64))].astype(f64)   # thresholds equal to a distance
    same = {"random": rng.random(P) < 0.3, "same": np.ones(P, bool), "different": np.zeros(P, bool)}[labels]
    return d, same, th


@pytest.mark.parametrize("P,nT", [(1, 1), (2047, 257), (2048, 256), (2049, 255), (100003, 30000), (2049, 30000),
                                  (1, 257), (100003, 1)])
@pytest.mark.parametrize("labels", ["random", "same", "different"])
def test_threshold_counts_are_numpy_exact(cuda_dev, P, nT, labels):
    d, same, th = _threshold_case(P, nT, labels, P + nT)
    tp, fp = verification.threshold_counts(torch.from_numpy(d).cuda(), torch.from_numpy(same).cuda(), th)
    rtp, rfp = threshold_reference(d, same, th)
    assert np.array_equal(tp, rtp) and np.array_equal(fp, rfp)
    if P * nT <= 2049 * 257:      # the sorted-search reference against the plain np.less counts
        below = np.less(d.astype(f64)[None, :], th[:, None])
        assert np.array_equal(rtp, (below & same).sum(1)) and np.array_equal(rfp, (below & ~same).sum(1))
