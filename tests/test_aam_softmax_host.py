"""AAM-softmax without a GPU: the fp64 oracle's explicit gradients against torch autograd of the textbook formula, and
an emulation of the arithmetic of the op's cosine GEMM (fp16 hi/lo operand halves concatenated along K, fp32
accumulation)."""
import numpy as np
import torch

from oracle import aam_softmax_oracle as A


def _case(N, C, D, seed, norm=10.0):
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(N, D, generator=g, dtype=torch.float64)
    E = norm * E / E.norm(dim=1, keepdim=True)
    W = torch.randn(C, D, generator=g, dtype=torch.float64) * 0.05
    return E, W, torch.randint(0, C, (N,), generator=g)


def _autograd(E, W, labels, m, s):
    Ed, Wd = E.clone().requires_grad_(True), W.clone().requires_grad_(True)
    loss = A.loss_autograd(Ed, Wd, labels, m, s)
    loss.backward()
    return loss.detach(), Ed.grad, Wd.grad


def test_oracle_gradients_equal_autograd():
    for m in (0.0, 0.2, 0.5):
        for s in (30.0, 64.0):
            E, W, labels = _case(48, 37, 64, seed=int(100 * m + s))
            wy = W[labels[:6]] / W[labels[:6]].norm(dim=1, keepdim=True)   # rows near the negated class centre
            E[:6] = -10.0 * wy + 0.1 * torch.randn(6, 64, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
            loss, gE_ref, gW_ref = _autograd(E, W, labels, m, s)
            oloss, cos, _ = A.forward(E, W, labels, m, s)
            gE, gW = A.backward(E, W, labels, m, s)
            if m > 0:                                       # the cos - mm branch is exercised
                assert bool((cos[torch.arange(6), labels[:6]] < A._consts(m)[2]).all())
            assert abs(float(oloss - loss)) <= 1e-12 * max(1.0, float(loss))
            assert float((gE - gE_ref).abs().max()) <= 1e-12 * float(gE_ref.abs().max())
            assert float((gW - gW_ref).abs().max()) <= 1e-12 * float(gW_ref.abs().max())


def test_oracle_gradient_at_sin_zero_is_finite_and_uses_cos_m():
    """A row exactly on its class centre: autograd of the textbook formula gives NaN there (sqrt at 0); the oracle's
    gradient is finite and equals autograd of the same loss whose phi has slope cos m at sin = 0."""
    m, s = 0.5, 30.0
    E, W, labels = _case(16, 9, 64, seed=7)
    u = torch.zeros(64, dtype=torch.float64)
    u[5] = 1.0
    W[labels[0]] = 0.3 * u
    E[0] = 10.0 * u                                         # cos = 1 exactly
    _, gE_nan, _ = _autograd(E, W, labels, m, s)
    assert not bool(torch.isfinite(gE_nan).all())
    gE, gW = A.backward(E, W, labels, m, s)
    assert bool(torch.isfinite(gE).all()) and bool(torch.isfinite(gW).all())

    cos_m, sin_m, th, mm = A._consts(m)

    def phi_rule(c):                                        # same values; derivative cos m where sin = 0
        x = torch.clamp(1.0 - c * c, 0.0, 1.0)
        sn = torch.sqrt(torch.where(x > 0, x, torch.ones_like(x))) * (x > 0)
        return torch.where(c > th, c * cos_m - sn * sin_m, c - mm)

    Ed, Wd = E.clone().requires_grad_(True), W.clone().requires_grad_(True)
    cos = torch.nn.functional.normalize(Ed) @ torch.nn.functional.normalize(Wd).T
    onehot = torch.nn.functional.one_hot(labels, 9).bool()
    torch.nn.functional.cross_entropy(s * torch.where(onehot, phi_rule(cos), cos), labels).backward()
    assert float((gE - Ed.grad).abs().max()) <= 1e-12 * float(Ed.grad.abs().max())
    assert float((gW - Wd.grad).abs().max()) <= 1e-12 * float(Wd.grad.abs().max())


def _f16(a):
    return a.astype(np.float16).astype(np.float64)


def _split(x32):
    hi = _f16(x32)
    return hi, _f16((x32.astype(np.float64) - hi).astype(np.float32))


def _gemm_fp32_acc(Aop, Bop, k_step=16):
    """A (N, K) B (C, K)^T with each 16-wide K step's products summed exactly and added to an fp32 accumulator."""
    acc = np.zeros((Aop.shape[0], Bop.shape[0]), np.float32)
    for k0 in range(0, Aop.shape[1], k_step):
        acc = (acc.astype(np.float64) + Aop[:, k0:k0 + k_step] @ Bop[:, k0:k0 + k_step].T).astype(np.float32)
    return acc.astype(np.float64)


def test_cosine_gemm_split_operand_arithmetic():
    """The cosine GEMM's operands are fp16 halves of the fp32 unit vectors, laid out [e_lo | e_hi | e_hi] against
    [w_hi | w_lo | w_hi] (K = 3D, lo-products first).  With fp32 accumulation that keeps max |dcos| <= 1e-6 against
    fp64; one fp16 pass does not."""
    rng = np.random.default_rng(0)
    N, C, D = 256, 1211, 512

    def unit(n):
        x = rng.standard_normal((n, D)).astype(np.float32)
        return x / np.sqrt((x.astype(np.float32) ** 2).sum(1, dtype=np.float32))[:, None]

    e, w = unit(N), unit(C)
    ref = e.astype(np.float64) @ w.astype(np.float64).T
    eh, el = _split(e)
    wh, wl = _split(w)
    got = _gemm_fp32_acc(np.concatenate([el, eh, eh], 1), np.concatenate([wh, wl, wh], 1))
    err = np.abs(got - ref).max()
    one_pass = np.abs(_gemm_fp32_acc(eh, wh) - ref).max()
    print(f"\nmax |dcos|: hi/lo lo-first {err:.2e}, one fp16 pass {one_pass:.2e}")
    assert err <= 1e-6
    assert one_pass > 1e-6
