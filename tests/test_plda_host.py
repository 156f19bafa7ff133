"""PLDA backend on the host (no GPU): the fp64 oracle against independent formulations (scipy's generalised
eigenproblem for LDA, the full-Gaussian two-covariance LLR), the library's batched EM against the oracle's class-by-class
EM, recovery of a known two-covariance model, and fit's argument errors."""
import numpy as np
import pytest
import scipy.linalg
import torch
from scipy.stats import multivariate_normal

from deepspeaker_pytorch_b200 import plda as P
from oracle import plda_oracle as O


def _labelled(rng, sizes, D, between=2.0, within=1.0):
    """Rows of len(sizes) classes (class c has sizes[c] rows): centre ~ N(0, between^2 I) + anisotropic noise."""
    lab = np.repeat(np.arange(len(sizes)), sizes)
    centres = rng.normal(size=(len(sizes), D)) * between
    scale = within * np.linspace(0.3, 1.5, D)
    X = centres[lab] + rng.normal(size=(lab.size, D)) * scale
    return X, lab


def _random_spd(rng, d, lo, hi):
    Q, _ = np.linalg.qr(rng.normal(size=(d, d)))
    return Q @ np.diag(np.linspace(lo, hi, d)) @ Q.T


def test_lda_oracle_matches_generalised_eigenproblem():
    rng = np.random.default_rng(0)
    X, lab = _labelled(rng, rng.integers(3, 12, size=40), 24)
    dim = 10
    _, _, b, w = O.lda_stats(X, lab)
    mu, L, lam = O.lda(X, lab, dim)
    ev, V = scipy.linalg.eigh(b, w)                       # b v = lambda w v, v^T w v = 1, ascending
    ev, V = ev[::-1], V[:, ::-1]
    assert np.all(np.diff(ev[:dim + 1]) < -1e-6), "the test needs distinct leading eigenvalues"
    np.testing.assert_allclose(lam[:dim], ev[:dim], rtol=1e-10, atol=1e-12)
    # the same vectors up to sign: rows of L are the generalised eigenvectors (both are w-orthonormal)
    Vs = O.sign_fix(V[:, :dim])
    Ls = O.sign_fix(L.T)
    np.testing.assert_allclose(Ls, Vs, rtol=0, atol=1e-10 * np.abs(Vs).max())
    np.testing.assert_allclose(L @ w @ L.T, np.eye(dim), atol=1e-10)


def test_diagonal_llr_equals_full_gaussian_form():
    rng = np.random.default_rng(1)
    d = 6
    B, W = _random_spd(rng, d, 0.5, 4.0), _random_spd(rng, d, 0.2, 1.5)
    Pm, psi = O.plda_diagonalise(W, B)
    np.testing.assert_allclose(Pm @ W @ Pm.T, np.eye(d), atol=1e-12)
    np.testing.assert_allclose(Pm @ B @ Pm.T, np.diag(psi), atol=1e-12)
    mean = rng.normal(size=d)
    model = {"plda_mean": mean, "plda_transform": Pm, "psi": psi}
    Y = mean + rng.normal(size=(8, d)) * 1.5
    T = O.plda_transform(model, Y, _normalize=False)
    joint = np.block([[B + W, B], [B, B + W]])
    worst = 0.0
    for i in range(4):
        for j in range(4, 8):
            u, v = Y[i] - mean, Y[j] - mean
            full = (multivariate_normal(np.zeros(2 * d), joint).logpdf(np.concatenate([u, v]))
                    - multivariate_normal(np.zeros(d), B + W).logpdf(u) - multivariate_normal(np.zeros(d), B + W).logpdf(v))
            diag = O.llr(psi, T[i], T[j])
            worst = max(worst, abs(diag - full) / (1 + abs(full)))
    print(f"diagonal vs full-Gaussian LLR: max rel err {worst:.2e}")
    assert worst < 1e-9


@pytest.mark.parametrize("sizes", [
    [5] * 30,                                             # one class size
    list(range(2, 32)),                                   # every size unique
    [2] * 10 + [7] * 5 + [3, 11, 40] + [1] * 4,           # repeated and unique sizes, singletons
])
def test_batched_em_equals_class_by_class_em(sizes):
    rng = np.random.default_rng(len(sizes))
    d = 8
    Y, lab = _labelled(rng, sizes, d, between=1.5, within=0.8)
    Pw_o, Pb_o, mbar = O.plda_em(Y, lab, iters=10)
    _, means, counts, Osc, _ = O.plda_stats(Y, lab)
    Pw, Pb = P.plda_em(Osc, means - mbar, counts, iters=10)
    for got, want, name in ((Pw, Pw_o, "phi_w"), (Pb, Pb_o, "phi_b")):
        rel = np.abs(got - want).max() / np.abs(want).max()
        print(f"{name}: rel {rel:.2e}")
        assert rel < 1e-10, name
    psi = P.diagonalise(Pw, Pb)[1]
    psi_o = O.plda_diagonalise(Pw_o, Pb_o)[1]
    np.testing.assert_allclose(psi, psi_o, rtol=1e-10)


def test_em_recovers_a_known_two_covariance_model():
    rng = np.random.default_rng(7)
    d, C, n = 6, 2000, 100                                # N = 200 000
    B, W = _random_spd(rng, d, 0.5, 3.0), _random_spd(rng, d, 0.2, 1.0)
    cls = rng.multivariate_normal(np.zeros(d), B, size=C)
    lab = np.repeat(np.arange(C), n)
    Y = cls[lab] + rng.multivariate_normal(np.zeros(d), W, size=C * n)
    _, means, counts, Osc, _ = O.plda_stats(Y, lab)
    Pw, Pb = P.plda_em(Osc, means - means.mean(axis=0), counts, iters=20)
    # statistical tolerance: phi_b rests on C = 2000 class means (relative sd about sqrt(2 / C) = 3 % per entry), phi_w
    # on N - C = 198 000 degrees of freedom (about 0.3 %); 3 to 4 standard deviations in the Frobenius norm
    eb = np.linalg.norm(Pb - B) / np.linalg.norm(B)
    ew = np.linalg.norm(Pw - W) / np.linalg.norm(W)
    print(f"recovery: phi_b rel Frobenius {eb:.3f}, phi_w {ew:.4f}")
    assert eb < 0.1 and ew < 0.015


def test_batched_lda_from_stats_matches_oracle():
    rng = np.random.default_rng(3)
    X, lab = _labelled(rng, rng.integers(2, 9, size=50), 32)
    _, tot, b, _ = O.lda_stats(X, lab)
    np.testing.assert_allclose(P.lda_from_stats(tot, b, 12), O.lda(X, lab, 12)[1], rtol=0, atol=1e-9)


def test_state_dict_round_trip():
    rng = np.random.default_rng(4)
    sd = {"mu": rng.normal(size=16), "lda": rng.normal(size=(4, 16)), "plda_mean": rng.normal(size=4),
          "plda_transform": rng.normal(size=(4, 4)), "psi": np.sort(rng.random(4))[::-1].copy()}
    be = P.PLDA.from_state_dict(sd)
    out = be.state_dict()
    assert set(out) == set(sd)
    for k in sd:
        assert out[k].dtype == torch.float64 and out[k].device.type == "cpu"
        np.testing.assert_array_equal(out[k].numpy(), sd[k])
    with pytest.raises(ValueError):
        P.PLDA.from_state_dict({k: v for k, v in sd.items() if k != "psi"})
    with pytest.raises(ValueError):
        P.PLDA.from_state_dict(dict(sd, psi=np.ones(5)))


class _FakeCuda(torch.Tensor):
    """A CPU tensor that claims to live on the GPU, so that fit's argument checks run without a device."""
    @property
    def is_cuda(self):
        return True


def test_fit_argument_errors():
    X = torch.zeros(12, 8).as_subclass(_FakeCuda)
    with pytest.raises(RuntimeError):
        P.fit(torch.zeros(12, 8), np.zeros(12))                              # not a CUDA tensor
    with pytest.raises(ValueError, match="2 classes"):
        P.fit(X, np.zeros(12), lda_dim=1)
    with pytest.raises(ValueError, match="2 or more"):
        P.fit(X, np.arange(12), lda_dim=1)
    with pytest.raises(ValueError, match="lda_dim"):
        P.fit(X, np.repeat(np.arange(3), 4), lda_dim=3)                     # C - 1 = 2
    with pytest.raises(ValueError, match="lda_dim"):
        P.fit(X, np.repeat(np.arange(3), 4), lda_dim=0)
    with pytest.raises(ValueError, match="lda_dim"):
        P.fit(torch.zeros(12, 2).as_subclass(_FakeCuda), np.arange(12) % 6, lda_dim=3)   # D = 2
    with pytest.raises(ValueError, match="labels"):
        P.fit(X, np.zeros(11), lda_dim=1)
