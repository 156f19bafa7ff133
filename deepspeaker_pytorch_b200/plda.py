"""A trained scoring backend: LDA and two-covariance PLDA, as in the Kaldi x-vector recipe (no reference
implementation exists; the reference scores Euclidean distances of triplet-trained embeddings).

``fit`` learns, from labelled training embeddings, the global mean, an LDA projection to ``lda_dim`` dimensions and a
two-covariance PLDA model of the length-normalised LDA outputs.  ``PLDA.transform`` takes embeddings through the
same steps into the PLDA's diagonal space, ``score_trials`` and ``score_matrix`` give log-likelihood ratios (higher =
same speaker).  ``enroll`` averages each speaker's raw embeddings, as Kaldi's ``ivector-mean`` does, and counts them:
an enrolment row of n utterances is transformed and scored with its count.

The N-sized passes run on the GPU in fp64 (class sums, the Gram on the fp64 tensor cores, the affine transforms, the
LLRs); the D x D and C x d model algebra (eigendecompositions, Cholesky, the EM iterations) runs in fp64 numpy on the
host.  ``oracle/plda_oracle.py`` states every step.

Fit memory on the device, beyond the (N, D) fp32 embeddings: the (N, d) fp32 LDA outputs, the (C, D) and (C, d)
fp64 class sums, at most 128 MiB for the transform and the Gram's split-K partials (about 1024 tiles of 32 KiB).
"""
from __future__ import annotations

import numpy as np
import torch

from . import engine
from .identification import speaker_csr

_KEYS = ("mu", "lda", "plda_mean", "plda_transform", "psi")


def _sign_fix(V):
    """Each column of V flipped so that its component of largest |.| is positive."""
    idx = np.argmax(np.abs(V), axis=0)
    s = np.sign(V[idx, np.arange(V.shape[1])])
    s[s == 0] = 1.0
    return V * s


def _eigh_desc(S):
    e, V = np.linalg.eigh(0.5 * (S + S.T))
    order = np.argsort(-e, kind="stable")
    return e[order], _sign_fix(V[:, order])


def lda_from_stats(tot, between, dim):
    """L (dim, D) from the total and between-class covariances: whiten the within-class covariance tot - between
    (eigenvalues floored at 1e-6 x the largest), then project on the leading eigenvectors of the whitened
    between-class covariance."""
    e, E = _eigh_desc(tot - between)
    e = np.maximum(e, 1e-6 * e.max())
    T = (E / np.sqrt(e)).T
    _, U = _eigh_desc(T @ between @ T.T)
    return U[:, :dim].T @ T


def diagonalise(phi_w, phi_b):
    """(P (d, d), psi (d,) descending, P^-1): P phi_w P^T = I and P phi_b P^T = diag(psi)."""
    Lc = np.linalg.cholesky(0.5 * (phi_w + phi_w.T))
    Cinv = np.linalg.inv(Lc)
    psi, V = _eigh_desc(Cinv @ phi_b @ Cinv.T)
    return V.T @ Cinv, psi, Lc @ V


def plda_em(O, means, counts, iters=10):
    """(phi_w, phi_b) after ``iters`` EM iterations of the two-covariance model from the offset scatter O (d, d), the
    class means centred on their mean (C, d) and the class sizes (C,), starting from phi_w = phi_b = I.

    Every iteration works in the basis P that diagonalises the current model (P phi_w P^T = I, P phi_b P^T =
    diag(psi)).  There a class of n utterances has the posterior covariance M = P^-1 diag(psi / (1 + n psi)) P^-T and
    the posterior mean w = P^-1 diag(n psi / (1 + n psi)) P m, so the statistics of all classes are two diagonal sums
    over the distinct class sizes and two (C, d) x (C, d) products:
      between = sum_c M_c + w_c w_c^T,  within = O + sum_c n_c (M_c + (m_c - w_c)(m_c - w_c)^T),
    divided by C and N."""
    means = np.asarray(means, dtype=np.float64)
    counts = np.asarray(counts, dtype=np.int64).reshape(-1)
    C, d = means.shape
    N = int(counts.sum())
    sizes, mult = np.unique(counts, return_counts=True)
    n = counts.astype(np.float64)[:, None]
    phi_w, phi_b = np.eye(d), np.eye(d)
    for _ in range(int(iters)):
        P, psi, Pinv = diagonalise(phi_w, phi_b)
        ns = sizes.astype(np.float64)[:, None]
        post = psi[None, :] / (1.0 + ns * psi[None, :])                    # (sizes, d): diag of M per class size
        sum_m = (mult[:, None] * post).sum(axis=0)
        sum_nm = (mult[:, None] * ns * post).sum(axis=0)
        mp = means @ P.T                                                   # P m_c
        gain = n * psi[None, :] / (1.0 + n * psi[None, :])
        q_b = mp * gain                                                    # P w_c
        q_w = mp * (1.0 - gain)                                            # P (m_c - w_c)
        between = Pinv @ (np.diag(sum_m) + q_b.T @ q_b) @ Pinv.T
        within = O + Pinv @ (np.diag(sum_nm) + q_w.T @ (n * q_w)) @ Pinv.T
        phi_w, phi_b = within / N, between / C
    return phi_w, phi_b


class PLDA:
    """A fitted LDA + PLDA backend.  Attributes are fp64 CPU tensors: ``mu`` (D,), ``lda`` (d, D), ``plda_mean``
    (d,), ``plda_transform`` (d, d) and ``psi`` (d,) (descending); the device copies are made on first use."""

    def __init__(self, mu, lda, plda_mean, plda_transform, psi):
        vals = [torch.as_tensor(v).detach().cpu().to(torch.float64).contiguous() for v in
                (mu, lda, plda_mean, plda_transform, psi)]
        self.mu, self.lda, self.plda_mean, self.plda_transform, self.psi = vals
        d, D = self.lda.shape
        if (self.mu.shape != (D,) or self.plda_mean.shape != (d,) or self.plda_transform.shape != (d, d)
                or self.psi.shape != (d,)):
            raise ValueError("PLDA: inconsistent shapes " + str({k: tuple(v.shape) for k, v in zip(_KEYS, vals)}))
        self._dev = {}

    @property
    def dim(self) -> int:
        return self.lda.shape[0]

    def state_dict(self) -> dict:
        return {k: getattr(self, k).clone() for k in _KEYS}

    @classmethod
    def from_state_dict(cls, sd):
        missing = [k for k in _KEYS if k not in sd]
        if missing:
            raise ValueError(f"PLDA.from_state_dict: missing {missing}")
        return cls(*(sd[k] for k in _KEYS))

    def _on(self, device):
        if device not in self._dev:
            self._dev[device] = {k: getattr(self, k).to(device) for k in _KEYS}
        return self._dev[device]

    def transform(self, emb, counts=None):
        """(U, d) fp32 on emb's device: subtract the mean, LDA, length-normalise to sqrt(d), then the PLDA transform
        with its scoring normalisation.  ``counts`` (U,): the utterances averaged into each row (``enroll``), None for
        single utterances."""
        if not isinstance(emb, torch.Tensor) or not emb.is_cuda:
            raise RuntimeError("PLDA.transform needs a CUDA embedding tensor; there is no CPU fallback")
        m = self._on(emb.device)
        y = engine.affine_norm_f64(emb, m["lda"], m["mu"], mode="length")
        return engine.affine_norm_f64(y, m["plda_transform"], m["plda_mean"], mode="plda", psi=m["psi"], counts=counts)

    def score_trials(self, Y, trials, counts=None):
        """(T,) fp32 LLRs of trials (T, 2) (enrolment, test) of row indices into the transformed rows Y; ``counts`` as
        given to ``transform`` (the enrolment side's; the test side is one utterance).  A bad index or count gives
        NaN."""
        return engine.plda_score_trials(Y, self._on(Y.device)["psi"], trials, counts)

    def score_matrix(self, Ya, Yb):
        """(M, N) fp32 LLRs of every transformed row of Ya against every transformed row of Yb (single utterances)."""
        return engine.plda_score_matrix(Ya, Yb, self._on(Ya.device)["psi"])


def enroll(emb, labels):
    """(means (S, D) fp32 on emb's device, counts (S,) int64 CPU tensor, speaker ids np.ndarray (S,) ascending): each
    speaker's mean of RAW embeddings (summed in fp64 in utterance order, divided by the count, rounded once).  Transform
    with ``be.transform(means, counts)`` and score with the same counts."""
    if not isinstance(emb, torch.Tensor) or not emb.is_cuda:
        raise RuntimeError("enroll needs a CUDA embedding tensor; there is no CPU fallback")
    if isinstance(labels, torch.Tensor) and labels.is_cuda:
        raise RuntimeError("enroll: labels must be CPU labels")
    order, offsets, ids = speaker_csr(labels)
    if order.size != emb.shape[0]:
        raise ValueError(f"enroll: {order.size} labels for {emb.shape[0]} embeddings")
    counts = torch.from_numpy(np.diff(offsets))
    sums = engine.class_sums_f64(emb, torch.from_numpy(order).to(emb.device), torch.from_numpy(offsets).to(emb.device))
    return (sums / counts.to(emb.device, torch.float64)[:, None]).float(), counts, ids


def _host(t, what):
    a = t.cpu().numpy()
    if not np.isfinite(a).all():
        raise ValueError(f"fit: {what} are not finite")
    return a


def fit(emb, labels, lda_dim: int = 200, iters: int = 10) -> PLDA:
    """Fit the backend on training embeddings ``emb`` (N, D) (a CUDA tensor) with CPU ``labels`` (N,).

    Device passes: the class sums (-> the global mean mu); the Gram and class sums of x - mu (-> the total and
    between-class covariances, LDA on the host); the LDA transform with length normalisation; the Gram and class sums
    of its outputs (-> the class means and the within-class scatter, PLDA EM on the host).  ValueError with fewer than
    2 classes, no class of 2 or more utterances, lda_dim outside [1, min(D, C - 1)], or a statistic that is not
    finite (checked on the host copies the algebra reads anyway)."""
    if not isinstance(emb, torch.Tensor) or not emb.is_cuda:
        raise RuntimeError("plda.fit needs a CUDA embedding tensor; there is no CPU fallback")
    if emb.dim() != 2:
        raise ValueError(f"fit: expected (N, D) embeddings, got shape {tuple(emb.shape)}")
    if isinstance(labels, torch.Tensor) and labels.is_cuda:
        raise RuntimeError("fit: labels must be CPU labels")
    order, offsets, _ = speaker_csr(labels)
    N, D = emb.shape
    if order.size != N:
        raise ValueError(f"fit: {order.size} labels for {N} embeddings")
    counts = np.diff(offsets)
    C = counts.size
    if C < 2:
        raise ValueError(f"fit: need at least 2 classes, got {C}")
    if counts.max() < 2:
        raise ValueError("fit: need a class with 2 or more utterances (the within-class covariance is not defined)")
    if not 1 <= int(lda_dim) <= min(D, C - 1):
        raise ValueError(f"fit: lda_dim must lie in [1, min(D, C - 1)] = [1, {min(D, C - 1)}], got {lda_dim}")
    if int(iters) < 0:
        raise ValueError(f"fit: iters must be >= 0, got {iters}")
    d = int(lda_dim)
    X = emb.detach().float().contiguous()
    dev = X.device
    order_d, offsets_d = torch.from_numpy(order).to(dev), torch.from_numpy(offsets).to(dev)
    # passes 1 and 2: mean, Gram and class sums of x - mu
    mu = engine.class_sums_f64(X, order_d, offsets_d).sum(dim=0) / N
    G = engine.gram_f64(X, mu)
    s = engine.class_sums_f64(X, order_d, offsets_d, mu)
    mu_h = _host(mu, "the embedding mean (a NaN or infinite training embedding)")
    G_h = _host(G, "the embedding covariance (a NaN or infinite training embedding)")
    s_h = _host(s, "the class sums (a NaN or infinite training embedding)")
    between = s_h.T @ (s_h / counts[:, None]) / N
    lda = lda_from_stats(G_h / N, between, d)
    if not np.isfinite(lda).all():
        raise ValueError("fit: the LDA transform is not finite (degenerate covariances)")
    # passes 3 and 4: length-normalised LDA outputs, their Gram and class sums
    Y = engine.affine_norm_f64(X, torch.from_numpy(lda).to(dev), mu, mode="length")
    Gy = _host(engine.gram_f64(Y), "the LDA outputs' scatter (an LDA output of zero norm)")
    sy = _host(engine.class_sums_f64(Y, order_d, offsets_d), "the LDA outputs' class sums (an LDA output of zero norm)")
    means = sy / counts[:, None]
    O = Gy - sy.T @ means
    mbar = means.mean(axis=0)
    phi_w, phi_b = plda_em(O, means - mbar, counts, iters)
    if not (np.isfinite(phi_w).all() and np.isfinite(phi_b).all()):
        raise ValueError("fit: the PLDA covariances are not finite")
    P, psi, _ = diagonalise(phi_w, phi_b)
    return PLDA(mu_h, lda, mbar, P, psi)
