"""fp64 restatement of the PLDA backend (LDA, length normalisation, two-covariance PLDA, LLR scoring) — TEST
INFRASTRUCTURE ONLY (the product never imports this module).

No reference implementation exists: this restates Kaldi's published algorithms in numpy, class by class and row by
row.  x_u are embeddings (D), C classes of n_c utterances, N = sum n_c; every statistic is fp64.

1. mu = (1/N) sum_u x_u.
2. LDA (``ivector-compute-lda --total-covariance-factor=0``, ``ComputeLdaTransform``): Sigma_tot = (1/N) sum_u
   (x_u - mu)(x_u - mu)^T, Sigma_b = (1/N) sum_c s_c s_c^T / n_c with s_c = sum_{u in c} (x_u - mu), Sigma_w =
   Sigma_tot - Sigma_b.  T = diag(e^-1/2) E^T from the eigendecomposition Sigma_w = E diag(e) E^T, e floored at 1e-6 x
   the largest (T Sigma_w T^T = I); U the eigenvectors of T Sigma_b T^T by descending eigenvalue; L = U[:, :d]^T T.
3. ``ivector-normalize-length``: y_u = sqrt(d) z_u / ||z_u||, z_u = L (x_u - mu).
4. ``PldaEstimator`` (10 EM iterations by default) on y with the same labels: class means m_c, offset scatter O =
   sum_c sum_{u in c} (y_u - m_c)(y_u - m_c)^T, m_bar = the mean of the class means, Phi_w = Phi_b = I; per
   iteration, within = O (count N - C), between = 0 (count 0), and for every class M = (Phi_b^-1 + n_c Phi_w^-1)^-1,
   m = m_c - m_bar, w = M n_c Phi_w^-1 m: between += M + w w^T, within += n_c (M + (m - w)(m - w)^T), each count + 1;
   Phi_w = within / count, Phi_b = between / count.  Then C = chol(Phi_w)^-1, C Phi_b C^T = V diag(psi) V^T (psi
   descending), P = V^T C (d x d).
   Sign convention of every eigendecomposition (E, U, V): each eigenvector's component of largest |.| is positive.
5. ``PLDA::TransformIvector`` (normalize_length, not simple_length_norm): t = P (y - m_bar), then t *= sqrt(d /
   sum_i t_i^2 / (psi_i + 1/n)), n the utterances averaged into the row (an enrolment row is the mean of the speaker's
   RAW embeddings, as ``ivector-mean`` takes it, carried through steps 1-5).
6. ``PLDA::LogLikelihoodRatio``: log N(t; a o e, diag(1 + psi / (n psi + 1))) - log N(t; 0, diag(1 + psi)),
   a = n psi / (n psi + 1), the test side always n = 1.

Parity with Kaldi itself is not pinned (Kaldi is not a dependency of the project).
"""
import numpy as np


def _f64(X):
    try:
        import torch

        if isinstance(X, torch.Tensor):
            return X.detach().cpu().double().numpy()
    except ImportError:
        pass
    return np.asarray(X, dtype=np.float64)


def sign_fix(V):
    """Columns of V flipped so that each column's component of largest |.| is positive (first such on a tie)."""
    V = np.array(V, dtype=np.float64)
    idx = np.argmax(np.abs(V), axis=0)
    s = np.sign(V[idx, np.arange(V.shape[1])])
    s[s == 0] = 1.0
    return V * s


def eigh_desc(S):
    """(eigenvalues descending, eigenvectors as columns, sign-fixed) of the symmetric S."""
    e, V = np.linalg.eigh(S)
    order = np.argsort(-e, kind="stable")
    return e[order], sign_fix(V[:, order])


def lda_stats(X, labels):
    """(mu, Sigma_tot, Sigma_b, Sigma_w) of step 2, class by class."""
    X = _f64(X)
    lab = np.asarray(labels).reshape(-1)
    N = X.shape[0]
    mu = X.mean(axis=0)
    Xc = X - mu
    tot = Xc.T @ Xc / N
    b = np.zeros_like(tot)
    for c in np.unique(lab):
        s = Xc[lab == c].sum(axis=0)
        b += np.outer(s, s) / np.count_nonzero(lab == c)
    b /= N
    return mu, tot, b, tot - b


def lda(X, labels, dim):
    """(mu (D,), L (dim, D), eigenvalues of T Sigma_b T^T descending (D,))."""
    mu, _, b, w = lda_stats(X, labels)
    e, E = eigh_desc(w)
    e = np.maximum(e, 1e-6 * e.max())
    T = (E / np.sqrt(e)).T
    lam, U = eigh_desc(T @ b @ T.T)
    return mu, U[:, :dim].T @ T, lam


def length_norm(Z):
    Z = _f64(Z)
    return np.sqrt(Z.shape[1]) * Z / np.linalg.norm(Z, axis=1, keepdims=True)


def plda_stats(Y, labels):
    """(class ids, class means (C, d), counts (C,), offset scatter O, m_bar)."""
    Y = _f64(Y)
    lab = np.asarray(labels).reshape(-1)
    ids = np.unique(lab)
    means, counts = [], []
    O = np.zeros((Y.shape[1], Y.shape[1]))
    for c in ids:
        Yc = Y[lab == c]
        m = Yc.mean(axis=0)
        O += (Yc - m).T @ (Yc - m)
        means.append(m)
        counts.append(Yc.shape[0])
    means = np.array(means)
    return ids, means, np.array(counts), O, means.mean(axis=0)


def plda_em(Y, labels, iters=10):
    """(Phi_w, Phi_b, m_bar) after ``iters`` EM iterations of step 4, class by class."""
    _, means, counts, O, mbar = plda_stats(Y, labels)
    d = means.shape[1]
    N, C = int(counts.sum()), means.shape[0]
    Pw, Pb = np.eye(d), np.eye(d)
    for _ in range(iters):
        within, wc = O.copy(), float(N - C)
        between, bc = np.zeros((d, d)), 0.0
        Wi, Bi = np.linalg.inv(Pw), np.linalg.inv(Pb)
        for mc, n in zip(means, counts):
            M = np.linalg.inv(Bi + n * Wi)
            m = mc - mbar
            w = M @ (n * Wi @ m)
            between += M + np.outer(w, w)
            bc += 1.0
            within += n * (M + np.outer(m - w, m - w))
            wc += 1.0
        Pw, Pb = within / wc, between / bc
    return Pw, Pb, mbar


def plda_diagonalise(Pw, Pb):
    """(P (d, d), psi (d,) descending): P Phi_w P^T = I, P Phi_b P^T = diag(psi)."""
    Cinv = np.linalg.inv(np.linalg.cholesky(Pw))
    psi, V = eigh_desc(Cinv @ Pb @ Cinv.T)
    return V.T @ Cinv, psi


def fit(X, labels, lda_dim=200, iters=10):
    """The fitted model as a dict of fp64 arrays: mu, lda, plda_mean, plda_transform, psi (and Phi_w, Phi_b)."""
    mu, L, _ = lda(X, labels, lda_dim)
    Y = length_norm((_f64(X) - mu) @ L.T)
    Pw, Pb, mbar = plda_em(Y, labels, iters)
    P, psi = plda_diagonalise(Pw, Pb)
    return {"mu": mu, "lda": L, "plda_mean": mbar, "plda_transform": P, "psi": psi, "phi_w": Pw, "phi_b": Pb}


def plda_transform(model, Y, counts=None, _normalize=True):
    """Step 5 on already length-normalised LDA outputs Y (rows).  ``_normalize=False`` skips the scoring
    normalisation (t = P (y - m_bar) only): a switch of this oracle for testing the LLR, not a library option."""
    Y = _f64(Y)
    t = (Y - model["plda_mean"]) @ model["plda_transform"].T
    if not _normalize:
        return t
    n = np.ones(Y.shape[0]) if counts is None else np.asarray(counts, dtype=np.float64).reshape(-1)
    dot = (t * t / (model["psi"][None, :] + 1.0 / n[:, None])).sum(axis=1)
    return t * np.sqrt(Y.shape[1] / dot)[:, None]


def transform(model, X, counts=None):
    """Steps 1-5 of raw embeddings X (rows): (U, d) fp64."""
    y = length_norm((_f64(X) - model["mu"]) @ model["lda"].T)
    return plda_transform(model, y, counts)


def llr(psi, e, t, n=1):
    """Step 6 for one enrolment row e (n utterances) and one test row t, as Kaldi's LogLikelihoodRatio computes it."""
    psi, e, t = (np.asarray(v, dtype=np.float64) for v in (psi, e, t))
    mean = n * psi / (n * psi + 1.0) * e
    var = 1.0 + psi / (n * psi + 1.0)
    given = -0.5 * (np.log(var).sum() + psi.size * np.log(2 * np.pi) + ((t - mean) ** 2 / var).sum())
    var0 = 1.0 + psi
    without = -0.5 * (np.log(var0).sum() + psi.size * np.log(2 * np.pi) + (t ** 2 / var0).sum())
    return given - without


def score_trials(psi, Y, trials, counts=None):
    """(T,) fp64 LLRs of trials (T, 2) (enrolment, test) into the transformed rows Y."""
    Y = _f64(Y)
    tr = np.asarray(trials, dtype=np.int64).reshape(-1, 2)
    n = np.ones(Y.shape[0]) if counts is None else np.asarray(counts, dtype=np.float64).reshape(-1)
    return np.array([llr(psi, Y[e], Y[t], n[e]) for e, t in tr])


def score_matrix(psi, Ya, Yb):
    """(M, N) fp64 n = 1 LLRs of every row of Ya against every row of Yb."""
    Ya, Yb = _f64(Ya), _f64(Yb)
    return np.array([[llr(psi, a, b) for b in Yb] for a in Ya])
