"""fp64 restatement of VBx, Bayesian HMM clustering of x-vector sequences — TEST INFRASTRUCTURE ONLY (the product
never imports this module).

No reference implementation exists: this follows the equations of Landini, Profant, Diez and Burget, "Bayesian HMM
clustering of x-vector sequences (VBx) in speaker diarization", Computer Speech & Language 2022.  Parity with BUT's
published VBx code is not pinned (it is not available to the project).

One recording: X (W, d) rows in the PLDA space, x_t = P (y_t - m_bar) without the scoring normalisation (within-speaker
covariance I, across-speaker covariance diag(Phi), Phi = psi), S speakers, the factors Fa, Fb, loop_p.

Once:
  G_t = -(|x_t|^2 + d ln 2 pi) / 2,  rho_t = x_t o sqrt(Phi),
  gamma^0 = the row softmax of init_smoothing one_hot(init_labels),  pi^0 = 1 / S.
Iteration i = 0, 1, ...:
  N_s = sum_t gamma_ts,
  invL_s = 1 / (1 + (Fa / Fb) N_s Phi)                                  (element-wise over d),
  alpha_s = (Fa / Fb) invL_s o sum_t gamma_ts rho_t,
  ln p_ts = Fa (rho_t . alpha_s - sum_l Phi_l (invL_sl + alpha_sl^2) / 2 + G_t),
  forward-backward in the log domain with the FULL S x S transition matrix A = loop_p I + (1 - loop_p) 1 pi^T and the
  initial distribution pi: ln a_0 = ln pi + ln p_0, ln a_t = ln p_t + logsumexp_i(ln a_{t-1,i} + ln A_i.),
  ln b_{W-1} = 0, ln b_t = logsumexp_j(ln A_.j + ln p_{t+1,j} + ln b_{t+1,j}), ln p(X) = logsumexp(ln a_{W-1}),
  gamma = exp(ln a + ln b - ln p(X)) (computed with messages normalised per window, see forward_backward),
  ELBO_i = ln p(X) + (Fb / 2) sum_s sum_l (ln invL_sl - invL_sl - alpha_sl^2 + 1),
  pi_s <- gamma_0s + (1 - loop_p) pi_s sum_{t>=1} exp(logsumexp(ln a_{t-1}) + ln p_ts + ln b_ts - ln p(X)), normalised
  to sum 1 (the second term is the expected number of switches into s; each summand is taken as
  exp(ln(1 - loop_p) + ln pi_s + ...), which is the same number, and the term is 0 at loop_p = 1, where there are no
  switches).
  Stop after iteration i when i >= 1 and ELBO_i - ELBO_{i-1} < epsilon, or when i + 1 = max_iters.
Output: gamma and pi as the last iteration left them (pi after its update), the ELBO history, the iterations run, and
labels = the argmax of each gamma row (ties to the lower speaker).
"""
import numpy as np
from scipy.special import logsumexp, softmax


def _f64(X):
    try:
        import torch

        if isinstance(X, torch.Tensor):
            return X.detach().cpu().double().numpy()
    except ImportError:
        pass
    return np.asarray(X, dtype=np.float64)


def log_transitions(pi, loop_p):
    """ln A (S, S), A = loop_p I + (1 - loop_p) 1 pi^T (ln 0 = -inf)."""
    A = loop_p * np.eye(pi.size) + (1.0 - loop_p) * np.asarray(pi, np.float64)[None, :]
    with np.errstate(divide="ignore"):
        return np.log(A)


def forward_backward(lnp, pi, loop_p):
    """The full-matrix forward-backward of emissions lnp (W, S) -> (gamma (W, S), ln p(X), ln a (W, S), ln b (W, S),
    switch (S,) = (1 - loop_p) pi_s sum_{t>=1} exp(logsumexp(ln a_{t-1}) + ln p_ts + ln b_ts - ln p(X))).

    The messages are normalised at every window: ln a_t here is ln alpha-hat_t - ln c_1..t and ln b_t is ln beta-hat_t
    - ln c_t+1..W-1, with ln c_t = logsumexp of the unnormalised ln a_t, so ln p(X) = sum_t ln c_t.  That is the same
    recursion (each step is still the full S x S logsumexp); it only keeps magnitudes of order ln p(X), which reach 10^6
    on long recordings, out of the exponentials, where their rounding would cost gamma about 1e-9 ln p(X)."""
    lnp = np.asarray(lnp, np.float64)
    pi = np.asarray(pi, np.float64)
    W, S = lnp.shape
    lnA = log_transitions(pi, loop_p)
    with np.errstate(divide="ignore"):
        lpi = np.log(pi)
    la = np.empty((W, S))
    lb = np.zeros((W, S))
    lc = np.empty(W)
    for t in range(W):
        x = lpi + lnp[0] if t == 0 else lnp[t] + logsumexp(la[t - 1][:, None] + lnA, axis=0)
        lc[t] = logsumexp(x)
        la[t] = x - lc[t]
    for t in range(W - 2, -1, -1):
        lb[t] = logsumexp(lnA + (lnp[t + 1] + lb[t + 1])[None, :], axis=1) - lc[t + 1]
    lpx = lc.sum()
    gamma = np.exp(la + lb)
    if loop_p == 1.0 or W == 1:
        switch = np.zeros(S)
    else:
        with np.errstate(divide="ignore"):
            lsw = np.log(1.0 - loop_p) + lpi
        # logsumexp(ln alpha-hat_{t-1}) + ln beta-hat_t - ln p(X) = ln b_t - ln c_t in the normalised messages
        switch = np.exp(lsw[None, :] + lnp[1:] + lb[1:] - lc[1:, None]).sum(axis=0)
    return gamma, lpx, la, lb, switch


def precompute(X, phi):
    """(G (W,), rho (W, d))."""
    X = _f64(X)
    phi = np.asarray(phi, np.float64)
    G = -0.5 * ((X ** 2).sum(axis=1) + X.shape[1] * np.log(2 * np.pi))
    return G, X * np.sqrt(phi)[None, :]


def initial_gamma(init_labels, S, init_smoothing):
    lab = np.asarray(init_labels, np.int64).reshape(-1)
    return softmax(init_smoothing * np.eye(S)[lab], axis=1)


def model(gamma, rho, phi, Fa, Fb):
    """(invL (S, d), alpha (S, d)) from the current gamma."""
    N = gamma.sum(axis=0)
    invL = 1.0 / (1.0 + Fa / Fb * N[:, None] * phi[None, :])
    alpha = Fa / Fb * invL * (gamma.T @ rho)
    return invL, alpha


def log_likelihoods(rho, G, invL, alpha, phi, Fa):
    return Fa * (rho @ alpha.T - 0.5 * (phi[None, :] * (invL + alpha ** 2)).sum(axis=1)[None, :] + G[:, None])


def vbx(X, phi, init_labels, Fa=0.3, Fb=17.0, loop_p=0.99, init_smoothing=5.0, max_iters=40, epsilon=1e-4, S=None):
    """One recording -> dict(gamma (W, S), pi (S,), elbo (iters,), iters, labels (W,)); S defaults to 1 + the
    largest initial label."""
    phi = np.asarray(phi, np.float64).reshape(-1)
    lab = np.asarray(init_labels, np.int64).reshape(-1)
    S = int(lab.max()) + 1 if S is None else int(S)
    G, rho = precompute(X, phi)
    gamma = initial_gamma(lab, S, init_smoothing)
    pi = np.full(S, 1.0 / S)
    elbo = []
    for i in range(int(max_iters)):
        invL, alpha = model(gamma, rho, phi, Fa, Fb)
        lnp = log_likelihoods(rho, G, invL, alpha, phi, Fa)
        gamma, lpx, _, _, switch = forward_backward(lnp, pi, loop_p)
        elbo.append(lpx + Fb / 2 * (np.log(invL) - invL - alpha ** 2 + 1).sum())
        num = gamma[0] + switch
        pi = num / num.sum()
        if (i >= 1 and elbo[-1] - elbo[-2] < epsilon) or i + 1 == max_iters:
            break
    return {"gamma": gamma, "pi": pi, "elbo": np.array(elbo), "iters": len(elbo), "labels": np.argmax(gamma, axis=1)}
