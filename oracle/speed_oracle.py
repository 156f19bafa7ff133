"""fp64 numpy restatement of speed perturbation (include/dsk.h ``dsk_wave_augment_speed``) - TEST INFRASTRUCTURE ONLY.

A factor alpha = p / q resamples the int16 utterance by a Hann-windowed sinc: output sample i reads the input at time
i alpha through the polyphase taps h_r[d] = fp32(h(r / q - d)), d = -24 .. 25, i p = m_i q + r_i, the sum over d in
fp64 in ascending order.  ``augment`` composes it with ``oracle/augment_oracle.py``: speed first, then reverb and noise.
"""
import math
from fractions import Fraction

import numpy as np

from oracle import augment_oracle as A

TAPS = 50
D0 = -24                      # the first tap's d
RHO, ZEROS = 0.99, 12


def h(tau, alpha):
    """The continuous kernel h(tau) = 2 f_c sinc(2 f_c tau) cos^2(pi tau / (2 Z_s)) for |tau| <= Z_s, in fp64 with the
    host math library, f_c = 0.5 rho min(1, 1 / alpha), Z_s = Z / (2 f_c)."""
    a = Fraction(alpha)
    fc = 0.5 * RHO * min(1.0, a.denominator / a.numerator)
    zs = ZEROS / (2.0 * fc)
    if abs(tau) > zs:
        return 0.0
    x = 2.0 * fc * tau
    sinc = 1.0 if x == 0.0 else math.sin(math.pi * x) / (math.pi * x)
    w = math.cos(math.pi * tau / (2.0 * zs))
    return 2.0 * fc * sinc * (w * w)


def taps(alpha):
    """(q, 50) fp32: row r = h(r / q - d) for d = -24 .. 25, each rounded once from fp64."""
    a = Fraction(alpha)
    q = a.denominator
    out = np.empty((q, TAPS), np.float32)
    for r in range(q):
        for j in range(TAPS):
            out[r, j] = np.float32(h(r / q - (j + D0), a))
    return out


def resample_sum(x, alpha, start, L, table=None):
    """The unscaled fp64 sums S_i = sum_d h_{r_i}[d] x[(start + m_i + d) mod n] (d ascending) for i in [0, L), and
    sum_d |h_{r_i}[d] x[...]| for error bounds; x is any 1-D array (int16 samples as stored)."""
    a = Fraction(alpha)
    p, q = a.numerator, a.denominator
    tab = taps(a) if table is None else table
    x = np.asarray(x, np.float64)
    n = x.size
    i = np.arange(L, dtype=np.int64)
    m, r = np.divmod(i * p, q)
    acc = np.zeros(L)
    mag = np.zeros(L)
    for j in range(TAPS):
        hv = tab[r, j].astype(np.float64)
        xv = x[(int(start) + m + (j + D0)) % n]
        acc = acc + hv * xv
        mag = mag + np.abs(hv * xv)
    return acc, mag


def speed(speech, soff, u, start, L, alpha):
    """The perturbed segment in fp64 (not rounded): S_i * 2^-15; alpha == 1 (or None) is the plain gather."""
    if alpha is None or Fraction(alpha) == 1:
        return A.gather(speech, soff, u, start, L)
    base, n = int(soff[u]), int(soff[u + 1] - soff[u])
    acc, _ = resample_sum(speech[base:base + n], alpha, start, L)
    return acc * 2.0 ** -15


def augment(speech, soff, u, start, L, alpha=None, rir=None, noise=None, noff=None, noise_idx=(), noise_start=(),
            snr_db=()):
    """One example of the definition in fp64: the segment perturbed by ``alpha`` and rounded to fp32 as the engine
    stores it, then ``augment_oracle``'s reverb and mix."""
    s = speed(speech, soff, u, start, L, alpha).astype(np.float32).astype(np.float64)
    r = A.reverb(s, rir)
    srcs, snrs = [], []
    for q, st, snr in zip(noise_idx, noise_start, snr_db):
        if q == -1:
            continue
        srcs.append(A.gather(noise, noff, int(q), int(st), L))
        snrs.append(float(snr))
    return A.mix(r, srcs, snrs)
