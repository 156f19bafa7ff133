"""fp64 stage-by-stage reference of the log-fbank front-end (``fbank_kernel``, csrc/fbank_kernels.cuh) and a bound on
every element the fp32 kernel writes, derived from its arithmetic.  Shared by tests/test_fbank_bound_host.py (the gate
against an fp32 emulation of the kernel, with seeded defects) and tests/test_gpu_fbank_bound.py (the gate on the GPU).

Reference.  From the fp32 samples x (n of them) at rate sr, in fp64 throughout:
  pre-emphasis   y_0 = x_0,  y_s = x_s - a x_{s-1} with a = fp32(0.97), the kernel's coefficient;
  frames         frame f is y[f step .. f step + flen), zero past sample n - 1, zero-padded to N = 512
                 (flen = round_half_up(0.025 sr), step = round_half_up(0.01 sr));
  power          X = rfft(frame, 512), p_k = |X_k|^2 / 512, k = 0 .. 256;
  mel            m_j = sum_k w_jk p_k with the oracle's fp64 weights FO.get_filterbanks(64, 512, sr);
  energy         E = sum_k p_k;
  log            20 log10(max(m_j, 1e-5)), eps where a filter output is 0;
  mean           the per-utterance column mean, subtracted.

Bound.  u = 2^-24, gamma_n = n u / (1 - n u).  The input domain is finite |x| <= 2^15, which holds un-normalised int16
audio; fp32 |X|^2 would overflow only at |x| of about 1e16 (|X| <= sum |y| <= 512 * 1.97 |x|), far outside it.
  Pre-emphasis.  y_s = fl(x_s - fl(a x_{s-1})), or one rounding when nvcc contracts it to an FMA: count two, so
      |dy_s| <= 2u(1+u) (|x_s| + a |x_{s-1}|), and ||dy||_1 is that summed over the frame (dy_0 = 0: x_0 is loaded as is).
  FFT.  Radix-2 decimation in time, 9 stages, twiddle w = exp(-i pi pos/half) from sincospif of an exact argument.
      CUDA's sinpif / cospif are within 1 ulp, so |w^ - w| <= mu = 2u.  One butterfly out = fl(a^ +- fl(c^ w^)): the
      complex product is off by at most sqrt(2) gamma_2 |c^||w^| and the add by u |a^ +- t^|.  By induction over the
      stages, if every stage-(s-1) value is within eps_{s-1} S of its exact value, S = sum |y^_j| over its inputs (which
      also bounds the exact value, |w| = 1), the stage-s value is within ((1 + eps_{s-1})(1 + eta) - 1) S with
          eta = mu + (1 + mu)(sqrt(2) gamma_2 + u (1 + sqrt(2) gamma_2)),
      so |X^_k - X_k| <= delta = ((1 + eta)^9 - 1)(||y||_1 + ||dy||_1) + ||dy||_1 for every bin of the frame.
  Power.  p^ = fl(fl(X^r^2) + X^i^2) / 512 (the / 512 is exact): |p^_k - p_k| <= dp_k =
      ((2|X_k| + delta) delta + gamma_2 (|X_k| + delta)^2) / 512.
  Mel.  m^_j = the fp32 FMA chain over k of p^_k fp32(w_jk); the n_j terms with w_jk != 0 round (an FMA with weight 0 is
      exact), the fp32 weight is within u w_jk:  |m^_j - m_j| <= B_j = sum_k w_jk dp_k + (u + gamma_{n_j}(1+u)) sum_k w_jk (p_k + dp_k).
      The linear output is m^_j, or fp32(eps) = fp32(2.220446049250313e-16) where m^_j == 0; so it must be non-zero and
      within B_j of m_j, or be fp32(eps) with m_j <= B_j.
  Log.  The output is fl(20 fl(log10f(max(m^', F)))) with F = fp32(1e-5) (1e-5 (1 - 2.5e-8); the interval below uses the
      kernel's own floor, so the fp32/fp64 floor difference needs no widening), m^' = m^ or eps.  max(m^', F) lies in
      [max(m - B, F), max(m + B, F)], so 20 log10 of it in [lo, hi] = 20 log10 of those ends.  log10f is within 2 ulp
      (CUDA programming guide), <= 4u |log10|, and the x20 rounds once: the output lies in [lo - e, hi + e],
      e = 20 R (5u + 9u^2), R = max(|log10 lo|, |log10 hi|).
  Mean.  From the engine's own un-subtracted output g (F frames): each 4-frame block partial is an fp32 sum of up to 4
      rows (3 roundings), the partials are added in double, divided by F in double and rounded to fp32, and the
      subtraction rounds once.  With mu_j = sum_f g_fj / F in fp64,
          |mean^_j - mu_j| <= M_j = (gamma_3 + (F/4 + 2) 2^-53) sum_f |g_fj| / F + u (|mu_j| + gamma_3 sum_f |g_fj| / F)
      and |out_fj - (g_fj - mu_j)| <= M_j + u (|g_fj - mu_j| + M_j).
  Energy (mk_mfb_batch_vad).  e^ = the fp32 sum of p^_0 .. p^_256 in bin order, 256 roundings:
      |e^ - E| <= sum_k dp_k + gamma_257 sum_k (p_k + dp_k); eps where e^ == 0, as for the mel outputs.
  Slack.  The fp64 reference itself is off by O(2^-53 log2 N) relative, covered by 2^-40 of the magnitude at each stage;
  gradual underflow adds at most 2^-150 per fp32 operation, covered by an absolute 2^-120 per stage.  Both are far below
  any value the tests look at.
"""
import numpy as np

from oracle import fbank_oracle as FO

NFFT, BINS, NMEL = 512, 257, 64
U = 2.0 ** -24
PREEMPH = float(np.float32(0.97))
FLOOR32 = float(np.float32(1e-5))
EPS32 = float(np.float32(2.220446049250313e-16))
REL = 2.0 ** -40            # fp64 reference slack, relative
TINY = 2.0 ** -120          # underflow slack, absolute


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1.0 - n * U)


MU = 2 * U                                                          # 1 ulp of sinpif / cospif, relative
ETA = MU + (1 + MU) * (np.sqrt(2) * gamma(2) + U * (1 + np.sqrt(2) * gamma(2)))
FFT_GROWTH = (1 + ETA) ** 9 - 1
PRE_ERR = 2 * U * (1 + U)


def geometry(sr):
    """(flen, step) of the 25 ms / 10 ms frames at ``sr``."""
    return FO.round_half_up(0.025 * sr), FO.round_half_up(0.01 * sr)


def num_frames(n, sr):
    flen, step = geometry(sr)
    return 1 if n <= flen else 1 + -(-(n - flen) // step)


def filterbank(sr):
    return FO.get_filterbanks(NMEL, NFFT, sr)


def isolated_filters(sr):
    """(filter, bin) of the filters that are one bin of weight exactly 1.0: their output is that bin's power."""
    W = filterbank(sr)
    out = []
    for j in range(NMEL):
        nz = np.flatnonzero(W[j])
        if nz.size == 1 and W[j, nz[0]] == 1.0:
            out.append((j, int(nz[0])))
    return out


def _frames(v, n, flen, step, f0, f1):
    idx = np.arange(f0, f1, dtype=np.int64)[:, None] * step + np.arange(flen, dtype=np.int64)[None, :]
    return np.where(idx < n, v[np.minimum(idx, n - 1)], 0.0)


class Reference:
    """The fp64 reference of one utterance and the per-element bounds of the kernel's outputs against it:
    ``m``, ``bm`` (F, 64) linear mel outputs and their bounds; ``E``, ``bE`` (F,) energies; ``p_iso``, ``bp_iso``
    (F, len(iso)) the power of the bins of the isolated filters ``iso`` and the per-bin power bound."""

    def __init__(self, x, sr):
        x = np.asarray(x, np.float32)
        n = x.size
        flen, step = geometry(sr)
        F = num_frames(n, sr)
        W = filterbank(sr)
        coef = U + gamma((W != 0).sum(1)) * (1 + U)
        self.iso = isolated_filters(sr)
        kiso = [k for _, k in self.iso]
        xd = x.astype(np.float64)
        y = xd.copy()
        y[1:] = xd[1:] - PREEMPH * xd[:-1]
        ay = np.zeros(n)
        ay[1:] = np.abs(xd[1:]) + PREEMPH * np.abs(xd[:-1])
        self.m, self.bm = np.empty((F, NMEL)), np.empty((F, NMEL))
        self.E, self.bE = np.empty(F), np.empty(F)
        self.p_iso, self.bp_iso = np.empty((F, len(kiso))), np.empty((F, len(kiso)))
        chunk = 8192
        for f0 in range(0, F, chunk):
            f1 = min(F, f0 + chunk)
            fy = _frames(y, n, flen, step, f0, f1)
            dl1 = PRE_ERR * _frames(ay, n, flen, step, f0, f1).sum(1, keepdims=True)
            l1 = np.abs(fy).sum(1, keepdims=True)
            delta = FFT_GROWTH * (l1 + dl1) + dl1 + REL * l1 + TINY
            X = np.abs(np.fft.rfft(fy, NFFT, axis=1))
            p = X * X / NFFT
            dp = ((2 * X + delta) * delta + gamma(2) * (X + delta) ** 2) / NFFT + REL * p + TINY
            m = p @ W.T
            self.m[f0:f1] = m
            self.bm[f0:f1] = dp @ W.T + coef * ((p + dp) @ W.T) + REL * m + TINY
            self.E[f0:f1] = p.sum(1)
            self.bE[f0:f1] = dp.sum(1) + gamma(BINS) * (p + dp).sum(1) + REL * p.sum(1) + TINY
            self.p_iso[f0:f1] = p[:, kiso]
            self.bp_iso[f0:f1] = dp[:, kiso]


def _linear_ratio(g, ref, bound):
    """err / bound of linear outputs that carry the eps substitution: inf for an output of 0 (the kernel never writes
    one), 0 for fp32(eps) where the reference is within the bound of 0."""
    g = np.asarray(g, np.float64)
    r = np.abs(g - ref) / bound
    r = np.where((g == EPS32) & (ref <= bound), 0.0, r)
    return np.where(g == 0, np.inf, r)


def mel_ratio(g, R):
    return _linear_ratio(g, R.m, R.bm)


def energy_ratio(e, R):
    return _linear_ratio(e, R.E, R.bE)


def iso_ratio(g, R):
    """The isolated filters' linear outputs against their bin's power and the per-bin power bound (no mel terms: an
    FMA by 1.0 into 0 and by 0 elsewhere is exact)."""
    if not R.iso:
        return np.zeros((R.m.shape[0], 0))
    return _linear_ratio(np.asarray(g)[:, [j for j, _ in R.iso]], R.p_iso, R.bp_iso)


def log_ratio(g, R):
    """The distance of g from the fp64 value 20 log10(max(m, F)) over the distance from it to the end of the widened
    dB interval on g's side: <= 1 inside the interval."""
    lo = np.log10(np.maximum(R.m - R.bm, FLOOR32))
    hi = np.log10(np.maximum(R.m + R.bm, FLOOR32))
    e = 20 * np.maximum(np.abs(lo), np.abs(hi)) * (5 * U + 9 * U * U + REL) + TINY
    lo, hi = 20 * lo - e, 20 * hi + e
    c = 20 * np.log10(np.maximum(R.m, FLOOR32))
    g = np.asarray(g, np.float64)
    return np.where(g >= c, (g - c) / (hi - c), (c - g) / (c - lo))


def mean_ratio(out, g):
    """The mean-subtracted output ``out`` against the engine's own un-subtracted output ``g`` of the same utterance."""
    g = np.asarray(g, np.float64)
    a = np.abs(g).sum(0) / g.shape[0]
    mu = g.sum(0) / g.shape[0]
    M = gamma(3) * a + U * (np.abs(mu) + gamma(3) * a) + (g.shape[0] / 4 + 2) * 2.0 ** -53 * a + REL * a + TINY
    bound = M + U * (np.abs(g - mu) + M)
    return np.abs(np.asarray(out, np.float64) - (g - mu)) / bound


# ---- the signals -------------------------------------------------------------------------------------------------------
def signal(kind, n, sr, seed=0):
    """fp32 test signal ``kind`` of n samples at ``sr`` (see ``batch``)."""
    g = np.random.default_rng(seed)
    i = np.arange(n)
    flen, step = geometry(sr)
    if kind == "tones":                  # two tones plus noise under a rising envelope (tests/test_fbank.py's signal)
        x = 0.3 * np.sin(2 * np.pi * 0.0275 * i) + 0.2 * np.sin(2 * np.pi * 0.14375 * i + 1.0) + 0.05 * g.standard_normal(n)
        x *= np.linspace(0.2, 1.0, n)
    elif kind == "int16":                # int16-quantised white noise, -32768 .. 32767 over 32768
        x = g.integers(-32768, 32768, n) / 32768.0
    elif kind == "int16_raw":            # un-normalised int16 values, up to +-32768
        x = g.integers(-32768, 32769, n).astype(np.float64)
    elif kind == "dc_step":              # pre-emphasis turns the step into an impulse
        x = np.where(i >= n // 2, 0.5, 0.0)
    elif kind == "nyquist":              # (-1)^n: seen by the energy and the bins next to 256 only
        x = 0.5 * (1 - 2 * (i & 1))
    elif kind.startswith("impulse_"):    # one impulse at frame 1's first sample, its last, or one in frames 1 and 2
        x = np.zeros(n)
        x[{"impulse_first": step, "impulse_last": step + flen - 1, "impulse_overlap": 2 * step}[kind]] = 1.0
    elif kind == "jump":                 # a tone that drops 80 dB at the start of frame 10
        x = np.sin(2 * np.pi * 0.0625 * i + 0.3) * np.where(i < 10 * step, 1.0, 1e-4)
    elif kind == "zeros":
        x = np.zeros(n)
    elif kind == "zero_gaps":            # noise with frames 4 .. 9 all zero (pre-emphasis leaks into frame 3)
        x = g.integers(-32768, 32768, n) / 32768.0
        x[3 * step:3 * step + 6 * step + flen] = 0.0
    elif kind == "lsb":                  # 1-LSB silence: -1, 0, 1 over 32768, below the 1e-5 floor
        x = g.integers(-1, 2, n) / 32768.0
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


SPECIAL = ("tones", "int16", "int16_raw", "dc_step", "nyquist", "impulse_first", "impulse_last", "impulse_overlap", "jump",
           "zeros", "zero_gaps", "lsb")


def batch(sr, seed=0, long=True):
    """The utterances of one batched call at ``sr``: a list of (signal class, fp32 samples).
      lengths 1, flen - 1, flen, flen + 1, flen + step - 1, flen + step, flen + step + 1, each followed by a loud
        un-normalised int16 neighbour (a frame that read past its utterance's end would see it);
      lengths of 8, 9, 10 and 11 frames (0 .. 3 mod the 4-frame block) whose last frame runs past the end, each also
        followed by a loud neighbour;
      every signal class of ``SPECIAL`` at 31 frames;
      with ``long``, 100 003 samples, and at 16 kHz one utterance of 2^24 + 12 345 samples."""
    flen, step = geometry(sr)
    kinds = ("tones", "int16", "nyquist", "dc_step", "lsb", "int16_raw", "tones")
    out = []
    s = seed
    shorts = [n for n in (1, flen - 1, flen, flen + 1, flen + step - 1, flen + step, flen + step + 1) if n >= 1]
    for j, n in enumerate(shorts):
        out.append((kinds[j % len(kinds)], signal(kinds[j % len(kinds)], n, sr, s)))
        out.append(("int16_raw", signal("int16_raw", flen + 3 * step, sr, s + 1)))
        s += 2
    for F, kind in zip((8, 9, 10, 11), ("tones", "int16", "nyquist", "jump")):
        out.append((kind, signal(kind, flen + (F - 2) * step + 1, sr, s)))
        out.append(("int16_raw", signal("int16_raw", flen + 3 * step, sr, s + 1)))
        s += 2
    for kind in SPECIAL:
        out.append((kind, signal(kind, flen + 29 * step + step // 2 + 1, sr, s)))
        s += 1
    if long:
        out.append(("tones", signal("tones", 100003, sr, s)))
        if sr == 16000:
            out.append(("int16", signal("int16", (1 << 24) + 12345, sr, s + 1)))
    return out
