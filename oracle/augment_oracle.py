"""fp64 numpy restatement of the waveform augmentation (include/dsk.h ``dsk_wave_augment``) - TEST INFRASTRUCTURE ONLY.

segment gather (int16 * 2^-15, wrapping), reverberation as the full convolution truncated to the segment
(``h`` used exactly as stored), and noise mixing at a target SNR with fp64 energies.  Features of the result come
through ``oracle/fbank_oracle.py``.
"""
import numpy as np


def gather(bank, offsets, u, start, L):
    """s[i] = bank[offsets[u] + (start + i) mod n_u] * 2^-15, fp64."""
    base, n = int(offsets[u]), int(offsets[u + 1] - offsets[u])
    return bank[base + (int(start) + np.arange(L)) % n].astype(np.float64) / 32768.0


def fft_convolve(s, h):
    """The first len(s) samples of the full linear convolution s * h, by one fp64 FFT of sufficient length."""
    L = s.size
    n = 1 << int(np.ceil(np.log2(L + h.size - 1)))
    return np.fft.irfft(np.fft.rfft(s, n) * np.fft.rfft(h, n), n)[:L]


def reverb(s, h):
    """r[i] = sum_{k=0}^{min(i, L_h - 1)} h[k] s[i - k] in fp64; h = None: r = s."""
    return np.array(s, np.float64) if h is None else fft_convolve(np.asarray(s, np.float64), np.asarray(h, np.float64))


def power(x):
    return float(np.sum(np.asarray(x, np.float64) ** 2) / x.size)


def gains(r, sources, snr_db):
    """g_j = sqrt(P(r) / (P(n_j) 10^(snr_j / 10))), 0 when P(n_j) = 0."""
    pr = power(r)
    out = []
    for n, snr in zip(sources, snr_db):
        pn = power(n)
        out.append(0.0 if pn == 0.0 else float(np.sqrt(pr / (pn * 10.0 ** (snr / 10.0)))))
    return out


def mix(r, sources, snr_db):
    """r + sum_j g_j n_j in fp64 (not rounded)."""
    out = np.array(r, np.float64)
    for g, n in zip(gains(r, sources, snr_db), sources):
        out = out + g * np.asarray(n, np.float64)
    return out


def augment(speech, soff, u, start, L, rir=None, noise=None, noff=None, noise_idx=(), noise_start=(), snr_db=()):
    """One example of the definition in fp64: ``rir`` is the RIR as stored (or None); the noise sources are
    (noise_idx[j], noise_start[j], snr_db[j]) with -1 = none."""
    r = reverb(gather(speech, soff, u, start, L), rir)
    srcs, snrs = [], []
    for q, st, snr in zip(noise_idx, noise_start, snr_db):
        if q == -1:
            continue
        srcs.append(gather(noise, noff, int(q), int(st), L))
        snrs.append(float(snr))
    return mix(r, srcs, snrs)


DEFECTS = ("drop_partition", "pair_shift", "sample_shift", "zero_last_block", "twiddle_sign")


def partitioned_convolve(s, h, P=1024, dtype=np.complex64, defect=None):
    """Uniformly partitioned overlap-save convolution as the kernels compute it, in ``dtype`` FFTs (complex64 = fp32):
    X_j = FFT(s[(j - 1) P .. (j + 1) P)), H_p = FFT(h[p P .. (p + 1) P) zero-padded to 2P), output block k the last P
    samples of IFFT(sum_{p <= k} X_{k - p} H_p) in partition order.  ``defect`` (one of DEFECTS) seeds a bug for the
    checker's self-test: partition 1 dropped, X_{k-p} paired with H_{p+1}, the output one sample late, the last block
    zeroed, or the middle block inverted with the forward twiddle sign.  Returns (r, X, H)."""
    import scipy.fft as sf

    rdt = np.float32 if dtype == np.complex64 else np.float64
    L, N = s.size, 2 * P
    nb, kp = -(-L // P), -(-h.size // P)
    sp = np.zeros((nb + 1) * P, rdt)
    sp[P:P + L] = s
    X = np.stack([sf.fft(sp[j * P:j * P + N].astype(dtype)) for j in range(nb)])
    hp = np.zeros(kp * P, rdt)
    hp[:h.size] = h
    H = np.stack([sf.fft(np.concatenate([hp[p * P:(p + 1) * P], np.zeros(P, rdt)]).astype(dtype)) for p in range(kp)])
    r = np.empty(nb * P, rdt)
    for k in range(nb):
        Y = np.zeros(N, dtype)
        for p in range(min(k + 1, kp)):
            if defect == "drop_partition" and p == 1:
                continue
            if defect == "pair_shift":
                if p + 1 < kp:
                    Y = Y + X[k - p] * H[p + 1]
                continue
            Y = Y + X[k - p] * H[p]
        y = sf.fft(Y) / N if defect == "twiddle_sign" and k == nb // 2 else sf.ifft(Y)
        r[k * P:(k + 1) * P] = y.real[P:].astype(rdt)
    if defect == "zero_last_block":
        r[(nb - 1) * P:] = 0
    if defect == "sample_shift":
        r[1:] = r[:-1].copy()
        r[0] = 0
    return r[:L], X, H


def reverb_bound(s, h, P=1024, c=None):
    """Per-sample error bound of the fp32 partitioned convolution, and its per-block L2 form (see
    tests/test_augment_host.py for the derivation): for output block k,
        bound_k = c log2(N) u sum_{p <= k} ||x_{k-p}||_2 ||h_p||_2,
    x_j = s[(j - 1) P .. (j + 1) P) (zero outside), h_p = h[p P .. (p + 1) P), N = 2P, u = 2^-24.
    Returns (bound per sample (L,), bound per block (nb,))."""
    c = 1.0 if c is None else c
    L, N = s.size, 2 * P
    nb, kp = -(-L // P), -(-h.size // P)
    sp = np.zeros((nb + 1) * P)
    sp[P:P + L] = s
    xn = np.array([np.linalg.norm(sp[j * P:j * P + N]) for j in range(nb)])
    hp = np.zeros(kp * P)
    hp[:h.size] = h
    hn = np.array([np.linalg.norm(hp[p * P:(p + 1) * P]) for p in range(kp)])
    u = 2.0 ** -24
    blk = np.array([sum(xn[k - p] * hn[p] for p in range(min(k + 1, kp))) for k in range(nb)])
    blk = c * np.log2(N) * u * blk
    return np.repeat(blk, P)[:L], blk


def reverb_error_ratios(r, s, h, P=1024):
    """(max_i |r_i - y_i| / bound_i, max_k ||r_k - y_k||_2 / bound_k) of a computed reverberation r of s by h against
    the fp64 result y; both must be <= 1."""
    s64, h64 = np.asarray(s, np.float64), np.asarray(h, np.float64)
    y = reverb(s64, h64)
    e = np.abs(np.asarray(r, np.float64) - y)
    per_sample, per_block = reverb_bound(s64, h64, P)
    nb = per_block.size
    ep = np.zeros(nb * P)
    ep[:e.size] = e
    with np.errstate(invalid="ignore", divide="ignore"):
        elem = np.max(np.where(e == 0, 0.0, e / per_sample))
        blk = np.max(np.where(ep.reshape(nb, P).any(1), np.linalg.norm(ep.reshape(nb, P), axis=1) / per_block, 0.0))
    return float(elem), float(blk)
