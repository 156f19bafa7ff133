// Waveform-domain augmentation of training segments (the MUSAN + RIR recipe of Kaldi x-vectors / voxceleb_trainer):
// a segment of int16 speech, reverberated by a room impulse response and mixed with noise sources at target SNRs.
// Definition in include/dsk.h (dsk_wave_augment).  The call runs, on one stream:
//   aug_check_kernel   per-example validity (indices, starts, RIR length, SNRs, speed factor), read from the banks'
//                      offsets only
//   aug_speed_kernel   s = the speed-perturbed segment into out (examples with a non-unit factor only)
//   aug_gather_kernel  s = bank[u][(start + i) mod n] * 2^-15 into out (the other examples; NaN rows for invalid ones)
//   aug_fft_in_kernel / aug_fft_rir_kernel / aug_conv_out_kernel
//                      uniformly partitioned overlap-save convolution, in place in out (examples with a RIR only)
//   aug_mix_kernel     fp64 energies and the mix, in place in out (when there are noise sources)
// No float atomics anywhere: every sum has a fixed order, so an example's bits depend on its own arguments only.
#pragma once
#include <stdint.h>

#include "../../include/dsk.h"

namespace dsk {

constexpr int kAugMaxSources = DSK_AUG_MAX_SOURCES;
constexpr int kAugMaxRir = DSK_AUG_MAX_RIR;
constexpr int kAugPart = 1024;         // partition length P
constexpr int kAugFft = 2 * kAugPart;  // N = 2P-point complex FFT
constexpr int kAugLogFft = 11;
constexpr int kAugBins = kAugPart + 1; // bins 0 .. N/2 of a real signal's spectrum; the rest are their conjugates
constexpr int kAugFftThreads = 512;
constexpr int kAugGatherThreads = 256;
constexpr int kAugGatherPerBlock = 4 * kAugGatherThreads;
constexpr int kAugMixThreads = 256;
constexpr int kSpeedMaxDen = DSK_SPEED_MAX_DEN;
constexpr int kSpeedTaps = DSK_SPEED_TAPS;       // d = -24 .. 25
constexpr int kSpeedMaxFactors = DSK_SPEED_MAX_FACTORS;
constexpr int kSpeedTapStride = 51;              // odd, so rows of different phases start in different bank pairs
constexpr int kSpeedMaxSpan = 2 * (kAugGatherPerBlock - 1) + 1 + kSpeedTaps;   // inputs of one tile at alpha = 2

// ok[b] codes written by aug_check_kernel
constexpr int kAugBad = 0, kAugGather = 1, kAugSpeed = 2;

__device__ __forceinline__ float aug_nan() { return __int_as_float(0x7fc00000); }

__device__ __forceinline__ bool aug_speed_ratio_ok(int p, int q) {
  if (q < 1 || q > kSpeedMaxDen || p < 1 || 2 * p < q || p > 2 * q) return false;
  int a = p, c = q;
  while (c) { const int t = a % c; a = c; c = t; }
  return a == 1;
}

// ok[b] = kAugBad unless every index and start of example b lies inside its bank, its RIR has 1 .. max_rir_len taps,
// the SNR of every used noise source is finite and its speed factor is -1 or a table entry whose ratio is within the
// limits; then kAugSpeed for a non-unit factor, else kAugGather.  Only offsets and ratios are read.
__global__ void aug_check_kernel(const int64_t* __restrict__ soff, int U, const int64_t* __restrict__ utt,
                                 const int64_t* __restrict__ start, int B, const int64_t* __restrict__ roff, int R,
                                 const int64_t* __restrict__ rir_idx, int max_rir_len, const int64_t* __restrict__ noff,
                                 int N, int M, const int64_t* __restrict__ noise_idx, const int64_t* __restrict__ noise_start,
                                 const double* __restrict__ snr_db, const int32_t* __restrict__ speed_ratio, int K,
                                 const int64_t* __restrict__ speed_idx, int* __restrict__ ok) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  bool good = false;
  const long u = utt[b], s = start[b];
  if (u >= 0 && u < U) {
    const long n = soff[u + 1] - soff[u];
    good = n >= 1 && s >= 0 && s < n;
  }
  if (good && rir_idx) {
    const long r = rir_idx[b];
    if (r >= 0 && r < R) {
      const long lh = roff[r + 1] - roff[r];
      good = lh >= 1 && lh <= max_rir_len;
    } else {
      good = r == -1;
    }
  }
  for (int j = 0; good && j < M; ++j) {
    const long q = noise_idx[static_cast<long>(b) * M + j];
    if (q == -1) continue;
    if (q < 0 || q >= N) { good = false; break; }
    const long n = noff[q + 1] - noff[q], st = noise_start[static_cast<long>(b) * M + j];
    good = n >= 1 && st >= 0 && st < n && isfinite(snr_db[static_cast<long>(b) * M + j]);
  }
  bool speed = false;
  if (good && K > 0) {
    const long k = speed_idx[b];
    if (k >= 0 && k < K) {
      const int p = speed_ratio[2 * k], q = speed_ratio[2 * k + 1];
      good = aug_speed_ratio_ok(p, q);
      speed = p != q;
    } else {
      good = k == -1;
    }
  }
  ok[b] = good ? (speed ? kAugSpeed : kAugGather) : kAugBad;
}

// out[b][i] = bank[soff[u] + (s + i) mod n] * 2^-15 (exact in fp32); NaN for an invalid example.
// grid = B * ceil(L / 1024), block = 256, four samples per thread.
__global__ void __launch_bounds__(kAugGatherThreads)
aug_gather_kernel(const int16_t* __restrict__ bank, const int64_t* __restrict__ soff, const int64_t* __restrict__ utt,
                  const int64_t* __restrict__ start, const int* __restrict__ ok, int L, float* __restrict__ out) {
  const int tiles = (L + kAugGatherPerBlock - 1) / kAugGatherPerBlock;
  const int b = blockIdx.x / tiles;
  const long i0 = static_cast<long>(blockIdx.x - b * tiles) * kAugGatherPerBlock;
  float* __restrict__ o = out + static_cast<long>(b) * L;
  if (ok[b] == kAugBad) {
    for (long i = i0 + threadIdx.x; i < L && i < i0 + kAugGatherPerBlock; i += kAugGatherThreads) o[i] = aug_nan();
    return;
  }
  if (ok[b] == kAugSpeed) return;      // written by aug_speed_kernel
  const long u = utt[b], base = soff[u], n = soff[u + 1] - base;
  long p = (start[b] + i0 + threadIdx.x) % n;
  for (long i = i0 + threadIdx.x; i < L && i < i0 + kAugGatherPerBlock; i += kAugGatherThreads) {
    o[i] = static_cast<float>(bank[base + p]) * (1.0f / 32768.0f);
    p += kAugGatherThreads;
    if (p >= n) p %= n;
  }
}

// Speed perturbation of the examples with ok[b] == kAugSpeed (definition in include/dsk.h): out[b][i] =
// fp32((sum_{d=-24}^{25} h_r[d] x[(start + m + d) mod n]) * 2^-15), i p = m q + r, the sum in fp64 in ascending d.
// grid = B * ceil(L / 1024) as aug_gather_kernel, block = 256, four outputs i0 + t + 256 j per thread.  The tile's
// m_last - m_first + 50 <= 2096 input samples are staged once into shared memory (coalesced, wrapped), so each bank
// sample is read about once per tile, together with the factor's q rows of taps; both as fp64, which makes every
// product h x exact and the fma chain the definition's sum.
__global__ void __launch_bounds__(kAugGatherThreads)
aug_speed_kernel(const int16_t* __restrict__ bank, const int64_t* __restrict__ soff, const int64_t* __restrict__ utt,
                 const int64_t* __restrict__ start, const int* __restrict__ ok, const int32_t* __restrict__ speed_ratio,
                 const float* __restrict__ speed_taps, const int64_t* __restrict__ speed_idx, int L,
                 float* __restrict__ out) {
  __shared__ double xs[kSpeedMaxSpan];
  __shared__ double hs[kSpeedMaxDen * kSpeedTapStride];
  const int tiles = (L + kAugGatherPerBlock - 1) / kAugGatherPerBlock;
  const int b = blockIdx.x / tiles;
  if (ok[b] != kAugSpeed) return;
  const long i0 = static_cast<long>(blockIdx.x - b * tiles) * kAugGatherPerBlock;
  const long i1 = min(static_cast<long>(L), i0 + kAugGatherPerBlock) - 1;
  const long k = speed_idx[b];
  const int p = speed_ratio[2 * k], q = speed_ratio[2 * k + 1];
  const long m0 = i0 * p / q, span = i1 * p / q - m0 + kSpeedTaps;
  const long u = utt[b], base = soff[u], n = soff[u + 1] - base;
  long pos = (start[b] + m0 - (kSpeedTaps / 2 - 1)) % n;           // x[start + m0 - 24], wrapped
  if (pos < 0) pos += n;
  pos = (pos + threadIdx.x) % n;
  for (long j = threadIdx.x; j < span; j += kAugGatherThreads) {
    xs[j] = static_cast<double>(bank[base + pos]);
    pos += kAugGatherThreads;
    if (pos >= n) pos %= n;
  }
  const float* __restrict__ h = speed_taps + k * kSpeedMaxDen * kSpeedTaps;
  for (int e = threadIdx.x; e < q * kSpeedTaps; e += kAugGatherThreads) {
    const int r = e / kSpeedTaps;
    hs[r * kSpeedTapStride + (e - r * kSpeedTaps)] = static_cast<double>(h[e]);
  }
  __syncthreads();
  float* __restrict__ o = out + static_cast<long>(b) * L;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long i = i0 + threadIdx.x + j * kAugGatherThreads;
    if (i > i1) break;
    const long ip = i * p, m = ip / q;
    const double* __restrict__ hr = hs + (ip - m * q) * kSpeedTapStride;
    const double* __restrict__ xr = xs + (m - m0);
    double acc = 0.0;
#pragma unroll
    for (int d = 0; d < kSpeedTaps; ++d) acc = fma(hr[d], xr[d], acc);
    o[i] = static_cast<float>(acc * (1.0 / 32768.0));
  }
}

// In-place radix-2 decimation-in-time FFT of N = 2048 points already in bit-reversed order, 512 threads, twiddles
// exp(sign * i pi pos / half) from sincospif as in fbank_kernel (sign = -1 forward, +1 inverse without the 1/N).
__device__ __forceinline__ void aug_fft2048(float2* buf, float sign) {
#pragma unroll 1
  for (int st = 1; st <= kAugLogFft; ++st) {
    const int half = 1 << (st - 1);
    for (int b = threadIdx.x; b < kAugFft / 2; b += kAugFftThreads) {
      const int grp = b / half, pos = b - grp * half;
      const int i0 = grp * 2 * half + pos, i1 = i0 + half;
      float sn, cs;
      sincospif(sign * static_cast<float>(pos) / static_cast<float>(half), &sn, &cs);
      const float2 a = buf[i0], c = buf[i1];
      const float2 w = make_float2(c.x * cs - c.y * sn, c.x * sn + c.y * cs);
      buf[i0] = make_float2(a.x + w.x, a.y + w.y);
      buf[i1] = make_float2(a.x - w.x, a.y - w.y);
    }
    __syncthreads();
  }
}

__device__ __forceinline__ int aug_brev(int i) { return static_cast<int>(__brev(static_cast<unsigned>(i)) >> (32 - kAugLogFft)); }

// The RIR's partition count: ceil(L_h / P) for an example that is valid and has a RIR, else 0.
__device__ __forceinline__ int aug_rir_parts(const int* ok, const int64_t* rir_idx, const int64_t* roff, int b) {
  if (!ok[b]) return 0;
  const long r = rir_idx[b];
  if (r < 0) return 0;
  return static_cast<int>((roff[r + 1] - roff[r] + kAugPart - 1) / kAugPart);
}

// X[b][j] = bins 0 .. P of FFT(s[(j - 1) P .. (j + 1) P)), s = 0 outside [0, L).  grid = B * nb, block = 512.
__global__ void __launch_bounds__(kAugFftThreads)
aug_fft_in_kernel(const float* __restrict__ seg, int L, int nb, const int* __restrict__ ok,
                  const int64_t* __restrict__ rir_idx, const int64_t* __restrict__ roff, float2* __restrict__ X) {
  __shared__ float2 buf[kAugFft];
  const int b = blockIdx.x / nb, j = blockIdx.x - b * nb;
  if (aug_rir_parts(ok, rir_idx, roff, b) == 0) return;
  const float* __restrict__ s = seg + static_cast<long>(b) * L;
  const long o = static_cast<long>(j - 1) * kAugPart;
  for (int i = threadIdx.x; i < kAugFft; i += kAugFftThreads) {
    const long t = o + i;
    buf[aug_brev(i)] = make_float2(t >= 0 && t < L ? s[t] : 0.f, 0.f);
  }
  __syncthreads();
  aug_fft2048(buf, -1.f);
  float2* __restrict__ x = X + (static_cast<long>(b) * nb + j) * kAugBins;
  for (int k = threadIdx.x; k < kAugBins; k += kAugFftThreads) x[k] = buf[k];
}

// H[b][p] = bins 0 .. P of FFT(h[p P .. (p + 1) P) zero-padded to N), h = RIR rir_idx[b] as stored.
// grid = B * kp, block = 512; partitions at or past ceil(L_h / P) are not written (and not read).
__global__ void __launch_bounds__(kAugFftThreads)
aug_fft_rir_kernel(const float* __restrict__ rir, const int64_t* __restrict__ roff, const int* __restrict__ ok,
                   const int64_t* __restrict__ rir_idx, int kp, float2* __restrict__ H) {
  __shared__ float2 buf[kAugFft];
  const int b = blockIdx.x / kp, p = blockIdx.x - b * kp;
  if (p >= aug_rir_parts(ok, rir_idx, roff, b)) return;
  const long r = rir_idx[b], base = roff[r], lh = roff[r + 1] - base;
  for (int i = threadIdx.x; i < kAugFft; i += kAugFftThreads) {
    const long t = static_cast<long>(p) * kAugPart + i;
    buf[aug_brev(i)] = make_float2(i < kAugPart && t < lh ? rir[base + t] : 0.f, 0.f);
  }
  __syncthreads();
  aug_fft2048(buf, -1.f);
  float2* __restrict__ h = H + (static_cast<long>(b) * kp + p) * kAugBins;
  for (int k = threadIdx.x; k < kAugBins; k += kAugFftThreads) h[k] = buf[k];
}

// Output block k of example b: Y = sum_{p = 0}^{min(k, parts - 1)} X[k - p] * H[p] in that order (bins 0 .. P, the
// others their conjugates), r[k P + i] = Re(IFFT(Y))[P + i] / N for i in [0, P) and k P + i < L, written over seg.
// grid = B * nb, block = 512.
__global__ void __launch_bounds__(kAugFftThreads)
aug_conv_out_kernel(const float2* __restrict__ X, const float2* __restrict__ H, int nb, int kp, const int* __restrict__ ok,
                    const int64_t* __restrict__ rir_idx, const int64_t* __restrict__ roff, int L, float* __restrict__ seg) {
  __shared__ float2 buf[kAugFft];
  const int b = blockIdx.x / nb, k = blockIdx.x - b * nb;
  const int parts = aug_rir_parts(ok, rir_idx, roff, b);
  if (parts == 0) return;
  const int np = min(k + 1, parts);
  const float2* __restrict__ xb = X + static_cast<long>(b) * nb * kAugBins;
  const float2* __restrict__ hb = H + static_cast<long>(b) * kp * kAugBins;
  for (int f = threadIdx.x; f < kAugBins; f += kAugFftThreads) {
    float2 y = make_float2(0.f, 0.f);
    for (int p = 0; p < np; ++p) {
      const float2 x = xb[static_cast<long>(k - p) * kAugBins + f], h = hb[static_cast<long>(p) * kAugBins + f];
      y.x = fmaf(x.x, h.x, fmaf(-x.y, h.y, y.x));
      y.y = fmaf(x.x, h.y, fmaf(x.y, h.x, y.y));
    }
    buf[aug_brev(f)] = y;
    if (f > 0 && f < kAugPart) buf[aug_brev(kAugFft - f)] = make_float2(y.x, -y.y);
  }
  __syncthreads();
  aug_fft2048(buf, 1.f);
  float* __restrict__ r = seg + static_cast<long>(b) * L;
  for (int i = threadIdx.x; i < kAugPart; i += kAugFftThreads) {
    const long t = static_cast<long>(k) * kAugPart + i;
    if (t < L) r[t] = buf[kAugPart + i].x * (1.0f / kAugFft);
  }
}

// Noise mixing, one block per example, in place: P(x) = sum x^2 / L in fp64 (thread-strided partial sums, then a fixed
// tree), g_j = sqrt(P(r) / (P(n_j) 10^(snr_j / 10))) (0 when P(n_j) = 0), out = (float)(r + sum_j g_j n_j) in fp64.
__global__ void __launch_bounds__(kAugMixThreads)
aug_mix_kernel(const int16_t* __restrict__ noise, const int64_t* __restrict__ noff, int M,
               const int64_t* __restrict__ noise_idx, const int64_t* __restrict__ noise_start,
               const double* __restrict__ snr_db, const int* __restrict__ ok, int L, float* out) {
  __shared__ double red[kAugMaxSources + 1][kAugMixThreads];
  __shared__ double gain[kAugMaxSources];
  __shared__ long nbase[kAugMaxSources], nlen[kAugMaxSources], nst[kAugMaxSources];
  const int b = blockIdx.x, t = threadIdx.x;
  if (!ok[b]) return;
  if (t < M) {
    const long q = noise_idx[static_cast<long>(b) * M + t];
    nbase[t] = q >= 0 ? noff[q] : 0;
    nlen[t] = q >= 0 ? noff[q + 1] - noff[q] : 0;
    nst[t] = q >= 0 ? noise_start[static_cast<long>(b) * M + t] : 0;
  }
  __syncthreads();
  float* r = out + static_cast<long>(b) * L;
  double acc[kAugMaxSources + 1];
  long pos[kAugMaxSources];     // (start + i) mod n of each source, advanced by the thread stride
#pragma unroll
  for (int j = 0; j <= kAugMaxSources; ++j) acc[j] = 0.0;
#pragma unroll
  for (int j = 0; j < kAugMaxSources; ++j) pos[j] = j < M && nlen[j] > 0 ? (nst[j] + t) % nlen[j] : 0;
  for (long i = t; i < L; i += kAugMixThreads) {
    const double v = r[i];
    acc[0] += v * v;
#pragma unroll
    for (int j = 0; j < kAugMaxSources; ++j) {
      if (j < M && nlen[j] > 0) {
        const double w = static_cast<double>(noise[nbase[j] + pos[j]]) * (1.0 / 32768.0);
        acc[j + 1] += w * w;
        pos[j] += kAugMixThreads;
        if (pos[j] >= nlen[j]) pos[j] %= nlen[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j <= kAugMaxSources; ++j) red[j][t] = acc[j];
  __syncthreads();
  for (int w = kAugMixThreads / 2; w > 0; w >>= 1) {
    if (t < w)
      for (int j = 0; j <= M; ++j) red[j][t] += red[j][t + w];
    __syncthreads();
  }
  if (t < M) {
    const double pn = red[t + 1][0] / L, pr = red[0][0] / L;
    gain[t] = nlen[t] > 0 && pn > 0.0 ? sqrt(pr / (pn * pow(10.0, snr_db[static_cast<long>(b) * M + t] / 10.0))) : 0.0;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kAugMaxSources; ++j) pos[j] = j < M && nlen[j] > 0 ? (nst[j] + t) % nlen[j] : 0;
  for (long i = t; i < L; i += kAugMixThreads) {
    double v = r[i];
#pragma unroll
    for (int j = 0; j < kAugMaxSources; ++j) {
      if (j < M && nlen[j] > 0) {
        v += gain[j] * (static_cast<double>(noise[nbase[j] + pos[j]]) * (1.0 / 32768.0));
        pos[j] += kAugMixThreads;
        if (pos[j] >= nlen[j]) pos[j] %= nlen[j];
      }
    }
    r[i] = static_cast<float>(v);
  }
}

}  // namespace dsk
