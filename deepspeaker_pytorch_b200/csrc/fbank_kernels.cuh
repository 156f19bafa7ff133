// Log mel-filterbank front-end of the reference (reference audio_processing.py:9-36 `mk_MFB`, constants.py:6-16):
//   filter_banks, _ = python_speech_features.fbank(audio, samplerate=16000, nfilt=64, winlen=0.025)     (:14)
//   filter_banks = 20 * log10(max(filter_banks, 1e-5))                                                  (:16-17)
//   filter_banks = filter_banks - mean(filter_banks, axis=0)          (normalize_frames, Scale=False)   (:29, :88-92)
// python_speech_features is NOT vendored in the reference and is absent from this image: its published algorithm
// (base.py `fbank` / sigproc.py, v0.6) is restated - pre-emphasis 0.97, frames of round(0.025 sr) samples every
// round(0.01 sr), rectangular window, zero-padded to NFFT = 512, power spectrum |rfft|^2 / NFFT, triangular mel filters
// on floor((NFFT + 1) * mel2hz(.) / sr) bin edges, zeros replaced by eps.  Parity against the package itself is unpinned;
// the oracle (oracle/fbank_oracle.py) is the numpy restatement of the same published algorithm.
// Output: (frames, 64) fp32 row-major - exactly the (T, 64) layout the network's (B, 1, T, 64) input is cropped from.
#pragma once
#include <stdint.h>

namespace dsk {

constexpr int kFbNfft = 512;
constexpr int kFbBins = kFbNfft / 2 + 1;  // 257
constexpr int kFbFilters = 64;
constexpr int kFbFramesPerBlock = 4;      // one warp-pair group of 64 threads per frame
constexpr int kFbThreads = 64 * kFbFramesPerBlock;

// feat[f][m] = 20 log10(max(sum_k pspec[f][k] * fb[m][k], floor)) for frame f; partial column sums per block for the
// mean.  audio: n samples; frame f covers samples [f*step, f*step + flen) of the PRE-EMPHASISED signal, zero beyond n.
// fb: [64][257] fp32.  grid = ceil(frames / 4), block = 256: thread group g = tid / 64 owns frame 4*blockIdx.x + g.
__global__ void __launch_bounds__(kFbThreads)
fbank_kernel(const float* __restrict__ audio, int n, int flen, int step, int frames, float preemph,
             const float* __restrict__ fb, int log_scale, float log_floor, float* __restrict__ feat,
             float* __restrict__ colsum_partial /* [gridDim.x][64] */) {
  __shared__ float2 buf[kFbFramesPerBlock][kFbNfft];     // complex FFT workspace per frame
  __shared__ float pspec[kFbFramesPerBlock][kFbBins + 3];
  __shared__ float rowfeat[kFbFramesPerBlock][kFbFilters];
  const int g = threadIdx.x >> 6, t = threadIdx.x & 63;
  const int f = blockIdx.x * kFbFramesPerBlock + g;
  const bool live = f < frames;
  // ---- load + pre-emphasis (y[0] = x[0], y[i] = x[i] - a x[i-1]) into bit-reversed order
  for (int i = t; i < kFbNfft; i += 64) {
    float v = 0.f;
    const long s = static_cast<long>(f) * step + i;
    if (live && i < flen && s < n) v = s == 0 ? audio[0] : audio[s] - preemph * audio[s - 1];
    buf[g][__brev(static_cast<unsigned>(i)) >> (32 - 9)] = make_float2(v, 0.f);
  }
  __syncthreads();
  // ---- radix-2 decimation-in-time FFT, 9 stages x 256 butterflies, 4 butterflies per thread and stage
#pragma unroll 1
  for (int st = 1; st <= 9; ++st) {
    const int half = 1 << (st - 1);
    for (int b = t; b < kFbNfft / 2; b += 64) {
      const int grp = b / half, pos = b - grp * half;
      const int i0 = grp * 2 * half + pos, i1 = i0 + half;
      float sn, cs;
      sincospif(-static_cast<float>(pos) / static_cast<float>(half), &sn, &cs);   // exp(-i pi pos / half)
      const float2 a = buf[g][i0], c = buf[g][i1];
      const float2 w = make_float2(c.x * cs - c.y * sn, c.x * sn + c.y * cs);
      buf[g][i0] = make_float2(a.x + w.x, a.y + w.y);
      buf[g][i1] = make_float2(a.x - w.x, a.y - w.y);
    }
    __syncthreads();
  }
  for (int k = t; k < kFbBins; k += 64) {
    const float2 z = buf[g][k];
    pspec[g][k] = (z.x * z.x + z.y * z.y) * (1.0f / kFbNfft);
  }
  __syncthreads();
  // ---- mel filterbank: thread t = filter t
  {
    const float* w = fb + t * kFbBins;
    float acc = 0.f;
    for (int k = 0; k < kFbBins; ++k) acc = fmaf(pspec[g][k], w[k], acc);
    if (acc == 0.f) acc = 2.220446049250313e-16f;           // numpy.finfo(float).eps, as fbank() substitutes
    if (log_scale) acc = 20.0f * log10f(fmaxf(acc, log_floor));
    rowfeat[g][t] = live ? acc : 0.f;
    if (live) feat[static_cast<long>(f) * kFbFilters + t] = acc;
  }
  __syncthreads();
  if (g == 0) {  // per-block column sums, fixed order
    float s = 0.f;
    for (int r = 0; r < kFbFramesPerBlock; ++r) s += rowfeat[r][t];
    colsum_partial[static_cast<long>(blockIdx.x) * kFbFilters + t] = s;
  }
}

// mean over frames (partials added in fixed order, in double) subtracted in place.  grid = ceil(frames / 64), block = 64 x 4
__global__ void fbank_mean_sub_kernel(float* __restrict__ feat, int frames, const float* __restrict__ colsum_partial, int nblk) {
  __shared__ float mean[kFbFilters];
  if (threadIdx.x < kFbFilters) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += colsum_partial[static_cast<long>(b) * kFbFilters + threadIdx.x];
    mean[threadIdx.x] = static_cast<float>(s / frames);
  }
  __syncthreads();
  const int m = threadIdx.x & 63;
  for (int f = blockIdx.x * 64 + (threadIdx.x >> 6); f < frames && f < (blockIdx.x + 1) * 64; f += blockDim.x >> 6)
    feat[static_cast<long>(f) * kFbFilters + m] -= mean[m];
}

}  // namespace dsk
