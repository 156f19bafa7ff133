// Log mel-filterbank front-end of the reference (reference audio_processing.py:9-36 `mk_MFB`, constants.py:6-16):
//   filter_banks, _ = python_speech_features.fbank(audio, samplerate=16000, nfilt=64, winlen=0.025)     (:14)
//   filter_banks = 20 * log10(max(filter_banks, 1e-5))                                                  (:16-17)
//   filter_banks = filter_banks - mean(filter_banks, axis=0)          (normalize_frames, Scale=False)   (:29, :88-92)
// python_speech_features is NOT vendored in the reference and is absent from this image: its published algorithm
// (base.py `fbank` / sigproc.py, v0.6) is restated - pre-emphasis 0.97, frames of round(0.025 sr) samples every
// round(0.01 sr), rectangular window, zero-padded to NFFT = 512, power spectrum |rfft|^2 / NFFT, triangular mel filters
// on floor((NFFT + 1) * mel2hz(.) / sr) bin edges, zeros replaced by eps.  Parity against the package itself is unpinned;
// the oracle (oracle/fbank_oracle.py) is the numpy restatement of the same published algorithm.
// Output: (frames, 64) fp32 row-major per utterance, a batch of utterances one after another - exactly the (T, 64) layout the network's (B, 1, T, 64) input is cropped from.
#pragma once
#include <stdint.h>

namespace dsk {

constexpr int kFbNfft = 512;
constexpr int kFbBins = kFbNfft / 2 + 1;  // 257
constexpr int kFbFilters = 64;
constexpr int kFbFramesPerBlock = 4;      // one warp-pair group of 64 threads per frame
constexpr int kFbThreads = 64 * kFbFramesPerBlock;

// A batch of U utterances: utterance u is samples [soff[u], soff[u+1]) of the concatenated audio, frames [foff[u],
// foff[u+1]) of feat and blocks [boff[u], boff[u+1]) of the grid, ceil(frames_u / 4) of them.  Every utterance starts on
// a block boundary, so each block, its frames and its column-sum partial are exactly those of a call on that utterance
// alone, wherever it sits in the batch.  The block's utterance: the largest u with boff[u] <= blk (boff is strictly
// increasing, boff[0] = 0).
__device__ __forceinline__ int fbank_block_utt(const int64_t* __restrict__ boff, int U, long blk) {
  int lo = 0, hi = U - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (boff[mid] <= blk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// feat[f][m] = 20 log10(max(sum_k pspec[f][k] * fb[m][k], floor)) for frame f of the block's utterance; partial column
// sums per block for the mean.  Utterance u: n samples; its frame f covers samples [f*step, f*step + flen) of the
// PRE-EMPHASISED signal, zero beyond n.  fb: [64][257] fp32.  grid = boff[U], block = 256: thread group g = tid / 64
// owns local frame 4*(blockIdx.x - boff[u]) + g.  energy_all (may be null): the frame energy E_f = pspec[f][0] +
// pspec[f][1] + ... + pspec[f][256] added in fp32 in bin order, 0 replaced by eps (python_speech_features' `energy`),
// one float per frame at foff[u] + f.
__global__ void __launch_bounds__(kFbThreads)
fbank_kernel(const float* __restrict__ audio_all, const int64_t* __restrict__ soff, const int64_t* __restrict__ foff,
             const int64_t* __restrict__ boff, int U, int flen, int step, float preemph,
             const float* __restrict__ fb, int log_scale, float log_floor, float* __restrict__ feat_all,
             float* __restrict__ colsum_partial /* [gridDim.x][64] */, float* __restrict__ energy_all = nullptr) {
  __shared__ float2 buf[kFbFramesPerBlock][kFbNfft];     // complex FFT workspace per frame
  __shared__ float pspec[kFbFramesPerBlock][kFbBins + 3];
  __shared__ float rowfeat[kFbFramesPerBlock][kFbFilters];
  const int u = fbank_block_utt(boff, U, blockIdx.x);
  const float* __restrict__ audio = audio_all + soff[u];
  const int n = static_cast<int>(soff[u + 1] - soff[u]);
  const int frames = static_cast<int>(foff[u + 1] - foff[u]);
  float* __restrict__ feat = feat_all + foff[u] * kFbFilters;
  const int g = threadIdx.x >> 6, t = threadIdx.x & 63;
  const int f = static_cast<int>(blockIdx.x - boff[u]) * kFbFramesPerBlock + g;
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
  if (energy_all && live && t == 0) {
    float e = 0.f;
    for (int k = 0; k < kFbBins; ++k) e += pspec[g][k];
    energy_all[foff[u] + f] = e == 0.f ? 2.220446049250313e-16f : e;
  }
  __syncthreads();
  if (g == 0) {  // per-block column sums, fixed order
    float s = 0.f;
    for (int r = 0; r < kFbFramesPerBlock; ++r) s += rowfeat[r][t];
    colsum_partial[static_cast<long>(blockIdx.x) * kFbFilters + t] = s;
  }
}

// per-utterance mean: mean[u][m] = the utterance's own partials added in block order, in double, over its frame count.
// One thread per (u, m); grid = ceil(64 U / 256), block = 256.
__global__ void fbank_mean_kernel(const float* __restrict__ colsum_partial, const int64_t* __restrict__ foff,
                                  const int64_t* __restrict__ boff, int U, float* __restrict__ mean) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(U) * kFbFilters) return;
  const int u = static_cast<int>(i / kFbFilters), m = static_cast<int>(i % kFbFilters);
  const int frames = static_cast<int>(foff[u + 1] - foff[u]);
  double s = 0.0;
  for (long b = boff[u]; b < boff[u + 1]; ++b) s += colsum_partial[b * kFbFilters + m];
  mean[i] = static_cast<float>(s / frames);
}

// the mean subtracted in place, over the fbank grid: grid = boff[U], block = 256 (frame 4*(blockIdx.x - boff[u]) + tid/64)
__global__ void __launch_bounds__(kFbThreads)
fbank_mean_sub_kernel(float* __restrict__ feat_all, const int64_t* __restrict__ foff, const int64_t* __restrict__ boff,
                      int U, const float* __restrict__ mean) {
  const int u = fbank_block_utt(boff, U, blockIdx.x);
  const int f = static_cast<int>(blockIdx.x - boff[u]) * kFbFramesPerBlock + (threadIdx.x >> 6), m = threadIdx.x & 63;
  if (f < foff[u + 1] - foff[u]) feat_all[(foff[u] + f) * kFbFilters + m] -= mean[static_cast<long>(u) * kFbFilters + m];
}

// Regular offsets of B equal segments of L samples and T frames each: soff[u] = u L, foff[u] = u T,
// boff[u] = u ceil(T / 4) for u in [0, B].  grid = ceil((B + 1) / 256), block = 256.
__global__ void fbank_regular_offsets_kernel(int B, int L, int T, int64_t* __restrict__ soff, int64_t* __restrict__ foff,
                                             int64_t* __restrict__ boff) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u > B) return;
  soff[u] = static_cast<int64_t>(u) * L;
  foff[u] = static_cast<int64_t>(u) * T;
  boff[u] = static_cast<int64_t>(u) * ((T + kFbFramesPerBlock - 1) / kFbFramesPerBlock);
}

// SpecAugment masks of crop b on bins 4q .. 4q+3 of its row t: all four zeroed when t lies in one of the n_time time
// masks, each one zeroed when it lies in one of the n_freq frequency masks ((start, width) int32 pairs).
__device__ __forceinline__ float4 fbank_apply_masks(float4 v, int b, int t, int q, const int* __restrict__ tmask,
                                                    int n_time, const int* __restrict__ fmask, int n_freq) {
  bool tm = false;
  for (int k = 0; k < n_time; ++k) {
    const long ms = tmask[(static_cast<long>(b) * n_time + k) * 2], mw = tmask[(static_cast<long>(b) * n_time + k) * 2 + 1];
    tm |= t >= ms && t < ms + mw;
  }
  if (tm) return make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 0; k < n_freq; ++k) {
    const long fs = fmask[(static_cast<long>(b) * n_freq + k) * 2], fe = fs + fmask[(static_cast<long>(b) * n_freq + k) * 2 + 1];
    const int m = 4 * q;
    if (m >= fs && m < fe) v.x = 0.f;
    if (m + 1 >= fs && m + 1 < fe) v.y = 0.f;
    if (m + 2 >= fs && m + 2 < fe) v.z = 0.f;
    if (m + 3 >= fs && m + 3 < fe) v.w = 0.f;
  }
  return v;
}

// The masks applied in place to (B, T, 64) features; grid = B * ceil(T / 16), block = 256, as fbank_crop_kernel.
constexpr int kCropRows = 16;
__global__ void __launch_bounds__(256)
fbank_mask_kernel(float* feat, int T, const int* __restrict__ tmask, int n_time, const int* __restrict__ fmask,
                  int n_freq) {
  const int tiles = (T + kCropRows - 1) / kCropRows;
  const int b = blockIdx.x / tiles;
  const int t = (blockIdx.x - b * tiles) * kCropRows + (threadIdx.x >> 4), q = threadIdx.x & 15;
  if (t >= T) return;
  float4* p = reinterpret_cast<float4*>(feat + (static_cast<long>(b) * T + t) * kFbFilters) + q;
  *p = fbank_apply_masks(*p, b, t, q, tmask, n_time, fmask, n_freq);
}

// Crops of a CSR feature bank (frames of U utterances concatenated, utterance u = rows [foff[u], foff[u+1]) of feat):
//   out[b][t][m] = feat[foff[u] + (s + t) mod n][m],  u = utt[b], s = start[b], n = foff[u+1] - foff[u],
// zeroed where t lies in one of the crop's n_time (start, width) time masks or m in one of its n_freq frequency masks.
// u outside [0, U) or s outside [0, n): the whole crop is NaN and feat is not read.  Each 256-thread block writes 16 rows
// of one crop, one float4 per thread; grid = B * ceil(T / 16).
__global__ void __launch_bounds__(256)
fbank_crop_kernel(const float* __restrict__ feat, const int64_t* __restrict__ foff, int U, const int64_t* __restrict__ utt,
                  const int64_t* __restrict__ start, int T, const int* __restrict__ tmask, int n_time,
                  const int* __restrict__ fmask, int n_freq, float* __restrict__ out) {
  const int tiles = (T + kCropRows - 1) / kCropRows;
  const int b = blockIdx.x / tiles;
  const int t = (blockIdx.x - b * tiles) * kCropRows + (threadIdx.x >> 4), q = threadIdx.x & 15;   // bins 4q .. 4q+3
  if (t >= T) return;
  const long u = utt[b], s = start[b];
  long base = 0, n = 0;
  bool ok = u >= 0 && u < U;
  if (ok) {
    base = foff[u];
    n = foff[u + 1] - base;
    ok = s >= 0 && s < n;
  }
  float4 v;
  if (!ok) {
    const float nan = __int_as_float(0x7fc00000);
    v = make_float4(nan, nan, nan, nan);
  } else {
    v = __ldg(reinterpret_cast<const float4*>(feat + (base + (s + t) % n) * kFbFilters) + q);
    v = fbank_apply_masks(v, b, t, q, tmask, n_time, fmask, n_freq);
  }
  reinterpret_cast<float4*>(out + (static_cast<long>(b) * T + t) * kFbFilters)[q] = v;
}

}  // namespace dsk
