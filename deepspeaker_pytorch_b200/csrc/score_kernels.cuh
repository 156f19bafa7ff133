// Cosine scoring with adaptive score normalisation (AS-norm): the row kernels around the tensor-core cosine GEMM of
// dsk_cosine_matrix / dsk_cohort_stats (dsk_api.cu; the GEMM and its hi/lo operand images are the AAM-softmax op's,
// aam_kernels.cuh) and the trial scorer.
//
// topk_select_stats_kernel: per row, the mean and standard deviation of the k largest values.  The k-th largest value
// tau is found exactly by a radix select (four 8-bit digits, most significant first) on order-preserving uint32 keys;
// the selected multiset is every value > tau plus (k - count_gt) copies of tau, so ties do not matter.  Both moments
// are fp64 sums in a fixed order (per thread in column order, then a fixed shuffle tree, then the warps in order): no
// float atomics, the same bits on every run and for every position of the row in the matrix.
#pragma once
#include <stdint.h>

namespace dsk {

constexpr int kTopkThreads = 256;       // one CTA per row
constexpr int kTopkStageCols = 16384;   // rows up to this many columns are staged in shared memory (read from HBM once)
constexpr int kScoreWarps = 8;          // trials per 256-thread CTA of score_trials_kernel
static_assert(kTopkThreads == 256, "topk_select_stats_kernel: one thread per histogram bin");

// Order-preserving key: a < b as numbers <=> key(a) < key(b) (-0 is taken as +0; NaN is screened out before use).
__device__ __forceinline__ uint32_t score_key(float x) {
  const uint32_t u = __float_as_uint(x + 0.f);  // -0 + 0 = +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float score_unkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Sum of one double per thread over the CTA in a fixed order; every thread gets the result.
__device__ __forceinline__ double topk_block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // red may still be read from the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = red[0];
  for (int w = 1; w < kTopkThreads / 32; ++w) s += red[w];
  return s;
}

// Row r of S (rows x cols, row stride ld): mean[r], std[r] of its k largest values (2 <= k <= cols; std with divisor
// k - 1), NaN for both if the row holds a NaN.  STAGED: the row is copied to dynamic shared memory (cols floats) first.
// grid rows, block kTopkThreads.
template <bool STAGED>
__global__ void __launch_bounds__(kTopkThreads)
topk_select_stats_kernel(const float* __restrict__ S, int cols, long ld, int k, float* __restrict__ mean,
                         float* __restrict__ stdev) {
  extern __shared__ float srow[];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t wsum[kTopkThreads / 32];
  __shared__ uint32_t sel_digit, sel_kr;
  __shared__ double red[kTopkThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* g = S + static_cast<size_t>(blockIdx.x) * ld;
  const float* x = g;
  if (STAGED) {
    int c0 = 0;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
      const int n4 = cols >> 2;
      const float4* g4 = reinterpret_cast<const float4*>(g);
      float4* s4 = reinterpret_cast<float4*>(srow);
#pragma unroll 4
      for (int c = tid; c < n4; c += kTopkThreads) s4[c] = __ldg(g4 + c);
      c0 = n4 << 2;
    }
    for (int c = c0 + tid; c < cols; c += kTopkThreads) srow[c] = __ldg(g + c);
    __syncthreads();
    x = srow;
  }
  // radix select of the k-th largest key: prefix / mask are its digits found so far, kr how many of the values that
  // share them still belong to the top k
  uint32_t prefix = 0, mask = 0, kr = static_cast<uint32_t>(k);
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[tid] = 0;
    __syncthreads();
    int nan = 0;
    if (shift == 24) {
      // the top digit (sign and exponent) takes few values: one atomic per distinct digit in the warp
      for (int c0 = 0; c0 < cols; c0 += kTopkThreads) {  // whole warps iterate together (__match_any_sync)
        const int c = c0 + tid;
        uint32_t dig = 256u + lane;
        if (c < cols) {
          const float v = x[c];
          nan |= v != v;
          dig = score_key(v) >> 24;
        }
        const uint32_t peers = __match_any_sync(0xffffffffu, dig);
        if (dig < 256u && (__ffs(peers) - 1) == lane) atomicAdd(&hist[dig], static_cast<uint32_t>(__popc(peers)));
      }
    } else {
      // later digits spread out, and most values no longer share the prefix
      for (int c = tid; c < cols; c += kTopkThreads) {
        const uint32_t key = score_key(x[c]);
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
    }
    if (shift == 24) {
      if (__syncthreads_or(nan)) {
        if (tid == 0) mean[blockIdx.x] = stdev[blockIdx.x] = __int_as_float(0x7fc00000);
        return;
      }
    } else {
      __syncthreads();
    }
    // inclusive scan of the counts from the top digit down: thread t holds digit 255 - t
    const uint32_t cnt = hist[255 - tid];
    uint32_t inc = cnt;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    for (int w = 0; w < warp; ++w) inc += wsum[w];
    const uint32_t exc = inc - cnt;
    if (exc < kr && kr <= inc) {  // exactly one digit holds the kr-th largest remaining value
      sel_digit = 255u - tid;
      sel_kr = kr - exc;
    }
    __syncthreads();
    prefix |= sel_digit << shift;
    mask |= 255u << shift;
    kr = sel_kr;
  }
  // prefix is the key of tau; kr copies of tau complete the k - kr values above it
  const double tau = score_unkey(prefix);
  double s = 0.0;
  for (int c = tid; c < cols; c += kTopkThreads) {
    const float v = x[c];
    if (score_key(v) > prefix) s += v;
  }
  s = topk_block_sum(s, red);
  const double mu = (s + static_cast<double>(kr) * tau) / k;
  double q = 0.0;
  for (int c = tid; c < cols; c += kTopkThreads) {
    const float v = x[c];
    if (score_key(v) > prefix) {
      const double d = v - mu;
      q += d * d;
    }
  }
  q = topk_block_sum(q, red);
  if (tid == 0) {
    const double d = tau - mu;
    mean[blockIdx.x] = static_cast<float>(mu);
    stdev[blockIdx.x] = static_cast<float>(sqrt((q + static_cast<double>(kr) * (d * d)) / (k - 1)));
  }
}

// Trial t = (e, u): raw[t] = x^_e . x^_u in fp64 from the fp32 rows (x^ = x / max(||x||, 1e-12)), and, when mean is
// non-NULL, normed[t] = 0.5 ((s - mean[e]) / std[e] + (s - mean[u]) / std[u]) in fp64 from the unrounded s.  An index
// outside [0, U) gives NaN in both and reads nothing.  One warp per trial, fixed order.  grid ceil(T / 8), block 256.
__global__ void __launch_bounds__(256)
score_trials_kernel(const float* __restrict__ X, int U, int D, const int64_t* __restrict__ trials, long long T,
                    const float* __restrict__ mean, const float* __restrict__ stdev, float* __restrict__ raw,
                    float* __restrict__ normed) {
  const long long t = static_cast<long long>(blockIdx.x) * kScoreWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int64_t e = trials[2 * t], u = trials[2 * t + 1];
  if (e < 0 || e >= U || u < 0 || u >= U) {
    if (lane == 0) {
      raw[t] = __int_as_float(0x7fc00000);
      if (mean) normed[t] = __int_as_float(0x7fc00000);
    }
    return;
  }
  const float* a = X + static_cast<size_t>(e) * D;
  const float* b = X + static_cast<size_t>(u) * D;
  double ab = 0.0, aa = 0.0, bb = 0.0;
  for (int d = lane; d < D; d += 32) {
    const double ad = a[d], bd = b[d];
    ab = fma(ad, bd, ab);
    aa = fma(ad, ad, aa);
    bb = fma(bd, bd, bb);
  }
  for (int o = 16; o > 0; o >>= 1) {
    ab += __shfl_xor_sync(0xffffffffu, ab, o);
    aa += __shfl_xor_sync(0xffffffffu, aa, o);
    bb += __shfl_xor_sync(0xffffffffu, bb, o);
  }
  if (lane != 0) return;
  const double s = ab / (fmax(sqrt(aa), 1e-12) * fmax(sqrt(bb), 1e-12));
  raw[t] = static_cast<float>(s);
  if (mean)
    normed[t] = static_cast<float>(0.5 * ((s - mean[e]) / static_cast<double>(stdev[e]) +
                                          (s - mean[u]) / static_cast<double>(stdev[u])));
}

}  // namespace dsk
