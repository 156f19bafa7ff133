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

#include "../../include/dsk.h"

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

// ---- identification: exact top-k with indices, the merge of two sorted lists, class centroids ----------------------
// The search order: a ranks above b <=> skey(a) > skey(b), or the keys are equal and a has the lower column.  -0 is
// taken as +0 and every NaN ranks below every number (-inf included).
constexpr int kSearchMaxK = DSK_SEARCH_MAX_K;

// Order-preserving key of the search: score_key for numbers (-inf has 0x007fffff), 0 for every NaN
__device__ __forceinline__ uint32_t search_key(float x) {
  if (x != x) return 0u;
  const uint32_t u = __float_as_uint(x + 0.f);  // -0 + 0 = +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// Sort entry of column c with key `key`: descending entries are in the search order (c < 2^16)
__device__ __forceinline__ unsigned long long search_entry(uint32_t key, int c) {
  return (static_cast<unsigned long long>(key) << 32) | (0xffffffffu - static_cast<uint32_t>(c));
}

// Row r of S (rows x cols, row stride ld): idx[r * ldo + i], val[r * ldo + i] for i < k are column col0 + c and value
// S[r][c] of the k first columns of the row in the search order.  1 <= k <= min(cols, kSearchMaxK), cols <= 65536.
// tau, the k-th key, comes from the radix select of topk_select_stats_kernel on search_key; every column with a key
// above tau is taken, then the kr lowest columns whose key is tau (an ordered compaction over tiles of kTopkThreads
// columns, no atomics), and the k entries are sorted by a bitonic sort in shared memory.  STAGED: the row is copied to
// dynamic shared memory (cols floats) first.  grid rows, block kTopkThreads.
template <bool STAGED>
__global__ void __launch_bounds__(kTopkThreads)
topk_indices_kernel(const float* __restrict__ S, int cols, long ld, int k, long long col0, int64_t* __restrict__ idx,
                    float* __restrict__ val, long ldo) {
  extern __shared__ float srow[];
  __shared__ unsigned long long ent[kSearchMaxK];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t wsum[kTopkThreads / 32];
  __shared__ uint32_t wcnt[2][kTopkThreads / 32];
  __shared__ uint32_t sel_digit, sel_kr;
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
  // radix select of the k-th largest key, as in topk_select_stats_kernel (NaN has a key here)
  uint32_t prefix = 0, mask = 0, kr = static_cast<uint32_t>(k);
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[tid] = 0;
    __syncthreads();
    if (shift == 24) {
      for (int c0 = 0; c0 < cols; c0 += kTopkThreads) {  // whole warps iterate together (__match_any_sync)
        const int c = c0 + tid;
        const uint32_t dig = c < cols ? search_key(x[c]) >> 24 : 256u + lane;
        const uint32_t peers = __match_any_sync(0xffffffffu, dig);
        if (dig < 256u && (__ffs(peers) - 1) == lane) atomicAdd(&hist[dig], static_cast<uint32_t>(__popc(peers)));
      }
    } else {
      for (int c = tid; c < cols; c += kTopkThreads) {
        const uint32_t key = search_key(x[c]);
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
    }
    __syncthreads();
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
    if (exc < kr && kr <= inc) {
      sel_digit = 255u - tid;
      sel_kr = kr - exc;
    }
    __syncthreads();
    prefix |= sel_digit << shift;
    mask |= 255u << shift;
    kr = sel_kr;
  }
  // emission in column order: slots [0, k - kr) take the keys above tau, slots [k - kr, k) the first kr columns at tau
  const uint32_t ngt = static_cast<uint32_t>(k) - kr, below = (1u << lane) - 1u;
  uint32_t base_gt = 0, base_eq = 0;
  // (the exit test is the same on every thread: the totals are the CTA's)
  for (int c0 = 0, par = 0; c0 < cols && !(base_gt == ngt && base_eq >= kr); c0 += kTopkThreads, par ^= 1) {
    const int c = c0 + tid;
    const uint32_t key = c < cols ? search_key(x[c]) : 0u;
    const bool gt = c < cols && key > prefix, eq = c < cols && key == prefix;
    const uint32_t bg = __ballot_sync(0xffffffffu, gt), be = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) wcnt[par][warp] = __popc(bg) | (__popc(be) << 16);
    __syncthreads();  // wcnt[par] is next written two tiles on, after every warp has passed the next barrier
    uint32_t before = 0, total = 0;
    for (int w = 0; w < kTopkThreads / 32; ++w) {
      const uint32_t v = wcnt[par][w];
      before += w < warp ? v : 0u;
      total += v;
    }
    if (gt) ent[base_gt + (before & 0xffffu) + __popc(bg & below)] = search_entry(key, c);
    if (eq) {
      const uint32_t p = base_eq + (before >> 16) + __popc(be & below);
      if (p < kr) ent[ngt + p] = search_entry(key, c);
    }
    base_gt += total & 0xffffu;
    base_eq += total >> 16;
  }
  int n = 1;
  while (n < k) n <<= 1;
  for (int i = k + tid; i < n; i += kTopkThreads) ent[i] = 0ull;  // below every entry of a column < 2^16
  __syncthreads();
  // bitonic sort, descending
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < n; i += kTopkThreads) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long a = ent[i], b = ent[j];
          if ((i & size) == 0 ? a < b : a > b) {
            ent[i] = b;
            ent[j] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  int64_t* oi = idx + static_cast<size_t>(blockIdx.x) * ldo;
  float* ov = val + static_cast<size_t>(blockIdx.x) * ldo;
  for (int i = tid; i < k; i += kTopkThreads) {
    const int c = static_cast<int>(0xffffffffu - static_cast<uint32_t>(ent[i]));
    oi[i] = col0 + c;
    ov[i] = x[c];
  }
}

// Row r: the running list idx / val [r * k, r * k + k) (sorted in the search order) and the new list nidx / nval
// [r * k, r * k + nb) (sorted, every column above the running list's) are merged; the k first entries replace the
// running list.  Ties go to the running list (its columns are lower).  Each entry's rank is its position in its own
// list plus a binary search in the other.  1 <= nb <= k <= kSearchMaxK.  grid rows, block kTopkThreads.
__global__ void __launch_bounds__(kTopkThreads)
topk_merge_kernel(int64_t* __restrict__ idx, float* __restrict__ val, const int64_t* __restrict__ nidx,
                  const float* __restrict__ nval, int k, int nb) {
  __shared__ uint32_t ak[kSearchMaxK], bk[kSearchMaxK];
  __shared__ float av[kSearchMaxK], bv[kSearchMaxK];
  __shared__ int64_t ai[kSearchMaxK], bi[kSearchMaxK];
  const size_t row = static_cast<size_t>(blockIdx.x) * k;
  for (int i = threadIdx.x; i < k; i += kTopkThreads) {
    av[i] = val[row + i];
    ai[i] = idx[row + i];
    ak[i] = search_key(av[i]);
  }
  for (int j = threadIdx.x; j < nb; j += kTopkThreads) {
    bv[j] = nval[row + j];
    bi[j] = nidx[row + j];
    bk[j] = search_key(bv[j]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < k; i += kTopkThreads) {  // new entries ranked above a[i]: keys > ak[i]
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (bk[mid] > ak[i]) lo = mid + 1; else hi = mid;
    }
    const int p = i + lo;
    if (p < k) {
      idx[row + p] = ai[i];
      val[row + p] = av[i];
    }
  }
  for (int j = threadIdx.x; j < nb; j += kTopkThreads) {  // running entries ranked above b[j]: keys >= bk[j]
    int lo = 0, hi = k;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ak[mid] >= bk[j]) lo = mid + 1; else hi = mid;
    }
    const int p = j + lo;
    if (p < k) {
      idx[row + p] = bi[j];
      val[row + p] = bv[j];
    }
  }
}

// Class s: out[s][d] = sum over u = order[offsets[s] .. offsets[s+1]) of x^_u[d] in fp64 in that order, divided by the
// count and rounded to fp32, with x^_u = X[u] / max(||X[u]||, 1e-12) in fp64 from the fp32 row (the norm one warp's
// fixed-order sum).  An empty segment gives a zero row, an index outside [0, U) a NaN row.  No float atomics.
// grid (S, ceil(D / 256)), block 256.
__global__ void __launch_bounds__(256)
class_centroids_kernel(const float* __restrict__ X, int U, int D, const int64_t* __restrict__ order,
                       const int64_t* __restrict__ offsets, float* __restrict__ out) {
  __shared__ double snrm[8];
  __shared__ int64_t srow[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = blockIdx.y * 256 + tid;
  const int64_t b = offsets[blockIdx.x], e = offsets[blockIdx.x + 1];
  double acc = 0.0;
  bool bad = false;
  for (int64_t u0 = b; u0 < e && !bad; u0 += 8) {
    const int n = e - u0 < 8 ? static_cast<int>(e - u0) : 8;
    if (warp < n) {
      const int64_t u = order[u0 + warp];
      double nr = -1.0;  // an index out of range
      if (u >= 0 && u < U) {
        const float* x = X + static_cast<size_t>(u) * D;
        double ss = 0.0;
        for (int i = lane; i < D; i += 32) {
          const double v = x[i];
          ss = fma(v, v, ss);
        }
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        nr = fmax(sqrt(ss), 1e-12);
      }
      if (lane == 0) {
        snrm[warp] = nr;
        srow[warp] = u;
      }
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
      const double nr = snrm[j];
      if (nr < 0.0) bad = true;  // the same on every thread
      else if (d < D) acc += static_cast<double>(X[static_cast<size_t>(srow[j]) * D + d]) / nr;
    }
    __syncthreads();
  }
  if (d < D)
    out[static_cast<size_t>(blockIdx.x) * D + d] =
        bad ? __int_as_float(0x7fc00000) : (e > b ? static_cast<float>(acc / static_cast<double>(e - b)) : 0.f);
}

}  // namespace dsk
