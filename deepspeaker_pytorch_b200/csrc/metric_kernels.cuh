// Verification-metric counting kernel: the threshold sweeps of the reference's eval_metrics.py
// (reference eval_metrics.py:16-37 calculate_roc over arange(0,30,0.01), :53-73 calculate_val over
// arange(0,30,0.001)) evaluate, for every threshold t, np.less(dist, t) against the same-speaker labels and count.
// The reference does 3 000 + 30 000 numpy passes over the distance array on the host; here one launch counts, for all
// thresholds at once, tp(t) = #{same & d < t} and fp(t) = #{different & d < t}; every other quantity of the sweep
// (tn, fn, tpr, fpr, accuracy, val, far) is integer arithmetic on these two counts plus n_same / n_diff.
// Comparison semantics = numpy's: the fp32 distance is promoted to double and compared with the double threshold,
// so the counts are exactly the reference's.
#pragma once
#include <stdint.h>

namespace dsk {

constexpr int kSweepThreads = 256;
constexpr int kSweepChunk = 2048;  // distances staged in shared memory per pass

// one thread = one threshold; the block walks all P distances through shared memory
__global__ void __launch_bounds__(kSweepThreads)
threshold_counts_kernel(const float* __restrict__ dist, const uint8_t* __restrict__ same, int P,
                        const double* __restrict__ thresholds, int nT, int32_t* __restrict__ tp,
                        int32_t* __restrict__ fp) {
  __shared__ float s_d[kSweepChunk];
  __shared__ uint8_t s_s[kSweepChunk];
  const int ti = blockIdx.x * kSweepThreads + threadIdx.x;
  const double thr = ti < nT ? thresholds[ti] : 0.0;
  int ctp = 0, cfp = 0;
  for (int base = 0; base < P; base += kSweepChunk) {
    const int n = P - base < kSweepChunk ? P - base : kSweepChunk;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kSweepThreads) {
      s_d[i] = dist[base + i];
      s_s[i] = same[base + i];
    }
    __syncthreads();
#pragma unroll 4
    for (int i = 0; i < n; ++i) {  // broadcast reads: every thread of the warp reads the same element
      const bool below = static_cast<double>(s_d[i]) < thr;
      const bool sm = s_s[i] != 0;
      ctp += (below && sm) ? 1 : 0;
      cfp += (below && !sm) ? 1 : 0;
    }
  }
  if (ti < nT) {
    tp[ti] = ctp;
    fp[ti] = cfp;
  }
}

}  // namespace dsk
