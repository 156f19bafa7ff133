// Frame-energy voice activity detection over the fbank's own frames, and the runs of kept frames of a CSR feature bank.
// The decision restates Kaldi's compute-vad rule (energy VAD as used by the VoxCeleb recipes); see include/dsk.h.
#pragma once
#include <stdint.h>

#include "fbank_kernels.cuh"

namespace dsk {

// ln E_f in fp64 for every frame, and per fbank block (4 frames of one utterance, the fbank grid's blocks) their sum in
// frame order.  One thread per block: grid = ceil(nblk / 256), block = 256.
__global__ void vad_log_energy_kernel(const float* __restrict__ energy, const int64_t* __restrict__ foff,
                                      const int64_t* __restrict__ boff, int U, int64_t nblk, double* __restrict__ loge,
                                      double* __restrict__ partial) {
  const int64_t blk = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (blk >= nblk) return;
  const int u = fbank_block_utt(boff, U, blk);
  const int64_t f0 = foff[u] + (blk - boff[u]) * kFbFramesPerBlock;
  const int64_t f1 = min(f0 + kFbFramesPerBlock, foff[u + 1]);
  double s = 0.0;
  for (int64_t f = f0; f < f1; ++f) {
    const double l = log(static_cast<double>(energy[f]));
    loge[f] = l;
    s += l;
  }
  partial[blk] = s;
}

// thr[u] = energy_threshold + mean_scale * (the utterance's block partials added in block order / n_u), as
// fbank_mean_kernel takes the feature mean: independent of the other utterances of the batch.  One thread per utterance.
__global__ void vad_threshold_kernel(const double* __restrict__ partial, const int64_t* __restrict__ foff,
                                     const int64_t* __restrict__ boff, int U, double energy_threshold, double mean_scale,
                                     double* __restrict__ thr) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= U) return;
  double s = 0.0;
  for (int64_t b = boff[u]; b < boff[u + 1]; ++b) s += partial[b];
  thr[u] = energy_threshold + mean_scale * (s / static_cast<double>(foff[u + 1] - foff[u]));
}

// speech[i] = 1 iff #{g in [max(0, f - c), min(n - 1, f + c)] : ln E_g > thr[u]} >= proportion * (window size), frame
// i = frame f of utterance u; the window never leaves the utterance.  One thread per frame: grid = ceil(F / 256).
__global__ void vad_decide_kernel(const double* __restrict__ loge, const int64_t* __restrict__ foff, int U,
                                  const double* __restrict__ thr, int64_t F, int64_t context, double proportion,
                                  uint8_t* __restrict__ speech) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const int u = fbank_block_utt(foff, U, i);     // the largest u with foff[u] <= i
  const int64_t base = foff[u], n = foff[u + 1] - base, f = i - base;
  const int64_t g0 = max(f - context, int64_t{0}), g1 = min(f + context, n - 1);
  const double t = thr[u];
  int64_t cnt = 0;
  for (int64_t g = g0; g <= g1; ++g) cnt += loge[base + g] > t;
  speech[i] = static_cast<double>(cnt) >= proportion * static_cast<double>(g1 - g0 + 1);
}

// ---- runs of kept frames ------------------------------------------------------------------------------------------------
// The K listed utterances utt[0..K) laid end to end: position p in [0, P) is local frame p - loff[j] of utterance
// utt[j], j the largest with loff[j] <= p (loff: K + 1 prefix sums of their frame counts).  A run starts at a kept frame
// that is its utterance's first or follows a dropped frame, and ends after a kept frame that is its utterance's last or
// precedes a dropped frame, so no run spans two utterances.  Each thread owns kRunItems consecutive positions of a tile
// of kRunTile; the run order is the position order, fixed by a count pass, one ordered scan of the block counts and a
// write pass that redoes the count.  No atomics.
constexpr int kRunThreads = 256;
constexpr int kRunItems = 16;
constexpr int kRunTile = kRunThreads * kRunItems;

struct RunFlags {
  bool kept, start, end;
  int64_t f;   // local frame
};

struct RunCursor {
  const uint8_t* mask;
  const int64_t *foff, *utt, *loff;
  int K;
  int64_t j, base, n;      // current list entry, its first bank row and frame count

  __device__ void seek(int64_t p) {
    int lo = 0, hi = K - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (loff[mid] <= p) lo = mid; else hi = mid - 1;
    }
    set(lo);
  }
  __device__ void set(int64_t jj) {
    j = jj;
    const int64_t u = utt[j];
    base = foff[u];
    n = foff[u + 1] - base;
  }
  __device__ RunFlags at(int64_t p) {
    while (p >= loff[j + 1]) set(j + 1);
    RunFlags r;
    r.f = p - loff[j];
    r.kept = mask[base + r.f] != 0;
    r.start = r.kept && (r.f == 0 || mask[base + r.f - 1] == 0);
    r.end = r.kept && (r.f == n - 1 || mask[base + r.f + 1] == 0);
    return r;
  }
};

// exclusive scan of one int64 per thread over the block (256 threads), in thread order; returns the block total
__device__ __forceinline__ int64_t run_block_scan(int64_t v, int64_t* sh, int64_t& excl) {
  const int t = threadIdx.x;
  sh[t] = v;
  __syncthreads();
  for (int d = 1; d < kRunThreads; d <<= 1) {
    const int64_t add = t >= d ? sh[t - d] : 0;
    __syncthreads();
    sh[t] += add;
    __syncthreads();
  }
  excl = sh[t] - v;
  const int64_t total = sh[kRunThreads - 1];
  __syncthreads();
  return total;
}

// per tile: the run starts and kept frames it holds.  grid = ceil(P / kRunTile), block = kRunThreads.
__global__ void __launch_bounds__(kRunThreads)
run_count_kernel(const uint8_t* __restrict__ mask, const int64_t* __restrict__ foff, const int64_t* __restrict__ utt,
                 const int64_t* __restrict__ loff, int K, int64_t P, int64_t* __restrict__ tile_starts,
                 int64_t* __restrict__ tile_kept) {
  __shared__ int64_t sh[kRunThreads];
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kRunTile + static_cast<int64_t>(threadIdx.x) * kRunItems;
  const int64_t p1 = min(p0 + kRunItems, P);
  int64_t starts = 0, kept = 0;
  if (p0 < P) {
    RunCursor c{mask, foff, utt, loff, K};
    c.seek(p0);
    for (int64_t p = p0; p < p1; ++p) {
      const RunFlags r = c.at(p);
      starts += r.start;
      kept += r.kept;
    }
  }
  int64_t ex;
  const int64_t ts = run_block_scan(starts, sh, ex);
  const int64_t tk = run_block_scan(kept, sh, ex);
  if (threadIdx.x == 0) {
    tile_starts[blockIdx.x] = ts;
    tile_kept[blockIdx.x] = tk;
  }
}

// exclusive prefix sums of the tile counts in tile order, in one block of kRunThreads threads (each a contiguous chunk);
// totals[0] = runs, totals[1] = kept frames; run_off[runs] = kept frames when runs <= capacity.
__global__ void __launch_bounds__(kRunThreads)
run_scan_kernel(int64_t* __restrict__ tile_starts, int64_t* __restrict__ tile_kept, int64_t ntiles, int64_t capacity,
                int64_t* __restrict__ run_off, int64_t* __restrict__ totals) {
  __shared__ int64_t sh[kRunThreads];
  const int64_t chunk = (ntiles + kRunThreads - 1) / kRunThreads;
  const int64_t b0 = min(static_cast<int64_t>(threadIdx.x) * chunk, ntiles), b1 = min(b0 + chunk, ntiles);
  int64_t s = 0, k = 0;
  for (int64_t b = b0; b < b1; ++b) {
    s += tile_starts[b];
    k += tile_kept[b];
  }
  int64_t es, ek;
  const int64_t ts = run_block_scan(s, sh, es);
  const int64_t tk = run_block_scan(k, sh, ek);
  for (int64_t b = b0; b < b1; ++b) {
    const int64_t vs = tile_starts[b], vk = tile_kept[b];
    tile_starts[b] = es;
    tile_kept[b] = ek;
    es += vs;
    ek += vk;
  }
  if (threadIdx.x == 0) {
    totals[0] = ts;
    totals[1] = tk;
    if (ts <= capacity) run_off[ts] = tk;
  }
}

// the run table: runs[r] = (j, first, end) local frames [first, end) of utterance utt[j], run_off[r] = the kept frames
// before it.  Rows at or past capacity are not written.  Same grid as run_count_kernel.
__global__ void __launch_bounds__(kRunThreads)
run_write_kernel(const uint8_t* __restrict__ mask, const int64_t* __restrict__ foff, const int64_t* __restrict__ utt,
                 const int64_t* __restrict__ loff, int K, int64_t P, const int64_t* __restrict__ tile_starts,
                 const int64_t* __restrict__ tile_kept, int64_t capacity, int64_t* __restrict__ runs,
                 int64_t* __restrict__ run_off) {
  __shared__ int64_t sh[kRunThreads];
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kRunTile + static_cast<int64_t>(threadIdx.x) * kRunItems;
  const int64_t p1 = min(p0 + kRunItems, P);
  RunCursor c{mask, foff, utt, loff, K};
  int64_t starts = 0, kept = 0;
  if (p0 < P) {
    c.seek(p0);
    for (int64_t p = p0; p < p1; ++p) {
      const RunFlags r = c.at(p);
      starts += r.start;
      kept += r.kept;
    }
  }
  int64_t es, ek;
  run_block_scan(starts, sh, es);
  run_block_scan(kept, sh, ek);
  if (p0 >= P) return;
  int64_t rs = tile_starts[blockIdx.x] + es, rk = tile_kept[blockIdx.x] + ek;   // runs started / frames kept before p
  c.seek(p0);
  for (int64_t p = p0; p < p1; ++p) {
    const RunFlags r = c.at(p);
    if (r.start) {
      if (rs < capacity) {
        runs[3 * rs] = c.j;
        runs[3 * rs + 1] = r.f;
        run_off[rs] = rk;
      }
      ++rs;
    }
    if (r.end && rs - 1 < capacity) runs[3 * (rs - 1) + 2] = r.f + 1;
    rk += r.kept;
  }
}

// rows of the new bank: row i of run r (run_off[r] <= i < run_off[r + 1]) is bank row foff[utt[j]] + first + i -
// run_off[r].  16 rows per 256-thread block, one float4 per thread; grid = ceil(rows / 16).
constexpr int kRunGatherRows = 16;
__global__ void __launch_bounds__(256)
run_gather_kernel(const float* __restrict__ feat, const int64_t* __restrict__ foff, const int64_t* __restrict__ utt,
                  const int64_t* __restrict__ runs, const int64_t* __restrict__ run_off, int64_t R, int64_t rows,
                  float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRunGatherRows + (threadIdx.x >> 4);
  const int q = threadIdx.x & 15;
  if (i >= rows) return;
  int64_t lo = 0, hi = R - 1;      // the largest r with run_off[r] <= i
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (run_off[mid] <= i) lo = mid; else hi = mid - 1;
  }
  const int64_t src = foff[utt[runs[3 * lo]]] + runs[3 * lo + 1] + (i - run_off[lo]);
  reinterpret_cast<float4*>(out + i * kFbFilters)[q] = __ldg(reinterpret_cast<const float4*>(feat + src * kFbFilters) + q);
}

}  // namespace dsk
