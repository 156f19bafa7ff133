// Agglomerative hierarchical clustering (average / complete linkage) by rounds of reciprocal-nearest-neighbour merges
// (the RAC scheme of Sumengen et al., 2021).  For a reducible linkage every pair of clusters that are each other's
// nearest cluster can be merged in the same round and the dendrogram is the one the sequential algorithm builds, so a
// round is one data-parallel pass over the live submatrix:
//
//   ahc_nn_kernel       one warp per live row: its nearest live column, ties to the smaller slot
//   ahc_decide_kernel   one block: the mutual pairs (in slot order), the threshold, the merge records, the
//                       bookkeeping of sizes and live flags, and the repack map when it is time to repack
//   ahc_update_kernel   the merged rows and columns, each entry computed once and written to (i, j) and (j, i)
//   ahc_compact_kernel  the live submatrix gathered into the other buffer (only in a repacking round)
//   ahc_finalize_kernel the per-slot arrays repacked, the stored dimension and the buffer switched
//
// Every size is read from the device-resident AhcState, so a batch of rounds is launched without the host knowing how
// many rounds are left; once `done` is set every kernel returns at once.  Slots are kept in the order of the clusters'
// representatives (smallest original index): a merge keeps the lower slot and repacking preserves order, so "ties to
// the smaller slot" is "ties to the smaller representative".  No float atomics; every value is computed by one thread
// in a fixed order, so two runs give the same bits.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace dsk {

constexpr int kAhcThreads = 256;
constexpr int kAhcDecideThreads = 1024;
constexpr int kAhcTile = 32;

struct AhcRecord {
  double height;
  int32_t rep_a, rep_b;  // the merged clusters' representatives, rep_a < rep_b
  int32_t size, round;
};

struct AhcState {
  double* mat[2];   // the working matrix (stored dimension n, row stride n) and the repack target
  int32_t cur;      // mat[cur] is live
  int32_t n;        // stored dimension
  int32_t n_active;
  int32_t M;        // pairs merged in this round
  int32_t compact;  // this round repacks into n_new slots
  int32_t n_new;
  int32_t done;
  int32_t round;
  int32_t n_rec;
  int32_t bad;      // a non-finite similarity in the upper triangle
  int32_t linkage;  // 0 average, 1 complete
  double stop_height;
};

// Per-slot arrays, all of capacity N (records N - 1).
struct AhcBufs {
  int32_t* rep;
  int32_t* size;
  int32_t* active;
  int32_t* nn;
  double* nnd;
  int32_t* pair_of;  // survivor slot -> index of its pair this round, -1 otherwise
  int32_t* pa;       // pair k: surviving slot (the lower one), merged-away slot, and their sizes before the merge
  int32_t* pb;
  int32_t* pna;
  int32_t* pnb;
  int32_t* map;      // repack: new slot -> old slot
  int32_t* tmp;      // repack scratch (2 N)
  AhcRecord* rec;
};

// D (N x N, fp64) from the strict upper triangle of S: D[i][j] = D[j][i] = 1 - (double)S[min][max], D[i][i] = 0.
// One 32 x 32 tile of S per block, for tiles on or above the diagonal; the mirrored tile is written through shared
// memory so both the read of S and the writes of D are coalesced.
__global__ void __launch_bounds__(kAhcTile * 8) ahc_init_matrix_kernel(const float* __restrict__ S, long long ld, int N,
                                                                       double* __restrict__ D, AhcState* st) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti > tj) return;
  __shared__ double t[kAhcTile][kAhcTile + 1];
  const int i0 = ti * kAhcTile, j0 = tj * kAhcTile;
  const int tx = threadIdx.x, ty = threadIdx.y;
  bool bad = false;
  for (int r = ty; r < kAhcTile; r += 8) {
    const int i = i0 + r, j = j0 + tx;
    double v = 0.0;
    if (i < N && j < N && i < j) {
      const float s = S[static_cast<long long>(i) * ld + j];
      bad |= !isfinite(s);
      v = 1.0 - static_cast<double>(s);
    }
    t[r][tx] = v;
  }
  __syncthreads();
  for (int r = ty; r < kAhcTile; r += 8) {
    const int i = i0 + r, j = j0 + tx;
    if (i < N && j < N) {
      // on a diagonal tile the lower half mirrors the upper one
      D[static_cast<size_t>(i) * N + j] = (ti == tj && r > tx) ? t[tx][r] : t[r][tx];
    }
  }
  if (ti != tj) {
    for (int r = ty; r < kAhcTile; r += 8) {
      const int i = j0 + r, j = i0 + tx;  // the mirrored tile: row j0 + r, column i0 + tx
      if (i < N && j < N) D[static_cast<size_t>(i) * N + j] = t[tx][r];
    }
  }
  if (__syncthreads_or(bad) && tx == 0 && ty == 0) st->bad = 1;
}

__global__ void ahc_init_state_kernel(AhcState* st, AhcBufs b, int N, double* mat0, double* mat1, int linkage,
                                      double stop_height) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int i = tid; i < N; i += gridDim.x * blockDim.x) {
    b.rep[i] = i;
    b.size[i] = 1;
    b.active[i] = 1;
    b.pair_of[i] = -1;
  }
  if (tid == 0) {
    st->mat[0] = mat0;
    st->mat[1] = mat1;
    st->cur = 0;
    st->n = N;
    st->n_active = N;
    st->M = 0;
    st->compact = 0;
    st->n_new = N;
    st->done = 0;
    st->round = 0;
    st->n_rec = 0;
    st->bad = 0;
    st->linkage = linkage;
    st->stop_height = stop_height;
  }
}

// Lexicographic (d, j) minimum across a warp.
__device__ __forceinline__ void ahc_warp_min(double& d, int& j) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, d, o);
    const int oj = __shfl_xor_sync(0xffffffffu, j, o);
    if (od < d || (od == d && oj < j)) {
      d = od;
      j = oj;
    }
  }
}

__global__ void __launch_bounds__(kAhcThreads) ahc_nn_kernel(AhcState* st, AhcBufs b) {
  if (st->done) return;
  const int n = st->n;
  const double* __restrict__ D = st->mat[st->cur];
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (kAhcThreads / 32);
  for (int i = blockIdx.x * (kAhcThreads / 32) + (threadIdx.x >> 5); i < n; i += warps) {
    if (!b.active[i]) continue;
    const double* row = D + static_cast<size_t>(i) * n;
    double best = __longlong_as_double(0x7ff0000000000000ll);  // +inf
    int bj = 0x7fffffff;
    for (int j = lane; j < n; j += 32) {  // ascending j per lane: strict < keeps the smaller slot on a tie
      if (j == i || !b.active[j]) continue;
      const double v = row[j];
      if (v < best) {
        best = v;
        bj = j;
      }
    }
    ahc_warp_min(best, bj);
    if (lane == 0) {
      b.nn[i] = bj;
      b.nnd[i] = best;
    }
  }
}

// Exclusive prefix sum of one int per thread over a 1024-thread block; returns the total.
__device__ __forceinline__ int ahc_block_scan(int v, int* excl, int* warp_tot) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[w] = x;
  __syncthreads();
  if (w == 0) {
    int t = warp_tot[lane];
    int s = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_tot[lane] = s - t;  // exclusive
    if (lane == 31) warp_tot[32] = s;
  }
  __syncthreads();
  *excl = warp_tot[w] + x - v;
  const int total = warp_tot[32];
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kAhcDecideThreads) ahc_decide_kernel(AhcState* st, AhcBufs b) {
  __shared__ int warp_tot[33];
  if (st->done) return;
  const int tid = threadIdx.x;
  const int n = st->n, n_active = st->n_active;
  const double stop_h = st->stop_height;
  for (int i = tid; i < n; i += kAhcDecideThreads) b.pair_of[i] = -1;
  // each thread owns a contiguous chunk of slots, so the pairs come out in slot order
  const int chunk = (n + kAhcDecideThreads - 1) / kAhcDecideThreads;
  const int c0 = min(n, tid * chunk), c1 = min(n, c0 + chunk);
  int cnt = 0;
  for (int i = c0; i < c1; ++i) {
    if (!b.active[i]) continue;
    const int j = b.nn[i];
    if (j <= i || j >= n || b.nn[j] != i || !(b.nnd[i] <= stop_h)) continue;
    ++cnt;
  }
  int excl;
  const int M = ahc_block_scan(cnt, &excl, warp_tot);
  if (M == 0) {  // the lowest mutual pair, the lowest live pair, lies above the threshold: every merge at or below it is done
    if (tid == 0) {
      st->M = 0;
      st->done = 1;
    }
    return;
  }
  for (int i = c0, k = excl; i < c1 && k < excl + cnt; ++i) {
    if (!b.active[i]) continue;
    const int j = b.nn[i];
    if (j <= i || j >= n || b.nn[j] != i || !(b.nnd[i] <= stop_h)) continue;
    b.pa[k] = i;
    b.pb[k] = j;
    ++k;
  }
  __syncthreads();
  const int round = st->round, n_rec = st->n_rec;
  for (int k = tid; k < M; k += kAhcDecideThreads) {
    const int a = b.pa[k], c = b.pb[k];
    const int na = b.size[a], nc = b.size[c];
    b.pna[k] = na;
    b.pnb[k] = nc;
    AhcRecord r;
    r.height = b.nnd[a];
    r.rep_a = b.rep[a];
    r.rep_b = b.rep[c];
    r.size = na + nc;
    r.round = round;
    b.rec[n_rec + k] = r;
    b.size[a] = na + nc;
    b.active[c] = 0;
    b.pair_of[a] = k;
  }
  const int left = n_active - M;
  const bool done = left == 1;
  const bool compact = !done && 2 * left < n;
  __syncthreads();
  if (compact) {  // new slot of every live slot, in order
    int live = 0;
    for (int i = c0; i < c1; ++i) live += b.active[i] != 0;
    int off;
    ahc_block_scan(live, &off, warp_tot);
    for (int i = c0; i < c1; ++i)
      if (b.active[i]) b.map[off++] = i;
  }
  if (tid == 0) {
    st->M = M;
    st->n_active = left;
    st->n_rec = n_rec + M;
    st->round = round + 1;
    st->compact = compact ? 1 : 0;
    st->n_new = left;
    st->done = done ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kAhcThreads) ahc_update_kernel(AhcState* st, AhcBufs b) {
  if (st->done) return;
  const int M = st->M, n = st->n, linkage = st->linkage;
  double* __restrict__ D = st->mat[st->cur];
  const long long total = static_cast<long long>(M) * n;
  for (long long idx = blockIdx.x * static_cast<long long>(kAhcThreads) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * kAhcThreads) {
    const int k = static_cast<int>(idx / n), j = static_cast<int>(idx - static_cast<long long>(k) * n);
    const int a = b.pa[k];
    if (j == a || !b.active[j]) continue;
    const int k2 = b.pair_of[j];
    if (k2 >= 0 && k2 < k) continue;  // two merged clusters: the pair of the lower slot computes their entry
    const double* ra = D + static_cast<size_t>(a) * n;
    const double* rb = D + static_cast<size_t>(b.pb[k]) * n;
    const double na = b.pna[k], nb = b.pnb[k];
    double v;
    if (k2 < 0) {  // A u B against an unmerged C
      const double dac = ra[j], dbc = rb[j];
      if (linkage == 0) {
        const double nc = b.size[j];
        v = __ddiv_rn(__dadd_rn(__dmul_rn(__dmul_rn(na, nc), dac), __dmul_rn(__dmul_rn(nb, nc), dbc)),
                      __dmul_rn(__dadd_rn(na, nb), nc));
      } else {
        v = fmax(dac, dbc);
      }
    } else {  // A u B against C u D, both merged this round; A < C, so the terms go AC, AD, BC, BD
      const int d = b.pb[k2];
      const double dac = ra[j], dad = ra[d], dbc = rb[j], dbd = rb[d];
      if (linkage == 0) {
        const double nc = b.pna[k2], nd = b.pnb[k2];
        double s = __dmul_rn(__dmul_rn(na, nc), dac);
        s = __dadd_rn(s, __dmul_rn(__dmul_rn(na, nd), dad));
        s = __dadd_rn(s, __dmul_rn(__dmul_rn(nb, nc), dbc));
        s = __dadd_rn(s, __dmul_rn(__dmul_rn(nb, nd), dbd));
        v = __ddiv_rn(s, __dmul_rn(__dadd_rn(na, nb), __dadd_rn(nc, nd)));
      } else {
        v = fmax(fmax(dac, dad), fmax(dbc, dbd));
      }
    }
    D[static_cast<size_t>(a) * n + j] = v;
    D[static_cast<size_t>(j) * n + a] = v;
  }
}

__global__ void __launch_bounds__(kAhcThreads) ahc_compact_kernel(AhcState* st, AhcBufs b) {
  if (!st->compact) return;
  const int n = st->n, m = st->n_new;
  const double* __restrict__ src = st->mat[st->cur];
  double* __restrict__ dst = st->mat[st->cur ^ 1];
  const long long total = static_cast<long long>(m) * m;
  for (long long idx = blockIdx.x * static_cast<long long>(kAhcThreads) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * kAhcThreads) {
    const int i = static_cast<int>(idx / m), j = static_cast<int>(idx - static_cast<long long>(i) * m);
    dst[idx] = src[static_cast<size_t>(b.map[i]) * n + b.map[j]];
  }
}

__global__ void __launch_bounds__(kAhcDecideThreads) ahc_finalize_kernel(AhcState* st, AhcBufs b) {
  if (!st->compact) return;
  const int m = st->n_new;
  for (int i = threadIdx.x; i < m; i += kAhcDecideThreads) {
    b.tmp[i] = b.rep[b.map[i]];
    b.tmp[m + i] = b.size[b.map[i]];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < m; i += kAhcDecideThreads) {
    b.rep[i] = b.tmp[i];
    b.size[i] = b.tmp[m + i];
    b.active[i] = 1;
  }
  if (threadIdx.x == 0) {
    st->n = m;
    st->cur ^= 1;
    st->compact = 0;
  }
}

}  // namespace dsk
