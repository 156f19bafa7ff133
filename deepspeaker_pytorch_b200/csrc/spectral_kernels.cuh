// Spectral clustering with NME-SC speaker counting (Park et al., IEEE SPL 2020): one call per recording, every pruning
// level p of the grid solved in the same launches.  oracle/spectral_oracle.py states the algorithm.
//
//   sc_rank_kernel     one CTA per row: for every p_t of the grid the exact threshold of the row's top p_t (a radix
//                      select of the p_t-th largest key, then the column of the last tied entry taken), and per column
//                      the code c_ij = the first t whose top p_t holds j (n_p if none)
//   sc_pair_kernel     W[i][j] = lo | hi << 8, lo / hi the min / max of c_ij and c_ji, so that
//                      A_{p_t}[i][j] = ([lo <= t] + [hi <= t]) / 2 for every t from one symmetric uint16 matrix
//   sc_degree_kernel   one CTA per row: d_i for every t from integer histograms of lo and hi
//   sc_setup_kernel    one CTA per problem: up = 2 max_i d_i (a Gershgorin bound of the spectrum)
// then per problem (t, kind): kind 0 wants the smallest eigenpairs of L_t, kind 1 the largest (as the smallest of
// up I - L_t), by Chebyshev-filtered subspace iteration (Zhou & Saad 2007) on a block of w columns:
//   sc_matvec_kernel   out = alpha Op(in) + beta in + gamma prev, Op(x) = D x - A x (or up x - D x + A x), the dense
//                      A tile decoded from W; fp64 FMA on the CUDA cores in a fixed order
//   sc_gram_kernel     the w x w partials of Xa^T Xb over splits of kScSplitRows rows
//   sc_resid_kernel    the per-column partials of |z - theta x|^2
//   sc_small_kernel    one CTA per problem: the partials summed in split order, then a (shifted) Cholesky and R^-1,
//                      or the Rayleigh-Ritz eigenproblem by cyclic Jacobi, or the convergence test and the next
//                      filter's cutoff and degree
//   sc_apply_kernel    out = in M for the w x w matrix of sc_small_kernel
//   sc_select_kernel   step 4 over the grid; sc_kmeans_kernel step 6 in one CTA
// No float atomics; every sum has a fixed order, so a call gives the same bits every time.  Problems that have
// converged are skipped by every later launch, so their Ritz vectors stay where the last check left them.
#pragma once
#include <stdint.h>

#include "score_kernels.cuh"

namespace dsk {

constexpr int kScGuard = 8;         // block columns beyond the wanted m, at least
constexpr int kScMinB = 40;         // and at least this many: a wider block moves the cutoff away from lambda_m
constexpr int kScTopWidth = 8;      // block width of the largest-eigenvalue problems
constexpr int kScMaxB = 48;         // >= DSK_SC_MAX_SPEAKERS + 1 + kScGuard
constexpr int kScRows = 64;         // matvec row tile
constexpr int kScK = 32;            // matvec K stage
constexpr int kScThreads = 256;
constexpr int kScSplitRows = 256;   // rows per partial of the Gram and residual passes
constexpr int kScMaxOuter = 1000;   // subspace iterations before a problem is declared not converged
constexpr int kScMaxDegree = 40;    // filter degree cap
constexpr double kScTol = 1e-10;    // every wanted residual ends <= kScTol * up

struct ScProb {
  int32_t t;      // grid index
  int32_t top;    // 0: smallest eigenpairs of L, 1: largest (smallest of up I - L)
  int32_t w;      // block width
  int32_t want;   // columns that must converge
  int32_t conv;
  int32_t deg;    // degree of the next filter
  int32_t iters;
  int32_t failed;
  int32_t lock;   // leading columns converged by residual: the filter leaves them as they are
  int32_t pad;
  double up;      // 2 max_i d_i
  double a;       // filter cutoff
  double res;     // largest wanted residual / up at the last check
};

// ---- ranks ---------------------------------------------------------------------------------------------------------
// Row i: keys in dynamic shared memory (N uint32, the diagonal 0 so it sorts last); bad set on a non-finite
// off-diagonal value.  grid N, block kScThreads.
__global__ void __launch_bounds__(kScThreads)
sc_rank_kernel(const float* __restrict__ S, int N, long long ld, const int32_t* __restrict__ pv, int n_p,
               uint8_t* __restrict__ code, int32_t* __restrict__ bad) {
  extern __shared__ uint32_t key[];
  __shared__ uint32_t hist[256], wsum[kScThreads / 32], wcnt[kScThreads / 32];
  __shared__ uint32_t sel_digit, sel_kr, tau[64];
  __shared__ int32_t colt[64];
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = S + static_cast<long long>(i) * ld;
  int nonfinite = 0;
  for (int c = tid; c < N; c += kScThreads) {
    const float v = row[c];
    if (c != i) nonfinite |= !isfinite(v);
    key[c] = c == i ? 0u : score_key(v);
  }
  if (__syncthreads_or(nonfinite)) {
    if (tid == 0) atomicOr(bad, 1);
    return;
  }
  for (int t = 0; t < n_p; ++t) {
    // radix select of the p_t-th largest key (as topk_select_stats_kernel)
    uint32_t prefix = 0, mask = 0, kr = static_cast<uint32_t>(pv[t]);
    for (int shift = 24; shift >= 0; shift -= 8) {
      hist[tid] = 0;
      __syncthreads();
      for (int c = tid; c < N; c += kScThreads) {
        const uint32_t k = key[c];
        if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
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
      __syncthreads();
    }
    // the kr-th column (in column order) whose key is tau: the last one in the top p_t
    uint32_t base = 0;
    for (int c0 = 0; c0 < N; c0 += kScThreads) {
      const int c = c0 + tid;
      const bool eq = c < N && key[c] == prefix;
      const uint32_t be = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) wcnt[warp] = __popc(be);
      __syncthreads();
      uint32_t before = 0, total = 0;
      for (int w = 0; w < kScThreads / 32; ++w) {
        before += w < warp ? wcnt[w] : 0u;
        total += wcnt[w];
      }
      if (eq && base + before + __popc(be & ((1u << lane) - 1u)) + 1 == kr) colt[t] = c;
      base += total;
      __syncthreads();
      if (base >= kr) break;
    }
    if (tid == 0) tau[t] = prefix;
    __syncthreads();
  }
  // code: the first t whose top p_t holds column c (the sets grow with t), n_p if none
  uint8_t* out = code + static_cast<size_t>(i) * N;
  for (int c = tid; c < N; c += kScThreads) {
    const uint32_t k = key[c];
    int lo = 0, hi = n_p;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (k > tau[mid] || (k == tau[mid] && c <= colt[mid])) hi = mid;
      else lo = mid + 1;
    }
    out[c] = static_cast<uint8_t>(c == i ? n_p : lo);
  }
}

// W[i][j] = min(c_ij, c_ji) | max(c_ij, c_ji) << 8 through a 32 x 32 shared tile.  grid (tiles, tiles), block (32, 8).
__global__ void sc_pair_kernel(const uint8_t* __restrict__ code, int N, uint16_t* __restrict__ W) {
  __shared__ uint8_t tr[32][33];
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  for (int r = ty; r < 32; r += 8) {  // the transposed tile: code[j0 + r][i0 + tx]
    const int a = j0 + r, b = i0 + tx;
    tr[r][tx] = (a < N && b < N) ? code[static_cast<size_t>(a) * N + b] : 0;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int i = i0 + r, j = j0 + tx;
    if (i >= N || j >= N) continue;
    const uint32_t x = code[static_cast<size_t>(i) * N + j], y = tr[tx][r];
    W[static_cast<size_t>(i) * N + j] = static_cast<uint16_t>(min(x, y) | (max(x, y) << 8));
  }
}

// deg[t][i] = sum_j ([lo_ij <= t] + [hi_ij <= t]) / 2 from integer histograms.  grid N, block kScThreads.
__global__ void __launch_bounds__(kScThreads)
sc_degree_kernel(const uint16_t* __restrict__ W, int N, int n_p, double* __restrict__ deg) {
  __shared__ uint32_t hl[65], hh[65];
  const int i = blockIdx.x, tid = threadIdx.x;
  if (tid < 65) hl[tid] = hh[tid] = 0;
  __syncthreads();
  const uint16_t* row = W + static_cast<size_t>(i) * N;
  for (int c = tid; c < N; c += kScThreads) {
    const uint32_t v = row[c];
    atomicAdd(&hl[v & 255u], 1u);
    atomicAdd(&hh[v >> 8], 1u);
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t cl = 0, ch = 0;
    for (int t = 0; t < n_p; ++t) {
      cl += hl[t];
      ch += hh[t];
      deg[static_cast<size_t>(t) * N + i] = 0.5 * (static_cast<double>(cl) + static_cast<double>(ch));
    }
  }
}

// Problem q: t = q % n_p, kind q / n_p; up = 2 max_i deg[t][i].  grid 2 n_p, block kScThreads.
__global__ void __launch_bounds__(kScThreads)
sc_setup_kernel(const double* __restrict__ deg, int N, int n_p, int m, int b, ScProb* __restrict__ probs) {
  __shared__ double red[kScThreads];
  const int q = blockIdx.x, t = q % n_p, tid = threadIdx.x;
  double mx = 0.0;
  for (int i = tid; i < N; i += kScThreads) mx = fmax(mx, deg[static_cast<size_t>(t) * N + i]);
  red[tid] = mx;
  __syncthreads();
  for (int o = kScThreads / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] = fmax(red[tid], red[tid + o]);
    __syncthreads();
  }
  if (tid == 0) {
    ScProb p;
    p.t = t;
    p.top = q >= n_p;
    p.w = p.top ? min(kScTopWidth, N) : b;
    p.want = p.top ? 1 : m;
    p.conv = 0;
    p.deg = 0;
    p.iters = 0;
    p.failed = 0;
    p.lock = 0;
    p.pad = 0;
    p.up = 2.0 * red[0];
    p.a = 0.0;
    p.res = 0.0;
    probs[q] = p;
  }
}

// Deterministic start: X[q][r][c] = a counter-based hash of (r, c) in [-1, 1) for c < w, 0 beyond.
__global__ void sc_init_kernel(double* __restrict__ X, int N, int B, const ScProb* __restrict__ probs) {
  const int q = blockIdx.y, w = probs[q].w;
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<long long>(N) * B) return;
  const int c = static_cast<int>(e % B);
  unsigned long long z = static_cast<unsigned long long>(e / B) * 0x9e3779b97f4a7c15ull + (c + 1) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  z ^= z >> 31;
  X[static_cast<size_t>(q) * N * B + e] = c < w ? static_cast<double>(z >> 11) * 0x1.0p-52 - 1.0 : 0.0;
}

__device__ __forceinline__ double sc_weight(uint32_t v, int t) {
  return 0.5 * (static_cast<double>((v & 255u) <= static_cast<uint32_t>(t)) +
                static_cast<double>((v >> 8) <= static_cast<uint32_t>(t)));
}

// Chebyshev step `step` of the scaled filter on [a, up] with the value at 0 kept at 1: the coefficients of
// out = alpha Op(in) + beta in + gamma prev.  step < 0: out = Op(in).
__device__ __forceinline__ void sc_cheb_coef(const ScProb& p, int step, double& alpha, double& beta, double& gamma) {
  if (step < 0) {
    alpha = 1.0;
    beta = gamma = 0.0;
    return;
  }
  const double e = 0.5 * (p.up - p.a), c = 0.5 * (p.up + p.a), s1 = -e / c;
  double s = s1;
  alpha = s1 / e;
  beta = -s1 * c / e;
  gamma = 0.0;
  for (int j = 1; j <= step; ++j) {
    const double sn = 1.0 / (2.0 / s1 - s);
    alpha = 2.0 * sn / e;
    beta = -2.0 * sn * c / e;
    gamma = -s * sn;
    s = sn;
  }
}

// One K stage of the matvec: thread (ty, tx) adds to rows 4 ty .. 4 ty + 3 and columns tx + 16 jj, jj < SLOTS.
template <int SLOTS>
__device__ __forceinline__ void sc_matvec_stage(const double (*wt)[kScK + 1], const double (*xs)[kScMaxB], int ty,
                                                int tx, double (&acc)[4][3]) {
#pragma unroll 8
  for (int k = 0; k < kScK; ++k) {
    double a[4], x[SLOTS];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) a[ii] = wt[4 * ty + ii][k];
#pragma unroll
    for (int jj = 0; jj < SLOTS; ++jj) x[jj] = xs[k][tx + 16 * jj];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int jj = 0; jj < SLOTS; ++jj) acc[ii][jj] = fma(a[ii], x[jj], acc[ii][jj]);
  }
}

// grid (P, ceil(N / kScRows)), block kScThreads: thread (ty, tx) owns rows 4 ty .. 4 ty + 3 of the tile and columns
// tx, tx + 16, tx + 32, of which only the ceil(w / 16) slots the block uses are computed.  A step at or past the problem's degree copies in to out.
__global__ void __launch_bounds__(kScThreads, 2)
sc_matvec_kernel(const uint16_t* __restrict__ W, const double* __restrict__ deg, const ScProb* __restrict__ probs,
                 int N, int B, int step, const double* __restrict__ in_all, const double* __restrict__ prev_all,
                 double* __restrict__ out_all) {
  __shared__ double wt[kScRows][kScK + 1];
  __shared__ double xs[kScK][kScMaxB];
  const int q = blockIdx.x;
  const ScProb p = probs[q];
  if (p.conv || p.failed) return;
  const int i0 = blockIdx.y * kScRows, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, w = p.w;
  const size_t base = static_cast<size_t>(q) * N * B;
  const double* in = in_all + base;
  double* out = out_all + base;
  if (step >= p.deg) {
    for (int e = tid; e < kScRows * B; e += kScThreads) {
      const int r = i0 + e / B;
      if (r < N) out[static_cast<size_t>(r) * B + e % B] = in[static_cast<size_t>(r) * B + e % B];
    }
    return;
  }
  double alpha, beta, gamma;
  sc_cheb_coef(p, step, alpha, beta, gamma);
  const int slots = (w + 15) / 16;  // column slots of 16 the block needs (1 for the largest-eigenvalue problems)
  double acc[4][3] = {};
  for (int j0 = 0; j0 < N; j0 += kScK) {
    for (int e = tid; e < kScRows * kScK; e += kScThreads) {
      const int r = e / kScK, k = e % kScK, i = i0 + r, j = j0 + k;
      wt[r][k] = (i < N && j < N) ? sc_weight(W[static_cast<size_t>(i) * N + j], p.t) : 0.0;
    }
    for (int e = tid; e < kScK * slots * 16; e += kScThreads) {
      const int k = e / (slots * 16), c = e % (slots * 16), j = j0 + k;
      xs[k][c] = (j < N && c < w) ? in[static_cast<size_t>(j) * B + c] : 0.0;
    }
    __syncthreads();
    if (slots == 1) {
      sc_matvec_stage<1>(wt, xs, ty, tx, acc);
    } else if (slots == 2) {
      sc_matvec_stage<2>(wt, xs, ty, tx, acc);
    } else {
      sc_matvec_stage<3>(wt, xs, ty, tx, acc);
    }
    __syncthreads();
  }
  const double* d = deg + static_cast<size_t>(p.t) * N;
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const int r = i0 + 4 * ty + ii;
    if (r >= N) continue;
    const double dr = d[r];
#pragma unroll
    for (int jj = 0; jj < 3; ++jj) {
      const int c = tx + 16 * jj;
      if (c >= w) continue;
      const size_t o = static_cast<size_t>(r) * B + c;
      const double xi = in[o];
      const double op = p.top ? (p.up - dr) * xi + acc[ii][jj] : dr * xi - acc[ii][jj];
      double v = alpha * op + beta * xi;
      if (gamma != 0.0) v += gamma * prev_all[base + o];
      out[o] = (step >= 0 && c < p.lock) ? xi : v;
    }
  }
}

// part[q][s][r][c] = sum over the rows u of split s, in order, of Xa[u][r] Xb[u][c] (r, c < w).
// grid (P, splits), block kScThreads.
__global__ void __launch_bounds__(kScThreads)
sc_gram_kernel(const double* __restrict__ Xa, const double* __restrict__ Xb, int N, int B,
               const ScProb* __restrict__ probs, double* __restrict__ part) {
  __shared__ double sa[kScK][kScMaxB], sb[kScK][kScMaxB];
  const int q = blockIdx.x, s = blockIdx.y, tid = threadIdx.x;
  const ScProb p = probs[q];
  if (p.conv || p.failed) return;
  const int w = p.w, u0 = s * kScSplitRows, u1 = min(N, u0 + kScSplitRows);
  const size_t base = static_cast<size_t>(q) * N * B;
  double acc[7] = {};  // entries tid + 256 e of the w x w block (w <= 41: 1681 <= 7 * 256)
  for (int k0 = u0; k0 < u1; k0 += kScK) {
    for (int e = tid; e < kScK * B; e += kScThreads) {
      const int k = e / B, c = e % B, u = k0 + k;
      sa[k][c] = u < u1 ? Xa[base + static_cast<size_t>(u) * B + c] : 0.0;
      sb[k][c] = u < u1 ? Xb[base + static_cast<size_t>(u) * B + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 7; ++e) {
      const int idx = tid + kScThreads * e;
      if (idx >= w * w) break;
      const int r = idx / w, c = idx % w;
      double v = acc[e];
      for (int k = 0; k < kScK; ++k) v = fma(sa[k][r], sb[k][c], v);
      acc[e] = v;
    }
    __syncthreads();
  }
  double* out = part + (static_cast<size_t>(q) * gridDim.y + s) * (kScMaxB * kScMaxB);
#pragma unroll
  for (int e = 0; e < 7; ++e) {
    const int idx = tid + kScThreads * e;
    if (idx < w * w) out[idx] = acc[e];
  }
}

// part[q][s][c] = sum over the rows of split s of (Z[u][c] - theta_c X[u][c])^2.  grid (P, splits), block kScMaxB.
__global__ void sc_resid_kernel(const double* __restrict__ X, const double* __restrict__ Z, int N, int B,
                                const ScProb* __restrict__ probs, const double* __restrict__ theta,
                                double* __restrict__ part) {
  const int q = blockIdx.x, s = blockIdx.y, c = threadIdx.x;
  const ScProb p = probs[q];
  if (p.conv || p.failed || c >= p.w) return;
  const double th = theta[q * kScMaxB + c];
  const size_t base = static_cast<size_t>(q) * N * B;
  double v = 0.0;
  for (int u = s * kScSplitRows; u < min(N, (s + 1) * kScSplitRows); ++u) {
    const double r = Z[base + static_cast<size_t>(u) * B + c] - th * X[base + static_cast<size_t>(u) * B + c];
    v = fma(r, r, v);
  }
  part[(static_cast<size_t>(q) * gridDim.y + s) * (kScMaxB * kScMaxB) + c] = v;
}

constexpr int kScModeChol = 0, kScModeRR = 1, kScModeRes = 2;

// One CTA per problem.  grid P, block kScThreads.
//   kScModeChol: G = sum of the partials; R^T R = G (+ s I when a pivot is not positive, the shift of shifted
//                CholeskyQR, Fukaya et al. 2020); mat = R^-1.
//   kScModeRR:   H = (G + G^T) / 2, cyclic Jacobi (one warp); theta ascending, mat = the eigenvectors in that order.
//   kScModeRes:  residual norms; conv when every wanted one is <= kScTol up; the next cutoff and degree.
__global__ void __launch_bounds__(kScThreads)
sc_small_kernel(const double* __restrict__ part, int splits, int N, ScProb* __restrict__ probs, int mode,
                double* __restrict__ mat_all, double* __restrict__ theta_all) {
  __shared__ double G[kScMaxB][kScMaxB + 1], V[kScMaxB][kScMaxB + 1];
  __shared__ int perm[kScMaxB];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  ScProb p = probs[q];
  if (p.conv || p.failed) return;
  const int w = p.w;
  const double* src = part + static_cast<size_t>(q) * splits * (kScMaxB * kScMaxB);
  double* mat = mat_all + static_cast<size_t>(q) * (kScMaxB * kScMaxB);
  double* theta = theta_all + q * kScMaxB;
  const int n_ent = mode == kScModeRes ? w : w * w;
  for (int e = tid; e < n_ent; e += kScThreads) {
    double v = 0.0;
    for (int s = 0; s < splits; ++s) v += src[static_cast<size_t>(s) * (kScMaxB * kScMaxB) + e];
    if (mode == kScModeRes) G[0][e] = v;
    else G[e / w][e % w] = v;
  }
  __syncthreads();
  if (mode == kScModeRes) {
    if (tid == 0) {
      double mx = 0.0;
      bool leading = true;
      int lock = 0;
      for (int c = 0; c < p.want; ++c) {
        const double r = sqrt(G[0][c]) / p.up;
        mx = fmax(mx, r);
        leading &= r <= kScTol;
        if (leading) lock = c + 1;
      }
      const bool done = mx <= kScTol;
      p.lock = min(lock, p.want - 1);
      p.res = mx;
      p.iters += 1;
      p.conv = done || w == N;
      if (!p.conv && p.iters >= kScMaxOuter) p.failed = 1;
      // the cutoff sits a little above the block's top Ritz value: when a cluster of equal eigenvalues reaches past
      // the block, a cutoff on the cluster itself would damp the components just above it no more than the
      // cluster's own, and the wanted columns would stop converging
      const double a = fmin(fmax(theta[w - 1] + 1e-3 * p.up, 0.01 * p.up), 0.99 * p.up);
      p.a = a;
      // degree: the first unlocked Ritz value amplified by at most ~1e6 over the cutoff (the active columns stay
      // well conditioned), and 0 by at most ~1e12: the locked directions regrow in the active columns from rounding
      // to no more than 1e-4 of them, and the three CholeskyQR passes, whose Gram puts the locked columns first,
      // project them out again (block Gram-Schmidt against the locked vectors, repeated)
      const double lo = fmin(fmax(theta[p.lock], 0.0), a);
      const double t_lo = (p.up + a - 2.0 * lo) / (p.up - a), t0 = (p.up + a) / (p.up - a);
      const double d1 = t_lo > 1.0 ? 14.5 / acosh(t_lo) : 1e9, d2 = 28.4 / acosh(t0);
      p.deg = max(1, min(kScMaxDegree, static_cast<int>(floor(fmin(d1, d2)))));
      probs[q] = p;
    }
    return;
  }
  if (mode == kScModeChol) {
    if (tid == 0) {
      double tr = 0.0;
      for (int i = 0; i < w; ++i) tr += G[i][i];
      double shift = 0.0;
      for (int attempt = 0; attempt < 2; ++attempt) {
        bool ok = true;
        for (int j = 0; j < w && ok; ++j) {  // upper R in V: G = R^T R
          double s = G[j][j] + shift;
          for (int k = 0; k < j; ++k) s -= V[k][j] * V[k][j];
          if (!(s > 0.0)) {
            ok = false;
            break;
          }
          const double rjj = sqrt(s);
          V[j][j] = rjj;
          for (int i = j + 1; i < w; ++i) {
            double x = G[j][i];
            for (int k = 0; k < j; ++k) x -= V[k][j] * V[k][i];
            V[j][i] = x / rjj;
          }
        }
        if (ok) break;
        shift = 11.0 * (static_cast<double>(N) * w + w * (w + 1.0)) * 1.1102230246251565e-16 * tr;
      }
      // R^-1 (upper) into G, column by column: R x = e_j
      for (int j = 0; j < w; ++j)
        for (int i = w - 1; i >= 0; --i) {
          double x = i == j ? 1.0 : 0.0;
          for (int k = i + 1; k <= j; ++k) x -= V[i][k] * G[k][j];
          G[i][j] = i > j ? 0.0 : x / V[i][i];
        }
    }
    __syncthreads();
    for (int e = tid; e < w * w; e += kScThreads) mat[e] = G[e / w][e % w];
    return;
  }
  // Rayleigh-Ritz: symmetrise, V = I, cyclic Jacobi sweeps by warp 0
  for (int e = tid; e < w * w; e += kScThreads) V[e / w][e % w] = 0.5 * (G[e / w][e % w] + G[e % w][e / w]);
  __syncthreads();
  for (int e = tid; e < w * w; e += kScThreads) {
    const int r = e / w, c = e % w;
    G[r][c] = V[r][c];
  }
  __syncthreads();
  for (int e = tid; e < w * w; e += kScThreads) {
    const int r = e / w, c = e % w;
    V[r][c] = r == c ? 1.0 : 0.0;
  }
  __syncthreads();
  if (tid < 32) {
    for (int sweep = 0; sweep < 30; ++sweep) {
      double off = 0.0, diag = 0.0;
      for (int e = lane; e < w * w; e += 32) {
        const int r = e / w, c = e % w;
        if (r != c) off += G[r][c] * G[r][c];
        else diag += G[r][c] * G[r][c];
      }
      for (int o = 16; o > 0; o >>= 1) {
        off += __shfl_xor_sync(0xffffffffu, off, o);
        diag += __shfl_xor_sync(0xffffffffu, diag, o);
      }
      off = __shfl_sync(0xffffffffu, off, 0);
      diag = __shfl_sync(0xffffffffu, diag, 0);
      if (off <= 1e-36 * diag || off == 0.0) break;
      for (int a = 0; a < w - 1; ++a)
        for (int b = a + 1; b < w; ++b) {
          const double hab = G[a][b];
          if (hab == 0.0) continue;
          const double haa = G[a][a], hbb = G[b][b];
          const double th = (hbb - haa) / (2.0 * hab);
          const double t = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
          const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
          __syncwarp();
          for (int k = lane; k < w; k += 32) {  // columns a, b of G
            const double ga = G[k][a], gb = G[k][b];
            G[k][a] = c * ga - s * gb;
            G[k][b] = s * ga + c * gb;
          }
          __syncwarp();
          for (int k = lane; k < w; k += 32) {  // rows a, b of G
            const double ga = G[a][k], gb = G[b][k];
            G[a][k] = c * ga - s * gb;
            G[b][k] = s * ga + c * gb;
          }
          for (int k = lane; k < w; k += 32) {
            const double va = V[k][a], vb = V[k][b];
            V[k][a] = c * va - s * vb;
            V[k][b] = s * va + c * vb;
          }
          __syncwarp();
        }
    }
    if (lane == 0) {  // ascending order, ties to the lower index
      for (int i = 0; i < w; ++i) perm[i] = i;
      for (int i = 0; i < w; ++i) {
        int best = i;
        for (int j = i + 1; j < w; ++j)
          if (G[perm[j]][perm[j]] < G[perm[best]][perm[best]]) best = j;
        const int tmp = perm[i];
        perm[i] = perm[best];
        perm[best] = tmp;
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < w * w; e += kScThreads) mat[e] = V[e / w][perm[e % w]];
  for (int c = tid; c < w; c += kScThreads) theta[c] = G[perm[c]][perm[c]];
}

// out[u][c] = sum_r in[u][r] mat[r][c] for c < w.  grid (P, ceil(N / kScRows)), block kScThreads.
__global__ void __launch_bounds__(kScThreads)
sc_apply_kernel(const double* __restrict__ in_all, double* __restrict__ out_all, int N, int B,
                const ScProb* __restrict__ probs, const double* __restrict__ mat_all) {
  __shared__ double M[kScMaxB * kScMaxB];
  __shared__ double xs[kScRows][kScMaxB + 1];
  const int q = blockIdx.x, tid = threadIdx.x;
  const ScProb p = probs[q];
  if (p.conv || p.failed) return;
  const int w = p.w, i0 = blockIdx.y * kScRows;
  const size_t base = static_cast<size_t>(q) * N * B;
  for (int e = tid; e < w * w; e += kScThreads) M[e] = mat_all[static_cast<size_t>(q) * (kScMaxB * kScMaxB) + e];
  for (int e = tid; e < kScRows * w; e += kScThreads) {
    const int r = e / w, c = e % w, u = i0 + r;
    xs[r][c] = u < N ? in_all[base + static_cast<size_t>(u) * B + c] : 0.0;
  }
  __syncthreads();
  for (int e = tid; e < kScRows * w; e += kScThreads) {
    const int r = e / w, c = e % w, u = i0 + r;
    if (u >= N) continue;
    double v = 0.0;
    for (int k = 0; k < w; ++k) v = fma(xs[r][k], M[k * w + c], v);
    out_all[base + static_cast<size_t>(u) * B + c] = v;
  }
}

// Step 4: eig (n_p, m) = the bottom Ritz values, lmax (n_p) = up - the top problem's least Ritz value, ratio (n_p);
// sel = {k, t}.  num_speakers 0: estimate.  grid 1, block 1.
__global__ void sc_select_kernel(const ScProb* __restrict__ probs, const double* __restrict__ theta, int n_p, int m,
                                 int N, const int32_t* __restrict__ pv, int num_speakers, double* __restrict__ eig,
                                 double* __restrict__ lmax, double* __restrict__ ratio, int32_t* __restrict__ sel) {
  double best = 0.0;
  int bt = -1, bk = 0;
  for (int t = 0; t < n_p; ++t) {
    const double* lam = theta + t * kScMaxB;
    const double lN = probs[n_p + t].up - theta[(n_p + t) * kScMaxB];
    for (int i = 0; i < m; ++i) eig[t * m + i] = lam[i];
    lmax[t] = lN;
    int k = num_speakers;
    if (k == 0) {
      k = 1;
      for (int i = 2; i < m; ++i)
        if (lam[i] - lam[i - 1] > lam[k] - lam[k - 1]) k = i;
    }
    const double g = (lam[k] - lam[k - 1]) / (lN + 1e-10);
    const double r = (static_cast<double>(pv[t]) / N) / (g + 1e-10);
    ratio[t] = r;
    if (bt < 0 || r < best) {
      best = r;
      bt = t;
      bk = k;
    }
  }
  sel[0] = bk;
  sel[1] = bt;
}

// Step 6 in one CTA on Y = the first k columns of the selected problem's Ritz vectors X (row stride B): maximin
// initialisation, Lloyd iterations, labels by smallest member; emb (N, ld_emb) gets Y and zeros, when not NULL.
// scratch: N doubles.  block 1024.
constexpr int kScKmThreads = 1024;

__device__ __forceinline__ void sc_argbest(double& v, int& i, bool maximise, double* rv, int* ri) {
  // block-wide (value, index) extremum, ties to the lower index; every thread gets the result
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if ((maximise ? ov > v : ov < v) || (ov == v && oi < i)) {
      v = ov;
      i = oi;
    }
  }
  __syncthreads();
  if (lane == 0) {
    rv[warp] = v;
    ri[warp] = i;
  }
  __syncthreads();
  v = rv[0];
  i = ri[0];
  for (int w = 1; w < kScKmThreads / 32; ++w)
    if ((maximise ? rv[w] > v : rv[w] < v) || (rv[w] == v && ri[w] < i)) {
      v = rv[w];
      i = ri[w];
    }
}

__global__ void __launch_bounds__(kScKmThreads)
sc_kmeans_kernel(const double* __restrict__ X_all, int N, int B, const int32_t* __restrict__ sel, int iters,
                 double* __restrict__ scratch, int32_t* __restrict__ labels, double* __restrict__ emb, int ld_emb) {
  __shared__ double C[32][33], mean[32], rv[32];
  __shared__ int ri[32], idx[32], map[32];
  const int tid = threadIdx.x, k = sel[0], t = sel[1];
  const double* Y = X_all + static_cast<size_t>(t) * N * B;
  if (emb)
    for (long long e = tid; e < static_cast<long long>(N) * ld_emb; e += kScKmThreads) {
      const int u = static_cast<int>(e / ld_emb), c = static_cast<int>(e % ld_emb);
      emb[e] = c < k ? Y[static_cast<size_t>(u) * B + c] : 0.0;
    }
  if (k <= 1) {
    for (int u = tid; u < N; u += kScKmThreads) labels[u] = 0;
    return;
  }
  auto dist2 = [&](int u, const double* c) {
    double s = 0.0;
    for (int d = 0; d < k; ++d) {
      const double x = Y[static_cast<size_t>(u) * B + d] - c[d];
      s = fma(x, x, s);
    }
    return s;
  };
  // the mean row: thread d sums column d in row order
  if (tid < k) {
    double s = 0.0;
    for (int u = 0; u < N; ++u) s += Y[static_cast<size_t>(u) * B + tid];
    mean[tid] = s / N;
  }
  __syncthreads();
  double v = -1.0;
  int bi = 0x7fffffff;
  for (int u = tid; u < N; u += kScKmThreads) {
    const double x = dist2(u, mean);
    if (x > v) {
      v = x;
      bi = u;
    }
  }
  sc_argbest(v, bi, true, rv, ri);
  if (tid == 0) idx[0] = bi;
  __syncthreads();
  for (int c = 1; c < k; ++c) {
    if (tid < k) C[c - 1][tid] = Y[static_cast<size_t>(idx[c - 1]) * B + tid];
    __syncthreads();
    v = -1.0;
    bi = 0x7fffffff;
    for (int u = tid; u < N; u += kScKmThreads) {
      const double x = dist2(u, C[c - 1]);
      const double nd = c == 1 ? x : fmin(scratch[u], x);
      scratch[u] = nd;
      if (nd > v) {
        v = nd;
        bi = u;
      }
    }
    sc_argbest(v, bi, true, rv, ri);
    if (tid == 0) idx[c] = bi;
    __syncthreads();
  }
  if (tid < k) C[k - 1][tid] = Y[static_cast<size_t>(idx[k - 1]) * B + tid];
  __syncthreads();
  for (int it = 0; it < iters; ++it) {
    int changed = 0;
    for (int u = tid; u < N; u += kScKmThreads) {
      int best = 0;
      double bd = dist2(u, C[0]);
      for (int c = 1; c < k; ++c) {
        const double x = dist2(u, C[c]);
        if (x < bd) {
          bd = x;
          best = c;
        }
      }
      if (it == 0 || labels[u] != best) changed = 1;
      labels[u] = best;
    }
    if (!__syncthreads_or(changed)) break;
    // thread (c, d) sums column d over the rows of cluster c in row order
    double s = 0.0;
    int n = 0;
    const int c = tid / 32, d = tid % 32;
    if (c < k && d < k) {
      for (int u = 0; u < N; ++u)
        if (labels[u] == c) {
          s += Y[static_cast<size_t>(u) * B + d];
          ++n;
        }
    }
    __syncthreads();
    if (c < k && d < k && n > 0) C[c][d] = s / n;
    __syncthreads();
  }
  // renumber by each cluster's smallest member
  if (tid == 0) {
    int next = 0;
    for (int c = 0; c < k; ++c) map[c] = -1;
    for (int u = 0; u < N; ++u) {
      const int l = labels[u];
      if (map[l] < 0) map[l] = next++;
      labels[u] = map[l];
    }
  }
}

}  // namespace dsk
