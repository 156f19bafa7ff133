// PLDA backend: the N-sized passes of an LDA + two-covariance PLDA fit and the PLDA log-likelihood-ratio scorers.
//
// Every statistic is fp64.  The three GEMM-shaped passes (the Gram of the centred embeddings, the affine transform of
// every row, the cross term of the score matrix) run on the fp64 tensor cores: mma.sync.m8n8k4.f64 (DMMA on sm_90a).
// They share one 64 x 64 CTA tile: 4 warps of 32 x 32, K staged through shared memory 32 at a time, one register stage
// of prefetch.  An operand is staged K-major ([k][m], the Gram: both operands are column slices of row-major rows) or
// M-major ([m][k], the other two: rows whose K is contiguous), padded so that both the stores and the fragment loads
// are free of bank conflicts.  The fixed K order makes each output a function of its own row and column only.
#pragma once
#include <stdint.h>

namespace dsk {

constexpr int kF64Tile = 64;                 // CTA output tile (rows and columns)
constexpr int kF64K = 32;                    // K per shared-memory stage
constexpr int kF64Threads = 128;             // 4 warps, 2 x 2 sub-tiles of 32 x 32
constexpr int kF64LdK = kF64Tile + 4;        // K-major stage row (doubles): 8-bank shift per k
constexpr int kF64LdM = kF64K + 4;           // M-major stage row (doubles): 8-bank shift per m
constexpr int kF64Stage = kF64Tile * kF64LdM;  // doubles per operand stage (>= kF64K * kF64LdK)
static_assert(kF64Stage >= kF64K * kF64LdK, "one stage size fits both layouts");
constexpr int kF64GramCtas = 1024;           // split-K target: upper tiles x splits (a function of (N, D) only)
constexpr int kPldaWarps = 8;                // trials / rows per 256-thread CTA of the warp-per-row kernels

__device__ __forceinline__ double f64_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

__device__ __forceinline__ void dmma_8x8x4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

template <bool KMAJOR>
__device__ __forceinline__ double f64_at(const double* s, int k, int m) {
  return KMAJOR ? s[k * kF64LdK + m] : s[m * kF64LdM + k];
}

// One shared-memory stage into the warp's 32 x 32 sub-tile (wm, wn in {0, 32}).  acc[i][j][r] is element
// (wm + 8 i + lane / 4, wn + 8 j + 2 (lane % 4) + r) of the tile: the m8n8k4 accumulator layout.
template <bool KM_A, bool KM_B>
__device__ __forceinline__ void f64_tile_mma(const double* sa, const double* sb, double (&acc)[4][4][2], int wm,
                                             int wn, int lane) {
  const int kq = lane & 3, mq = lane >> 2;
#pragma unroll
  for (int k0 = 0; k0 < kF64K; k0 += 4) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = f64_at<KM_A>(sa, k0 + kq, wm + 8 * i + mq);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = f64_at<KM_B>(sb, k0 + kq, wn + 8 * j + mq);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma_8x8x4(acc[i][j], a[i], b[j]);
  }
}

// M-major staging of rows r0 .. r0 + 63 of a row-major (rows, K) matrix P (row stride ld), columns k0 .. k0 + 31:
// thread t covers k = t % 32 for rows t / 32 + 4 i.  Out of range elements are 0.
template <class T>
__device__ __forceinline__ void f64_load_mmajor(const T* __restrict__ P, long long rows, int K, long long ld,
                                                long long r0, int k0, T (&reg)[16]) {
  const int k = k0 + (threadIdx.x & 31), m0 = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const long long r = r0 + m0 + 4 * i;
    reg[i] = (r < rows && k < K) ? P[r * ld + k] : T(0);
  }
}

// ---- Gram: G (D x D) = sum_u (x_u - mu)(x_u - mu)^T ----------------------------------------------------------------
// grid (upper tiles, splits), block kF64Threads.  CTA (t, s) computes tile t = (bi <= bj) of the split-s rows
// [s * rows_per, (s + 1) * rows_per) into ws[s][t][64][64]; gram_reduce_kernel sums the splits in order.
__device__ __forceinline__ void f64_tile_coords(int t, int tiles, int& bi, int& bj) {
  bi = 0;
  while (t >= tiles - bi) {
    t -= tiles - bi;
    ++bi;
  }
  bj = bi + t;
}

__global__ void __launch_bounds__(kF64Threads)
gram_f64_kernel(const float* __restrict__ X, long long N, int D, const double* __restrict__ mu, long long rows_per,
                double* __restrict__ ws) {
  __shared__ double sa[kF64Stage], sb[kF64Stage];
  const int tiles = (D + kF64Tile - 1) / kF64Tile;
  int bi, bj;
  f64_tile_coords(blockIdx.x, tiles, bi, bj);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const long long u0 = static_cast<long long>(blockIdx.y) * rows_per;
  const long long u1 = u0 + rows_per < N ? u0 + rows_per : N;
  // K-major staging: thread t covers column m = t % 64 of rows t / 64 + 2 i
  const int m = tid & 63, kr = tid >> 6;
  const int ca = bi * kF64Tile + m, cb = bj * kF64Tile + m;
  const double mua = (ca < D && mu) ? mu[ca] : 0.0, mub = (cb < D && mu) ? mu[cb] : 0.0;
  float ra[16], rb[16];
  auto load = [&](long long k0) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const long long u = k0 + kr + 2 * i;
      const bool in = u < u1;
      ra[i] = (in && ca < D) ? X[u * D + ca] : 0.f;
      rb[i] = (in && cb < D) ? X[u * D + cb] : 0.f;
    }
  };
  double acc[4][4][2] = {};
  if (u0 < u1) load(u0);
  for (long long k0 = u0; k0 < u1; k0 += kF64K) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const bool in = k0 + kr + 2 * i < u1;  // padding rows stay exactly 0
      sa[(kr + 2 * i) * kF64LdK + m] = (in && ca < D) ? static_cast<double>(ra[i]) - mua : 0.0;
      sb[(kr + 2 * i) * kF64LdK + m] = (in && cb < D) ? static_cast<double>(rb[i]) - mub : 0.0;
    }
    __syncthreads();
    if (k0 + kF64K < u1) load(k0 + kF64K);
    f64_tile_mma<true, true>(sa, sb, acc, wm, wn, lane);
  }
  double* out = ws + (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * (kF64Tile * kF64Tile);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = wm + 8 * i + (lane >> 2), c = wn + 8 * j + 2 * (lane & 3);
      out[r * kF64Tile + c] = acc[i][j][0];
      out[r * kF64Tile + c + 1] = acc[i][j][1];
    }
}

// G[i][j] = G[j][i] = the sum of the splits' partials of element (i, j), i <= j, in split order: exactly symmetric.
// grid (upper tiles), block 256.
__global__ void __launch_bounds__(256)
gram_reduce_kernel(const double* __restrict__ ws, int D, int splits, double* __restrict__ G) {
  const int tiles = (D + kF64Tile - 1) / kF64Tile, nt = gridDim.x;
  int bi, bj;
  f64_tile_coords(blockIdx.x, tiles, bi, bj);
  for (int e = threadIdx.x; e < kF64Tile * kF64Tile; e += 256) {
    const int r = e / kF64Tile, c = e % kF64Tile;
    const int gi = bi * kF64Tile + r, gj = bj * kF64Tile + c;
    if (gi >= D || gj >= D || (bi == bj && r > c)) continue;
    const double* p = ws + static_cast<size_t>(blockIdx.x) * (kF64Tile * kF64Tile) + e;
    double s = 0.0;
    for (int k = 0; k < splits; ++k) s += p[static_cast<size_t>(k) * nt * (kF64Tile * kF64Tile)];
    G[static_cast<size_t>(gi) * D + gj] = s;
    G[static_cast<size_t>(gj) * D + gi] = s;
  }
}

// ---- class sums: out[c] (C x D) = sum over u = order[offsets[c] .. offsets[c+1]) of x_u - mu, in that order -------
// An index outside [0, N) gives a NaN row.  grid (C, ceil(D / 256)), block 256.
__global__ void __launch_bounds__(256)
class_sums_f64_kernel(const float* __restrict__ X, long long N, int D, const int64_t* __restrict__ order,
                      const int64_t* __restrict__ offsets, const double* __restrict__ mu, double* __restrict__ out) {
  const int d = blockIdx.y * 256 + threadIdx.x;
  if (d >= D) return;
  const int64_t b = offsets[blockIdx.x], e = offsets[blockIdx.x + 1];
  const double m = mu ? mu[d] : 0.0;
  double acc = 0.0;
  bool bad = false;
  int64_t u = b;
  for (; u + 4 <= e; u += 4) {  // four independent loads in flight, added in order
    int64_t r[4];
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      r[i] = order[u + i];
      bad |= r[i] < 0 || r[i] >= N;
    }
    if (bad) break;
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = X[r[i] * D + d];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc += static_cast<double>(v[i]) - m;
  }
  for (; u < e && !bad; ++u) {
    const int64_t r = order[u];
    if (r < 0 || r >= N) bad = true;
    else acc += static_cast<double>(X[r * D + d]) - m;
  }
  out[static_cast<size_t>(blockIdx.x) * D + d] = bad ? f64_nan() : acc;
}

// ---- affine transform: Z (rows x d) fp64 = (x_u - c) A^T -----------------------------------------------------------
// X rows r0 .. r0 + rows of (N, D) fp32; A (d, D) fp64; c (D,) fp64 or NULL.  grid (ceil(d / 64), ceil(rows / 64)),
// block kF64Threads.
__global__ void __launch_bounds__(kF64Threads)
affine_f64_kernel(const float* __restrict__ X, long long rows, int D, const double* __restrict__ A, int d,
                  const double* __restrict__ c, double* __restrict__ Z) {
  __shared__ double sa[kF64Stage], sb[kF64Stage];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const long long r0 = static_cast<long long>(blockIdx.y) * kF64Tile;
  const int o0 = blockIdx.x * kF64Tile;
  const int kk = tid & 31, m0 = tid >> 5;
  float ra[16];
  double rb[16];
  double acc[4][4][2] = {};
  f64_load_mmajor<float>(X, rows, D, D, r0, 0, ra);
  f64_load_mmajor<double>(A, d, D, D, o0, 0, rb);
  for (int k0 = 0; k0 < D; k0 += kF64K) {
    const double ck = (k0 + kk < D && c) ? c[k0 + kk] : 0.0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const bool in = r0 + m0 + 4 * i < rows && k0 + kk < D;
      sa[(m0 + 4 * i) * kF64LdM + kk] = in ? static_cast<double>(ra[i]) - ck : 0.0;
      sb[(m0 + 4 * i) * kF64LdM + kk] = rb[i];
    }
    __syncthreads();
    if (k0 + kF64K < D) {
      f64_load_mmajor<float>(X, rows, D, D, r0, k0 + kF64K, ra);
      f64_load_mmajor<double>(A, d, D, D, o0, k0 + kF64K, rb);
    }
    f64_tile_mma<false, false>(sa, sb, acc, wm, wn, lane);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long r = r0 + wm + 8 * i + (lane >> 2);
      const int o = o0 + wn + 8 * j + 2 * (lane & 3);
      if (r < rows) {
        if (o < d) Z[r * d + o] = acc[i][j][0];
        if (o + 1 < d) Z[r * d + o + 1] = acc[i][j][1];
      }
    }
}

// Row u of Z (rows x d): Y[u] = fp32(s_u z_u).  mode 0: s = 1; 1: s = sqrt(d) / ||z||; 2: s = sqrt(d / sum_l z_l^2 /
// (psi_l + 1 / n_u)), n_u = counts[u] (1 without counts; a count < 1 gives a NaN row).  The sums are one warp's fixed
// order.  grid ceil(rows / 8), block 256.
__global__ void __launch_bounds__(256)
affine_scale_kernel(const double* __restrict__ Z, long long rows, int d, int mode, const double* __restrict__ psi,
                    const int32_t* __restrict__ counts, float* __restrict__ Y) {
  const long long u = static_cast<long long>(blockIdx.x) * kPldaWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (u >= rows) return;
  const double* z = Z + u * d;
  double s = 1.0;
  if (mode != 0) {
    const int n = counts ? counts[u] : 1;
    const double inv_n = 1.0 / n;
    double ss = 0.0;
    for (int l = lane; l < d; l += 32) {
      const double v = z[l];
      ss += mode == 1 ? v * v : v * v / (psi[l] + inv_n);
    }
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    s = mode == 1 ? sqrt(static_cast<double>(d)) / sqrt(ss) : sqrt(static_cast<double>(d) / ss);
    if (n < 1) s = f64_nan();
  }
  for (int l = lane; l < d; l += 32) Y[u * d + l] = static_cast<float>(z[l] * s);
}

// ---- PLDA scoring -------------------------------------------------------------------------------------------------
// Trial t = (e, u) of rows of Y (U x dim): the LLR of test row u against enrolment row e of n = counts[e] utterances
// (n = 1 without counts), sum over l of
//   -0.5 (log v1 + (y_u - a y_e)^2 / v1) + 0.5 (log v0 + y_u^2 / v0),  a = n psi / (n psi + 1), v1 = 1 + psi / (n psi
//   + 1), v0 = 1 + psi,
// in fp64, one warp per trial in a fixed order.  An index outside [0, U) or a count < 1 gives NaN and reads no row.
// grid ceil(T / 8), block 256.
__global__ void __launch_bounds__(256)
plda_trials_kernel(const float* __restrict__ Y, int U, int dim, const double* __restrict__ psi,
                   const int32_t* __restrict__ counts, const int64_t* __restrict__ trials, long long T,
                   float* __restrict__ llr) {
  const long long t = static_cast<long long>(blockIdx.x) * kPldaWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int64_t e = trials[2 * t], u = trials[2 * t + 1];
  if (e < 0 || e >= U || u < 0 || u >= U || (counts && counts[e] < 1)) {
    if (lane == 0) llr[t] = __int_as_float(0x7fc00000);
    return;
  }
  const double n = counts ? counts[e] : 1;
  const float* ye = Y + e * dim;
  const float* yu = Y + u * dim;
  double s = 0.0;
  for (int l = lane; l < dim; l += 32) {
    const double p = psi[l], ev = ye[l], tv = yu[l];
    const double v1 = 1.0 + p / (n * p + 1.0), v0 = 1.0 + p;
    const double diff = tv - n * p / (n * p + 1.0) * ev;
    s += -0.5 * (log(v1) + diff * diff / v1) + 0.5 * (log(v0) + tv * tv / v0);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) llr[t] = static_cast<float>(s);
}

// The n = 1 LLR in expanded form: S_ij = k + q(a_i) + q(b_j) + sum_l beta_l a_il b_jl with
//   q(y) = sum_l w_l y_l^2, w_l = -0.5 psi^2 / ((1 + psi)(2 psi + 1)), beta_l = psi / (2 psi + 1),
//   k = 0.5 sum_l (log(1 + psi) - log((2 psi + 1) / (1 + psi))).
// plda_coef_kernel: coef = [w (dim), beta (dim), k], one warp.
__global__ void plda_coef_kernel(const double* __restrict__ psi, int dim, double* __restrict__ coef) {
  const int lane = threadIdx.x;
  double k = 0.0;
  for (int l = lane; l < dim; l += 32) {
    const double p = psi[l];
    coef[l] = -0.5 * p * p / ((1.0 + p) * (2.0 * p + 1.0));
    coef[dim + l] = p / (2.0 * p + 1.0);
    k += 0.5 * (log(1.0 + p) - log((2.0 * p + 1.0) / (1.0 + p)));
  }
  for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
  if (lane == 0) coef[2 * dim] = k;
}

// q[r] = q(row r) for the rows of Ya (M) then Yb (N), one warp per row.  grid ceil((M + N) / 8), block 256.
__global__ void __launch_bounds__(256)
plda_q_kernel(const float* __restrict__ Ya, int M, const float* __restrict__ Yb, int N, int dim,
              const double* __restrict__ coef, double* __restrict__ q) {
  const long long r = static_cast<long long>(blockIdx.x) * kPldaWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= static_cast<long long>(M) + N) return;
  const float* y = r < M ? Ya + r * dim : Yb + (r - M) * dim;
  double s = 0.0;
  for (int l = lane; l < dim; l += 32) {
    const double v = y[l];
    s += coef[l] * v * v;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) q[r] = s;
}

// S (M x N, row stride ld) fp32 = k + q_a[i] + q_b[j] + (beta o a_i) . b_j, the cross term on the fp64 tensor cores.
// grid (ceil(N / 64), ceil(M / 64)), block kF64Threads.
__global__ void __launch_bounds__(kF64Threads)
plda_matrix_kernel(const float* __restrict__ Ya, int M, const float* __restrict__ Yb, int N, int dim,
                   const double* __restrict__ coef, const double* __restrict__ q, float* __restrict__ S, long long ld) {
  __shared__ double sa[kF64Stage], sb[kF64Stage];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int i0 = blockIdx.y * kF64Tile, j0 = blockIdx.x * kF64Tile;
  const int kk = tid & 31, m0 = tid >> 5;
  const double* beta = coef + dim;
  float ra[16], rb[16];
  double acc[4][4][2] = {};
  f64_load_mmajor<float>(Ya, M, dim, dim, i0, 0, ra);
  f64_load_mmajor<float>(Yb, N, dim, dim, j0, 0, rb);
  for (int k0 = 0; k0 < dim; k0 += kF64K) {
    const double bk = k0 + kk < dim ? beta[k0 + kk] : 0.0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      sa[(m0 + 4 * i) * kF64LdM + kk] = bk * static_cast<double>(ra[i]);
      sb[(m0 + 4 * i) * kF64LdM + kk] = rb[i];
    }
    __syncthreads();
    if (k0 + kF64K < dim) {
      f64_load_mmajor<float>(Ya, M, dim, dim, i0, k0 + kF64K, ra);
      f64_load_mmajor<float>(Yb, N, dim, dim, j0, k0 + kF64K, rb);
    }
    f64_tile_mma<false, false>(sa, sb, acc, wm, wn, lane);
  }
  const double k = coef[2 * dim];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = i0 + wm + 8 * i + (lane >> 2);
      const int c = j0 + wn + 8 * j + 2 * (lane & 3);
      if (r >= M) continue;
      const double qr = k + q[r];
      if (c < N) S[r * ld + c] = static_cast<float>(qr + q[M + c] + acc[i][j][0]);
      if (c + 1 < N) S[r * ld + c + 1] = static_cast<float>(qr + q[M + c + 1] + acc[i][j][1]);
    }
}

}  // namespace dsk
