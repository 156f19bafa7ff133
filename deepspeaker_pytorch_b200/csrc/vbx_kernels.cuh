// VBx: variational-Bayes HMM clustering of window embeddings in the PLDA space (Landini et al., "Bayesian HMM
// clustering of x-vector sequences (VBx) in speaker diarization", 2022), batched over recordings.
//
// oracle/vbx_oracle.py states the iteration.  Per recording r (rows t = offsets[r] .. offsets[r+1], S_r speakers):
//   prep:      G_t = -(|x_t|^2 + d ln 2 pi) / 2, rho_t = x_t o sqrt(phi), the bad flag and S_r;
//   gamma0:    gamma = rowwise softmax(init_smoothing one_hot(label));
// then per iteration:
//   stats:     the partial sums over a split of kVbxSplitRows rows of gamma^T [rho | 1] on the fp64 tensor cores (the
//              f64_tile_mma tile of plda_kernels.cuh); column d is N_s;
//   model:     one warp per (r, s): the splits summed in order, invL, alpha, the constant c_s and the KL term of s;
//   loglik:    ln p_ts = Fa (rho_t . alpha_s - c_s + G_t), the cross term on the same fp64 tile;
//   fb:        one warp per recording: the forward-backward of the rank-one transition matrix in the log domain,
//              gamma, ln p(X), the switch sums, then the pi update, the ELBO and the done flag.
// Every sum has a fixed order and no float atomics are used, and nothing a kernel computes for one recording reads
// another recording's rows, so a recording's outputs are the same bits in any batch.  A recording whose done flag is
// set (converged, or a bad input) is skipped by every kernel of the later iterations.
#pragma once
#include <stdint.h>

#include "plda_kernels.cuh"

namespace dsk {

constexpr int kVbxSplitRows = 256;   // rows per split of the statistics pass (8 K stages)
constexpr int kVbxMaxStates = 4;     // states per lane of the forward-backward warp (128 speakers)

__device__ __forceinline__ double vbx_warp_sum(double v) {  // fixed tree, lane 0's result on every lane
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}

__device__ __forceinline__ double vbx_warp_max(double v) {
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return __shfl_sync(0xffffffffu, v, 0);
}

// The recording of row t: the r with off[r] <= t < off[r + 1].
__device__ __forceinline__ int vbx_recording(const int64_t* __restrict__ off, int R, long long t) {
  int lo = 0, hi = R - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= t) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One warp per row: rho, G, and per recording the bad flag (a non-finite element or a label outside [0, S)) and
// S_r = 1 + the largest label (integer atomics only).  grid ceil(W / 8), block 256.
__global__ void __launch_bounds__(256)
vbx_prep_kernel(const float* __restrict__ X, long long W, int d, const int64_t* __restrict__ off, int R,
                const int32_t* __restrict__ labels, int S, const double* __restrict__ phi, double* __restrict__ rho,
                double* __restrict__ G, int32_t* __restrict__ rec_S, int32_t* __restrict__ bad) {
  const long long t = static_cast<long long>(blockIdx.x) * kPldaWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= W) return;
  double ss = 0.0;
  bool finite = true;
  for (int l = lane; l < d; l += 32) {
    const double x = X[t * d + l];
    finite &= isfinite(x);
    rho[t * d + l] = x * sqrt(phi[l]);
    ss += x * x;
  }
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  finite = __all_sync(0xffffffffu, finite);
  if (lane == 0) {
    G[t] = -0.5 * (ss + d * 1.8378770664093453);  // ln 2 pi
    const int r = vbx_recording(off, R, t);
    const int32_t lab = labels[t];
    if (!finite || lab < 0 || lab >= S) atomicOr(&bad[r], 1);
    else atomicMax(&rec_S[r], lab + 1);
  }
}

// One thread per recording: done = bad, iters 0, pi = 1 / S_r (NaN rows for a bad recording), the ELBO row NaN.
__global__ void vbx_rec_init_kernel(int R, int S, int max_iters, const int32_t* __restrict__ rec_S,
                                    const int32_t* __restrict__ bad, int32_t* __restrict__ done,
                                    int32_t* __restrict__ n_done, double* __restrict__ pi, double* __restrict__ elbo,
                                    int32_t* __restrict__ iters) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const bool b = bad[r] != 0;
  done[r] = b;
  if (b) atomicAdd(n_done, 1);
  iters[r] = 0;
  const int Sr = rec_S[r];
  for (int s = 0; s < S; ++s) pi[static_cast<size_t>(r) * S + s] = b ? f64_nan() : (s < Sr ? 1.0 / Sr : 0.0);
  for (int i = 0; i < max_iters; ++i) elbo[static_cast<size_t>(r) * max_iters + i] = f64_nan();
}

// One thread per row: gamma0 = softmax(sm one_hot(label)) over the recording's S_r speakers, 0 past them.
__global__ void vbx_gamma0_kernel(long long W, const int64_t* __restrict__ off, int R, const int32_t* __restrict__ labels,
                                  int S, double sm, const int32_t* __restrict__ rec_S, const int32_t* __restrict__ bad,
                                  double* __restrict__ gamma) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= W) return;
  const int r = vbx_recording(off, R, t);
  if (bad[r]) return;
  const int Sr = rec_S[r], lab = labels[t];
  const double e = exp(-sm), inv = 1.0 / (1.0 + (Sr - 1) * e);  // the label's entry exp(0), the others exp(-sm)
  for (int s = 0; s < S; ++s) gamma[t * S + s] = s >= Sr ? 0.0 : (s == lab ? inv : e * inv);
}

// Statistics: part[e][tile] (64 x 64) = sum over the split's rows u of gamma[u][s] [rho_u | 1][c], s in the tile's
// speaker block, c in its column block of d + 1 (column d is 1: N_s).  Entry e = (r, split) of tab.
// grid (entries, speaker tiles x column tiles), block kF64Threads.
__global__ void __launch_bounds__(kF64Threads)
vbx_stats_kernel(const double* __restrict__ gamma, int S, const double* __restrict__ rho, int d,
                 const int64_t* __restrict__ off, const int32_t* __restrict__ tab, const int32_t* __restrict__ rec_S,
                 const int32_t* __restrict__ done, double* __restrict__ part) {
  __shared__ double sa[kF64Stage], sb[kF64Stage];
  const int r = tab[2 * blockIdx.x], split = tab[2 * blockIdx.x + 1];
  if (done[r]) return;
  const int tiles_c = (d + 1 + kF64Tile - 1) / kF64Tile;
  const int bi = blockIdx.y / tiles_c, bj = blockIdx.y % tiles_c;
  const int Sr = rec_S[r];
  if (bi * kF64Tile >= Sr) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const long long u0 = off[r] + static_cast<long long>(split) * kVbxSplitRows;
  const long long u1 = min(u0 + kVbxSplitRows, static_cast<long long>(off[r + 1]));
  // K-major staging: thread t covers column m = t % 64 of rows t / 64 + 2 i
  const int m = tid & 63, kr = tid >> 6;
  const int sa_col = bi * kF64Tile + m, sb_col = bj * kF64Tile + m;
  double ra[16], rb[16];
  auto load = [&](long long k0) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const long long u = k0 + kr + 2 * i;
      const bool in = u < u1;
      ra[i] = (in && sa_col < Sr) ? gamma[u * S + sa_col] : 0.0;
      rb[i] = !in ? 0.0 : sb_col < d ? rho[u * d + sb_col] : sb_col == d ? 1.0 : 0.0;
    }
  };
  double acc[4][4][2] = {};
  load(u0);
  for (long long k0 = u0; k0 < u1; k0 += kF64K) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      sa[(kr + 2 * i) * kF64LdK + m] = ra[i];
      sb[(kr + 2 * i) * kF64LdK + m] = rb[i];
    }
    __syncthreads();
    if (k0 + kF64K < u1) load(k0 + kF64K);
    f64_tile_mma<true, true>(sa, sb, acc, wm, wn, lane);
  }
  double* out = part + (static_cast<size_t>(blockIdx.x) * gridDim.y + blockIdx.y) * (kF64Tile * kF64Tile);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int rr = wm + 8 * i + (lane >> 2), c = wn + 8 * j + 2 * (lane & 3);
      out[rr * kF64Tile + c] = acc[i][j][0];
      out[rr * kF64Tile + c + 1] = acc[i][j][1];
    }
}

// Model: one warp per (r, s < S_r).  F_sl = the splits' partials summed in split order (column d: N_s), invL_l =
// 1 / (1 + (Fa / Fb) N_s phi_l), alpha_sl = (Fa / Fb) invL_l F_sl, cst[r][s] = sum_l phi_l (invL_l + alpha_sl^2) / 2,
// kl[r][s] = sum_l (ln invL_l - invL_l - alpha_sl^2 + 1).  grid (R, ceil(S / 8)), block 256.
__global__ void __launch_bounds__(256)
vbx_model_kernel(const double* __restrict__ part, const int64_t* __restrict__ off, const int32_t* __restrict__ split_base,
                 int S, int d, const double* __restrict__ phi, double ratio, const int32_t* __restrict__ rec_S,
                 const int32_t* __restrict__ done, double* __restrict__ alpha, double* __restrict__ cst,
                 double* __restrict__ kl) {
  const int r = blockIdx.x, s = blockIdx.y * kPldaWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (done[r] || s >= rec_S[r]) return;
  const int tiles_c = (d + 1 + kF64Tile - 1) / kF64Tile, tiles = (S + kF64Tile - 1) / kF64Tile * tiles_c;
  const int base = split_base[r], splits = split_base[r + 1] - base;
  const int bi = s / kF64Tile, sr = s % kF64Tile;
  auto total = [&](int c) {
    const double* p = part + (static_cast<size_t>(base) * tiles + bi * tiles_c + c / kF64Tile) * (kF64Tile * kF64Tile) +
                      sr * kF64Tile + c % kF64Tile;
    double v = 0.0;
    for (int k = 0; k < splits; ++k) v += p[static_cast<size_t>(k) * tiles * (kF64Tile * kF64Tile)];
    return v;
  };
  const double N = total(d);
  double* a = alpha + (static_cast<size_t>(r) * S + s) * d;
  double cs = 0.0, k = 0.0;
  for (int l = lane; l < d; l += 32) {
    const double invL = 1.0 / (1.0 + ratio * N * phi[l]);
    const double al = ratio * invL * total(l);
    a[l] = al;
    cs += phi[l] * (invL + al * al);
    k += log(invL) - invL - al * al + 1.0;
  }
  for (int o = 16; o > 0; o >>= 1) {
    cs += __shfl_xor_sync(0xffffffffu, cs, o);
    k += __shfl_xor_sync(0xffffffffu, k, o);
  }
  if (lane == 0) {
    cst[static_cast<size_t>(r) * S + s] = 0.5 * cs;
    kl[static_cast<size_t>(r) * S + s] = k;
  }
}

// Log-likelihoods: lnp[t][s] = Fa ((rho_t . alpha_s - cst_s) + G_t) for the 64 rows of entry e = (r, row tile) of tab
// and the 64 speakers of blockIdx.y (s < S_r only).  grid (entries, speaker tiles), block kF64Threads.
__global__ void __launch_bounds__(kF64Threads)
vbx_loglik_kernel(const double* __restrict__ rho, int d, const double* __restrict__ alpha, const double* __restrict__ cst,
                  const double* __restrict__ G, int S, double Fa, const int64_t* __restrict__ off,
                  const int32_t* __restrict__ tab, const int32_t* __restrict__ rec_S, const int32_t* __restrict__ done,
                  double* __restrict__ lnp) {
  __shared__ double sa[kF64Stage], sb[kF64Stage];
  const int r = tab[2 * blockIdx.x];
  if (done[r]) return;
  const int Sr = rec_S[r], s0 = blockIdx.y * kF64Tile;
  if (s0 >= Sr) return;
  const long long t0 = off[r], Wr = off[r + 1] - t0, m0 = static_cast<long long>(tab[2 * blockIdx.x + 1]) * kF64Tile;
  const double* A = rho + t0 * d;
  const double* B = alpha + static_cast<size_t>(r) * S * d;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int kk = tid & 31, mm = tid >> 5;
  double ra[16], rb[16];
  double acc[4][4][2] = {};
  f64_load_mmajor<double>(A, Wr, d, d, m0, 0, ra);
  f64_load_mmajor<double>(B, Sr, d, d, s0, 0, rb);
  for (int k0 = 0; k0 < d; k0 += kF64K) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      sa[(mm + 4 * i) * kF64LdM + kk] = ra[i];
      sb[(mm + 4 * i) * kF64LdM + kk] = rb[i];
    }
    __syncthreads();
    if (k0 + kF64K < d) {
      f64_load_mmajor<double>(A, Wr, d, d, m0, k0 + kF64K, ra);
      f64_load_mmajor<double>(B, Sr, d, d, s0, k0 + kF64K, rb);
    }
    f64_tile_mma<false, false>(sa, sb, acc, wm, wn, lane);
  }
  const double* c = cst + static_cast<size_t>(r) * S;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long row = m0 + wm + 8 * i + (lane >> 2);
      const int s = s0 + wn + 8 * j + 2 * (lane & 3);
      if (row >= Wr) continue;
      const double g = G[t0 + row];
      double* out = lnp + (t0 + row) * S;
      if (s < Sr) out[s] = Fa * ((acc[i][j][0] - c[s]) + g);
      if (s + 1 < Sr) out[s + 1] = Fa * ((acc[i][j][1] - c[s + 1]) + g);
    }
}

// ln(e^a + e^b), -inf when both are, NaN when either is.
__device__ __forceinline__ double vbx_logaddexp(double a, double b) {
  const double mx = fmax(a, b), mn = fmin(a, b);
  if (isnan(a) || isnan(b)) return a + b;
  return mn == -__longlong_as_double(0x7ff0000000000000ll) ? mx : mx + log1p(exp(mn - mx));
}

// Forward-backward, pi update, ELBO and stop test of iteration `it`: one warp per recording, state j = lane + 32 k.
// Transitions A = loop_p I + (1 - loop_p) 1 pi^T, so sum_i a_i A_ij = loop_p a_j + (1 - loop_p) pi_j sum_i a_i.  The
// messages are scaled and kept as logarithms: a linear message of a state that is behind by more than fp64's range
// would underflow to 0 and never recover at loop_p = 1, though the state may win later.
//   forward:  la_j = ln p_tj + ln pred_j, ln pred = ln pi at t = 0, else logaddexp(ln loop_p + ln at_{t-1},
//             ln(1 - loop_p) + ln pi) (at_{t-1} sums to 1); m = max_j la_j, c = sum_j exp(la_j - m); ln at_t =
//             la - m - ln c goes to gamma, ln C_t = m + ln c to lnc, ln p(X) = sum_t ln C_t.
//   backward: ln bt_{W-1} = 0; gamma_t = exp(ln at_t + ln bt_t); for t >= 1, lu_j = ln p_tj + ln bt_tj - ln C_t (the
//             switch term of the pi update at t is exp(ln(1 - loop_p) + ln pi_j + lu_j)), ln q = logsumexp_i(ln pi_i +
//             lu_i), ln bt_{t-1,j} = logaddexp(ln loop_p + lu_j, ln(1 - loop_p) + ln q).
// at and bt are the scaled messages: alpha-hat_t / prod_{u<=t} C_u and beta-hat_t / prod_{u>t} C_u.
// grid R, block 32.
__global__ void __launch_bounds__(32)
vbx_fb_kernel(const int64_t* __restrict__ off, int S, const double* __restrict__ lnp, double* __restrict__ gamma,
              double* __restrict__ lnc, const double* __restrict__ kl, double loop_p, double Fb, double epsilon, int it,
              int max_iters, const int32_t* __restrict__ rec_S, int32_t* __restrict__ done,
              int32_t* __restrict__ n_done, double* __restrict__ pi, double* __restrict__ elbo,
              int32_t* __restrict__ iters) {
  const int r = blockIdx.x, lane = threadIdx.x;
  if (done[r]) return;
  const int Sr = rec_S[r], nk = (Sr + 31) / 32;
  const long long t0 = off[r], W = off[r + 1] - t0;
  const double ninf = -__longlong_as_double(0x7ff0000000000000ll);
  const double lst = log(loop_p), lsw = log(1.0 - loop_p);
  double p[kVbxMaxStates], lpi[kVbxMaxStates];
  bool v[kVbxMaxStates];
#pragma unroll
  for (int k = 0; k < kVbxMaxStates; ++k) {
    const int j = lane + 32 * k;
    v[k] = k < nk && j < Sr;
    p[k] = v[k] ? pi[static_cast<size_t>(r) * S + j] : 0.0;
    lpi[k] = log(p[k]);
  }
  auto load = [&](const double* base, long long t, double (&x)[kVbxMaxStates]) {
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) x[k] = v[k] ? base[(t0 + t) * S + lane + 32 * k] : ninf;
  };
  // forward
  double prev[kVbxMaxStates], nxt[kVbxMaxStates], lnpx = 0.0;
  load(lnp, 0, nxt);
  for (long long t = 0; t < W; ++t) {
    double la[kVbxMaxStates];
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) la[k] = nxt[k];
    if (t + 1 < W) load(lnp, t + 1, nxt);
    double m = ninf;
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) {
      if (v[k]) la[k] += t == 0 ? lpi[k] : vbx_logaddexp(lst + prev[k], lsw + lpi[k]);
      m = fmax(m, la[k]);
    }
    m = vbx_warp_max(m);
    double c = 0.0;
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) c += v[k] ? exp(la[k] - m) : 0.0;
    c = vbx_warp_sum(c);
    const double lC = m + log(c);
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) {
      prev[k] = la[k] - lC;
      if (v[k]) gamma[(t0 + t) * S + lane + 32 * k] = prev[k];
    }
    if (lane == 0) lnc[t0 + t] = lC;
    lnpx += lC;
  }
  // backward
  double lb[kVbxMaxStates], swsum[kVbxMaxStates], g0[kVbxMaxStates];
#pragma unroll
  for (int k = 0; k < kVbxMaxStates; ++k) {
    lb[k] = v[k] ? 0.0 : ninf;
    swsum[k] = 0.0;
  }
  double na[kVbxMaxStates], nl[kVbxMaxStates], nc = lnc[t0 + W - 1];
  load(gamma, W - 1, na);
  load(lnp, W - 1, nl);
  for (long long t = W - 1;; --t) {
    double la[kVbxMaxStates], lp[kVbxMaxStates];
    const double lC = nc;
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) {
      la[k] = na[k];
      lp[k] = nl[k];
    }
    if (t > 0) {
      load(gamma, t - 1, na);
      load(lnp, t - 1, nl);
      nc = lnc[t0 + t - 1];
    }
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) {
      const double g = v[k] ? exp(la[k] + lb[k]) : 0.0;
      if (v[k]) gamma[(t0 + t) * S + lane + 32 * k] = g;
      g0[k] = g;
    }
    if (t == 0) break;
    double lu[kVbxMaxStates], M = ninf;
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) {
      lu[k] = lp[k] + lb[k] - lC;
      if (v[k]) {
        swsum[k] += exp(lsw + lpi[k] + lu[k]);
        M = fmax(M, lpi[k] + lu[k]);
      }
    }
    M = vbx_warp_max(M);
    double q = 0.0;
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) q += v[k] ? exp(lpi[k] + lu[k] - M) : 0.0;
    const double lq = M + log(vbx_warp_sum(q));
#pragma unroll
    for (int k = 0; k < kVbxMaxStates; ++k) lb[k] = v[k] ? vbx_logaddexp(lst + lu[k], lsw + lq) : ninf;
  }
  // pi update, ELBO, stop test
  double num[kVbxMaxStates], tot = 0.0, kls = 0.0;
#pragma unroll
  for (int k = 0; k < kVbxMaxStates; ++k) {
    num[k] = v[k] ? g0[k] + swsum[k] : 0.0;
    tot += num[k];
    kls += v[k] ? kl[static_cast<size_t>(r) * S + lane + 32 * k] : 0.0;
  }
  tot = vbx_warp_sum(tot);
  kls = vbx_warp_sum(kls);
#pragma unroll
  for (int k = 0; k < kVbxMaxStates; ++k)
    if (v[k]) pi[static_cast<size_t>(r) * S + lane + 32 * k] = num[k] / tot;
  if (lane == 0) {
    double* e = elbo + static_cast<size_t>(r) * max_iters;
    const double cur = lnpx + 0.5 * Fb * kls;
    e[it] = cur;
    if ((it >= 1 && cur - e[it - 1] < epsilon) || it + 1 == max_iters) {
      done[r] = 1;
      iters[r] = it + 1;
      atomicAdd(n_done, 1);
    }
  }
}

// One thread per row: labels = the argmax of the gamma row over s < S_r (ties to the lower index); a bad recording
// gets label -1 and a NaN gamma row.
__global__ void vbx_labels_kernel(long long W, const int64_t* __restrict__ off, int R, int S,
                                  const int32_t* __restrict__ rec_S, const int32_t* __restrict__ bad,
                                  double* __restrict__ gamma, int32_t* __restrict__ labels) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= W) return;
  const int r = vbx_recording(off, R, t);
  double* g = gamma + t * S;
  if (bad[r]) {
    for (int s = 0; s < S; ++s) g[s] = f64_nan();
    labels[t] = -1;
    return;
  }
  const int Sr = rec_S[r];
  int best = 0;
  for (int s = 1; s < Sr; ++s)
    if (g[s] > g[best]) best = s;
  labels[t] = best;
}

}  // namespace dsk
