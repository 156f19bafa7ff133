// Supervised-contrastive loss (Khosla et al., NeurIPS 2020, the L_out form; with labels = the utterance of each view it
// is SimCLR's NT-Xent) over the batch's own cosine matrix: the row kernels around the AAM-softmax plan's tensor-core
// GEMMs (dsk_supcon / dsk_supcon_bwd in dsk_api.cu).  The plan is the AAM op's for (N, N, D) with E in place of the
// class weights: cos = E^ E^T, and the backward's two products dC E^ and dC^T E^ are its gE^ and gW^ GEMMs.
//
// A row's sums (the softmax denominator, the positive sum and count) are fp64, in a fixed order: each thread adds its
// columns in ascending order, then the warps are added in a fixed tree and the 8 warp sums in warp order.
#pragma once
#include <stdint.h>

#include "aam_kernels.cuh"

namespace dsk {

// The block-wide sums of a, b, c (block 256), the same on every thread; red [3][8] is free again on return.
__device__ __forceinline__ void supcon_block_sum3(double& a, double& b, double& c, double (*red)[8]) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = a;
    red[1][threadIdx.x >> 5] = b;
    red[2][threadIdx.x >> 5] = c;
  }
  __syncthreads();
  a = red[0][0];
  b = red[1][0];
  c = red[2][0];
  for (int k = 1; k < 8; ++k) {
    a += red[0][k];
    b += red[1][k];
    c += red[2][k];
  }
  __syncthreads();
}

// exp(s_ij - lse_i) with s = cos / tau, the exponent formed in fp64 (at tau = 0.01 both terms reach 100, and an fp32
// difference would lose 1e-5 of every probability)
__device__ __forceinline__ float supcon_exp(float c, double inv_tau, double l) {
  return expf(static_cast<float>(static_cast<double>(c) * inv_tau - l));
}

// fp64 cosine of the fp32 rows e and w (D wide) with F.normalize's 1e-12 floors, by one warp in a fixed order (lane-
// strided sums, then a fixed butterfly); every lane returns it.
__device__ __forceinline__ double supcon_cos64_warp(const float* __restrict__ e, const float* __restrict__ w, int D) {
  const int lane = threadIdx.x & 31;
  double ew = 0.0, ee = 0.0, ww = 0.0;
  for (int d = lane; d < D; d += 32) {
    const double ed = e[d], wd = w[d];
    ew = fma(ed, wd, ew);
    ee = fma(ed, ed, ee);
    ww = fma(wd, wd, ww);
  }
  for (int o = 16; o > 0; o >>= 1) {
    ew += __shfl_xor_sync(0xffffffffu, ew, o);
    ee += __shfl_xor_sync(0xffffffffu, ee, o);
    ww += __shfl_xor_sync(0xffffffffu, ww, o);
  }
  return ew / (fmax(sqrt(ee), 1e-12) * fmax(sqrt(ww), 1e-12));
}

// Forward rows.  First the positive pairs' cosines (j != i with y_j = y_i) are recomputed in fp64 from the fp32 rows of
// E and rounded once into the GEMM output G (two views of one utterance sit close, cos near 1, where the tensor cores'
// truncated accumulation errs most; as aam_rows_kernel's target column): warp w takes the columns [32 k, 32 k + 32)
// with k = w mod 8 and computes their positives one after another.  Then cos_out[i][j] = G[i][j] (the diagonal holds
// the GEMM's value), and over j != i: cmax = the largest cosine (NaN skipped by fmaxf; a NaN term still reaches the sum
// below), lse = cmax / tau + log sum_j exp((c_ij - cmax) / tau) in fp64, rounded once; |P(i)| and the positive sum of
// c_ip; row_loss[i] = lse - (sum_p c_ip) / (tau |P(i)|) on a valid row (|P(i)| > 0), else 0.  grid N, block 256.
__global__ void __launch_bounds__(256)
supcon_rows_kernel(float* __restrict__ G, int ldg, const float* __restrict__ E, int D,
                   const int64_t* __restrict__ labels, int N, double inv_tau, float* __restrict__ cos_out,
                   float* __restrict__ lse, float* __restrict__ row_loss) {
  __shared__ float redf[8];
  __shared__ double red[3][8];
  const int i = blockIdx.x, lane = threadIdx.x & 31;
  float* g = G + static_cast<size_t>(i) * ldg;
  float* co = cos_out + static_cast<size_t>(i) * N;
  const int64_t y = labels[i];
  const float* ei = E + static_cast<size_t>(i) * D;
  for (int j0 = threadIdx.x & ~31; j0 < N; j0 += blockDim.x) {
    const int j = j0 + lane;
    unsigned m = __ballot_sync(0xffffffffu, j < N && j != i && labels[j] == y);
    while (m) {
      const int jj = j0 + __ffs(m) - 1;
      m &= m - 1;
      const double v = supcon_cos64_warp(ei, E + static_cast<size_t>(jj) * D, D);
      if (lane == 0) g[jj] = static_cast<float>(v);
    }
  }
  __syncthreads();
  float cmax = -INFINITY;
  double psum = 0.0, pcnt = 0.0;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float c = g[j];
    co[j] = c;
    if (j == i) continue;
    cmax = fmaxf(cmax, c);
    if (labels[j] == y) {
      psum += c;
      pcnt += 1.0;
    }
  }
  cmax = block_reduce_max(cmax, redf);
  double z = 0.0;
  for (int j = threadIdx.x; j < N; j += blockDim.x)
    if (j != i) z += expf(static_cast<float>((static_cast<double>(g[j]) - cmax) * inv_tau));
  supcon_block_sum3(z, psum, pcnt, red);
  if (threadIdx.x == 0) {
    const double l = cmax * inv_tau + log(z);
    lse[i] = static_cast<float>(l);
    row_loss[i] = pcnt > 0.0 ? static_cast<float>(l - psum * inv_tau / pcnt) : 0.f;
  }
}

// Backward rows: with e_j = exp(s_ij - lse_i) over j != i, Z = sum_j e_j (the saved lse's rounding cancels in e_j / Z),
// E+ and E- the sums over the positives and the negatives (fp64):
//   dS_ij = e_j / Z (negative j),  ((e_p - E+ / |P|) - E- / |P|) / Z (positive p): p_p - 1/|P| without the cancellation
//   of 1/|P| against p_p (exactly -E- / Z at |P| = 1, NT-Xent's positive);
//   dC_ij = grad_loss / (V tau) dS_ij, exactly 0 on the diagonal, on invalid rows and past N.
// dC goes to the fp32 workspace dcos [Np][Cp] and, times the row's power of two 2^e (rinv[i] = 2^-e), to the K-sliced
// A-side image dimg [Np][3 Cp] = [lo | hi | hi] of gE^ = dC E^, as aam_dcos_kernel writes them.  grid Np, block 256.
__global__ void __launch_bounds__(256)
supcon_dcos_kernel(const float* __restrict__ cos, const float* __restrict__ lse, const int64_t* __restrict__ labels,
                   int N, int V, double inv_tau, const float* __restrict__ grad_loss, int Cp, float* __restrict__ dcos,
                   uint16_t* __restrict__ dimg, float* __restrict__ rinv) {
  __shared__ float redf[8];
  __shared__ double red[3][8];
  const int i = blockIdx.x;
  float* d = dcos + static_cast<size_t>(i) * Cp;
  const int Np = gridDim.x;
  if (i >= N) {
    for (int c = threadIdx.x; c < Cp; c += blockDim.x) {
      d[c] = 0.f;
      dimg[aam_kslice_off(i, Np, 0, c, Cp)] = dimg[aam_kslice_off(i, Np, 1, c, Cp)] =
          dimg[aam_kslice_off(i, Np, 2, c, Cp)] = 0;
    }
    if (threadIdx.x == 0) rinv[i] = 1.f;
    return;
  }
  const float* co = cos + static_cast<size_t>(i) * N;
  const int64_t y = labels[i];
  const double l = lse[i];
  double ep = 0.0, en = 0.0, cnt = 0.0;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    if (j == i) continue;
    const float e = supcon_exp(co[j], inv_tau, l);
    if (labels[j] == y) {
      ep += e;
      cnt += 1.0;
    } else {
      en += e;
    }
  }
  supcon_block_sum3(ep, en, cnt, red);
  const bool valid = cnt > 0.0;
  const double coef = static_cast<double>(grad_loss[0]) * inv_tau / V / (ep + en);
  const double pm = valid ? ep / cnt : 0.0, nm = valid ? en / cnt : 0.0;
  float mx = 0.f;
  for (int j = threadIdx.x; j < Cp; j += blockDim.x) {
    float v = 0.f;
    if (valid && j < N && j != i) {
      const double e = supcon_exp(co[j], inv_tau, l);
      v = static_cast<float>(coef * (labels[j] == y ? (e - pm) - nm : e));
    }
    d[j] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  const int e = aam_scale_exp(block_reduce_max(mx, redf));
  if (threadIdx.x == 0) rinv[i] = aam_pow2(-e);
  const float S = aam_pow2(e);
  for (int c = threadIdx.x; c < Cp; c += blockDim.x) {
    uint16_t hi, lo;
    aam_split16(d[c] * S, hi, lo);
    dimg[aam_kslice_off(i, Np, 0, c, Cp)] = lo;
    dimg[aam_kslice_off(i, Np, 1, c, Cp)] = hi;
    dimg[aam_kslice_off(i, Np, 2, c, Cp)] = hi;
  }
}

}  // namespace dsk
