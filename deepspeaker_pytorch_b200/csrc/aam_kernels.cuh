// Additive angular margin softmax (ArcFace / AAM-softmax) over a cosine classifier: the element-wise and row kernels
// around the tensor-core cosine GEMMs (dsk_aam_softmax_sc / dsk_aam_softmax_sc_bwd in dsk_api.cu, of which
// dsk_aam_softmax / _bwd are the K = 1, topk = 0 calls).
//
// The three GEMMs (cos = E^ W^T, gE^ = dcos W^, gW^ = dcos^T E^) run on conv_umma_kernel as plain GEMMs with fp16
// operands split into hi/lo halves (x = hi + lo, 22 significant bits) and concatenated along K, so that one fp32
// accumulator sums lo*hi + hi*lo + hi*hi.  The "A" side of a GEMM is laid out [lo | hi | hi], the "B" side
// [hi | lo | hi]: the two small lo-products come first in K (they are summed while the accumulator is still small).
// The tensor cores add each 16-wide K step to the fp32 accumulator with truncation, so the error grows with the number
// of steps times the accumulator's size.  The backward GEMMs (K = 3 Cp and 3 Np) therefore run in K slices of
// kAamSlice classes / utterances, each slice a GEMM of its own into its own fp32 output, summed in slice order by the
// Jacobian kernel (deterministic split K); and the target column's cosine, where an embedding sits close to its class
// centre, is recomputed in fp64 from the fp32 inputs.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "head_kernels.cuh"

namespace dsk {

constexpr int kAamSlice = 512;  // classes (gE^) or utterances (gW^) per K slice of a backward GEMM

// Element (row, seg, k) of a K-sliced backward operand image over Kp columns: slice s = k / kAamSlice holds columns
// [s kAamSlice, s kAamSlice + w) as a [rows][3w] image (segments seg = 0, 1, 2 of width w), slices one after another
// kAamSlice * 3 * rows elements apart.
__device__ __forceinline__ size_t aam_kslice_off(int row, int rows, int seg, int k, int Kp) {
  const int sl = k / kAamSlice, kk = k - sl * kAamSlice;
  const int w = Kp - sl * kAamSlice < kAamSlice ? Kp - sl * kAamSlice : kAamSlice;
  return static_cast<size_t>(sl) * kAamSlice * 3 * rows + static_cast<size_t>(row) * 3 * w + seg * w + kk;
}

struct AamMargin {
  float cos_m, sin_m;  // cos m, sin m
  float th, mm;        // cos(pi - m), sin(pi - m) * m: below th the target logit is cos - mm (non-"easy" margin)
  float s;             // scale
  float cos_t, sin_t;  // cos m', sin m' of the inter-top-k margin
};

// phi(cos) of the target column
__device__ __forceinline__ float aam_phi(float c, const AamMargin& a) {
  const float sn = sqrtf(fminf(fmaxf(1.f - c * c, 0.f), 1.f));
  return c > a.th ? c * a.cos_m - sn * a.sin_m : c - a.mm;
}
// d phi / d cos; at sin = 0 (a row on its class centre) the finite limit cos m
__device__ __forceinline__ float aam_dphi(float c, const AamMargin& a) {
  if (!(c > a.th)) return 1.f;
  const float sn = sqrtf(fminf(fmaxf(1.f - c * c, 0.f), 1.f));
  return sn > 0.f ? a.cos_m + a.sin_m * c / sn : a.cos_m;
}
// psi(cos) = cos(theta - m') of a class in the row's top-k set
__device__ __forceinline__ float aam_psi(float c, const AamMargin& a) {
  const float sn = sqrtf(fminf(fmaxf(1.f - c * c, 0.f), 1.f));
  return c * a.cos_t + sn * a.sin_t;
}
// d psi / d cos; at sin = 0 the finite value cos m', as aam_dphi
__device__ __forceinline__ float aam_dpsi(float c, const AamMargin& a) {
  const float sn = sqrtf(fminf(fmaxf(1.f - c * c, 0.f), 1.f));
  return sn > 0.f ? a.cos_t - a.sin_t * c / sn : a.cos_t;
}

// Key of class c with class cosine v in the top-k order: a larger key ranks first.  Larger cosines first, ties to the
// lower class, -0 == +0, and NaN after every number (-inf included), as dsk_topk_indices orders.  Keys are distinct and
// nonzero.
__device__ __forceinline__ unsigned long long aam_topk_key(float v, int c) {
  uint32_t u = __float_as_uint(v == 0.f ? 0.f : v);
  u = isnan(v) ? 0u : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));
  return (static_cast<unsigned long long>(u) << 32) | (0xffffffffu - static_cast<uint32_t>(c));
}
__device__ __forceinline__ unsigned long long block_reduce_max_u64(unsigned long long v, unsigned long long* red) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t > v ? t : v;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long t = red[0];
  for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) t = red[i] > t ? red[i] : t;
  __syncthreads();
  return t;
}

// fp64 cosine of the fp32 rows e and w (D wide) with F.normalize's 1e-12 floors, summed in a fixed order; the value is
// that of thread 0 (0 elsewhere).  Block 256; red3 [3][8] is free again on return.
__device__ double aam_cos64(const float* __restrict__ e, const float* __restrict__ w, int D, double (*red3)[8]) {
  double ew = 0.0, ee = 0.0, ww = 0.0;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
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
  if ((threadIdx.x & 31) == 0) {
    red3[0][threadIdx.x >> 5] = ew;
    red3[1][threadIdx.x >> 5] = ee;
    red3[2][threadIdx.x >> 5] = ww;
  }
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0) {
    for (int k = 1; k < static_cast<int>(blockDim.x >> 5); ++k) {
      ew += red3[0][k];
      ee += red3[1][k];
      ww += red3[2][k];
    }
    r = ew / (fmax(sqrt(ee), 1e-12) * fmax(sqrt(ww), 1e-12));
  }
  __syncthreads();
  return r;
}

// Sub-centre max: v replaces the running best b when b is a number and v is NaN or larger (ties keep the lower k, the
// first NaN wins and stays)
template <typename T>
__device__ __forceinline__ bool aam_sub_better(T v, T b) {
  return !isnan(b) && (isnan(v) || v > b);
}

__device__ __forceinline__ void aam_split16(float x, uint16_t& hi, uint16_t& lo) {
  const __half h = __float2half_rn(x);
  hi = __half_as_ushort(h);
  lo = __half_as_ushort(__float2half_rn(x - __half2float(h)));  // x - hi is exact in fp32
}

// Exponent e of the power of two 2^e that puts max|v| of a row (column) of dcos at [256, 512): the hi/lo halves of the
// scaled values stay in fp16's normal range.  0 for an all-zero or non-finite row.
__device__ __forceinline__ int aam_scale_exp(float m) {
  if (!(m > 0.f) || !isfinite(m)) return 0;
  const int e = static_cast<int>(floorf(log2f(512.f / m)));
  return e < -24 ? -24 : (e > 100 ? 100 : e);
}
// 2^e for |e| <= 100, exactly
__device__ __forceinline__ float aam_pow2(int e) { return __int_as_float((127 + e) << 23); }

// nrm[r] = max(||X[r]||, 1e-12) (F.normalize's denominator); one warp per row, fixed order.  grid ceil(rows / 8), block 256.
__global__ void __launch_bounds__(256) aam_norm_kernel(const float* __restrict__ X, int rows, int D, float* __restrict__ nrm) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* x = X + static_cast<size_t>(r) * D;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) s = fmaf(x[d], x[d], s);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) nrm[r] = fmaxf(sqrtf(s), 1e-12f);
}

// x^ = X[r] / nrm[r] split into fp16 hi/lo operand images; rows in [rows, rows_pad) are zero.
//   img  (may be NULL): [rows_pad][3D], [lo | hi | hi] (lo_first, the A side) or [hi | lo | hi] (B side)
//   imgT (may be NULL): [D][3 rows_pad] K-sliced (aam_kslice_off), [hi | lo | hi]: the transposed B-side image of the
//                       backward GEMMs
// grid (D / 64, rows_pad / 32), block 256.
__global__ void __launch_bounds__(256)
aam_split_kernel(const float* __restrict__ X, const float* __restrict__ nrm, int rows, int rows_pad, int D, int lo_first,
                 uint16_t* __restrict__ img, uint16_t* __restrict__ imgT) {
  __shared__ float t[32][65];
  const int r0 = blockIdx.y * 32, d0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 63;
  for (int rr = threadIdx.x >> 6; rr < 32; rr += 4) {
    const int r = r0 + rr;
    const float v = r < rows ? X[static_cast<size_t>(r) * D + d0 + tx] / nrm[r] : 0.f;
    t[rr][tx] = v;
    if (img) {
      uint16_t hi, lo;
      aam_split16(v, hi, lo);
      uint16_t* o = img + static_cast<size_t>(r) * 3 * D + d0 + tx;
      o[0] = lo_first ? lo : hi;
      o[D] = lo_first ? hi : lo;
      o[2 * D] = hi;
    }
  }
  if (!imgT) return;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < 64; k += 8) {
    uint16_t hi, lo;
    aam_split16(t[lane][k], hi, lo);
    imgT[aam_kslice_off(d0 + k, D, 0, r0 + lane, rows_pad)] = hi;
    imgT[aam_kslice_off(d0 + k, D, 1, r0 + lane, rows_pad)] = lo;
    imgT[aam_kslice_off(d0 + k, D, 2, r0 + lane, rows_pad)] = hi;
  }
}

// Forward rows over C classes of K sub-centres each (columns c K + k of the GEMM's padded output G; K = 1 and topk = 0
// is the plain AAM-softmax):
//   cos_out[i][c] = max_k G[i][cK + k] and sub[i][c] (may be NULL) its argmax, by aam_sub_better; on the target column
//     all K cosines are recomputed in fp64 from E[i] and W[yK + k] (a row near its class centre has cos ~ 1 there, where
//     the GEMM's accumulation error is largest), the max taken in fp64 and rounded once;
//   top[i] (topk of them) = the non-target classes first in aam_topk_key's order, by topk block arg-max passes (each the
//     largest key below the previous one); a class is in the set when its key is at least the last one's;
//   logits s cos, s phi on the target column, s psi in the top-k set; lse[i] = logsumexp over all C in a fixed order,
//   row_loss[i] = lse[i] - s*phi (NaN for a label outside [0, C)).  grid N, block 256.
__global__ void __launch_bounds__(256)
aam_rows_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ E, const float* __restrict__ W, int D,
                const int64_t* __restrict__ labels, int C, int K, int topk, AamMargin a, float* __restrict__ cos_out,
                uint8_t* __restrict__ sub, int32_t* __restrict__ top, float* __restrict__ lse,
                float* __restrict__ row_loss) {
  __shared__ float red[8];
  __shared__ double red3[3][8];
  __shared__ unsigned long long redk[8];
  __shared__ float tcos;
  __shared__ int tsub;
  const int i = blockIdx.x;
  const float* g = G + static_cast<size_t>(i) * ldg;
  float* co = cos_out + static_cast<size_t>(i) * C;
  const int64_t y = labels[i];
  const bool ok = y >= 0 && y < C;
  if (ok) {
    const float* e = E + static_cast<size_t>(i) * D;
    double best = 0.0;
    int bk = 0;
    for (int k = 0; k < K; ++k) {
      const double v = aam_cos64(e, W + (static_cast<size_t>(y) * K + k) * D, D, red3);
      if (k == 0 || aam_sub_better(v, best)) {
        best = v;
        bk = k;
      }
    }
    if (threadIdx.x == 0) {
      tcos = static_cast<float>(best);
      tsub = bk;
    }
    __syncthreads();
  }
  float m = -INFINITY;  // the row's largest logit; without a top-k set taken in the same pass
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float cv;
    int ak = 0;
    const bool tgt = ok && c == y;
    if (tgt) {
      cv = tcos;
      ak = tsub;
    } else {
      const float* gc = g + static_cast<size_t>(c) * K;
      cv = gc[0];
      for (int k = 1; k < K; ++k)
        if (aam_sub_better(gc[k], cv)) {
          cv = gc[k];
          ak = k;
        }
    }
    co[c] = cv;
    if (sub) sub[static_cast<size_t>(i) * C + c] = static_cast<uint8_t>(ak);
    if (topk == 0) m = fmaxf(m, a.s * (tgt ? aam_phi(cv, a) : cv));
  }
  unsigned long long thr = ~0ull;
  if (topk > 0) {
    __syncthreads();  // the row's class cosines, written above by every thread
    for (int j = 0; j < topk; ++j) {
      unsigned long long b = 0;
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        if (ok && c == y) continue;
        const unsigned long long kc = aam_topk_key(co[c], c);
        if (kc < thr && kc > b) b = kc;
      }
      thr = block_reduce_max_u64(b, redk);
      if (threadIdx.x == 0) top[static_cast<size_t>(i) * topk + j] = static_cast<int32_t>(0xffffffffu - static_cast<uint32_t>(thr));
    }
  }
  auto logit = [&](int c) {
    const float cv = co[c];
    if (ok && c == y) return aam_phi(cv, a);
    return topk > 0 && aam_topk_key(cv, c) >= thr ? aam_psi(cv, a) : cv;
  };
  if (topk > 0)
    for (int c = threadIdx.x; c < C; c += blockDim.x) m = fmaxf(m, a.s * logit(c));
  m = block_reduce_max(m, red);
  float sum = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) sum += expf(a.s * logit(c) - m);
  sum = block_reduce_sum(sum, red);
  if (threadIdx.x == 0) {
    const float l = m + logf(sum);
    lse[i] = l;
    row_loss[i] = ok ? l - a.s * aam_phi(tcos, a) : __int_as_float(0x7fc00000);
  }
}

// Backward rows: the class gradient dc[i][c] = s (softmax - onehot) grad_loss / N, times dphi/dcos on the target column
// and dpsi/dcos in the top-k set (the classes whose key is at least that of top[i][topk - 1]), goes to column
// c K + sub[i][c] of the fp32 workspace dcos [Np][Cp] (sub may be NULL when K = 1); the other K - 1 columns of the class
// are 0.  dcos is also written, multiplied by the row's power of two 2^e (rinv[i] = 2^-e), into the K-sliced A-side
// image dimg [Np][3 Cp] = [lo | hi | hi] of gE^ = dcos W^.  The probabilities are e_c / sum_c e_c with
// e_c = exp(logit - lse): the division removes the rounding of the saved lse, and the target's softmax - 1 is minus the
// sum over the other classes, which keeps its relative accuracy in rows that are already well classified.  Rows i >= N
// and columns past C K are zero.  grid Np, block 256.
__global__ void __launch_bounds__(256)
aam_dcos_kernel(const float* __restrict__ cos, const uint8_t* __restrict__ sub, const int32_t* __restrict__ top,
                const float* __restrict__ lse, const int64_t* __restrict__ labels, int N, int C, int K, int Cp, int topk,
                AamMargin a, const float* __restrict__ grad_loss, float* __restrict__ dcos, uint16_t* __restrict__ dimg,
                float* __restrict__ rinv) {
  __shared__ float red[8];
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
  const float* co = cos + static_cast<size_t>(i) * C;
  const int64_t y = labels[i];
  const bool ok = y >= 0 && y < C;
  const float l = lse[i];
  unsigned long long thr = ~0ull;
  if (topk > 0) {
    const int t = top[static_cast<size_t>(i) * topk + topk - 1];
    if (t >= 0 && t < C) thr = aam_topk_key(co[t], t);
  }
  auto in_top = [&](int c, float cv) { return topk > 0 && aam_topk_key(cv, c) >= thr; };
  float sig = 0.f, other = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const bool tgt = ok && c == y;
    const float cv = co[c];
    const float e = expf(a.s * (tgt ? aam_phi(cv, a) : (in_top(c, cv) ? aam_psi(cv, a) : cv)) - l);
    sig += e;
    if (!tgt) other += e;
  }
  sig = block_reduce_sum(sig, red);
  other = block_reduce_sum(other, red);
  const float coef = grad_loss[0] / static_cast<float>(N) * a.s / sig;
  const uint8_t* sb = sub ? sub + static_cast<size_t>(i) * C : nullptr;
  const int CK = C * K;
  float mx = 0.f;
  for (int j = threadIdx.x; j < Cp; j += blockDim.x) {
    float v = 0.f;
    const int c = K == 1 ? j : j / K;
    if (j < CK && (K == 1 || j - c * K == sb[c])) {
      const float cv = co[c];
      if (ok && c == y) v = -other * coef * aam_dphi(cv, a);
      else if (in_top(c, cv)) v = expf(a.s * aam_psi(cv, a) - l) * coef * aam_dpsi(cv, a);
      else v = expf(a.s * cv - l) * coef;
    }
    d[j] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  const int e = aam_scale_exp(block_reduce_max(mx, red));
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

// Each row's fp64 cosines to the K sub-centres of its own class, rounded once: out[i][k] = cos(E[i], W[y_i K + k]),
// the forward's target recompute (NaN for a label outside [0, C)).  grid N, block 256.
__global__ void __launch_bounds__(256)
aam_subcentre_cos_kernel(const float* __restrict__ E, const float* __restrict__ W, const int64_t* __restrict__ labels,
                         int C, int K, int D, float* __restrict__ out) {
  __shared__ double red3[3][8];
  const int i = blockIdx.x;
  const int64_t y = labels[i];
  float* o = out + static_cast<size_t>(i) * K;
  if (!(y >= 0 && y < C)) {
    if (threadIdx.x < K) o[threadIdx.x] = __int_as_float(0x7fc00000);
    return;
  }
  for (int k = 0; k < K; ++k) {
    const double v = aam_cos64(E + static_cast<size_t>(i) * D, W + (static_cast<size_t>(y) * K + k) * D, D, red3);
    if (threadIdx.x == 0) o[k] = static_cast<float>(v);
  }
}

// The A-side image of gW^ = dcos^T E^: K-sliced dimgT [Cp][3 Np] = [lo | hi | hi] of column c of dcos times its own power of two
// 2^e_c (cinv[c] = 2^-e_c; a per-column scale keeps classes whose every probability is small out of fp16's subnormals).
// grid Cp / 32, block 256.
__global__ void __launch_bounds__(256)
aam_dcos_t_kernel(const float* __restrict__ dcos, int Np, int Cp, uint16_t* __restrict__ dimgT, float* __restrict__ cinv) {
  __shared__ float tile[32][33];
  __shared__ float red[8][32];
  __shared__ float scl[32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32;
  float mx = 0.f;
  for (int i = ty; i < Np; i += 8) mx = fmaxf(mx, fabsf(dcos[static_cast<size_t>(i) * Cp + c0 + tx]));
  red[ty][tx] = mx;
  __syncthreads();
  if (ty == 0) {
    for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k][tx]);
    const int e = aam_scale_exp(mx);
    scl[tx] = aam_pow2(e);
    cinv[c0 + tx] = aam_pow2(-e);
  }
  __syncthreads();
  const float* src = dcos + static_cast<size_t>(ty) * Cp + c0 + tx;
  for (int i0 = 0; i0 < Np; i0 += 32) {
#pragma unroll
    for (int r = 0; r < 32; r += 8) tile[ty + r][tx] = src[static_cast<size_t>(i0 + r) * Cp];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 32; r += 8) {
      uint16_t hi, lo;
      aam_split16(tile[tx][ty + r] * scl[ty + r], hi, lo);
      dimgT[aam_kslice_off(c0 + ty + r, Cp, 0, i0 + tx, Np)] = lo;
      dimgT[aam_kslice_off(c0 + ty + r, Cp, 1, i0 + tx, Np)] = hi;
      dimgT[aam_kslice_off(c0 + ty + r, Cp, 2, i0 + tx, Np)] = hi;
    }
    __syncthreads();
  }
}

// The F.normalize Jacobian: out[r] = (g - x^ (x^ . g)) / nrm[r] with x^ = X[r] / nrm[r] and g = the sum of the K
// slices' GEMM rows G[s][r] (slices `slice_elems` apart, added in slice order) times ginv[r] (un-scaling by its exact
// power of two).  One warp per row, fixed order.  grid ceil(rows / 8), block 256.
__global__ void __launch_bounds__(256)
aam_normalize_bwd_kernel(const float* __restrict__ X, const float* __restrict__ nrm, const float* __restrict__ G,
                         int slices, long slice_elems, const float* __restrict__ ginv, int rows, int D,
                         float* __restrict__ out) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* x = X + static_cast<size_t>(r) * D;
  const float* g = G + static_cast<size_t>(r) * D;
  const float n = nrm[r], gi = ginv[r];
  auto grad = [&](int d) {
    float v = g[d];
    for (int s = 1; s < slices; ++s) v += g[s * slice_elems + d];
    return v * gi;
  };
  float dot = 0.f;
  for (int d = lane; d < D; d += 32) dot = fmaf(x[d] / n, grad(d), dot);
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  float* y = out + static_cast<size_t>(r) * D;
  for (int d = lane; d < D; d += 32) y[d] = (grad(d) - (x[d] / n) * dot) / n;
}

// ---- the class-sharded op (dsk_aam_shard_*): rank r holds the classes [c0, c0 + Cr) of C, all N gathered rows --------
// Local class c is global class c0 + c; c0 is a multiple of kAamShardBlock, so the 128-class blocks of a shard are
// blocks of the global class axis and the block partials below do not depend on the split.
constexpr int kAamShardBlock = 128;

// The logit of local class c with class cosine cv: s phi on the row's target (local index yl, -1 when the target is
// on another rank or the label is invalid), s psi when the global key is at least the top-k threshold thr, else s cos.
__device__ __forceinline__ float aam_shard_logit(float cv, int c, int yl, int c0, int topk, unsigned long long thr,
                                                 const AamMargin& a) {
  if (c == yl) return a.s * aam_phi(cv, a);
  return a.s * (topk > 0 && aam_topk_key(cv, c0 + c) >= thr ? aam_psi(cv, a) : cv);
}

__device__ __forceinline__ int aam_shard_target(int64_t y, int c0, int Cr) {
  return y >= c0 && y < static_cast<int64_t>(c0) + Cr ? static_cast<int>(y - c0) : -1;
}

// Stage 1: class cosines and sub-centre argmax of the shard (aam_rows_kernel's first pass over the shard's columns of
// the padded GEMM output G, the target recomputed in fp64 when it is local), then the row's local top-k candidate keys
// keys[i] (topk of them, global class ids, target excluded, ranked by topk block arg-max passes; 0 once the shard has
// no candidate left).  grid N, block 256.
__global__ void __launch_bounds__(256)
aam_shard_cos_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ E, const float* __restrict__ W,
                     int D, const int64_t* __restrict__ labels, int c0, int Cr, int K, int topk,
                     float* __restrict__ cos_out, uint8_t* __restrict__ sub, unsigned long long* __restrict__ keys) {
  __shared__ double red3[3][8];
  __shared__ unsigned long long redk[8];
  __shared__ float tcos;
  __shared__ int tsub;
  const int i = blockIdx.x;
  const float* g = G + static_cast<size_t>(i) * ldg;
  float* co = cos_out + static_cast<size_t>(i) * Cr;
  const int yl = aam_shard_target(labels[i], c0, Cr);
  if (yl >= 0) {
    const float* e = E + static_cast<size_t>(i) * D;
    double best = 0.0;
    int bk = 0;
    for (int k = 0; k < K; ++k) {
      const double v = aam_cos64(e, W + (static_cast<size_t>(yl) * K + k) * D, D, red3);
      if (k == 0 || aam_sub_better(v, best)) {
        best = v;
        bk = k;
      }
    }
    if (threadIdx.x == 0) {
      tcos = static_cast<float>(best);
      tsub = bk;
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < Cr; c += blockDim.x) {
    float cv;
    int ak = 0;
    if (c == yl) {
      cv = tcos;
      ak = tsub;
    } else {
      const float* gc = g + static_cast<size_t>(c) * K;
      cv = gc[0];
      for (int k = 1; k < K; ++k)
        if (aam_sub_better(gc[k], cv)) {
          cv = gc[k];
          ak = k;
        }
    }
    co[c] = cv;
    if (sub) sub[static_cast<size_t>(i) * Cr + c] = static_cast<uint8_t>(ak);
  }
  if (topk == 0) return;
  __syncthreads();
  unsigned long long thr = ~0ull;
  for (int j = 0; j < topk; ++j) {
    unsigned long long b = 0;
    for (int c = threadIdx.x; c < Cr; c += blockDim.x) {
      if (c == yl) continue;
      const unsigned long long kc = aam_topk_key(co[c], c0 + c);
      if (kc < thr && kc > b) b = kc;
    }
    thr = block_reduce_max_u64(b, redk);
    if (threadIdx.x == 0) keys[static_cast<size_t>(i) * topk + j] = thr;
  }
}

// Stage 2: the global top-k of row i from every rank's candidates keys_all [R][N][topk] (the topk largest keys, by topk
// block arg-max passes: the keys are distinct but for the 0 sentinels, and topk <= C - 1 real ones exist), top[i] their
// global class ids and thr[i] the last key; then mloc[i], the largest logit of the shard's classes.  grid N, block 256.
__global__ void __launch_bounds__(256)
aam_shard_merge_kernel(const float* __restrict__ cos, const int64_t* __restrict__ labels,
                       const unsigned long long* __restrict__ keys_all, int R, int N, int c0, int Cr, int topk,
                       AamMargin a, int32_t* __restrict__ top, unsigned long long* __restrict__ thr_out,
                       float* __restrict__ mloc) {
  __shared__ float red[8];
  __shared__ unsigned long long redk[8];
  const int i = blockIdx.x;
  const int yl = aam_shard_target(labels[i], c0, Cr);
  unsigned long long thr = ~0ull;
  if (topk > 0) {
    for (int j = 0; j < topk; ++j) {
      unsigned long long b = 0;
      for (int t = threadIdx.x; t < R * topk; t += blockDim.x) {
        const int r = t / topk;
        const unsigned long long kc = keys_all[(static_cast<size_t>(r) * N + i) * topk + (t - r * topk)];
        if (kc < thr && kc > b) b = kc;
      }
      thr = block_reduce_max_u64(b, redk);
      if (threadIdx.x == 0) top[static_cast<size_t>(i) * topk + j] = static_cast<int32_t>(0xffffffffu - static_cast<uint32_t>(thr));
    }
    if (threadIdx.x == 0) thr_out[i] = thr;
  }
  const float* co = cos + static_cast<size_t>(i) * Cr;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < Cr; c += blockDim.x) m = fmaxf(m, aam_shard_logit(co[c], c, yl, c0, topk, thr, a));
  m = block_reduce_max(m, red);
  if (threadIdx.x == 0) mloc[i] = m;
}

// Stage 3: m[i] = the largest of the ranks' maxima maxima [R][N] (exact in any order), and the record of row i over
// the shard: rec[i] = [S_b, S_other_b] for b < nb, then the target logit and the flags (as float bits), 2 nb + 2 floats.
// S_b is the sum of exp(logit - m) over the classes of the shard's block b (one thread per class, a fixed tree: the sum
// depends on the block's classes only), S_other_b the same without the target; blocks past the shard are +0.  A NaN
// term sets flag 1 and is left out of the sums; flag 2: the target is on this shard and rec[2 nb] = s phi(cos_target);
// bits 8 and up: the shard's block count ceil(Cr / 128), which places its blocks on the global block axis in stage 4.
// grid N, block kAamShardBlock.
__global__ void __launch_bounds__(kAamShardBlock)
aam_shard_partials_kernel(const float* __restrict__ cos, const int64_t* __restrict__ labels,
                          const unsigned long long* __restrict__ thr_in, const float* __restrict__ maxima, int R, int N,
                          int c0, int Cr, int topk, int nb, AamMargin a, float* __restrict__ m_out,
                          float* __restrict__ rec) {
  __shared__ float red[2][kAamShardBlock / 32];
  const int i = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int yl = aam_shard_target(labels[i], c0, Cr);
  float m = maxima[i];
  for (int r = 1; r < R; ++r) m = fmaxf(m, maxima[static_cast<size_t>(r) * N + i]);
  const unsigned long long thr = topk > 0 ? thr_in[i] : ~0ull;
  const float* co = cos + static_cast<size_t>(i) * Cr;
  float* out = rec + static_cast<size_t>(i) * (2 * nb + 2);
  int nan = 0;
  for (int blk = 0; blk < nb; ++blk) {
    const int c = blk * kAamShardBlock + threadIdx.x;
    float s = 0.f, so = 0.f;
    if (c < Cr) {
      const float e = expf(aam_shard_logit(co[c], c, yl, c0, topk, thr, a) - m);
      if (isnan(e)) {
        nan = 1;
      } else {
        s = e;
        so = c == yl ? 0.f : e;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      so += __shfl_xor_sync(0xffffffffu, so, o);
    }
    if (lane == 0) {
      red[0][w] = s;
      red[1][w] = so;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int k = 1; k < kAamShardBlock / 32; ++k) {
        s += red[0][k];
        so += red[1][k];
      }
      out[2 * blk] = s;
      out[2 * blk + 1] = so;
    }
    __syncthreads();
  }
  nan = __syncthreads_or(nan);
  if (threadIdx.x == 0) {
    out[2 * nb] = yl >= 0 ? a.s * aam_phi(co[yl], a) : 0.f;
    const int nbr = (Cr + kAamShardBlock - 1) / kAamShardBlock;
    out[2 * nb + 1] = __int_as_float((nan ? 1 : 0) | (yl >= 0 ? 2 : 0) | (nbr << 8));
    m_out[i] = m;
  }
}

// Stage 4, on every rank alike: the records of all ranks rec_all [R][N][2 nb + 2] summed in fp64 in an order fixed by
// the global block index g alone (rank r's blocks are g = its predecessors' block counts + b), so the sums do not depend
// on R or the split: lane g mod 32 adds its blocks in ascending g, then a fixed butterfly over the 32 lanes.  lse[i] =
// m + log S rounded once, row_loss[i] = lse - the target logit (NaN for a label outside [0, C)), den[i] = (S, S_other)
// in fp32; a NaN flag makes all four NaN.  One warp per row, lane-contiguous loads; grid ceil(N / 8), block 256.
__global__ void __launch_bounds__(256)
aam_shard_finish_kernel(const float* __restrict__ rec_all, const float* __restrict__ m, const int64_t* __restrict__ labels,
                        int R, int N, int C, int nb, float* __restrict__ lse, float* __restrict__ row_loss,
                        float* __restrict__ den) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= N) return;
  const size_t w = 2 * static_cast<size_t>(nb) + 2;
  auto rec = [&](int r) { return rec_all + (static_cast<size_t>(r) * N + i) * w; };
  auto flags_of = [&](int r) { return __float_as_int(rec(r)[2 * nb + 1]); };
  int fl = 0, total = 0;
  float t = 0.f;
  for (int r = lane; r < R; r += 32) {
    const int f = flags_of(r);
    fl |= f & 3;
    total += f >> 8;
    if (f & 2) t = rec(r)[2 * nb];
  }
  const unsigned own = __ballot_sync(0xffffffffu, fl & 2);
  t = own ? __shfl_sync(0xffffffffu, t, __ffs(own) - 1) : 0.f;
  const int flags = __reduce_or_sync(0xffffffffu, fl);
  total = __reduce_add_sync(0xffffffffu, total);
  double S = 0.0, So = 0.0;
  int r = 0, off = 0, cnt = flags_of(0) >> 8;
  for (int g = lane; g < total; g += 32) {
    while (g >= off + cnt) {
      off += cnt;
      cnt = flags_of(++r) >> 8;
    }
    const float* p = rec(r) + 2 * (g - off);
    S += p[0];
    So += p[1];
  }
  for (int o = 16; o > 0; o >>= 1) {
    S += __shfl_xor_sync(0xffffffffu, S, o);
    So += __shfl_xor_sync(0xffffffffu, So, o);
  }
  if (lane) return;
  const float qnan = __int_as_float(0x7fc00000);
  const int64_t y = labels[i];
  const bool nan = flags & 1;
  const float l = nan ? qnan : static_cast<float>(static_cast<double>(m[i]) + log(S));
  lse[i] = l;
  row_loss[i] = y >= 0 && y < C && (flags & 2) ? l - t : qnan;
  den[2 * i] = nan ? qnan : static_cast<float>(S);
  den[2 * i + 1] = nan ? qnan : static_cast<float>(So);
}

// Backward dcos over the shard's columns for all N rows: aam_dcos_kernel's values with the probabilities
// exp(logit - m) / S and the target's softmax - 1 = -S_other / S from the forward's den = (S, S_other); the row's
// power-of-two scale is that of the shard's columns.  grid Np, block 256.
__global__ void __launch_bounds__(256)
aam_shard_dcos_kernel(const float* __restrict__ cos, const uint8_t* __restrict__ sub,
                      const unsigned long long* __restrict__ thr_in, const float* __restrict__ m_in,
                      const float* __restrict__ den, const int64_t* __restrict__ labels, int N, int c0, int Cr, int K,
                      int Cp, int topk, AamMargin a, const float* __restrict__ grad_loss, float* __restrict__ dcos,
                      uint16_t* __restrict__ dimg, float* __restrict__ rinv) {
  __shared__ float red[8];
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
  const float* co = cos + static_cast<size_t>(i) * Cr;
  const int yl = aam_shard_target(labels[i], c0, Cr);
  const unsigned long long thr = topk > 0 ? thr_in[i] : ~0ull;
  const float m = m_in[i], S = den[2 * i], So = den[2 * i + 1];
  const float coef = grad_loss[0] / static_cast<float>(N) * a.s / S;
  const uint8_t* sb = sub ? sub + static_cast<size_t>(i) * Cr : nullptr;
  const int CK = Cr * K;
  float mx = 0.f;
  for (int j = threadIdx.x; j < Cp; j += blockDim.x) {
    float v = 0.f;
    const int c = K == 1 ? j : j / K;
    if (j < CK && (K == 1 || j - c * K == sb[c])) {
      const float cv = co[c];
      if (c == yl) v = -So * coef * aam_dphi(cv, a);
      else if (topk > 0 && aam_topk_key(cv, c0 + c) >= thr) v = expf(a.s * aam_psi(cv, a) - m) * coef * aam_dpsi(cv, a);
      else v = expf(a.s * cv - m) * coef;
    }
    d[j] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  const int e = aam_scale_exp(block_reduce_max(mx, red));
  if (threadIdx.x == 0) rinv[i] = aam_pow2(-e);
  const float sc = aam_pow2(e);
  for (int c = threadIdx.x; c < Cp; c += blockDim.x) {
    uint16_t hi, lo;
    aam_split16(d[c] * sc, hi, lo);
    dimg[aam_kslice_off(i, Np, 0, c, Cp)] = lo;
    dimg[aam_kslice_off(i, Np, 1, c, Cp)] = hi;
    dimg[aam_kslice_off(i, Np, 2, c, Cp)] = hi;
  }
}

// The shard's partial gradient w.r.t. the normalised rows: part[i][d] = (the K slices of G summed in slice order)
// times rinv[i], un-scaled by its power of two.  grid ceil(N D / 256), block 256.
__global__ void __launch_bounds__(256)
aam_shard_gpart_kernel(const float* __restrict__ G, int slices, size_t slice_elems, const float* __restrict__ rinv,
                       int N, int D, float* __restrict__ part) {
  const size_t t = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<size_t>(N) * D) return;
  float v = G[t];
  for (int s = 1; s < slices; ++s) v += G[s * slice_elems + t];
  part[t] = v * rinv[t / D];
}

// gE of this rank's n rows X: g = the R ranks' partials parts [R][n][D] added in rank order, then the F.normalize
// Jacobian (g - x^ (x^ . g)) / nrm with nrm taken as aam_norm_kernel takes it.  One warp per row; grid ceil(n / 8),
// block 256.
__global__ void __launch_bounds__(256)
aam_shard_rows_bwd_kernel(const float* __restrict__ X, const float* __restrict__ parts, int R, int n, int D,
                          float* __restrict__ out) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* x = X + static_cast<size_t>(r) * D;
  float ss = 0.f;
  for (int d = lane; d < D; d += 32) ss = fmaf(x[d], x[d], ss);
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float nr = fmaxf(sqrtf(ss), 1e-12f);
  auto grad = [&](int d) {
    float v = parts[static_cast<size_t>(r) * D + d];
    for (int q = 1; q < R; ++q) v += parts[(static_cast<size_t>(q) * n + r) * D + d];
    return v;
  };
  float dot = 0.f;
  for (int d = lane; d < D; d += 32) dot = fmaf(x[d] / nr, grad(d), dot);
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  float* y = out + static_cast<size_t>(r) * D;
  for (int d = lane; d < D; d += 32) y[d] = (grad(d) - (x[d] / nr) * dot) / nr;
}

}  // namespace dsk
