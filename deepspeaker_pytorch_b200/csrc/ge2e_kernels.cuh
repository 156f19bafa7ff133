// Generalised end-to-end (GE2E) loss against in-batch speaker centroids: the row kernels around the AAM-softmax op's
// cosine GEMMs (dsk_ge2e_rows / _mean / _dcos_rows / _bwd_rows in dsk_api.cu, and dsk_ge2e / dsk_ge2e_bwd composed of
// them).  The row kernels work on a row range [row0, row0 + rows) of the batch; the centroids, norms and speaker sums
// are always those of the whole batch, so every row's bits are the same whichever range it is computed in.
//
// The inclusive centroids are class_centroids_kernel's; the (N, P) cosines and both backward products (gE^ = dcos C^,
// gC^ = dcos^T E^) run on the AAM plan's hi/lo GEMMs with the centroids in place of W.  What is GE2E's own is here:
// the target column, scored against the leave-one-out (exclusive) centroid of the row's speaker, recomputed in fp64 from
// the fp32 rows; the softmax / contrast rows and their derivatives; and the gradient that reaches every member of a
// speaker through the centroids.  Every sum over a speaker's members runs over the CSR `order[offsets[k] ..
// offsets[k+1])` in that order (ascending row index, as the host builds it).  No float atomics.
#pragma once
#include <stdint.h>

#include "aam_kernels.cuh"

namespace dsk {

enum { kGe2eSoftmax = 0, kGe2eContrast = 1 };

__device__ __forceinline__ double block_reduce_sum_f64(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) t += red[i];
  __syncthreads();
  return t;
}

__device__ __forceinline__ float ge2e_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// nr[r] = max(||X[r]||, 1e-12) in fp64 from the fp32 row (class_centroids_kernel's norm: one warp, the same order).
// grid ceil(rows / 8), block 256.
__global__ void __launch_bounds__(256) ge2e_norm64_kernel(const float* __restrict__ X, int rows, int D, double* __restrict__ nr) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* x = X + static_cast<size_t>(r) * D;
  double ss = 0.0;
  for (int i = lane; i < D; i += 32) {
    const double v = x[i];
    ss = fma(v, v, ss);
  }
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) nr[r] = fmax(sqrt(ss), 1e-12);
}

// Element d of the sum of x^_u over the members u != i of the speaker [b, e) of the CSR, in fp64, in CSR order.
__device__ __forceinline__ double ge2e_excl_sum(const float* __restrict__ X, const double* __restrict__ nr, int D,
                                                const int64_t* __restrict__ order, int64_t b, int64_t e, int64_t i, int d) {
  double s = 0.0;
  for (int64_t q = b; q < e; ++q) {
    const int64_t u = order[q];
    if (u != i) s += static_cast<double>(X[static_cast<size_t>(u) * D + d]) / nr[u];
  }
  return s;
}

// Forward rows of the row range [row0, row0 + gridDim.x) of the batch; G, cos_out, rec and row_loss are indexed by the
// row's place r = i - row0 in the range, X, nr and the CSR by the batch row i.  cos_out[r] = G[r][0, P) (the GEMM's
// padded output) except the target column y = col[i], which for a row of a speaker with n >= 2 rows is e^_i . c^(-i)^
// recomputed in fp64 (c^(-i) the mean of the speaker's other normalised rows, wherever they sit in the batch) and
// rounded once; a singleton row keeps the inclusive (GEMM) cosine there.  S = max(w, 1e-6) cos + b;
//   softmax:  rec[r] = lse_i = logsumexp_k S_ik,          row_loss[r] = lse_i - S_iy;
//   contrast: rec[r] = k* = argmax_{k != y} sigmoid(S_ik) (ties to the lowest column, stored as a float),
//             row_loss[r] = 1 - sigmoid(S_iy) + sigmoid(S_ik*).
// row_loss is 0 on rows of singleton speakers.  grid rows, block 256.
__global__ void __launch_bounds__(256)
ge2e_rows_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ X, int D, const double* __restrict__ nr,
                 const int64_t* __restrict__ order, const int64_t* __restrict__ offsets, const int64_t* __restrict__ col,
                 int P, const float* __restrict__ w, const float* __restrict__ bias, int method, int row0,
                 float* __restrict__ cos_out, float* __restrict__ rec, float* __restrict__ row_loss) {
  __shared__ float red[8];
  __shared__ double red64[8];
  __shared__ unsigned long long redk[8];
  const int r = blockIdx.x, i = row0 + r;
  const int y = static_cast<int>(col[i]);
  const int64_t b = offsets[y], e = offsets[y + 1];
  const bool valid = e - b >= 2;
  const float* g = G + static_cast<size_t>(r) * ldg;
  float* co = cos_out + static_cast<size_t>(r) * P;
  float tcos = g[y];
  if (valid) {
    double ew = 0.0, cc = 0.0;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      const double s = ge2e_excl_sum(X, nr, D, order, b, e, i, d);
      ew = fma(static_cast<double>(X[static_cast<size_t>(i) * D + d]) / nr[i], s, ew);
      cc = fma(s, s, cc);
    }
    ew = block_reduce_sum_f64(ew, red64);
    cc = block_reduce_sum_f64(cc, red64);
    const double m = static_cast<double>(e - b - 1);
    tcos = static_cast<float>((ew / m) / fmax(sqrt(cc) / m, 1e-12));
  }
  const float we = fmaxf(w[0], 1e-6f), bb = bias[0];
  const float sy = fmaf(we, tcos, bb);
  if (method == kGe2eSoftmax) {
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < P; c += blockDim.x) {
      const float cv = c == y ? tcos : g[c];
      co[c] = cv;
      mx = fmaxf(mx, fmaf(we, cv, bb));
    }
    mx = block_reduce_max(mx, red);
    float sum = 0.f;
    for (int c = threadIdx.x; c < P; c += blockDim.x) sum += expf(fmaf(we, c == y ? tcos : g[c], bb) - mx);
    sum = block_reduce_sum(sum, red);
    if (threadIdx.x == 0) {
      const float l = mx + logf(sum);
      rec[r] = l;
      row_loss[r] = valid ? l - sy : 0.f;
    }
  } else {
    // key: the sigmoid's bits (non-negative: ordered as integers) above the complement of the column
    unsigned long long best = 0ull;
    for (int c = threadIdx.x; c < P; c += blockDim.x) {
      const float cv = c == y ? tcos : g[c];
      co[c] = cv;
      if (c == y) continue;
      const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(ge2e_sigmoid(fmaf(we, cv, bb)))) << 32) |
                                     (0xffffffffu - static_cast<unsigned>(c));
      best = key > best ? key : best;
    }
    best = block_reduce_max_u64(best, redk);
    if (threadIdx.x == 0) {
      const int ks = static_cast<int>(0xffffffffu - static_cast<unsigned>(best & 0xffffffffull));
      rec[r] = static_cast<float>(ks);
      row_loss[r] = valid ? 1.f - ge2e_sigmoid(sy) + __uint_as_float(static_cast<unsigned>(best >> 32)) : 0.f;
    }
  }
}

// Row r of the K-sliced A-side image dimg [Rp][3 Pp] = [lo | hi | hi] of gE^ = dcos C^ from the fp32 dcos row d (Pp
// columns), scaled by the power of two 2^e that puts the row's max |dcos| = mx at [256, 512) (rinv[r] = 2^-e).  Every
// thread of the block calls it; thread t reads the columns it wrote to d itself.
__device__ __forceinline__ void ge2e_dcos_image_row(const float* d, int Pp, float mx, int r, int Rp,
                                                    uint16_t* __restrict__ dimg, float* __restrict__ rinv) {
  const int ex = aam_scale_exp(mx);
  if (threadIdx.x == 0) rinv[r] = aam_pow2(-ex);
  const float S = aam_pow2(ex);
  for (int c = threadIdx.x; c < Pp; c += blockDim.x) {
    uint16_t hi, lo;
    aam_split16(d[c] * S, hi, lo);
    dimg[aam_kslice_off(r, Rp, 0, c, Pp)] = lo;
    dimg[aam_kslice_off(r, Rp, 1, c, Pp)] = hi;
    dimg[aam_kslice_off(r, Rp, 2, c, Pp)] = hi;
  }
}

// Backward rows of the row range [row0, row0 + gridDim.x): dS_ik = grad_loss / V * dL_i / dS_ik on rows of speakers
// with >= 2 rows (0 elsewhere), dcos = max(w, 1e-6) dS.  cos, rec and the outputs are indexed by the row's place r in the
// range.  The target column's dcos goes to tdc[r] and is zeroed in dcos (row stride ldd), so that the GEMMs carry only
// the inclusive-centroid terms.  part[r] = sum_k dS_ik cos_ik and part[rows + r] = sum_k dS_ik in fp64 (the row's
// shares of dL/dw and dL/db).  Softmax probabilities are e_k / sum_k e_k with e_k = exp(S_ik - lse_i) (the division
// removes the rounding of the saved lse); the target's p - 1 is minus the sum over the other columns.
// dimg == NULL: dcos (rows, ldd = P).  dimg != NULL (the whole batch, row0 = 0): dcos is the zero-padded workspace
// [Np][ldd = Pp] with columns [P, Pp) written as 0, and the row's gE^ image goes to dimg [Rp][3 Pp] and rinv, as
// ge2e_dcos_img_kernel would build them from the unpadded rows.  grid rows, block 256.
__global__ void __launch_bounds__(256)
ge2e_dcos_rows_kernel(const float* __restrict__ cos, const float* __restrict__ rec, const int64_t* __restrict__ offsets,
                      const int64_t* __restrict__ col, int row0, int P, int V, const float* __restrict__ w,
                      const float* __restrict__ bias, int method, const float* __restrict__ grad_loss,
                      float* __restrict__ dcos, int ldd, float* __restrict__ tdc, double* __restrict__ part,
                      int Pp, int Rp, uint16_t* __restrict__ dimg, float* __restrict__ rinv) {
  __shared__ float red[8];
  __shared__ double red64[8];
  const int r = blockIdx.x, rows = gridDim.x, i = row0 + r;
  float* d = dcos + static_cast<size_t>(r) * ldd;
  const float* co = cos + static_cast<size_t>(r) * P;
  const int y = static_cast<int>(col[i]);
  const bool valid = offsets[y + 1] - offsets[y] >= 2;
  const float we = fmaxf(w[0], 1e-6f), bb = bias[0];
  const float g = valid ? grad_loss[0] / static_cast<float>(V) : 0.f;
  float coef = 0.f, other = 0.f, lse = 0.f, dsk_ = 0.f, dsy = 0.f;
  int ks = -1;
  if (method == kGe2eSoftmax) {
    lse = rec[r];
    float sig = 0.f;
    for (int c = threadIdx.x; c < P; c += blockDim.x) {
      const float ex = expf(fmaf(we, co[c], bb) - lse);
      sig += ex;
      if (c != y) other += ex;
    }
    sig = block_reduce_sum(sig, red);
    other = block_reduce_sum(other, red);
    coef = g / sig;
    dsy = -other * coef;
  } else {
    ks = static_cast<int>(rec[r]);
    const float s1 = ge2e_sigmoid(fmaf(we, co[y], bb)), s2 = ge2e_sigmoid(fmaf(we, co[ks], bb));
    dsy = -g * s1 * (1.f - s1);
    dsk_ = g * s2 * (1.f - s2);
  }
  const int cols = dimg ? Pp : P;
  float mx = 0.f;
  double pw = 0.0, pb = 0.0;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float ds = 0.f;
    if (c < P) {
      if (c == y) ds = dsy;
      else if (method == kGe2eSoftmax) ds = expf(fmaf(we, co[c], bb) - lse) * coef;
      else if (c == ks) ds = dsk_;
      pw = fma(static_cast<double>(ds), static_cast<double>(co[c]), pw);
      pb += ds;
    }
    const float v = c == y ? 0.f : we * ds;
    d[c] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  pw = block_reduce_sum_f64(pw, red64);
  pb = block_reduce_sum_f64(pb, red64);
  if (threadIdx.x == 0) {
    tdc[r] = we * dsy;
    part[r] = pw;
    part[rows + r] = pb;
  }
  if (dimg) ge2e_dcos_image_row(d, Pp, block_reduce_max(mx, red), r, Rp, dimg, rinv);
}

// The operands of gE^ = dcos C^ and gC^ = dcos^T E^ from dcos (N, P) of the whole batch: the zero-padded fp32
// workspace ws [Np][Pp] (aam_dcos_t_kernel's input) for every row, and for the rows i of the range [row0, row0 + rows)
// the K-sliced A-side image dimg [Rp][3 Pp] = [lo | hi | hi] of row r = i - row0, scaled by the row's own power of two
// (rinv[r] = 2^-e).  Rows [rows, Rp) of dimg are left as they are (the plan zeroes them once).  grid Np, block 256.
__global__ void __launch_bounds__(256)
ge2e_dcos_img_kernel(const float* __restrict__ dcos, int N, int P, int Pp, int row0, int rows, int Rp,
                     float* __restrict__ ws, uint16_t* __restrict__ dimg, float* __restrict__ rinv) {
  __shared__ float red[8];
  const int i = blockIdx.x, r = i - row0;
  float* d = ws + static_cast<size_t>(i) * Pp;
  const float* src = dcos + static_cast<size_t>(i) * P;
  float mx = 0.f;
  for (int c = threadIdx.x; c < Pp; c += blockDim.x) {
    const float v = i < N && c < P ? src[c] : 0.f;
    d[c] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  if (r < 0 || r >= rows) return;
  ge2e_dcos_image_row(d, Pp, block_reduce_max(mx, red), r, Rp, dimg, rinv);
}

// The exclusive-centroid terms of row j of a speaker with n >= 2 rows, in fp64 from the fp32 rows, with t = tdc[j] the
// target column's dcos and c = c^(-j) (the mean of the speaker's other normalised rows), c^ = c / max(||c||, 1e-12):
//   own[j] = t c^                                                   (the direct term of the target column)
//   xg[j]  = (t e^_j - c^ (c^ . t e^_j)) / max(||c||, 1e-12) / (n - 1)  (the Jacobian at c^(-j), shared by the others)
// Both are zero for a singleton speaker's row.  For the row range [row0, row0 + rows): own (rows, D) is written for the
// rows j of the range (at j - row0), xg (N, D) for every member j of a speaker with a row in the range (what the range's
// gather reads); other blocks return at once.  grid N, block 256.
__global__ void __launch_bounds__(256)
ge2e_excl_bwd_kernel(const float* __restrict__ X, int D, const double* __restrict__ nr, const int64_t* __restrict__ order,
                     const int64_t* __restrict__ offsets, const int64_t* __restrict__ col, const float* __restrict__ tdc,
                     int row0, int rows, float* __restrict__ own, float* __restrict__ xg) {
  __shared__ double red64[8];
  const int j = blockIdx.x;
  const int y = static_cast<int>(col[j]);
  const int64_t b = offsets[y], e = offsets[y + 1];
  const bool mine = j >= row0 && j - row0 < rows;
  bool needed = false;
  for (int64_t q = b; q < e && !needed; ++q) needed = order[q] >= row0 && order[q] - row0 < rows;
  if (!needed) return;
  float* oj = mine ? own + static_cast<size_t>(j - row0) * D : nullptr;
  float* xj = xg + static_cast<size_t>(j) * D;
  if (e - b < 2) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      if (mine) oj[d] = 0.f;
      xj[d] = 0.f;
    }
    return;
  }
  const float* x = X + static_cast<size_t>(j) * D;
  const double m = static_cast<double>(e - b - 1), t = tdc[j], nj = nr[j];
  double ew = 0.0, cc = 0.0;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const double s = ge2e_excl_sum(X, nr, D, order, b, e, j, d);
    ew = fma(static_cast<double>(x[d]) / nj, s, ew);
    cc = fma(s, s, cc);
  }
  ew = block_reduce_sum_f64(ew, red64);
  cc = block_reduce_sum_f64(cc, red64);
  const double cn = fmax(sqrt(cc) / m, 1e-12);
  const double tdot = t * ((ew / m) / cn);  // c^ . (t e^_j)
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const double ch = ge2e_excl_sum(X, nr, D, order, b, e, j, d) / m / cn;
    if (mine) oj[d] = static_cast<float>(t * ch);
    xj[d] = static_cast<float>((t * (static_cast<double>(x[d]) / nj) - ch * tdot) / cn / m);
  }
}

// gê of row u = row0 + r of the range, in place in own (rows, D) at row r: the K slices of the GEMM dcos C^ (rows of
// the range, added in slice order, times rinv[r]), then own[r] (the target's direct term), gc[k] / n_k (the inclusive
// centroid's Jacobian, k = col[u]), then xg[j] of every other member j of the speaker in CSR order.
// grid (rows, ceil(D / 256)), block 256.
__global__ void __launch_bounds__(256)
ge2e_gather_kernel(const float* __restrict__ Gs, int slices, long slice_elems, const float* __restrict__ rinv,
                   const float* __restrict__ gc, const int64_t* __restrict__ order, const int64_t* __restrict__ offsets,
                   const int64_t* __restrict__ col, const float* __restrict__ xg, int D, int row0,
                   float* __restrict__ own) {
  const int r = blockIdx.x, u = row0 + r, d = blockIdx.y * 256 + threadIdx.x;
  if (d >= D) return;
  const int y = static_cast<int>(col[u]);
  const int64_t b = offsets[y], e = offsets[y + 1];
  const size_t o = static_cast<size_t>(r) * D + d;
  float v = Gs[o];
  for (int s = 1; s < slices; ++s) v += Gs[s * slice_elems + o];
  v = v * rinv[r] + own[o];
  v += gc[static_cast<size_t>(y) * D + d] / static_cast<float>(e - b);
  for (int64_t q = b; q < e; ++q) {
    const int64_t j = order[q];
    if (j != u) v += xg[static_cast<size_t>(j) * D + d];
  }
  own[o] = v;
}

// Over the rows of a range (part [2][rows], ge2e_dcos_rows_kernel's): gw = sum_r part[r] where w >= 1e-6 (torch.clamp's
// gradient), else 0; gb = sum_r part[rows + r] for contrast and exactly 0 for softmax (b cancels out of the softmax
// loss).  fp64, fixed order, rounded once.  grid 1, block 256.
__global__ void __launch_bounds__(256)
ge2e_scalars_kernel(const double* __restrict__ part, int rows, const float* __restrict__ w, int method,
                    float* __restrict__ gw, float* __restrict__ gb) {
  __shared__ double red64[8];
  double a = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    a += part[i];
    c += part[rows + i];
  }
  a = block_reduce_sum_f64(a, red64);
  c = block_reduce_sum_f64(c, red64);
  if (threadIdx.x == 0) {
    gw[0] = w[0] >= 1e-6f ? static_cast<float>(a) : 0.f;
    gb[0] = method == kGe2eSoftmax ? 0.f : static_cast<float>(c);
  }
}

}  // namespace dsk
