// Layout converters and (below) the training-mode kernels: batch-statistics BatchNorm, backward passes.
#pragma once
#include "dsk_ptx.cuh"

namespace dsk {

// fp32 NCHW -> 16-bit NHWC (boundary / test helper).
template <bool BF16>
__global__ void nchw_to_nhwc16_kernel(const float* __restrict__ in, uint16_t* __restrict__ out, int B, int C, int HW) {
  const long total = static_cast<long>(B) * C * HW;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = i % C;
    const long r = i / C;
    const int hw = r % HW;
    const int b = r / HW;
    out[i] = to16<BF16>(in[(static_cast<long>(b) * C + c) * HW + hw]);
  }
}

// 16-bit NHWC -> fp32 NCHW.
template <bool BF16>
__global__ void nhwc16_to_nchw_kernel(const uint16_t* __restrict__ in, float* __restrict__ out, int B, int C, int HW) {
  const long total = static_cast<long>(B) * C * HW;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = i % C;
    const long r = i / C;
    const int hw = r % HW;
    const int b = r / HW;
    out[(static_cast<long>(b) * C + c) * HW + hw] = from16<BF16>(in[i]);
  }
}

__global__ void nhwc_f32_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int HW) {
  const long total = static_cast<long>(B) * C * HW;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = i % C;
    const long r = i / C;
    const int hw = r % HW;
    const int b = r / HW;
    out[(static_cast<long>(b) * C + c) * HW + hw] = in[i];
  }
}

}  // namespace dsk

// =================================================================================================
// Training mode.  BatchNorm2d with batch statistics (reference model.py:59,62,94,99,103,107 in
// train mode, called once per a/p/n forward: train_triplet.py:215) and the backward of every non-conv op.
//
// Elementwise kernels work on tiles of 64 pixels x 64 channels of an NHWC 16-bit tensor viewed as
// [M pixels][C]; thread t handles pixels {t/8, t/8+32} and the 8 channels (16 bytes) t%8 of the chunk.
// Reductions are two-stage and deterministic: per-block partials, then a fixed-order finalize.
// =================================================================================================
namespace dsk {

constexpr int kEwTilePix = 64;

template <bool BF16>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack2<BF16>(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack2<BF16>(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack2<BF16>(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack2<BF16>(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool BF16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack2<BF16>(f[0], f[1]);
  o.y = pack2<BF16>(f[2], f[3]);
  o.z = pack2<BF16>(f[4], f[5]);
  o.w = pack2<BF16>(f[6], f[7]);
  return o;
}

__device__ __forceinline__ void load8f(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// ---- forward: per-channel sum / sum of squares of the raw conv output --------------------------------------
// Two pairs of sums per channel: of x itself (stats 0, 1) and of x - k_c around the pivot k_c = the channel's first
// element, row 0 of raw (stats 2, 3).  E[x^2] - mean^2 from the plain fp32 sums loses (mean/std)^2 ulps of the variance
// (1e-3 relative at mean/std 300); bn_finalize_kernel takes the shifted sums where that matters.
// grid (gx, C/64); partial[(bx*4 + stat)*C + c]
__global__ void __launch_bounds__(256)
bn_stats_partial_kernel(const float* __restrict__ raw, long M, int C, float* __restrict__ partial) {
  __shared__ float red[4][32][65];
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + q * 8;
  float s[8], ss[8], sd[8], ssd[8], k[8];
  load8f(raw + c0, k);
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = ss[e] = sd[e] = ssd[e] = 0.f;
  for (long m = blockIdx.x * 32L + p; m < M; m += 32L * gridDim.x) {
    float f[8];
    load8f(raw + m * C + c0, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s[e] += f[e];
      ss[e] = fmaf(f[e], f[e], ss[e]);
      const float d = f[e] - k[e];
      sd[e] += d;
      ssd[e] = fmaf(d, d, ssd[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    red[0][p][q * 8 + e] = s[e];
    red[1][p][q * 8 + e] = ss[e];
    red[2][p][q * 8 + e] = sd[e];
    red[3][p][q * 8 + e] = ssd[e];
  }
  __syncthreads();
  {
    const int stat = threadIdx.x >> 6, c = threadIdx.x & 63;
    float t = 0.f;
    for (int i = 0; i < 32; ++i) t += red[stat][i][c];
    partial[(static_cast<long>(blockIdx.x) * 4 + stat) * C + blockIdx.y * 64 + c] = t;
  }
}

// Sum of the per-block partials of 32 channels by one 1024-thread block: thread (slice, channel) adds every 32nd
// partial row in double, the slices are combined in fixed order (deterministic).  A single thread per channel walking
// all ~1000 rows took ~50 us per launch, a quarter of the training step.
// Rows of block b are b*rows + row0 (s) and b*rows + row0 + 1 (ss).  Every thread of the block must call it.
// Returns the totals to the threads of slice 0 (threadIdx.x < 32); the others get ok == false.
__device__ __forceinline__ bool bn_partial_totals(const float* __restrict__ partial, int nblk, int C, int c, double& s,
                                                  double& ss, int rows = 2, int row0 = 0) {
  __shared__ double red[2][32][33];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  __syncthreads();  // a previous call's readers are done with red
  double a = 0.0, b2 = 0.0;
  if (c < C) {
    int b = sl;
    for (; b + 96 < nblk; b += 128) {  // four rows in flight per thread
      float t0[4], t1[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        t0[j] = partial[(static_cast<long>(b + 32 * j) * rows + row0) * C + c];
        t1[j] = partial[(static_cast<long>(b + 32 * j) * rows + row0 + 1) * C + c];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        a += t0[j];
        b2 += t1[j];
      }
    }
    for (; b < nblk; b += 32) {
      a += partial[(static_cast<long>(b) * rows + row0) * C + c];
      b2 += partial[(static_cast<long>(b) * rows + row0 + 1) * C + c];
    }
  }
  red[0][sl][lane] = a;
  red[1][sl][lane] = b2;
  __syncthreads();
  if (sl != 0 || c >= C) return false;
  s = 0.0;
  ss = 0.0;
  for (int i = 0; i < 32; ++i) {
    s += red[0][i][lane];
    ss += red[1][i][lane];
  }
  return true;
}

// running = (1 - momentum) * running + momentum * batch, with the roundings pinned (one multiply, one FMA) so that the
// in-kernel update of bn_finalize_kernel and the deferred bn_running_commit_kernel produce the same bits
__device__ __forceinline__ float bn_momentum_update(float running, float batch, float momentum) {
  return __fmaf_rn(momentum, batch, __fmul_rn(1.f - momentum, running));
}

// mean / biased var -> rstd, scale = gamma*rstd, shift = beta - mean*scale; running stats (momentum, unbiased var).
// `raw` is the tensor bn_stats_partial_kernel reduced: its row 0 holds the pivots of the shifted sums.  Channels with
// mean^2 <= 1024 var keep the plain sums: their cancellation costs at most 10 bits (variance error <= 4e-5 relative in an
// emulation of this summation order), and they reproduce the earlier kernels' bits, which a training run depends on (its
// last bits compound over the steps).  The others, where E[x^2] - mean^2 would cancel more, use mean = k + sd/M,
// var = ssd/M - (sd/M)^2.
// grid ceil(C/32), block 1024
__global__ void bn_finalize_kernel(const float* __restrict__ partial, const float* __restrict__ raw, int nblk, int C, long M,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
                                   float eps, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                   float* __restrict__ scale_out, float* __restrict__ shift_out,
                                   float* __restrict__ unbiased_out, int update_running) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  double s, ss, sd, ssd;
  const bool ok = bn_partial_totals(partial, nblk, C, c, s, ss, 4, 0);
  if (!bn_partial_totals(partial, nblk, C, c, sd, ssd, 4, 2) || !ok) return;
  double mean = s / static_cast<double>(M);
  double var = ss / static_cast<double>(M) - mean * mean;
  if (mean * mean > 1024.0 * var) {
    const double dmean = sd / static_cast<double>(M);  // mean - k_c
    mean = static_cast<double>(raw[c]) + dmean;
    var = ssd / static_cast<double>(M) - dmean * dmean;
  }
  if (var < 0.0) var = 0.0;
  const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const float sc = gamma[c] * rstd;
  mean_out[c] = static_cast<float>(mean);
  rstd_out[c] = rstd;
  scale_out[c] = sc;
  shift_out[c] = beta[c] - static_cast<float>(mean) * sc;
  const double unbiased = M > 1 ? var * static_cast<double>(M) / static_cast<double>(M - 1) : var;
  if (unbiased_out) unbiased_out[c] = static_cast<float>(unbiased);
  if (update_running) {
    running_mean[c] = bn_momentum_update(running_mean[c], static_cast<float>(mean), momentum);
    running_var[c] = bn_momentum_update(running_var[c], static_cast<float>(unbiased), momentum);
  }
}

// Deferred running-statistics update of ONE train-mode forward (all 12 BatchNorm layers in one launch): when several
// forwards of a step run concurrently on different streams (DeepSpeakerModel.forward_triplet) their in-place
// read-modify-writes of running_mean / running_var would race, so bn_finalize only records the batch mean and unbiased
// variance and this kernel applies the momentum update afterwards, one forward after the other, in the order the
// reference's sequential calls would have (train_triplet.py:215: a, p, n) - same operations, same bits.
struct BnCommitParams {
  const float* mean[12];
  const float* unbiased[12];
  float* running_mean[12];
  float* running_var[12];
  int C[12];
  float momentum;
};
__global__ void bn_running_commit_kernel(const BnCommitParams p) {
  const int layer = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.C[layer]) return;
  float* rm = p.running_mean[layer];
  float* rv = p.running_var[layer];
  rm[c] = bn_momentum_update(rm[c], p.mean[layer][c], p.momentum);
  rv[c] = bn_momentum_update(rv[c], p.unbiased[layer][c], p.momentum);
}

// ---- forward: y = clip(raw*scale + shift (+res), 0, hi), NHWC 16-bit ---------------------------------------------
// grid (ceil(M/64), C/64)
template <bool BF16>
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ raw, const float* __restrict__ scale, const float* __restrict__ shift,
                const uint16_t* __restrict__ res, uint16_t* __restrict__ y, long M, int C, float clip_hi) {
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + q * 8;
  const long m0 = static_cast<long>(blockIdx.x) * kEwTilePix;
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    sc[e] = scale[c0 + e];
    sh[e] = shift[c0 + e];
  }
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const long m = m0 + p + 32 * half;
    if (m >= M) continue;
    float f[8];
    load8f(raw + m * C + c0, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = fmaf(f[e], sc[e], sh[e]);
    if (res) {
      float r[8];
      unpack8<BF16>(*reinterpret_cast<const uint4*>(res + m * C + c0), r);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] += r[e];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = fminf(fmaxf(f[e], 0.f), clip_hi);
    *reinterpret_cast<uint4*>(y + m * C + c0) = pack8<BF16>(f);
  }
}

// ---- backward: dbeta = sum g_z, dgamma = sum g_z * xhat, with g_z = g_y * 1[0 < y < hi] -----------------------
template <bool BF16>
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const uint16_t* __restrict__ gy, const uint16_t* __restrict__ y, const float* __restrict__ raw,
                     const float* __restrict__ mean, const float* __restrict__ rstd, long M, int C, float clip_hi,
                     float* __restrict__ partial) {
  __shared__ float red[2][32][65];
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + q * 8;
  float mu[8], rs[8], s[8], ss[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = mean[c0 + e];
    rs[e] = rstd[c0 + e];
    s[e] = ss[e] = 0.f;
  }
  for (long m = blockIdx.x * 32L + p; m < M; m += 32L * gridDim.x) {
    float g[8], yy[8], r[8];
    unpack8<BF16>(*reinterpret_cast<const uint4*>(gy + m * C + c0), g);
    unpack8<BF16>(*reinterpret_cast<const uint4*>(y + m * C + c0), yy);
    load8f(raw + m * C + c0, r);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float gz = (yy[e] > 0.f && yy[e] < clip_hi) ? g[e] : 0.f;
      s[e] += gz;
      ss[e] = fmaf(gz, (r[e] - mu[e]) * rs[e], ss[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    red[0][p][q * 8 + e] = s[e];
    red[1][p][q * 8 + e] = ss[e];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int stat = threadIdx.x >> 6, c = threadIdx.x & 63;
    float t = 0.f;
    for (int i = 0; i < 32; ++i) t += red[stat][i][c];
    partial[(static_cast<long>(blockIdx.x) * 2 + stat) * C + blockIdx.y * 64 + c] = t;
  }
}

// dgamma, dbeta (unscaled by 1/S) and the three per-channel coefficients of
// g_raw = a * (g_z - b - xhat * d),  a = gamma*rstd, b = dbeta/M, d = dgamma/M.
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ partial, int nblk, int C, long M,
                                       const float* __restrict__ gamma, const float* __restrict__ rstd,
                                       float inv_loss_scale, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       float* __restrict__ coef /*[3][C]*/, const float* __restrict__ dyn = nullptr) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  double s, ss;
  if (!bn_partial_totals(partial, nblk, C, c, s, ss)) return;
  if (dyn) inv_loss_scale *= dyn[1];  // device-side loss scale of this backward: {S, 1/S}
  dbeta[c] = static_cast<float>(s) * inv_loss_scale;
  dgamma[c] = static_cast<float>(ss) * inv_loss_scale;
  coef[c] = gamma[c] * rstd[c];
  coef[C + c] = static_cast<float>(s / static_cast<double>(M));
  coef[2 * C + c] = static_cast<float>(ss / static_cast<double>(M));
}

// g_raw -> G (NHWC); optionally g_z -> gres (NHWC) for the skip branch.   grid (ceil(M/64), C/64)
template <bool BF16>
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const uint16_t* __restrict__ gy, const uint16_t* __restrict__ y, const float* __restrict__ raw,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ coef,
                    uint16_t* __restrict__ G, uint16_t* __restrict__ gres, long M, int C, float clip_hi) {
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + q * 8;
  const long m0 = static_cast<long>(blockIdx.x) * kEwTilePix;
  float mu[8], rs[8], ca[8], cb[8], cd[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = mean[c0 + e];
    rs[e] = rstd[c0 + e];
    ca[e] = coef[c0 + e];
    cb[e] = coef[C + c0 + e];
    cd[e] = coef[2 * C + c0 + e];
  }
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const long m = m0 + p + 32 * half;
    if (m >= M) continue;
    float g[8], yy[8], r[8];
    unpack8<BF16>(*reinterpret_cast<const uint4*>(gy + m * C + c0), g);
    unpack8<BF16>(*reinterpret_cast<const uint4*>(y + m * C + c0), yy);
    load8f(raw + m * C + c0, r);
    float gz[8], gr[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gz[e] = (yy[e] > 0.f && yy[e] < clip_hi) ? g[e] : 0.f;
      gr[e] = ca[e] * (gz[e] - cb[e] - (r[e] - mu[e]) * rs[e] * cd[e]);
    }
    *reinterpret_cast<uint4*>(G + m * C + c0) = pack8<BF16>(gr);
    if (gres) *reinterpret_cast<uint4*>(gres + m * C + c0) = pack8<BF16>(gz);
  }
}

// ---- tail backward ---------------------------------------------------------------------------------------------
// emb = alpha * x / sqrt(sum x^2 + 1e-10)  =>  g_x = alpha*inv * (g - xhat * (xhat . g)), xhat = x*inv.
__global__ void l2norm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ inv_norm,
                                  const float* __restrict__ g, float* __restrict__ gx, int E, float alpha) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float inv = inv_norm[b];
  const float* xr = x + static_cast<long>(b) * E;
  const float* gr = g + static_cast<long>(b) * E;
  float s = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) s = fmaf(xr[i] * inv, gr[i], s);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float dot = red[0];
  for (int i = threadIdx.x; i < E; i += blockDim.x)
    gx[static_cast<long>(b) * E + i] = alpha * inv * (gr[i] - xr[i] * inv * dot);
}

// dW[e][c*4+w] = sum_b gy[b][e] * pooled[b][w*512+c]  (written in the PyTorch fc.weight layout), db[e] = sum_b gy[b][e].
// grid (E/8, K/256), block 256: thread = one k, 8 e's.
__global__ void __launch_bounds__(256)
fc_bwd_weight_kernel(const float* __restrict__ gy, const float* __restrict__ pooled, float* __restrict__ dW,
                     float* __restrict__ db, int B, int K, int E, int Cch, int Wd) {
  const int e0 = blockIdx.x * 8;
  const int k = blockIdx.y * 256 + threadIdx.x;  // index in (w, c) order
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  float bsum = 0.f;
  for (int b = 0; b < B; ++b) {
    const float pv = pooled[static_cast<long>(b) * K + k];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(gy[static_cast<long>(b) * E + e0 + j], pv, acc[j]);
    if (blockIdx.y == 0 && threadIdx.x < 8) bsum += gy[static_cast<long>(b) * E + e0 + threadIdx.x];
  }
  const int wi = k / Cch, c = k % Cch;
#pragma unroll
  for (int j = 0; j < 8; ++j) dW[static_cast<long>(e0 + j) * K + c * Wd + wi] = acc[j];
  if (blockIdx.y == 0 && threadIdx.x < 8) db[e0 + threadIdx.x] = bsum;
}

// dP[b][k] = sum_e gy[b][e] * wq[e][k]   grid (B, K/256)
__global__ void __launch_bounds__(256)
fc_bwd_input_kernel(const float* __restrict__ gy, const float* __restrict__ wq, float* __restrict__ dP, int K, int E) {
  extern __shared__ float sg[];  // [E]
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < E; i += blockDim.x) sg[i] = gy[static_cast<long>(b) * E + i];
  __syncthreads();
  const int k = blockIdx.y * 256 + threadIdx.x;
  float acc = 0.f;
  for (int e = 0; e < E; ++e) acc = fmaf(sg[e], wq[static_cast<long>(e) * K + k], acc);
  dP[static_cast<long>(b) * K + k] = acc;
}

// g_y[b][h][w][c] = loss_scale * dP[b][w*C + c] / H  (mean over time backward) -> 16-bit NHWC
template <bool BF16>
__global__ void pool_bwd_kernel(const float* __restrict__ dP, uint16_t* __restrict__ gy, int H, int WC, float mult,
                                const float* __restrict__ dyn = nullptr) {
  const int b = blockIdx.x;
  if (dyn) mult *= dyn[0];  // device-side loss scale of this backward: {S, 1/S}
  for (int i = threadIdx.x; i < WC; i += blockDim.x) {
    const uint16_t v = to16<BF16>(dP[static_cast<long>(b) * WC + i] * mult);
    for (int h = 0; h < H; ++h) gy[(static_cast<long>(b) * H + h) * WC + i] = v;
  }
}

// ---- conv1 weight gradient (Cin = 1): dW[co][r][s] = sum_pix G[pix][co] * x[2h-2+r][2w-2+s] -----------------------
// grid B * ceil(hout/8); block 256 = 8 warps.  Same shape as the SIMT conv1 forward: block = 8 output rows of one
// utterance with their 19 x 68 input patch in shared memory, warp = one output row, lane = 2 output channels with
// 2 x 25 accumulators in registers; four pixels per iteration share three float4 patch loads per filter row.
// partial[blk][co][25]; summed by sum_partials_kernel.
template <bool BF16>
__global__ void __launch_bounds__(256)
conv1_wgrad_partial_kernel(const uint16_t* __restrict__ G, const float* __restrict__ x, int B, int T,
                           float* __restrict__ partial) {
  constexpr int WIN = 64, WOUT = 32, ROWS = 8, PATCH_ROWS = 2 * ROWS + 3, PATCH_W = WIN + 4;
  __shared__ __align__(16) float patch[PATCH_ROWS][PATCH_W];
  __shared__ float red[64 * 25];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int hout = T / 2;
  const int tiles_h = (hout + ROWS - 1) / ROWS;
  const int n = blockIdx.x / tiles_h;
  const int h0 = (blockIdx.x % tiles_h) * ROWS;
  const float* xin = x + static_cast<long>(n) * T * WIN;
  {
    constexpr int NEL = PATCH_ROWS * PATCH_W, NIT = (NEL + 255) / 256;
    float t[NIT];
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = threadIdx.x + 256 * j;
      const int pr = i / PATCH_W, pc = i % PATCH_W;
      const int ih = 2 * h0 - 2 + pr, iw = pc - 2;
      t[j] = (i < NEL && ih >= 0 && ih < T && iw >= 0 && iw < WIN) ? xin[ih * WIN + iw] : 0.0f;
    }
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = threadIdx.x + 256 * j;
      if (i < NEL) patch[i / PATCH_W][i % PATCH_W] = t[j];
    }
  }
  for (int i = threadIdx.x; i < 64 * 25; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
  float a0[25], a1[25];
#pragma unroll
  for (int t = 0; t < 25; ++t) a0[t] = a1[t] = 0.f;
  const int oh = h0 + warp;
  if (oh < hout) {
    const uint32_t* g32 = reinterpret_cast<const uint32_t*>(G) + ((static_cast<long>(n) * hout + oh) * WOUT) * 32 + lane;
#pragma unroll 1
    for (int ow = 0; ow < WOUT; ow += 4) {
      float2 g[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) g[q] = unpack2<BF16>(g32[(ow + q) * 32]);
#pragma unroll
      for (int r = 0; r < 5; ++r) {
        const float4* prow = reinterpret_cast<const float4*>(&patch[2 * warp + r][2 * ow]);
        const float4 v0 = prow[0], v1 = prow[1], v2 = prow[2];
        const float v[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
#pragma unroll
        for (int s2 = 0; s2 < 5; ++s2) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            a0[r * 5 + s2] = fmaf(g[q].x, v[2 * q + s2], a0[r * 5 + s2]);
            a1[r * 5 + s2] = fmaf(g[q].y, v[2 * q + s2], a1[r * 5 + s2]);
          }
        }
      }
    }
  }
  // warp w adds in round w so the shared-memory sum has a fixed order (deterministic)
  for (int w = 0; w < 8; ++w) {
    if (warp == w) {
#pragma unroll
      for (int t = 0; t < 25; ++t) {
        red[(lane * 2) * 25 + t] += a0[t];
        red[(lane * 2 + 1) * 25 + t] += a1[t];
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 64 * 25; i += blockDim.x) partial[static_cast<long>(blockIdx.x) * 1600 + i] = red[i];
}

// out[i] = mult * sum_b partial[b][i].  grid ceil(n/32), block 1024: thread (slice, i) adds every 32nd row in double,
// slices are combined in fixed order.
__global__ void sum_partials_kernel(const float* __restrict__ partial, int nblk, int n, float mult,
                                    float* __restrict__ out, const float* __restrict__ dyn = nullptr) {
  __shared__ double red[32][33];
  if (dyn) mult *= dyn[1];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + lane;
  double t = 0.0;
  if (i < n) {
    int b = sl;
    for (; b + 96 < nblk; b += 128) {
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = partial[static_cast<long>(b + 32 * j) * n + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) t += v[j];
    }
    for (; b < nblk; b += 32) t += partial[static_cast<long>(b) * n + i];
  }
  red[sl][lane] = t;
  __syncthreads();
  if (sl != 0 || i >= n) return;
  double tot = 0.0;
  for (int k = 0; k < 32; ++k) tot += red[k][lane];
  out[i] = static_cast<float>(tot) * mult;
}

// K-split partial weight gradients fp32 [ksplit][tap][co][ci] (one slice per split of the wgrad GEMM) -> OIHW
// [co][ci][tap], slices added in fixed order (deterministic), scaled by mult.  Reads are coalesced along ci.
__global__ void unpack_wgrad_kernel(const float* __restrict__ in, float* __restrict__ out, int cout, int cin, int taps,
                                    float mult, int ksplit, long slice_elems, const float* __restrict__ dyn = nullptr) {
  const long total = static_cast<long>(cout) * cin * taps;
  if (dyn) mult *= dyn[1];
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ci = i % cin;
    const long r = i / cin;
    const int co = r % cout;
    const int tap = r / cout;
    float acc = in[i];
    for (int k = 1; k < ksplit; ++k) acc += in[k * slice_elems + i];
    out[(static_cast<long>(co) * cin + ci) * taps + tap] = acc * mult;
  }
}

// Loss scale of ONE backward, chosen on the device (no host round trip): 16-bit gradient tensors are multiplied by a
// power of two S inside the backward and every parameter gradient is divided by it again.  S puts the largest incoming
// gradient max|dL/d(fc output)| at ~2^9 - the operating point of round 1's static rule 2^(9 + log2 B) on a fresh network,
// but following the loss as it shrinks during training (a static scale lets late-training gradients sink into fp16
// subnormals: tests/test_gpu_train.py::test_fp16_backward_survives_small_gradients).  fixed > 0 overrides (bf16: 1).
// ls = {S, 1/S}.  grid 1, block 1024.
__global__ void loss_scale_kernel(const float* __restrict__ g, long n, float fixed, float* __restrict__ ls) {
  __shared__ float red[32];
  float m = 0.f;
  for (long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(g[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
    float S = fixed;
    if (!(S > 0.f)) {
      S = 1.f;
      if (m > 0.f && isfinite(m)) {
        S = exp2f(floorf(log2f(512.f / m)));
        S = fminf(fmaxf(S, 5.9604645e-8f /*2^-24*/), 1.0995116e12f /*2^40*/);
      }
    }
    ls[0] = S;
    ls[1] = 1.f / S;
  }
}

// ---- synchronised BatchNorm: per-utterance records ----------------------------------------------------------------
// Under data parallelism with synchronised BatchNorm every rank normalises with the statistics of the GLOBAL batch.  The
// ranks exchange one record per utterance instead of per-rank totals: a record is summed in an order fixed by the
// utterance's own pixel count, and the finalize kernels combine all N records in global utterance order, so the
// statistics - and everything a rank computes for its own utterances - do not depend on how the batch is split.
//
// Forward record of utterance u (fp32 words, 3C + 1): [0, C) the pivots k_c = the utterance's first pixel,
// [C, 2C) sum (x - k_c), [2C, 3C) sum (x - k_c)^2, [3C] the pixel count HW (int32 bits).  The pixels of u are the rows
// [u HW, (u + 1) HW) of the NHWC raw conv output.
// Backward record (2C words): [0, C) sum g_z, [C, 2C) sum g_z xhat, xhat from the global mean / rstd.
//
// Record sums: lane p (0..31) of the block walks pixels p, p + 32, ... of the utterance, then the 32 lanes are added by
// a fixed tree.  grid (B, C/64), block 256; thread = lane p = t/8, 8 channels (t%8)*8 of the 64-channel group.
__device__ __forceinline__ void utt_tree_sum(float (*red)[32][65], int nstat, int p, int q, float (*v)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e)
    for (int st = 0; st < nstat; ++st) red[st][p][q * 8 + e] = v[st][e];
  __syncthreads();
  for (int half = 16; half > 0; half >>= 1) {
    if (p < half) {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        for (int st = 0; st < nstat; ++st) red[st][p][q * 8 + e] += red[st][p + half][q * 8 + e];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
bn_utt_record_kernel(const float* __restrict__ raw, int HW, int C, float* __restrict__ rec) {
  __shared__ float red[2][32][65];
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int u = blockIdx.x;
  const int c0 = blockIdx.y * 64 + q * 8;
  const float* base = raw + static_cast<long>(u) * HW * C;
  float k[8], v[2][8];
  load8f(base + c0, k);
#pragma unroll
  for (int e = 0; e < 8; ++e) v[0][e] = v[1][e] = 0.f;
  for (int m = p; m < HW; m += 32) {
    float f[8];
    load8f(base + static_cast<long>(m) * C + c0, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = f[e] - k[e];
      v[0][e] += d;
      v[1][e] = fmaf(d, d, v[1][e]);
    }
  }
  utt_tree_sum(red, 2, p, q, v);
  float* r = rec + static_cast<long>(u) * (3 * C + 1);
  if (p == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      r[c0 + e] = k[e];
      r[C + c0 + e] = red[0][0][q * 8 + e];
      r[2 * C + c0 + e] = red[1][0][q * 8 + e];
    }
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) r[3 * C] = __int_as_float(HW);
}

// The global statistics from the gathered forward records of all N utterances, combined in double in utterance order
// around K = record 0's pivot (slice sl of 32 adds utterances sl, sl + 32, ..., the slices are added in fixed order):
// S1 = sum_u sd_u + n_u (k_u - K),  S2 = sum_u ssd_u + 2 (k_u - K) sd_u + n_u (k_u - K)^2,  mean = K + S1/M,
// var = S2/M - (S1/M)^2.  Then rstd, scale / shift and the running statistics as bn_finalize_kernel; *count_out = M.
// grid ceil(C/32), block 1024
__global__ void __launch_bounds__(1024)
bn_record_finalize_kernel(const float* __restrict__ rec, int N, int C, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float* __restrict__ running_mean,
                          float* __restrict__ running_var, float momentum, float eps, float* __restrict__ mean_out,
                          float* __restrict__ rstd_out, float* __restrict__ scale_out, float* __restrict__ shift_out,
                          float* __restrict__ unbiased_out, long long* __restrict__ count_out, int update_running) {
  __shared__ double red[3][32][33];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const long S = 3L * C + 1;
  double a1 = 0.0, a2 = 0.0, an = 0.0, K = 0.0;
  if (c < C) {
    K = rec[c];
    for (int u = sl; u < N; u += 32) {
      const float* r = rec + u * S;
      const double dk = static_cast<double>(r[c]) - K;
      const double sd = r[C + c], ssd = r[2 * C + c];
      const double n = static_cast<double>(__float_as_int(r[3 * C]));
      a1 += sd + n * dk;
      a2 += ssd + 2.0 * dk * sd + n * dk * dk;
      an += n;
    }
  }
  red[0][sl][lane] = a1;
  red[1][sl][lane] = a2;
  red[2][sl][lane] = an;
  __syncthreads();
  if (sl != 0 || c >= C) return;
  double s1 = 0.0, s2 = 0.0, M = 0.0;
  for (int i = 0; i < 32; ++i) {
    s1 += red[0][i][lane];
    s2 += red[1][i][lane];
    M += red[2][i][lane];
  }
  const double dmean = s1 / M;
  const double mean = K + dmean;
  double var = s2 / M - dmean * dmean;
  if (var < 0.0) var = 0.0;
  const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const float sc = gamma[c] * rstd;
  mean_out[c] = static_cast<float>(mean);
  rstd_out[c] = rstd;
  scale_out[c] = sc;
  shift_out[c] = beta[c] - static_cast<float>(mean) * sc;
  const double unbiased = M > 1.0 ? var * M / (M - 1.0) : var;
  if (unbiased_out) unbiased_out[c] = static_cast<float>(unbiased);
  if (update_running) {
    running_mean[c] = bn_momentum_update(running_mean[c], static_cast<float>(mean), momentum);
    running_var[c] = bn_momentum_update(running_var[c], static_cast<float>(unbiased), momentum);
  }
  if (c == 0 && count_out) *count_out = static_cast<long long>(M);
}

// Backward record of every utterance: sum g_z, sum g_z xhat (the terms of bn_bwd_reduce_kernel).  grid (B, C/64)
template <bool BF16>
__global__ void __launch_bounds__(256)
bn_bwd_utt_record_kernel(const uint16_t* __restrict__ gy, const uint16_t* __restrict__ y, const float* __restrict__ raw,
                         const float* __restrict__ mean, const float* __restrict__ rstd, int HW, int C, float clip_hi,
                         float* __restrict__ rec) {
  __shared__ float red[2][32][65];
  const int q = threadIdx.x & 7, p = threadIdx.x >> 3;
  const int u = blockIdx.x;
  const int c0 = blockIdx.y * 64 + q * 8;
  const long off = static_cast<long>(u) * HW * C + c0;
  float mu[8], rs[8], v[2][8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = mean[c0 + e];
    rs[e] = rstd[c0 + e];
    v[0][e] = v[1][e] = 0.f;
  }
  for (int m = p; m < HW; m += 32) {
    const long i = off + static_cast<long>(m) * C;
    float g[8], yy[8], r[8];
    unpack8<BF16>(*reinterpret_cast<const uint4*>(gy + i), g);
    unpack8<BF16>(*reinterpret_cast<const uint4*>(y + i), yy);
    load8f(raw + i, r);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float gz = (yy[e] > 0.f && yy[e] < clip_hi) ? g[e] : 0.f;
      v[0][e] += gz;
      v[1][e] = fmaf(gz, (r[e] - mu[e]) * rs[e], v[1][e]);
    }
  }
  utt_tree_sum(red, 2, p, q, v);
  if (p == 0) {
    float* r = rec + static_cast<long>(u) * 2 * C;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      r[c0 + e] = red[0][0][q * 8 + e];
      r[C + c0 + e] = red[1][0][q * 8 + e];
    }
  }
}

// Backward finalize from the records: the coefficients of bn_bwd_apply_kernel from the GLOBAL sums over the N gathered
// records (b = sum g_z / M, d = sum g_z xhat / M with M the forward's global pixel count), dgamma / dbeta from this rank's
// own n records (the data-parallel gradient reduction adds the ranks' shares), divided by the loss scale dyn[1].
// grid ceil(C/32), block 1024
__global__ void __launch_bounds__(1024)
bn_bwd_record_finalize_kernel(const float* __restrict__ gathered, int N, const float* __restrict__ local, int n, int C,
                              const long long* __restrict__ count, const float* __restrict__ gamma,
                              const float* __restrict__ rstd, const float* __restrict__ dyn, float* __restrict__ dgamma,
                              float* __restrict__ dbeta, float* __restrict__ coef /*[3][C]*/) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  double gs, gss, ls, lss;
  const bool ok = bn_partial_totals(gathered, N, C, c, gs, gss);
  if (!bn_partial_totals(local, n, C, c, ls, lss) || !ok) return;
  const double M = static_cast<double>(*count);
  dbeta[c] = static_cast<float>(ls) * dyn[1];
  dgamma[c] = static_cast<float>(lss) * dyn[1];
  coef[c] = gamma[c] * rstd[c];
  coef[C + c] = static_cast<float>(gs / M);
  coef[2 * C + c] = static_cast<float>(gss / M);
}

// max |g| of every row of a (B, E) matrix: the loss-scale record of one utterance (loss_scale_kernel over the gathered
// maxima picks the S of the single-device backward over the union).  grid B, block 128
__global__ void __launch_bounds__(128) row_absmax_kernel(const float* __restrict__ g, int E, float* __restrict__ out) {
  __shared__ float red[4];
  const float* r = g + static_cast<long>(blockIdx.x) * E;
  float m = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) m = fmaxf(m, fabsf(r[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) out[blockIdx.x] = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
}

// ---- weight repack of a training step: ONE launch for all eleven tensor-core convs -----------------------------------
// A training step changes every parameter, so the 16-bit operand images are rebuilt once per step, on the caller's
// stream, before the three forwards fork, in one launch rather than 44 small ones with strided 4-byte gathers.  Here a block owns a 16 (cout) x 32 (cin) x taps tile of one layer: it reads the
// OIHW fp32 rows contiguously, keeps the rounded 16-bit values in shared memory and writes both images the training path
// reads - [tap][cout][cin] for the forward / weight-gradient convs and [tap'][cin][cout] (filter turned by 180 degrees
// for stride 1) for the data gradient - in 64- and 32-byte runs.  The last block copies conv1's 64x25 fp32 filter.
struct PackTrainTable {
  const float* w[12];
  uint16_t* fwd[12];
  uint16_t* dgrad[12];
  int cout[12], cin[12], taps[12], rotate[12];
  int first_block[13];   // first_block[i] .. first_block[i+1]: the blocks of layer i (i = 1..11); [12] = conv1 block
  float* conv1_dst;
};
constexpr int kPackCo = 16, kPackCi = 32;
template <bool BF16>
__global__ void __launch_bounds__(256) pack_train_weights_kernel(const PackTrainTable t) {
  __shared__ uint16_t sm[kPackCo][kPackCi * 25 + 2];
  const int b = blockIdx.x;
  if (b >= t.first_block[12]) {
    for (int i = threadIdx.x; i < 64 * 25; i += blockDim.x) t.conv1_dst[i] = t.w[0][i];
    return;
  }
  int l = 1;
  while (b >= t.first_block[l + 1]) ++l;
  const int cout = t.cout[l], cin = t.cin[l], taps = t.taps[l];
  const int lb = b - t.first_block[l];
  const int ci_tiles = cin / kPackCi;
  const int co0 = (lb / ci_tiles) * kPackCo, ci0 = (lb % ci_tiles) * kPackCi;
  const int row = kPackCi * taps;                     // contiguous floats of one cout row of the tile
  const float* __restrict__ w = t.w[l];
  for (int i = threadIdx.x; i < kPackCo * row; i += blockDim.x) {
    const int r = i / row, j = i - r * row;
    sm[r][j] = to16<BF16>(w[(static_cast<long>(co0 + r) * cin + ci0) * taps + j]);
  }
  __syncthreads();
  uint16_t* __restrict__ of = t.fwd[l];
  for (int i = threadIdx.x; i < taps * kPackCo * kPackCi; i += blockDim.x) {
    const int ci = i % kPackCi, r = (i / kPackCi) % kPackCo, tap = i / (kPackCi * kPackCo);
    of[(static_cast<long>(tap) * cout + co0 + r) * cin + ci0 + ci] = sm[r][ci * taps + tap];
  }
  uint16_t* __restrict__ od = t.dgrad[l];
  const int rot = t.rotate[l];
  for (int i = threadIdx.x; i < taps * kPackCo * kPackCi; i += blockDim.x) {
    const int r = i % kPackCo, ci = (i / kPackCo) % kPackCi, tap = i / (kPackCi * kPackCo);
    od[(static_cast<long>(tap) * cin + ci0 + ci) * cout + co0 + r] = sm[r][ci * taps + (rot ? taps - 1 - tap : tap)];
  }
}

}  // namespace dsk
