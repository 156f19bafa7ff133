// Classifier head + cross-entropy of the reference's hard-triplet branch and the fused optimizer step.
//
//   * Linear(512, C) of DeepSpeakerModel.forward_classifier (reference model.py:167,220-223) and its backward:
//     three small fp32 GEMMs (M = 3k selected utterances <= 1536, N = C classes (1211 for VoxCeleb1), K = 512;
//     0.24 GFLOP each at k = 128).  They are latency-sized and feed a log-softmax whose loss must match the fp32
//     reference to 1e-3, so they run in fp32 on the CUDA cores (one 64x64 tile per CTA, fixed summation order:
//     deterministic) instead of rounding embeddings and logit gradients to 16 bit for the tensor cores.
//   * nn.CrossEntropyLoss()(cat[cls_a, cls_p, cls_n], cat[label_p, label_p, label_n])
//     (reference train_triplet.py:281-285): row-wise log-sum-exp + NLL, mean over rows; backward
//     (softmax - onehot) * g / M.
//   * torch.optim.Adagrad(lr, lr_decay, weight_decay) step (reference train_triplet.py:369-383, called at
//     :224,291) over ONE flat parameter / gradient / state bucket, fused with the post-allreduce scale:
//       g = grad / div (/ max(*denom, 1e-30));  g += wd * p;  G = fma(g, g, G);  p += (g * -clr) / (sqrt(G) + eps)
//     — after the scale, the operation order of torch's foreach implementation, so results are bit-identical to
//     torch.optim.Adagrad stepping on the divided gradient.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dsk {

// ---- fp32 GEMM with generic strides ------------------------------------------------------------------------------
// C[i][j] = sum_k A(i,k) * B(k,j) (+ bias[j]),  A(i,k) = A[i*a_i + k*a_k],  B(k,j) = B[k*b_k + j*b_j],  C row-major.
// 64x64 tile per CTA, 16-deep K slices, 256 threads x (4x4) outputs; k runs in ascending order (deterministic).
constexpr int kGemmTile = 64, kGemmK = 16;

__global__ void __launch_bounds__(256)
sgemm_strided_kernel(const float* __restrict__ A, long a_i, long a_k, const float* __restrict__ B, long b_k, long b_j,
                     const float* __restrict__ bias, float* __restrict__ C, int M, int N, int K) {
  __shared__ float sa[kGemmK][kGemmTile + 4];
  __shared__ float sb[kGemmK][kGemmTile + 4];
  const int i0 = blockIdx.y * kGemmTile, j0 = blockIdx.x * kGemmTile;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  // loader mapping: when the k stride is 1 consecutive threads walk k (coalesced rows), otherwise they walk i / j
  const bool a_kfast = a_k == 1, b_kfast = b_k == 1;
  for (int k0 = 0; k0 < K; k0 += kGemmK) {
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const int e = threadIdx.x + 256 * l;  // 1024 elements per operand slice
      {
        const int kk = a_kfast ? (e & 15) : (e >> 6), ii = a_kfast ? (e >> 4) : (e & 63);
        const int gi = i0 + ii, gk = k0 + kk;
        sa[kk][ii] = (gi < M && gk < K) ? A[gi * a_i + gk * a_k] : 0.f;
      }
      {
        const int kk = b_kfast ? (e & 15) : (e >> 6), jj = b_kfast ? (e >> 4) : (e & 63);
        const int gj = j0 + jj, gk = k0 + kk;
        sb[kk][jj] = (gj < N && gk < K) ? B[gk * b_k + gj * b_j] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGemmK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&sa[kk][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&sb[kk][tx * 4]);
      const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(a4[r], b4[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int gi = i0 + ty * 4 + r;
    if (gi >= M) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int gj = j0 + tx * 4 + c;
      if (gj < N) C[static_cast<long>(gi) * N + gj] = acc[r][c] + (bias ? bias[gj] : 0.f);
    }
  }
}

// out[j] = sum_i G[i][j]   (bias gradient; one thread per column, ascending i: deterministic)
__global__ void colsum_kernel(const float* __restrict__ G, int M, int N, float* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  float s = 0.f;
  for (int i = 0; i < M; ++i) s += G[static_cast<long>(i) * N + j];
  out[j] = s;
}

// ---- cross-entropy ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = red[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
  __syncthreads();
  return t;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
  __syncthreads();
  return t;
}

// one block per row: lse[i] = log sum_j exp(logits[i][j]); row_loss[i] = lse[i] - logits[i][label[i]]
// (a label outside [0, C) gives NaN, which poisons the mean instead of reading out of bounds)
__global__ void __launch_bounds__(256)
ce_rows_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int C, float* __restrict__ lse,
               float* __restrict__ row_loss) {
  __shared__ float red[8];
  const float* row = logits + static_cast<long>(blockIdx.x) * C;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < C; j += blockDim.x) m = fmaxf(m, row[j]);
  m = block_reduce_max(m, red);
  float s = 0.f;
  for (int j = threadIdx.x; j < C; j += blockDim.x) s += expf(row[j] - m);
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) {
    const float l = m + logf(s);
    const int64_t y = labels[blockIdx.x];
    lse[blockIdx.x] = l;
    row_loss[blockIdx.x] = (y >= 0 && y < C) ? l - row[y] : __int_as_float(0x7fc00000);
  }
}

// loss = sum(row_loss[0, M)) / count   (single block, fixed order; count = M is the mean, count < M the mean over the
// rows that carry a term when the others hold 0)
__global__ void __launch_bounds__(1024)
mean_rows_kernel(const float* __restrict__ v, int M, int count, float* __restrict__ out) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < M; i += blockDim.x) s += v[i];
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) out[0] = s / static_cast<float>(count);
}

// dlogits[i][j] = (exp(logits - lse) - [j == label]) * g / M; a row whose label is outside [0, C) is NaN, like its loss
__global__ void ce_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels,
                              const float* __restrict__ lse, const float* __restrict__ grad_loss, int M, int C,
                              float* __restrict__ dlogits) {
  const long total = static_cast<long>(M) * C;
  const float g = grad_loss[0] / static_cast<float>(M);
  for (long e = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(e / C), j = static_cast<int>(e - static_cast<long>(i) * C);
    const int64_t y = labels[i];
    const float p = expf(logits[e] - lse[i]);
    dlogits[e] = (y >= 0 && y < C) ? (p - (y == j ? 1.f : 0.f)) * g : __int_as_float(0x7fc00000);
  }
}

// ---- fused Adagrad over a flat bucket -------------------------------------------------------------------------------
// Explicit round-to-nearest intrinsics pin the operation order (no re-association / contraction beyond the one fma
// torch's foreach addcmul kernel performs).
// The post-allreduce scale divides, as GradBucket's div_ does: g / div, then g / max(*denom, 1e-30) (torch's
// clamp_min, NaN passes).  A product with the rounded reciprocal differs from the quotient in the last bit for a fifth
// to a half of the elements when the divisor is 3, 5, 6, 7 or 37; with *denom = 0 it would be 0 * inf = NaN.
__global__ void __launch_bounds__(256)
adagrad_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sum, long n, float div,
                    const float* __restrict__ denom, float minus_clr, float eps, float wd) {
  float dd = 1.0f;
  if (denom) dd = denom[0] < 1e-30f ? 1e-30f : denom[0];
  const long n4 = n >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float4* s4 = reinterpret_cast<float4*>(sum);
  auto upd = [&](float& pv, float gv, float& sv) {
    if (div != 1.0f) gv = __fdiv_rn(gv, div);
    if (denom) gv = __fdiv_rn(gv, dd);
    if (wd != 0.f) gv = __fmaf_rn(pv, wd, gv);        // grad.add(param, alpha=wd)
    sv = __fmaf_rn(gv, gv, sv);                       // state_sum.addcmul_(grad, grad, value=1)
    const float std_ = __fadd_rn(__fsqrt_rn(sv), eps);  // sqrt().add_(eps)
    pv = __fadd_rn(pv, __fdiv_rn(__fmul_rn(gv, minus_clr), std_));  // param.addcdiv_(grad * -clr, std)
  };
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    float4 pv = p4[i], sv = s4[i];
    const float4 gv = g4[i];
    upd(pv.x, gv.x, sv.x);
    upd(pv.y, gv.y, sv.y);
    upd(pv.z, gv.z, sv.z);
    upd(pv.w, gv.w, sv.w);
    p4[i] = pv;
    s4[i] = sv;
  }
  for (long i = (n4 << 2) + blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    float pv = p[i], sv = sum[i];
    upd(pv, g[i], sv);
    p[i] = pv;
    sum[i] = sv;
  }
}

}  // namespace dsk
