// CUDA-core kernels around the tensor-core convs: weight repack, BN folding, the Cin=1 first conv,
// temporal mean-pool + fc + L2-norm tail.  NHWC 16-bit activations (fp16 or bf16 via template).
#pragma once
#include "dsk_ptx.cuh"

namespace dsk {

// ---------------------------------------------------------------------------------------------
// OIHW fp32 -> [tap][cout][cin] 16-bit (tap = r*S + s). One-time at weight load.
// ---------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, uint16_t* __restrict__ out, int cout, int cin,
                                        int taps) {
  const long total = static_cast<long>(cout) * cin * taps;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ci = i % cin;
    const long r = i / cin;
    const int co = r % cout;
    const int tap = r / cout;
    out[i] = to16<BF16>(w[(static_cast<long>(co) * cin + ci) * taps + tap]);
  }
}

// [slot][cout][cin] with slot -> original tap perm[slot] (plane-major tap order of the halo 5x5 s2 conv).
template <bool BF16>
__global__ void pack_conv_weight_perm_kernel(const float* __restrict__ w, uint16_t* __restrict__ out, int cout, int cin,
                                             int taps, const int* __restrict__ perm) {
  const long total = static_cast<long>(cout) * cin * taps;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ci = i % cin;
    const long r = i / cin;
    const int co = r % cout;
    const int slot = r / cout;
    out[i] = to16<BF16>(w[(static_cast<long>(co) * cin + ci) * taps + perm[slot]]);
  }
}

// Same with cin/cout swapped (the weight of "data-gradient as a convolution"): out[tap'][ci][co] =
// w[co][ci][rotate ? taps-1-tap' : tap'].  rotate=1 (filter turned by 180 degrees) for stride-1 convs; the
// stride-2 data-gradient picks its taps by index and keeps the original order.
template <bool BF16>
__global__ void pack_conv_weight_dgrad_kernel(const float* __restrict__ w, uint16_t* __restrict__ out, int cout,
                                              int cin, int taps, int rotate) {
  const long total = static_cast<long>(cout) * cin * taps;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int co = i % cout;
    const long r = i / cout;
    const int ci = r % cin;
    const int tap = r / cin;
    out[i] = to16<BF16>(w[(static_cast<long>(co) * cin + ci) * taps + (rotate ? taps - 1 - tap : tap)]);
  }
}

// Eval-mode BatchNorm folded to y = x*scale + bias  (reference model.py:59,62,94,99,103,107;
// torch defaults eps=1e-5).
__global__ void bn_fold_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ mean, const float* __restrict__ var, float eps,
                               float* __restrict__ scale, float* __restrict__ bias, int c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c) {
    const float s = gamma[i] / sqrtf(var[i] + eps);
    scale[i] = s;
    bias[i] = beta[i] - mean[i] * s;
  }
}

// ---------------------------------------------------------------------------------------------
// conv1: 5x5 s2 p2, Cin=1 -> 64 (reference model.py:93, used at :187), + affine (+clip).
// x fp32 (B, T, 64) [= NCHW with C=1]; out NHWC 16-bit (B, T/2, 32, 64).
// Block = 4 output rows of one utterance; warp = 16 pixels; lane = 2 output channels, whose
// 50 filter weights live in registers; the input patch is broadcast from shared memory.
// ---------------------------------------------------------------------------------------------
template <bool BF16, bool OUT_F32 = false>
__global__ void __launch_bounds__(256)
conv1_kernel(const float* __restrict__ x, const float* __restrict__ w /*[64][25]*/, const float* __restrict__ scale,
             const float* __restrict__ bias, void* __restrict__ out, int T, int do_clip, float clip_hi, int padded) {
  constexpr int WIN = 64, WOUT = 32, ROWS = 8, PATCH_ROWS = 2 * ROWS + 3, PATCH_W = WIN + 4;
  __shared__ __align__(16) float patch[PATCH_ROWS][PATCH_W];  // PATCH_W * 4 B is a multiple of 16
  __shared__ float wsm[64 * 25];
  pdl_launch_dependents();
  pdl_wait();  // the output buffer may still be read by the previous forward's kernels
  const int hout = T / 2;
  const int tiles_h = (hout + ROWS - 1) / ROWS;
  const int n = blockIdx.x / tiles_h;
  const int h0 = (blockIdx.x % tiles_h) * ROWS;
  const float* xin = x + static_cast<long>(n) * T * WIN;
  {
    constexpr int NEL = PATCH_ROWS * PATCH_W, NIT = (NEL + 255) / 256;
    float t[NIT];
#pragma unroll
    for (int j = 0; j < NIT; ++j) {  // all loads first (independent), then the stores
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
  {
    float t[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) t[j] = (threadIdx.x + 256 * j < 64 * 25) ? w[threadIdx.x + 256 * j] : 0.f;
#pragma unroll
    for (int j = 0; j < 7; ++j)
      if (threadIdx.x + 256 * j < 64 * 25) wsm[threadIdx.x + 256 * j] = t[j];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = lane * 2;
  float w0[25], w1[25];
#pragma unroll
  for (int t = 0; t < 25; ++t) {
    w0[t] = wsm[c0 * 25 + t];
    w1[t] = wsm[(c0 + 1) * 25 + t];
  }
  const float s0 = scale[c0], s1 = scale[c0 + 1], b0 = bias[c0], b1 = bias[c0 + 1];
  uint32_t* o32 = reinterpret_cast<uint32_t*>(out);
  const int oh = h0 + warp;  // one output row per warp
  if (oh >= hout) return;
  // padded NHWC layout (conv3x3_halo.cuh): row n*(H+1)+h+1, W+1 pixels per row, column 0 is the zero pad
  const long pix0 = padded ? (static_cast<long>(n) * (hout + 1) + oh + 1) * (WOUT + 1) + 1
                           : (static_cast<long>(n) * hout + oh) * WOUT;
  // four output pixels per iteration: their 5x11 input window is 3 aligned float4 broadcast loads per filter row
  // (15 shared loads feed 200 FMAs; one load per tap would make the loop load-issue bound)
#pragma unroll 1
  for (int ow = 0; ow < WOUT; ow += 4) {
    float a[4][2];
#pragma unroll
    for (int q = 0; q < 4; ++q) a[q][0] = a[q][1] = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const float4* prow = reinterpret_cast<const float4*>(&patch[2 * warp + r][2 * ow]);
      const float4 v0 = prow[0], v1 = prow[1], v2 = prow[2];
      const float v[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
#pragma unroll
      for (int s = 0; s < 5; ++s) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          a[q][0] = fmaf(v[2 * q + s], w0[r * 5 + s], a[q][0]);
          a[q][1] = fmaf(v[2 * q + s], w1[r * 5 + s], a[q][1]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float a0 = fmaf(a[q][0], s0, b0);
      float a1 = fmaf(a[q][1], s1, b1);
      if (do_clip) {
        a0 = relu_clip(a0, clip_hi);
        a1 = relu_clip(a1, clip_hi);
      }
      if constexpr (OUT_F32)
        reinterpret_cast<float2*>(out)[(pix0 + ow + q) * 32 + lane] = make_float2(a0, a1);
      else
        o32[(pix0 + ow + q) * 32 + lane] = pack2<BF16>(a0, a1);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Tail: temporal mean (reference model.py:111,207-208) -> fc (:164,209) -> l2_norm*alpha
// (:172-183,210-213).
// pooled[b][w*C + c] = mean_h act[b][h][w][c]   (act NHWC 16-bit, W=4, C=512)
// The fc weight is repacked once to the same (w, c) column order: wq[e][w*C + c] = W[e][c*4 + w].
// ---------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(256)
pool_time_kernel(const uint16_t* __restrict__ act, float* __restrict__ pooled, int H, int WC, int C, int padded) {
  // grid (B, WC/512): thread = 2 adjacent channels (one 32-bit load per time step), loads independent in h
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const int i = blockIdx.y * 256 + threadIdx.x;  // index of the channel pair
  if (i >= WC / 2) return;
  // dense: rows of W*C; padded layout: rows of (W+1)*C with a leading zero pixel, images H+1 rows apart, first row is a pad
  const long row_pitch = padded ? (WC + C) / 2 : WC / 2;
  const uint32_t* a = reinterpret_cast<const uint32_t*>(act) +
                      (padded ? (static_cast<long>(b) * (H + 1) + 1) * row_pitch + C / 2 : static_cast<long>(b) * H * row_pitch) + i;
  const float inv = 1.0f / static_cast<float>(H);
  float s0 = 0.f, s1 = 0.f;
  int h = 0;
  for (; h + 4 <= H; h += 4) {
    uint32_t u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = a[static_cast<long>(h + j) * row_pitch];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = unpack2<BF16>(u[j]);
      s0 += v.x;
      s1 += v.y;
    }
  }
  for (; h < H; ++h) {
    const float2 v = unpack2<BF16>(a[static_cast<long>(h) * row_pitch]);
    s0 += v.x;
    s1 += v.y;
  }
  pooled[static_cast<long>(b) * WC + 2 * i] = s0 * inv;
  pooled[static_cast<long>(b) * WC + 2 * i + 1] = s1 * inv;
}

__global__ void pack_fc_weight_kernel(const float* __restrict__ w /*[E][C*4+w]*/, float* __restrict__ out, int E,
                                      int C, int W) {
  const long total = static_cast<long>(E) * C * W;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = i % C;
    const long r = i / C;
    const int wi = r % W;
    const int e = r / W;
    out[i] = w[(static_cast<long>(e) * C + c) * W + wi];
  }
}

// part[z][b][e] = sum_{k in slice z} pooled[b][k] * wq[e][k].  grid (ceil(B/64), E/32, kFcSplit), block 256.
// Block = 64 utterances x 32 output features x one K slice of 128: both operand slices sit in shared memory (rows
// padded by 4 floats so that the float4 reads of 8 consecutive rows hit 8 different bank groups); thread = 4 utterances
// x 2 features (f and f+16), six float4 shared loads per 32 FMAs.  Operand traffic from L2 is (64+32)*128*4 B per
// block, 12 MB per forward at B=64 (a 16x16 tile moves 32 MB and was bandwidth-bound at 15 us).  The K split gives the
// tail 256 blocks; the slices are summed in fixed order (plus the bias) by l2norm_kernel, so the result does not
// depend on scheduling.
constexpr int kFcUtt = 64, kFcFeat = 32, kFcSlice = 128, kFcSplit = 2048 / kFcSlice, kFcPitch = kFcSlice + 4;
__global__ void __launch_bounds__(256)
fc_kernel(const float* __restrict__ pooled, const float* __restrict__ wq, float* __restrict__ part, int B, int K, int E) {
  extern __shared__ __align__(16) float fc_smem[];
  float* sp = fc_smem;                      // [kFcUtt][kFcPitch]
  float* sw = fc_smem + kFcUtt * kFcPitch;  // [kFcFeat][kFcPitch]
  const int b0 = blockIdx.x * kFcUtt, e0 = blockIdx.y * kFcFeat, k0 = blockIdx.z * kFcSlice;
  const int tid = threadIdx.x;
  pdl_launch_dependents();
  // fill: (64 + 32) rows x 32 float4; thread = float4 column (tid & 31) of rows (tid >> 5) + 8 i; all loads in flight
  {
    const int c4 = tid & 31, r0 = tid >> 5;
    float4 tw[kFcFeat / 8], tp[kFcUtt / 8];
#pragma unroll
    for (int i = 0; i < kFcFeat / 8; ++i)  // parameters: safe before the dependency wait
      tw[i] = reinterpret_cast<const float4*>(wq + static_cast<long>(e0 + r0 + 8 * i) * K + k0)[c4];
    pdl_wait();
#pragma unroll
    for (int i = 0; i < kFcUtt / 8; ++i) {
      const int u = b0 + r0 + 8 * i;
      tp[i] = u < B ? reinterpret_cast<const float4*>(pooled + static_cast<long>(u) * K + k0)[c4]
                    : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < kFcFeat / 8; ++i) reinterpret_cast<float4*>(sw + (r0 + 8 * i) * kFcPitch)[c4] = tw[i];
#pragma unroll
    for (int i = 0; i < kFcUtt / 8; ++i) reinterpret_cast<float4*>(sp + (r0 + 8 * i) * kFcPitch)[c4] = tp[i];
  }
  __syncthreads();
  const int tf = tid & 15, tu = tid >> 4;  // features tf, tf+16; utterances 4*tu .. 4*tu+3
  float acc[4][2];
#pragma unroll
  for (int u = 0; u < 4; ++u) acc[u][0] = acc[u][1] = 0.f;
  const float4* w0 = reinterpret_cast<const float4*>(sw + tf * kFcPitch);
  const float4* w1 = reinterpret_cast<const float4*>(sw + (tf + 16) * kFcPitch);
  const float4* p0 = reinterpret_cast<const float4*>(sp + (4 * tu) * kFcPitch);
#pragma unroll 4
  for (int k4 = 0; k4 < kFcSlice / 4; ++k4) {
    const float4 a = w0[k4], b = w1[k4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4 pv = p0[u * (kFcPitch / 4) + k4];
      acc[u][0] = fmaf(a.x, pv.x, acc[u][0]);
      acc[u][0] = fmaf(a.y, pv.y, acc[u][0]);
      acc[u][0] = fmaf(a.z, pv.z, acc[u][0]);
      acc[u][0] = fmaf(a.w, pv.w, acc[u][0]);
      acc[u][1] = fmaf(b.x, pv.x, acc[u][1]);
      acc[u][1] = fmaf(b.y, pv.y, acc[u][1]);
      acc[u][1] = fmaf(b.z, pv.z, acc[u][1]);
      acc[u][1] = fmaf(b.w, pv.w, acc[u][1]);
    }
  }
  float* pz = part + static_cast<long>(blockIdx.z) * B * E;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int ub = b0 + 4 * tu + u;
    if (ub < B) {
      pz[static_cast<long>(ub) * E + e0 + tf] = acc[u][0];
      pz[static_cast<long>(ub) * E + e0 + tf + 16] = acc[u][1];
    }
  }
}

// y[b][:] = bias + sum_z part[z][b][:] (fixed order; written out for the backward pass), then
// out[b][:] = alpha * y[b][:] / sqrt(sum(y^2) + 1e-10)   (reference model.py:172-183,210-213)
// also writes inv_norm[b] = 1/sqrt(sum+1e-10) when inv_norm != nullptr (saved for backward).
__global__ void l2norm_kernel(const float* __restrict__ part, int nsplit, const float* __restrict__ bias,
                              float* __restrict__ y, float* __restrict__ out, float* __restrict__ inv_norm, int B, int E,
                              float alpha) {
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  float* yr = y + static_cast<long>(b) * E;
  float s = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    float v = bias[i];
    const float* pp = part + static_cast<long>(b) * E + i;
    const long zs = static_cast<long>(B) * E;
    int z = 0;
    for (; z + 8 <= nsplit; z += 8) {  // eight independent loads, added in slice order
      float t[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = pp[(z + j) * zs];
#pragma unroll
      for (int j = 0; j < 8; ++j) v += t[j];
    }
    for (; z < nsplit; ++z) v += pp[z * zs];
    yr[i] = v;  // re-read below by the same thread
    s = fmaf(v, v, s);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float norm = sqrtf(red[0] + 1e-10f);
  if (threadIdx.x == 0 && inv_norm) inv_norm[b] = 1.0f / norm;
  for (int i = threadIdx.x; i < E; i += blockDim.x) out[static_cast<long>(b) * E + i] = (yr[i] / norm) * alpha;
}

}  // namespace dsk
