// Stage-entry conv1 of the eval forward — 5x5 stride-2 pad-2, 1 -> 64 channels, + folded bn1 + clipped ReLU
// (reference model.py:94-97 used at :187-189) — on the Hopper tensor cores (wgmma) at fp32-level accuracy.
//
// The SIMT form of this layer is FP32-issue bound (1600 FMAs per output pixel).  Here a CTA builds the im2col operand
// of 128 output pixels in shared memory (one thread = one pixel = one 128-byte K-major SWIZZLE_128B row) and lets
// wgmma do the math (each K16 step twice, rows 0-63 and 64-127):
//   x = x_hi + x_lo, w = w_hi + w_lo (each half a 16-bit float);  x*w ~= x_hi*w_hi + x_lo*w_hi + x_hi*w_lo
//   A row  = [ x_hi(taps 0..24), 0 x 7 | x_lo(taps 0..24), 0 x 7 ]                      (K = 64)
//   B1 row = [ w_hi,             0 x 7 | w_hi,             0 x 7 ]  -> 4 K16 steps (K = 64): (x_hi + x_lo) * w_hi
//   B2 row = [ w_lo,             0 x 7 |        unused            ]  -> 2 K16 steps (K = 32):  x_hi * w_lo
// The dropped x_lo*w_lo term is 2^-22 relative (fp16 halves; 2^-16 with bf16 halves), far below the 16-bit
// rounding of the activation this kernel stores.  Accumulation is fp32 in registers.
// 128 threads (one warpgroup) and ~55 KB of shared memory per CTA: several CTAs share an SM, so one CTA's operand
// build overlaps another's MMA / epilogue.
#pragma once
#include "conv_umma.cuh"

namespace dsk {

constexpr int kConv1ImgHalfs = 2 * 64 * 64;  // B1 | B2, each 64 rows x 64 halfs, pre-swizzled

// w [64][25] fp32 -> the pre-swizzled shared-memory image of B1 | B2 (byte offset of element (n, k) inside a
// matrix: n*128 + ((k/8) ^ (n&7))*16 + (k%8)*2 — the SWIZZLE_128B K-major layout TMA would have produced).
template <bool BF16>
__global__ void pack_conv1_umma_kernel(const float* __restrict__ w, uint16_t* __restrict__ img) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kConv1ImgHalfs; i += gridDim.x * blockDim.x) {
    const int mat = i / (64 * 64), n = (i / 64) % 64, k = i % 64;
    const int tap = k & 31;
    uint16_t v = 0;
    if (tap < 25 && (mat == 0 || k < 32)) {
      const float wf = w[n * 25 + tap];
      const uint16_t hi = to16<BF16>(wf);
      v = mat == 0 ? hi : to16<BF16>(wf - from16<BF16>(hi));
    }
    img[mat * 64 * 64 + n * 64 + (((k >> 3) ^ (n & 7)) << 3) + (k & 7)] = v;
  }
}

// x (B, T, 64) fp32 through tmX: 3-D tensor map (64 bins, T frames, B utterances), box {64, 11, 1}, no swizzle - the 11
// input rows an output-row quad needs arrive as ONE TMA box; rows above / below the utterance are the map's
// out-of-bounds zero fill (the conv's zero padding in time), the two padding columns per side are predicated reads.
// out: zero-padded NHWC 16-bit activation (rows n*(T/2+1)+h+1, 33 pixels per row, 64 channels).
// Tiles: 4 output rows x 32 pixels; n_tiles = B * (T/2) / 4 (T/2 must be a multiple of 4).
//
// Persistent over the CTA's tiles t_0, t_1, ... (tile = blockIdx.x + k * gridDim.x):
//     iteration i :  wait patch(t_i)  ->  build A[i&1]  ->  prefetch patch(t_{i+2})  ->  MMA(t_i)  ->  epilogue(t_i)
// so the fbank rows of tile i+2 are in flight while tile i is computed.  The weight image and the barriers are set up
// once per CTA instead of once per tile.
constexpr int kConv1Threads = 128;
constexpr int kConv1PatchRows = 11;
constexpr int kConv1SmemBytes = 2 * 128 * 128 /*A*/ + 2 * 64 * 128 /*B*/ + 2 * kConv1PatchRows * 64 * 4 /*patch*/ + 1024 /*align*/;

template <bool BF16>
__global__ void __launch_bounds__(kConv1Threads)
conv1_umma_kernel(const __grid_constant__ CUtensorMap tmX, const uint4* __restrict__ wimg, const float* __restrict__ scale,
                  const float* __restrict__ bias, uint16_t* __restrict__ out, int T, int n_tiles, float clip_hi) {
  constexpr int WOUT = 32, ROWS = 4, PR = kConv1PatchRows;
  extern __shared__ uint8_t c1_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(c1_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                   // [2][128 rows x 128 B], SWIZZLE_128B K-major
  uint8_t* sB = sA + 2 * 128 * 128;                     // B1 | B2
  float* patch = reinterpret_cast<float*>(sB + 2 * 64 * 128);   // [2][11][64]
  __shared__ float s_scale[64], s_bias[64];
  __shared__ __align__(8) uint64_t patch_full[2];

  const int tid = threadIdx.x;
  const int hout = T / 2, tiles_h = hout / ROWS;
  pdl_launch_dependents();
  if (tid == 32) {
    tma_prefetch_desc(&tmX);
    mbar_init(&patch_full[0], 1);
    mbar_init(&patch_full[1], 1);
    fence_barrier_init();
  }
  // parameters are safe to read before the dependency wait; the input batch may come from the preceding kernel of
  // the stream and the output buffer is still read by the previous forward
#pragma unroll
  for (int i = 0; i < 8; ++i) reinterpret_cast<uint4*>(sB)[tid + 128 * i] = wimg[tid + 128 * i];
  if (tid < 64) {
    s_scale[tid] = scale[tid];
    s_bias[tid] = bias[tid];
  }
  fence_proxy_async_smem();  // B image: generic-proxy writes -> visible to the tensor core's async proxy
  __syncthreads();
  pdl_wait();

  const int my_tiles = (n_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  auto tile_of = [&](int i) { return static_cast<int>(blockIdx.x) + i * static_cast<int>(gridDim.x); };
  auto load_patch = [&](int i) {  // one thread: the 11 x 64 fp32 rows of tile t_i, zero-filled outside the utterance
    const int t = tile_of(i), n = t / tiles_h, h0 = (t - n * tiles_h) * ROWS;
    const int b = i & 1;
    mbar_arrive_expect_tx(&patch_full[b], PR * 64 * 4);
    tma_load_3d(patch + b * PR * 64, &tmX, &patch_full[b], 0, 2 * h0 - 2, n);
  };
  if (tid == 0) {
    if (my_tiles > 0) load_patch(0);
    if (my_tiles > 1) load_patch(1);
  }

  const int fr = frag_row(), fc = frag_col();
  for (int i = 0; i < my_tiles; ++i) {
    const int b = i & 1;
    mbar_wait(&patch_full[b], (i >> 1) & 1);
    // ---- operand build: thread = output pixel (r, ow) of the tile = row tid of A[b]
    {
      const float* pt = patch + b * PR * 64;
      const int r = tid >> 5, ow = tid & 31;
      uint32_t hi[16], lo[16];  // 32 halfs each, taps 25..31 are zero
#pragma unroll
      for (int q = 0; q < 16; ++q) hi[q] = lo[q] = 0u;
#pragma unroll
      for (int ii = 0; ii < 5; ++ii) {
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const int tap = ii * 5 + j;
          const int iw = 2 * ow + j - 2;
          const float v = (static_cast<unsigned>(iw) < 64u) ? pt[(2 * r + ii) * 64 + iw] : 0.0f;
          const uint16_t h16 = to16<BF16>(v);
          const uint16_t l16 = to16<BF16>(v - from16<BF16>(h16));
          hi[tap >> 1] |= static_cast<uint32_t>(h16) << ((tap & 1) * 16);
          lo[tap >> 1] |= static_cast<uint32_t>(l16) << ((tap & 1) * 16);
        }
      }
      // A[b] is free: its last reader, the cooperative store of tile i-2's epilogue, ended before the previous
      // iteration's last __syncthreads
      uint8_t* row = sA + b * 128 * 128 + tid * 128;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        *reinterpret_cast<uint4*>(row + ((c ^ (tid & 7)) << 4)) = make_uint4(hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]);
        *reinterpret_cast<uint4*>(row + (((c + 4) ^ (tid & 7)) << 4)) = make_uint4(lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]);
      }
    }
    fence_proxy_async_smem();  // generic-proxy writes of A -> visible to the tensor core's async proxy
    __syncthreads();           // A[b] complete; patch[b] consumed by every thread
    if (tid == 0 && i + 2 < my_tiles) load_patch(i + 2);
    // ---- MMA: rows 0-63 and 64-127 of the tile, fp32 accumulators in registers
    float acc[2][32];
    {
      const uint64_t da = gmma_desc_sw128(smem_u32(sA + b * 128 * 128));
      const uint64_t db1 = gmma_desc_sw128(smem_u32(sB));
      const uint64_t db2 = gmma_desc_sw128(smem_u32(sB + 64 * 128));
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int e = 0; e < 32; ++e) acc[m][e] = 0.0f;
      wgmma_fence();
#pragma unroll
      for (int m = 0; m < 2; ++m) {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_f16<64, BF16>(acc[m], da + m * kDescRows64 + 2 * k, db1 + 2 * k, k > 0 ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < 2; ++k) wgmma_f16<64, BF16>(acc[m], da + m * kDescRows64 + 2 * k, db2 + 2 * k, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc[0]);
      wgmma_fence_acc(acc[1]);
    }
    __syncthreads();  // every warp's MMAs have read A[b]: it becomes the staging tile
    // ---- epilogue: folded BN, clip, 16-bit pack into A[b], then cooperative stores: 8 lanes write one 128-byte pixel
    // row, so a warp store covers four full lines
    {
      const int t = tile_of(i), n = t / tiles_h, h0 = (t - n * tiles_h) * ROWS;
      uint8_t* stage = sA + b * 128 * 128;
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = 64 * m + fr + 8 * h, c = 8 * g + fc;
            const float f0 = relu_clip(fmaf(acc[m][4 * g + 2 * h], s_scale[c], s_bias[c]), clip_hi);
            const float f1 = relu_clip(fmaf(acc[m][4 * g + 2 * h + 1], s_scale[c + 1], s_bias[c + 1]), clip_hi);
            *reinterpret_cast<uint32_t*>(stage + sw128_off16(row, c)) = pack2<BF16>(f0, f1);
          }
      __syncthreads();
      const int chunk = tid & 7;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int row = k * 16 + (tid >> 3);
        const uint4 val = *reinterpret_cast<const uint4*>(stage + row * 128 + ((chunk ^ (row & 7)) << 4));
        const long pix = (static_cast<long>(n) * (hout + 1) + h0 + (row >> 5) + 1) * (WOUT + 1) + 1 + (row & 31);
        reinterpret_cast<uint4*>(out + pix * 64)[chunk] = val;
      }
      __syncthreads();  // the staging tile is the next-but-one operand tile: every row has been copied out before it is rebuilt
    }
  }
}

}  // namespace dsk
