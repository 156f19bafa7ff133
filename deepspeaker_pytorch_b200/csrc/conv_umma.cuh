// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the cuDNN calls the reference reaches through nn.Conv2d for the 3x3 s1 p1 convs inside
// BasicBlock (reference model.py:47-50,58,61 used at :69,73) and the 5x5 s2 p2 stage-entry
// convs conv2..conv4 (reference model.py:98,102,106 used at :192,197,202), with the
// BatchNorm affine (:59,62,99,103,107), the residual add (:79) and the clipped ReLU (:36-39)
// folded into the epilogue.
//
// Data layout: activations are NHWC, 16-bit (fp16 or bf16).  GEMM view: M = output pixels,
// N = output channels, K = taps x input channels.  One K-step = one filter tap x 64 input channels:
//   A tile  (128 pixels x 64 ch)   one TMA box {64, wt, 1, hb, nb} of the (tap-shifted) input; zero padding
//                                  comes from TMA out-of-bounds fill
//   B tile  (N_TILE cout x 64 ch)  one TMA box of the [tap][cout][cin] weight tensor
// both land in 128B-swizzled shared memory and feed wgmma (M=64, N=N_TILE, K=16) x 4 in each of two consumer
// warpgroups (rows 0-63 and 64-127 of the tile).  The fp32 accumulators stay in the consumers' registers; the same
// warpgroups then apply scale/bias (+residual) (+clip), convert to 16 bit and TMA-store NHWC through a swizzled
// staging tile.
#pragma once
#include "dsk_ptx.cuh"

namespace dsk {

constexpr int kMaxTaps = 25;
constexpr int kTileM = 128;
constexpr int kKStep = 64;               // 16-bit elements per K-step = 128 bytes = one swizzle row
constexpr int kATileBytes = kTileM * 128;  // 16 KB

enum ConvFlags : int {
  CONV_RESIDUAL = 1,  // add residual tile (same shape as output) before the clip
  CONV_CLIP = 2,      // clamp to [0, clip_hi]
};

struct ConvParams {
  // tile geometry
  int tiles_w, tiles_h, tiles_n, tiles_c;  // output tile grid: width, height, batch, cout
  int wt, hb, nb;                          // pixels per tile along w, h, batch (wt*hb*nb == 128)
  int taps, cin_chunks;
  int cout;
  int flags;
  float clip_hi;
  const float* scale;  // [cout] or nullptr (=1)
  const float* bias;   // [cout] or nullptr (=0)
  // output placement in the 5-D output view (c, w, ph, h, n): channel base and parity row.  Plain NHWC
  // outputs use (0, 0); the stride-2 data-gradient writes parity class (ph, pw) with out_c_base = pw*C.
  int out_c_base, out_ph;
  // per-tap source offsets in the 5-D input view (c, w2, ph, h2, n) and weight slice index
  int16_t tap_c[kMaxTaps];
  int8_t tap_w[kMaxTaps];
  int8_t tap_dw[kMaxTaps];
  int8_t tap_ph[kMaxTaps];
  int8_t tap_dh[kMaxTaps];
};

constexpr int kConvThreads = 384;  // warpgroup 0: TMA producer (warp 0) and residual prefetcher (warp 3); 1, 2: consumers

// Position of accumulator element d[4*i + 2*h + e] of a wgmma fragment (dsk_ptx.cuh) inside its warpgroup's 64 x N
// slice: row frag_row() + 8*h, column 8*i + frag_col() + e.
__device__ __forceinline__ int frag_row() { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2); }
__device__ __forceinline__ int frag_col() { return 2 * (threadIdx.x & 3); }
// byte offset of 16-bit element (row, col) (col < 64) in a 128-row x 128-byte SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_off16(int row, int col) {
  return static_cast<uint32_t>(row * 128 + ((((col >> 3) ^ row) & 7) << 4) + (col & 7) * 2);
}
// byte offset of fp32 element (row, col) (col < 32) in a 128-row x 128-byte SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_off32(int row, int col) {
  return static_cast<uint32_t>(row * 128 + ((((col >> 2) ^ row) & 7) << 4) + (col & 3) * 4);
}

template <int N_TILE>
struct ConvSmem {
  static_assert(N_TILE == 64 || N_TILE == 128, "a consumer thread holds N_TILE / 2 fp32 accumulators");
  static constexpr int kStages = N_TILE == 64 ? 6 : 4;
  static constexpr int kBTileBytes = N_TILE * 128;
  static constexpr int kStageBytes = kATileBytes + kBTileBytes;
  static constexpr int kStagingBytes = 2 * kATileBytes;  // two 128-row x 128-byte output chunks
  static constexpr int kResBytes = 2 * kATileBytes;      // residual tiles, prefetched by their own warp
  static constexpr int kScaleBiasBytes = 2 * 512 * 4;
  static constexpr int kBarBytes = 256;
  static constexpr int kTotal =
      kStages * kStageBytes + kStagingBytes + kResBytes + kScaleBiasBytes + kBarBytes + 1024;
};

// OUT_F32: the epilogue stores fp32 (no residual / clip): used for the pre-BatchNorm conv output of the
// train-mode forward, which must not be rounded to 16 bit before the batch statistics are applied.
template <int N_TILE, bool BF16, bool OUT_F32 = false>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes,
                 const ConvParams p) {
  using S = ConvSmem<N_TILE>;
  constexpr int kStages = S::kStages;
  constexpr int kChunks = N_TILE / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kATileBytes;
  uint8_t* smem_stg = smem + kStages * S::kStageBytes;
  uint8_t* smem_res = smem_stg + S::kStagingBytes;
  float* smem_scale = reinterpret_cast<float*>(smem_res + S::kResBytes);
  float* smem_bias = smem_scale + 512;
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(smem_scale) + S::kScaleBiasBytes);
  uint64_t* full_bar = bars;                  // [kStages]
  uint64_t* empty_bar = bars + kStages;       // [kStages]
  uint64_t* res_full = empty_bar + kStages;   // [2]
  uint64_t* res_empty = res_full + 2;         // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  const int ksteps = p.taps * p.cin_chunks;
  const int tiles_m = p.tiles_w * p.tiles_h * p.tiles_n;
  const int num_tiles = tiles_m * p.tiles_c;

  // ---- one-time setup -------------------------------------------------------------------------
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmOut);
    if (p.flags & CONV_RESIDUAL) tma_prefetch_desc(&tmRes);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&res_full[i], 1);
      mbar_init(&res_empty[i], 8);  // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < p.cout && i < 512; i += blockDim.x) {
    smem_scale[i] = p.scale ? p.scale[i] : 1.0f;
    smem_bias[i] = p.bias ? p.bias[i] : 0.0f;
  }
  __syncthreads();
  pdl_wait();  // everything above touched only parameters; activations of the previous kernel are read/written below

  // tile -> coordinates. Tile order: cout tile fastest so CTAs running concurrently share the A tile in L2.
  auto decode = [&](int tile, int& c0, int& w0, int& h0, int& n0) {
    int ct = tile % p.tiles_c;
    int mt = tile / p.tiles_c;
    int wt_i = mt % p.tiles_w;
    int r = mt / p.tiles_w;
    int ht_i = r % p.tiles_h;
    int nt_i = r / p.tiles_h;
    c0 = ct * N_TILE;
    w0 = wt_i * p.wt;
    h0 = ht_i * p.hb;
    n0 = nt_i * p.nb;
  };

  if (warp == 0) {
    // ===================== TMA producer (warp-converged loop, one elected lane issues) =====================
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int c0, w0, h0, n0;
      decode(tile, c0, w0, h0, n0);
      for (int ks = 0; ks < ksteps; ++ks) {
        const int tap = ks / p.cin_chunks;
        const int ch = ks - tap * p.cin_chunks;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
          tma_load_5d(smem_a + stage * kATileBytes, &tmA, &full_bar[stage], p.tap_c[tap] + ch * kKStep,
                      w0 + p.tap_dw[tap], p.tap_ph[tap], h0 + p.tap_dh[tap], n0);
          tma_load_3d(smem_b + stage * S::kBTileBytes, &tmB, &full_bar[stage], ch * kKStep, c0, p.tap_w[tap]);
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp == 3) {
    // ===================== residual prefetcher: one 128 x 64 tile per output chunk, two buffers =====================
    if (!OUT_F32 && (p.flags & CONV_RESIDUAL)) {
      int rb = 0;
      uint32_t rph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int c0, w0, h0, n0;
        decode(tile, c0, w0, h0, n0);
        for (int j = 0; j < kChunks; ++j) {
          mbar_wait(&res_empty[rb], rph ^ 1);
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&res_full[rb], kATileBytes);
            tma_load_5d(smem_res + rb * kATileBytes, &tmRes, &res_full[rb], p.out_c_base + c0 + j * 64, w0, p.out_ph, h0, n0);
          }
          __syncwarp();
          if (++rb == 2) {
            rb = 0;
            rph ^= 1;
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup cg = rows [64*cg, 64*cg+64) of every tile: MMA, then epilogue ==========
    const int cg = (warp >> 2) - 1;
    const int etid = threadIdx.x - 128;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const bool has_res = (p.flags & CONV_RESIDUAL) != 0;
    const bool do_clip = (p.flags & CONV_CLIP) != 0;
    const int fr = 64 * cg + frag_row();
    const int fc = frag_col();
    float acc[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.0f;
    int stage = 0;
    uint32_t phase = 0;
    int rb = 0;
    uint32_t rph = 0;
    int buf = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int c0, w0, h0, n0;
      decode(tile, c0, w0, h0, n0);
      int prev = -1;
      for (int ks = 0; ks < ksteps; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = gmma_desc_sw128(smem_u32(smem_a + stage * kATileBytes)) + cg * kDescRows64;
        const uint64_t db = gmma_desc_sw128(smem_u32(smem_b + stage * S::kBTileBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kKStep / 16; ++k)
          // advancing 16 elements (32 B) along K inside the swizzle atom = +2 in the (addr>>4) field
          wgmma_f16<N_TILE, BF16>(acc, da + 2 * k, db + 2 * k, (ks > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous K-step's MMAs are done: its stage goes back to the producer
        if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue: both warpgroups fill one 128-row staging tile per 64-channel chunk, one thread TMA-stores it
#pragma unroll
      for (int j = 0; j < kChunks; ++j) {
        const float* sc = smem_scale + c0 + j * 64;
        const float* bi = smem_bias + c0 + j * 64;
        if constexpr (OUT_F32) {
          // fp32 output: columns 0-31 / 32-63 of the chunk fill one 128-row x 32-float staging buffer each
          if (etid == 0) tma_store_wait_read<0>();
          named_bar_sync(1, 256);
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = fr + 8 * h, col = 8 * i + fc;
              const float v0 = fmaf(acc[(8 * j + i) * 4 + 2 * h], sc[col], bi[col]);
              const float v1 = fmaf(acc[(8 * j + i) * 4 + 2 * h + 1], sc[col + 1], bi[col + 1]);
              *reinterpret_cast<float2*>(smem_stg + (col >> 5) * kATileBytes + sw128_off32(row, col & 31)) =
                  make_float2(v0, v1);
            }
          fence_proxy_async_smem();
          named_bar_sync(1, 256);
          if (etid == 0) {
            tma_store_5d(&tmOut, smem_stg, p.out_c_base + c0 + j * 64, w0, p.out_ph, h0, n0);
            tma_store_5d(&tmOut, smem_stg + kATileBytes, p.out_c_base + c0 + j * 64 + 32, w0, p.out_ph, h0, n0);
            tma_store_commit();
          }
        } else {
          uint8_t* stg = smem_stg + buf * kATileBytes;
          // staging buffer `buf` was last used two chunks ago: its TMA store must have finished reading smem
          if (etid == 0) tma_store_wait_read<1>();
          named_bar_sync(1, 256);
          if (has_res) mbar_wait(&res_full[rb], rph);
          const uint8_t* res = smem_res + rb * kATileBytes;
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = fr + 8 * h, col = 8 * i + fc;
              const uint32_t off = sw128_off16(row, col);
              float f0 = fmaf(acc[(8 * j + i) * 4 + 2 * h], sc[col], bi[col]);
              float f1 = fmaf(acc[(8 * j + i) * 4 + 2 * h + 1], sc[col + 1], bi[col + 1]);
              if (has_res) {
                const float2 t = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(res + off));
                f0 += t.x;
                f1 += t.y;
              }
              if (do_clip) {
                f0 = fminf(fmaxf(f0, 0.0f), p.clip_hi);
                f1 = fminf(fmaxf(f1, 0.0f), p.clip_hi);
              }
              *reinterpret_cast<uint32_t*>(stg + off) = pack2<BF16>(f0, f1);
            }
          fence_proxy_async_smem();
          if (has_res) {  // residual buffer consumed: hand it back to the prefetcher
            __syncwarp();
            if (lane == 0) mbar_arrive(&res_empty[rb]);
            if (++rb == 2) {
              rb = 0;
              rph ^= 1;
            }
          }
          named_bar_sync(1, 256);
          if (etid == 0) {
            tma_store_5d(&tmOut, stg, p.out_c_base + c0 + j * 64, w0, p.out_ph, h0, n0);
            tma_store_commit();
          }
          buf ^= 1;
        }
      }
    }
    if (etid == 0) tma_store_wait_all<0>();
  }
}

}  // namespace dsk
