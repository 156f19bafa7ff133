// Weight-gradient GEMM on the Hopper tensor cores (wgmma, sm_90a).
//
// Replaces cuDNN's convolution-backward-filter reached by autograd for every nn.Conv2d of the
// ResCNN (reference model.py:58,61,98,102,106; backward triggered at train_triplet.py:223).
//
//   dW[tap][co][ci] = sum over pixels  G[pix][co] * X[pix shifted by tap][ci]
//
// The reduction index is the pixel, and both tensors are NHWC (channels contiguous), so both operands are
// "MN-major" for the tensor core: a TMA box of 128 pixels x 64 channels lands in shared memory as 128 rows of
// 128 bytes (SWIZZLE_128B) and is consumed as one 64-wide operand atom (descriptor: leading byte offset = atom
// stride, stride byte offset = 1024 B between 8-pixel groups; wgmma's transpose flags mark both operands MN-major).
// Two consumer warpgroups each own one 64-row atom of the 128-row A tile and keep their accumulators in registers.  The tap shift and the zero padding
// are TMA coordinates on the outer (w, h) dims exactly as in the forward conv, so no transposed copies exist.
//
// Work item = (tap, 128 output channels, N_TILE input channels, K split).  Every K split writes its partial tile with
// plain stores into its OWN slice dw[ks][tap][cout][cin]; unpack_wgrad_kernel then adds the slices in fixed order, so
// the weight gradient is bit-reproducible from run to run (no atomics, no pre-zeroing).  Layers with 64 output
// channels use the swapped form (M = two taps x 64 input channels, N = 64 output channels) so that the MMA still
// has M = 128 (one tap per consumer warpgroup).
#pragma once
#include "conv_umma.cuh"

namespace dsk {

constexpr int kAtomBytes = 128 * 128;  // 128 pixels x 64 channels x 2 B

struct WgradParams {
  int swapped;              // 0: A = G (2 atoms of 64 co), B = X;  1: A = X for two taps, B = G (cout == 64)
  int taps, co_tiles, ci_tiles, ksplit;
  int cout, cin;
  int chunks_w, chunks_h, chunks_n;  // K-chunk grid; chunk = pixel box {wt, hb, nb} of 128 pixels
  int wt, hb, nb;
  int16_t tap_c[kMaxTaps];  // X view: channel offset (parity column), w/h offsets, parity row
  int8_t tap_dw[kMaxTaps];
  int8_t tap_ph[kMaxTaps];
  int8_t tap_dh[kMaxTaps];
  float* dw;                // fp32 [ksplit][tap][cout][cin]: one slice per K split, every element written exactly once
  long slice_elems;         // taps * cout * cin
};

template <int N_TILE>
struct WgradSmem {
  static constexpr int kBAtoms = N_TILE / 64;
  static constexpr int kStageBytes = (2 + kBAtoms) * kAtomBytes;
  static constexpr int kStages = (N_TILE == 64) ? 4 : 3;
  static constexpr int kTotal = kStages * kStageBytes + 256 + 1024;
};
constexpr int kWgradThreads = 384;  // warp 0: TMA producer; warpgroups 1, 2: consumers (MMA + epilogue)

// MN-major SWIZZLE_128B operand descriptor (see header comment)
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(kAtomBytes >> 4) << 16;  // leading byte offset: next 64-channel atom
  d |= static_cast<uint64_t>(1024 >> 4) << 32;        // stride byte offset: next group of 8 pixel rows
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

template <int N_TILE, bool BF16>
__global__ void __launch_bounds__(kWgradThreads, 1)
wgrad_umma_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX,
                  const WgradParams p) {
  using S = WgradSmem<N_TILE>;
  constexpr int kStages = S::kStages;
  constexpr int kBAtoms = S::kBAtoms;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_chunks = p.chunks_w * p.chunks_h * p.chunks_n;
  const int tap_units = p.swapped ? (p.taps + 1) / 2 : p.taps;
  const int num_items = tap_units * p.co_tiles * p.ci_tiles * p.ksplit;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmG);
    tma_prefetch_desc(&tmX);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  // item -> (tap unit, co tile, ci tile, K range); K split fastest
  auto decode = [&](int item, int& tu, int& co0, int& ci0, int& k_begin, int& k_end) -> int {
    const int ks = item % p.ksplit;
    int r = item / p.ksplit;
    const int cit = r % p.ci_tiles;
    r /= p.ci_tiles;
    const int cot = r % p.co_tiles;
    tu = r / p.co_tiles;
    co0 = cot * kTileM;
    ci0 = cit * N_TILE;
    const int per = (total_chunks + p.ksplit - 1) / p.ksplit;
    k_begin = ks * per;
    k_end = k_begin + per < total_chunks ? k_begin + per : total_chunks;
    return ks;
  };

  if (warp == 0) {
    // TMA producer: warp-converged loop, one elected lane issues
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int tu, co0, ci0, kb, ke;
      decode(item, tu, co0, ci0, kb, ke);
      for (int k = kb; k < ke; ++k) {
        const int cw = k % p.chunks_w;
        const int r = k / p.chunks_w;
        const int chh = r % p.chunks_h;
        const int cn = r / p.chunks_h;
        const int w0 = cw * p.wt, h0 = chh * p.hb, n0 = cn * p.nb;
        uint8_t* sa = smem + stage * S::kStageBytes;
        uint8_t* sb = sa + 2 * kAtomBytes;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
          if (!p.swapped) {
            tma_load_5d(sa, &tmG, &full_bar[stage], co0, w0, 0, h0, n0);
            tma_load_5d(sa + kAtomBytes, &tmG, &full_bar[stage], co0 + 64, w0, 0, h0, n0);
#pragma unroll
            for (int j = 0; j < kBAtoms; ++j)
              tma_load_5d(sb + j * kAtomBytes, &tmX, &full_bar[stage], p.tap_c[tu] + ci0 + 64 * j, w0 + p.tap_dw[tu],
                          p.tap_ph[tu], h0 + p.tap_dh[tu], n0);
          } else {
            const int t0 = 2 * tu, t1 = (2 * tu + 1 < p.taps) ? 2 * tu + 1 : 2 * tu;
            tma_load_5d(sa, &tmX, &full_bar[stage], p.tap_c[t0], w0 + p.tap_dw[t0], p.tap_ph[t0], h0 + p.tap_dh[t0], n0);
            tma_load_5d(sa + kAtomBytes, &tmX, &full_bar[stage], p.tap_c[t1], w0 + p.tap_dw[t1], p.tap_ph[t1],
                        h0 + p.tap_dh[t1], n0);
            tma_load_5d(sb, &tmG, &full_bar[stage], 0, w0, 0, h0, n0);
          }
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    // consumers: warpgroup cg multiplies A atom cg (64 rows of the 128) by the whole B tile, then stores its rows
    const int cg = (warp >> 2) - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int fr = frag_row();  // row within this warpgroup's 64 (+ 8 for the odd register pairs)
    const int fc = frag_col();
    float acc[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.0f;
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int tu, co0, ci0, kb, ke;
      const int ks = decode(item, tu, co0, ci0, kb, ke);
      int prev = -1;
      for (int k = kb; k < ke; ++k) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = gmma_desc_mn_sw128(smem_u32(smem + stage * S::kStageBytes + cg * kAtomBytes));
        const uint64_t db = gmma_desc_mn_sw128(smem_u32(smem + stage * S::kStageBytes + 2 * kAtomBytes));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)  // 128 pixels = 8 x K16; one K16 step = 16 rows x 128 B = +128 in the addr field
          wgmma_f16<N_TILE, BF16, 1, 1>(acc, da + 128 * kk, db + 128 * kk, (k > kb || kk > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
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
      // destination of D[row][col] inside this K split's slice; an empty K range (split rounding) stores zeros
      float* dst = p.dw + static_cast<long>(ks) * p.slice_elems;
      const bool empty = ke <= kb;
      if (!p.swapped) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = co0 + 64 * cg + fr + 8 * h;
          if (co < p.cout) {
            float* drow = dst + (static_cast<long>(tu) * p.cout + co) * p.cin + ci0 + fc;
#pragma unroll
            for (int i = 0; i < N_TILE / 8; ++i)
              *reinterpret_cast<float2*>(drow + 8 * i) =
                  empty ? make_float2(0.f, 0.f) : make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
          }
        }
      } else {
        const int tap = 2 * tu + cg;  // [tap][co = col][ci = row % 64]
        if (tap < p.taps) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float* dcol = dst + static_cast<long>(tap) * p.cout * p.cin + fr + 8 * h;
#pragma unroll
            for (int i = 0; i < N_TILE / 8; ++i) {
              dcol[static_cast<long>(8 * i + fc) * p.cin] = empty ? 0.f : acc[4 * i + 2 * h];
              dcol[static_cast<long>(8 * i + fc + 1) * p.cin] = empty ? 0.f : acc[4 * i + 2 * h + 1];
            }
          }
        }
      }
    }
  }
}

}  // namespace dsk
