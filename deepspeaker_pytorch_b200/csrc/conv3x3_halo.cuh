// 3x3 stride-1 convolution on the Hopper tensor cores (wgmma) with halo-tile reuse (sm_90a) — the eval-forward kernel for
// the eight BasicBlock convs (reference model.py:47-50,58,61 used at :69,73), with the folded BatchNorm
// affine (:59,62), the residual add (:79) and the clipped ReLU (:36-39) in the epilogue.
//
// Why a second conv kernel: the generic kernel issues one 16 KB A box per tap, so every input pixel crosses L2 -> shared
// memory nine times.  Here:
//   * activations live in a ZERO-PADDED NHWC layout: rows R = n*(H+1)+h+1 (row 0 and the row after every image are
//     zero), W+1 pixels per row (column 0 is zero), so position Q = R*(W+1) + w+1 and the 3x3 neighbourhood of Q is
//     Q + (r-1)*(W+1) + (s-1) for every pixel, including image borders (the pads are real zeros in memory);
//   * an output tile is 128 CONSECUTIVE padded positions; its A operand for one 64-channel
//     chunk is ONE contiguous TMA box of tile + 2W + 4 rows (the halo), and every filter tap reads it through a wgmma descriptor whose start
//     address is shifted by (r*(W+1)+s) rows (row-shifted SWIZZLE_128B descriptors: the swizzle follows the address);
//   * weights arrive as one box per filter row (3 taps x N_TILE x 64 ch); with 64 channels all 9 taps stay resident;
//   * junk outputs (pad positions, 1/(W+1) + 1/(H+1) of the rows) are written as zeros, which keeps the pads zero.
#pragma once
#include "conv_umma.cuh"

namespace dsk {

// The same kernel runs the 5x5 stride-2 stage-entry convs (model.py:98,102,106): their input is stored PARITY-PLANAR
// (four planes (h&1, w&1), each a zero-padded grid at the OUTPUT resolution), so that every tap (r, s) reads plane
// (r&1, s&1) at a fixed shift ((r-2)>>1, (s-2)>>1) of the output position: one halo box per (64-channel chunk, plane)
// serves all taps of that plane.  The weight BOXES (<= 3 taps each, packed consecutively in plane-major tap order) are
// listed in a table the producer walks; the consumers run the same sequence from a compile-time plan (HaloPlan).
constexpr int kHaloMaxBoxes = 9;  // 5x5 s2: 3 + 2 + 2 + 2 three-tap boxes
constexpr int kHaloMaxStages = 4;

struct HaloParams {
  int W, H, N;            // OUTPUT image geometry (real pixels); tiles run over its padded position space
  int q_begin;            // first position of tile 0 (= W+1: first real row)
  int tiles_m, tiles_c;   // HaloSmem::kTileRows-position tiles, N_TILE channel tiles
  int chunks;             // Cin / 64
  int cout;
  // shared-memory carve (runtime): ring depths and buffer counts chosen by the host per layer
  int a_stage_bytes;      // halo tile rows * 128 rounded up to 1024
  int a_stages, b_stages; // <= kHaloMaxStages
  int stg_bufs;           // output staging buffers (1 or 2)
  // K-loop table (per 64-channel chunk)
  int nboxes;
  int plane_positions;                     // positions per input plane (parity-planar input), 0 for a single plane
  int8_t box_plane[kHaloMaxBoxes];         // input plane of the box's taps
  int8_t box_first[kHaloMaxBoxes];         // first box of its plane group: load the plane's halo tile
  int16_t box_wtap[kHaloMaxBoxes];         // first packed tap index of the box
  // output: standard padded layout (TMA store) or parity-planar (3x3 only; staged, then copied out in 128-byte rows;
  // feeds a stride-2 conv)
  int out_planar;
  uint16_t* out_ptr;                       // planar destination base
  int out_plane_positions;                 // positions per output plane
  int out_C;
  int flags;              // CONV_RESIDUAL | CONV_CLIP
  float clip_hi;
  // folded eval-BN affine of the layer's output channels, carried in the kernel parameters: the epilogue reads it
  // through the constant cache (warp-uniform addresses) instead of spending shared-memory bandwidth, which is the
  // resource the MMA operand fetch already saturates
  float scale_c[512];
  float bias_c[512];
  int b_resident;         // all weight boxes of a CTA's channel tile fit the B ring: load once
  // floor(2^64/d)+1 for d = W+1 and H+1: q/d == __umul64hi(q, magic) for every q < 2^32 (the error of the rounded-up
  // reciprocal, q (magic d - 2^64) / (d 2^64) < q / 2^64, stays below 1/d).  A 32-bit reciprocal is exact only for
  // q < 2^32/d, which the image index R / (H+1) of a long batch of long utterances passes.
  unsigned long long pitch_magic, img_magic;
  const uint16_t* res_ptr;  // residual tensor (padded layout, cout channels per position): read straight from global / L2
};

// Compile-time K-loop plans for the MMA issuer (the producer still walks the runtime tables, which say the same).
// KIND 1: 3x3, one plane, boxes = filter rows.  KIND 2: planar 5x5 s2, packed tap n = 3*box + t, planes start at
// packed taps 0 / 9 / 15 / 21 and have 3x3, 3x2, 2x3, 2x2 taps; tap (i, j) of a plane reads halo row i*(W+1) + j.
template <int KIND>
struct HaloPlan {
  static constexpr int TPB = 3;  // taps per weight box
  static constexpr int kTaps = KIND == 1 ? 9 : 25;
  static constexpr int kBoxes = (kTaps + TPB - 1) / TPB;  // plane starts 0/9/15/21 are multiples of 3: boxes never straddle planes
  __host__ __device__ static constexpr int plane_of(int n) { return KIND == 1 ? 0 : (n < 9 ? 0 : n < 15 ? 1 : n < 21 ? 2 : 3); }
  __host__ __device__ static constexpr int plane_start(int pl) { return pl == 0 ? 0 : pl == 1 ? 9 : pl == 2 ? 15 : 21; }
  __host__ __device__ static constexpr int plane_end(int pl) { return KIND == 1 ? 9 : (pl == 0 ? 9 : pl == 1 ? 15 : pl == 2 ? 21 : 25); }
  __host__ __device__ static constexpr int cols(int pl) { return (KIND == 2 && (pl & 1)) ? 2 : 3; }
  __host__ __device__ static constexpr int ntaps(int b) { return kTaps - TPB * b < TPB ? kTaps - TPB * b : TPB; }
  __host__ __device__ static constexpr bool first(int b) { return TPB * b == plane_start(plane_of(TPB * b)); }
  __host__ __device__ static constexpr bool last(int b) { return TPB * b + ntaps(b) == plane_end(plane_of(TPB * b)); }
  __host__ __device__ static constexpr int row_i(int b, int t) {
    return (TPB * b + t - plane_start(plane_of(TPB * b + t))) / cols(plane_of(TPB * b + t));
  }
  __host__ __device__ static constexpr int col_j(int b, int t) {
    return (TPB * b + t - plane_start(plane_of(TPB * b + t))) % cols(plane_of(TPB * b + t));
  }
};

// One CTA per SM: 384 threads, up to 227 KB of shared memory; each of the two consumer warpgroups computes one 64-row
// slice of a tile and holds its 64 x N_TILE fp32 accumulators in registers.
template <int N_TILE>
struct HaloSmem {
  static constexpr int kTileRows = 128;  // positions per tile: 64 per consumer warpgroup
  static constexpr int kBStageBytes = 3 * N_TILE * 128;  // weight box: 3 taps (48 KB at 128 channels)
  static constexpr int kFixedBytes = 512 + 1024;  // barriers + alignment slack
};

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}

// tmIn : 2-D (C, positions) view of the padded input, box {64, kTileRows + 2W + 4}
// tmW  : 3-D (cin, cout, 9 taps) packed weights, box {64, N_TILE, 3}
// tmOut : 2-D (C, positions) view of the padded output, box {64, kTileRows}   (the residual is read from global memory
//         through HaloParams::res_ptr)
constexpr int kHaloThreads = 384;  // one control warpgroup + two consumer warpgroups

// KIND: the compile-time tap plan the consumers run - 1 = 3x3 (HaloPlan<1>), 2 = parity-planar 5x5 s2 (HaloPlan<2>).
// One plan per instantiation (and the resident-weights burst only where it can occur, 64-channel 3x3): each
// instantiation carries only what it runs.
template <int N_TILE, bool BF16, int KIND>
__global__ void __launch_bounds__(kHaloThreads, 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmW,
                    const __grid_constant__ CUtensorMap tmOut, const HaloParams p) {
  using S = HaloSmem<N_TILE>;
  constexpr int kEpiThreads = 256;
  constexpr int kCG = 2;        // consumer warpgroups
  constexpr int kMW = 1;        // 64-row slices of the tile per consumer warpgroup
  constexpr int kTM = S::kTileRows;
  const int kAStages = p.a_stages, kBStages = p.b_stages;
  constexpr int kChunksOut = N_TILE / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + kAStages * p.a_stage_bytes;
  uint8_t* smem_stg = smem_b + kBStages * S::kBStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_stg + p.stg_bufs * kATileBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kHaloMaxStages;
  uint64_t* b_full = a_empty + kHaloMaxStages;
  uint64_t* b_empty = b_full + kHaloMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  const int pitch = p.W + 1;
  const int halo_rows = kTM + 2 * p.W + 4;
  const int num_tiles = p.tiles_m * p.tiles_c;

  // channel tile slowest: a CTA's consecutive tiles (stride gridDim.x) mostly share the weight tile
  auto decode = [&](int tile, int& c0, int& q0) {
    const int ct = tile / p.tiles_m;
    const int mt = tile - ct * p.tiles_m;
    c0 = ct * N_TILE;
    q0 = p.q_begin + mt * kTM;
  };
  // a CTA's tiles: blockIdx.x, blockIdx.x + gridDim.x, ...; each runs units (weight box b of chunk ch) 0 .. units-1
  const int units = p.chunks * p.nboxes;

  // Prologue, split over two warps so that the two first-use descriptor fetches overlap: warp 0 sets up the weight ring
  // and issues the first weight boxes (parameters: no dependency wait), warp 3 sets up the halo ring and issues the first
  // halo tile right after the dependency wait.
  int pre_b = 0;  // weight boxes of the first tile already issued (producer warp only)
  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&tmW);
      for (int i = 0; i < kBStages; ++i) {
        mbar_init(&b_full[i], 1);
        mbar_init(&b_empty[i], kCG);  // one arrive per consumer warpgroup
      }
      fence_barrier_init();
    }
    __syncwarp();
    if (static_cast<int>(blockIdx.x) < num_tiles) {
      int c0, q0;
      decode(blockIdx.x, c0, q0);
      pre_b = units < kBStages ? units : kBStages;
      if (elect_one_sync()) {
        for (int i = 0; i < pre_b; ++i) {
          const int ch = i / p.nboxes, b = i - ch * p.nboxes;
          mbar_arrive_expect_tx(&b_full[i], S::kBStageBytes);
          tma_load_3d(smem_b + i * S::kBStageBytes, &tmW, &b_full[i], ch * 64, c0, p.box_wtap[b]);
        }
      }
      __syncwarp();
    }
  }
  if (warp == 3) {
    if (lane == 0) {
      tma_prefetch_desc(&tmIn);
      for (int i = 0; i < kAStages; ++i) {
        mbar_init(&a_full[i], 1);
        mbar_init(&a_empty[i], kCG);
      }
      fence_barrier_init();
    }
    __syncwarp();
    if (static_cast<int>(blockIdx.x) < num_tiles) {
      int c0, q0;
      decode(blockIdx.x, c0, q0);
      pdl_wait();  // activations of the previous kernel are read below
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&a_full[0], halo_rows * 128);
        tma_load_2d(smem_a, &tmIn, &a_full[0], 0, p.box_plane[0] * p.plane_positions + q0 - (p.W + 2));
      }
      __syncwarp();
    }
  }
  if (warp == 1 && lane == 0) tma_prefetch_desc(&tmOut);
  __syncthreads();
  pdl_wait();  // everything above (but the producer's first halo tile) touched only parameters

  if (warp == 0) {
    // ===================== TMA producer (warp-converged loop, one elected lane issues) =====================
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    bool first = true;
    bool a_pre = true;  // the first halo tile was issued in the prologue
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int c0, q0;
      decode(tile, c0, q0);
      for (int u = 0; u < units; ++u) {
        const int ch = u / p.nboxes, b = u - ch * p.nboxes;
        if (p.box_first[b]) {  // a plane's halo tile: at its first box
          if (a_pre) {
            a_pre = false;
          } else {
            mbar_wait(&a_empty[as], aph ^ 1);
            if (elect_one_sync()) {
              mbar_arrive_expect_tx(&a_full[as], halo_rows * 128);
              tma_load_2d(smem_a + as * p.a_stage_bytes, &tmIn, &a_full[as], ch * 64,
                          p.box_plane[b] * p.plane_positions + q0 - (p.W + 2));
            }
            __syncwarp();
          }
          if (++as == kAStages) {
            as = 0;
            aph ^= 1;
          }
        }
        if (!p.b_resident || first) {
          if (pre_b > 0) {
            --pre_b;
          } else {
            mbar_wait(&b_empty[bs], bph ^ 1);
            if (elect_one_sync()) {
              mbar_arrive_expect_tx(&b_full[bs], S::kBStageBytes);
              tma_load_3d(smem_b + bs * S::kBStageBytes, &tmW, &b_full[bs], ch * 64, c0, p.box_wtap[b]);
            }
            __syncwarp();
          }
          if (++bs == kBStages) {
            bs = 0;
            bph ^= 1;
          }
        }
      }
      first = false;
    }
  } else if (warp >= 4) {
    // ===================== consumers: MMA of a tile, then its epilogue ======================================
    // Warpgroup cg computes the 64-row slices cg*kMW .. cg*kMW + kMW - 1 of every tile (thread rows: frag_row() + 8*h
    // of each slice).
    const int cg = (warp >> 2) - 1;
    const int etid = threadIdx.x - 128;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int fr = frag_row(), fc = frag_col();
    const bool has_res = (p.flags & CONV_RESIDUAL) != 0;
    const bool do_clip = (p.flags & CONV_CLIP) != 0;
    const int rows_real_end = p.N * (p.H + 1) + 1;  // first row index past the last image
    const uint32_t clip_hi2 = pack2<BF16>(p.clip_hi, p.clip_hi);
    float acc[kMW][N_TILE / 2];
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    bool first = true;
    int buf = 0;
    // stages read by the last committed weight box: handed back to the producer once a later wait shows it complete
    int pend_b = -1, pend_a = -1;
    auto release_pending = [&]() {
      if (wg_leader) {
        if (pend_b >= 0) mbar_arrive(&b_empty[pend_b]);
        if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
      }
      pend_b = pend_a = -1;
    };
    // all taps of one weight box on the halo tile at da0 (committed, not waited for): scale_d = 0 for the first K16 step
    // when `zero`
    auto mma_box = [&](uint64_t da0, uint64_t db0, int ntaps_, const int16_t* shifts, bool zero) {
      wgmma_fence();
#pragma unroll
      for (int m = 0; m < kMW; ++m) {
        const uint64_t dam = da0 + static_cast<uint64_t>(cg * kMW + m) * kDescRows64;
        for (int t = 0; t < ntaps_; ++t) {
          const uint64_t da = dam + static_cast<uint64_t>(shifts[t]) * kDescRow;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_f16<N_TILE, BF16>(acc[m], da + 2 * k, db0 + (t * (N_TILE * 8) + 2 * k), (t > 0 || k > 0 || !zero) ? 1u : 0u);
        }
      }
      wgmma_commit();
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int c0, q0;
      decode(tile, c0, q0);
      // ---------------- MMA over the units of this tile ----------------
      {
        constexpr bool kResident = N_TILE == 64 && KIND == 1;  // the only shape whose 9 taps fit the ring
        bool resident = false;
        if constexpr (kResident) resident = p.b_resident != 0;
        if (resident) {
          // 64-channel 3x3: all nine weight taps stay resident (three 3-tap boxes); one burst of 36 K16 steps per tile
          mbar_wait(&a_full[as], aph);
          if (first)
            for (int b = 0; b < 3; ++b) mbar_wait(&b_full[b], 0);
          const uint64_t da0 = gmma_desc_sw128(smem_u32(smem_a + as * p.a_stage_bytes));
          const uint64_t db0 = gmma_desc_sw128(smem_u32(smem_b));
          wgmma_fence();
#pragma unroll
          for (int m = 0; m < kMW; ++m) {
            const uint64_t dam = da0 + static_cast<uint64_t>(cg * kMW + m) * kDescRows64;
#pragma unroll
            for (int b = 0; b < 3; ++b)
#pragma unroll
              for (int t = 0; t < 3; ++t)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                  wgmma_f16<N_TILE, BF16>(acc[m], dam + static_cast<uint64_t>(b * pitch + t) * kDescRow + 2 * k,
                                          db0 + ((b * 3 + t) * (N_TILE * 8) + 2 * k), (b > 0 || t > 0 || k > 0) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          if (wg_leader) mbar_arrive(&a_empty[as]);
          if (++as == kAStages) {
            as = 0;
            aph ^= 1;
          }
        } else {
          using Plan = HaloPlan<KIND>;
          // unit u = box b of chunk ch.  The host's table has Plan::kBoxes boxes per chunk, so u < units holds for every
          // box; the per-box bound stays because without it ptxas gives the 64-channel forms some 20 more registers.
          for (int ch = 0; ch * Plan::kBoxes < units; ++ch) {
            uint64_t da0 = 0;
#pragma unroll
            for (int b = 0; b < Plan::kBoxes; ++b) {
              if (ch * Plan::kBoxes + b >= units) continue;
              if (Plan::first(b)) {
                mbar_wait(&a_full[as], aph);
                da0 = gmma_desc_sw128(smem_u32(smem_a + as * p.a_stage_bytes));
              }
              mbar_wait(&b_full[bs], bph);
              const bool rel_a = Plan::last(b);
              int16_t shifts[3];
#pragma unroll
              for (int t = 0; t < Plan::ntaps(b); ++t) shifts[t] = static_cast<int16_t>(Plan::row_i(b, t) * pitch + Plan::col_j(b, t));
              mma_box(da0, gmma_desc_sw128(smem_u32(smem_b + bs * S::kBStageBytes)), Plan::ntaps(b), shifts, ch == 0 && b == 0);
              wgmma_wait<1>();  // the previous box's MMAs are done: its stages go back to the producer
              release_pending();
              pend_b = bs;
              pend_a = rel_a ? as : -1;
              if (++bs == kBStages) {
                bs = 0;
                bph ^= 1;
              }
              if (rel_a) {
                if (++as == kAStages) {
                  as = 0;
                  aph ^= 1;
                }
              }
            }
          }
          wgmma_wait<0>();
          release_pending();
        }
        first = false;
#pragma unroll
        for (int m = 0; m < kMW; ++m) wgmma_fence_acc(acc[m]);
      }
      // ---------------- epilogue ----------------
      // this thread's rows: slice m, half h -> tile row (cg*kMW + m)*64 + fr + 8h; padded position q0 + row
      // padded position q0 + row: junk (a pad position) or, for a parity-planar output, its destination (nullptr = junk)
      auto is_junk = [&](int row, int& R, int& cc, int& img) -> bool {
        const int q = q0 + row;
        R = static_cast<int>(__umul64hi(static_cast<unsigned>(q), p.pitch_magic));
        cc = q - R * pitch;
        img = static_cast<int>(__umul64hi(static_cast<unsigned>(R), p.img_magic));
        return (cc == 0) || (R - img * (p.H + 1) == 0) || (R >= rows_real_end);
      };
      // parity-planar destination of a position (only when the consumer is a stride-2 conv): pixel (n, h, w) ->
      // plane (h&1, w&1), padded position of (n, h>>1, w>>1) on the half-resolution grid
      auto planar_dst = [&](int row) -> uint16_t* {
        int R, cc, img;
        if (is_junk(row, R, cc, img)) return nullptr;
        const int n = img;  // R = n*(H+1) + h + 1 with h < H  =>  img == n for real rows
        const int hh = R - 1 - n * (p.H + 1), ww = cc - 1;
        const int H2 = p.H >> 1, W2 = p.W >> 1;
        const long q2 = static_cast<long>(n * (H2 + 1) + (hh >> 1) + 1) * (W2 + 1) + (ww >> 1) + 1;
        const long plane = (hh & 1) * 2 + (ww & 1);
        return p.out_ptr + (plane * p.out_plane_positions + q2) * p.out_C + c0;
      };
      bool junk[kMW][2];
#pragma unroll
      for (int m = 0; m < kMW; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int R, cc, img;
          junk[m][h] = is_junk((cg * kMW + m) * 64 + fr + 8 * h, R, cc, img);
        }
      // A planar output is staged like the padded one and then copied out row by row: thread etid moves the 16-byte
      // pieces etid + i * kEpiThreads (row = piece / 8), so each warp writes four whole 128-byte rows.  (Stored straight
      // from the accumulator fragment, every warp store touched 8 positions with 16 bytes each.)
      // Only the 3x3 form writes a planar output (a block's last conv feeding the next stage's 5x5 s2 conv; the host
      // rejects it for the 5x5 form), so the 5x5 instantiations carry none of this code.
      const bool out_planar = KIND == 1 && p.out_planar;
      constexpr int kCopyIters = kTM * 8 / kEpiThreads;
      static_assert(kCopyIters * kEpiThreads == kTM * 8, "the copy-out covers the staging tile");
#pragma unroll
      for (int j = 0; j < kChunksOut; ++j) {
        uint8_t* stg = smem_stg + buf * kATileBytes;
        if (!out_planar) {
          // staging buffer `buf`: its previous TMA store (stg_bufs chunks ago) has finished reading it
          if (etid == 0) {
            if (p.stg_bufs == 2) tma_store_wait_read<1>();
            else tma_store_wait_read<0>();
          }
          named_bar_sync(1, kEpiThreads);
        } else if (p.stg_bufs == 1) {
          named_bar_sync(1, kEpiThreads);  // the previous chunk's copy-out has read the one staging buffer
        }
#pragma unroll
        for (int m = 0; m < kMW; ++m)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = (cg * kMW + m) * 64 + fr + 8 * h;
            const uint32_t* res = has_res ? reinterpret_cast<const uint32_t*>(p.res_ptr + static_cast<size_t>(q0 + row) * p.cout + c0 + j * 64) : nullptr;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int col = 8 * i + fc;  // within the 64-channel chunk
              const int cabs = c0 + j * 64 + col;
              float f0 = fmaf(acc[m][(8 * j + i) * 4 + 2 * h], p.scale_c[cabs], p.bias_c[cabs]);
              float f1 = fmaf(acc[m][(8 * j + i) * 4 + 2 * h + 1], p.scale_c[cabs + 1], p.bias_c[cabs + 1]);
              if (has_res) {
                const float2 t = unpack2<BF16>(__ldg(res + (col >> 1)));
                f0 += t.x;
                f1 += t.y;
              }
              uint32_t o = pack2<BF16>(f0, f1);
              if (do_clip) o = clip2<BF16>(o, 0u, clip_hi2);  // on the packed pair: same result as an fp32 clamp (0 and 20 are exact)
              if (junk[m][h]) o = 0u;                         // pad positions stay zero
              *reinterpret_cast<uint32_t*>(stg + sw128_off16(row, col)) = o;
            }
          }
        if (out_planar) {
          // with two staging buffers, the barrier after this chunk's writes also orders the copy-out of the chunk before
          // (same buffer as the next chunk) ahead of the next chunk's writes
          named_bar_sync(1, kEpiThreads);
          const uint32_t stg_s = smem_u32(stg);
#pragma unroll
          for (int i = 0; i < kCopyIters; ++i) {
            const int piece = i * kEpiThreads + etid;
            const int row = piece >> 3, k = piece & 7;
            uint16_t* dst = planar_dst(row);  // recomputed per chunk: a few integer ops, no registers held across the MMAs
            if (dst != nullptr) {
              const uint4 v = lds128(stg_s + row * 128 + (((k ^ row) & 7) << 4));
              *reinterpret_cast<uint4*>(dst + j * 64 + k * 8) = v;
            }
          }
          if (p.stg_bufs == 2) buf ^= 1;
        } else {
          fence_proxy_async_smem();
          named_bar_sync(1, kEpiThreads);
          if (etid == 0) {
            tma_store_2d(&tmOut, stg, c0 + j * 64, q0);
            tma_store_commit();
          }
          if (p.stg_bufs == 2) buf ^= 1;
        }
      }
    }
    if (etid == 0) tma_store_wait_all<0>();
  }
}

}  // namespace dsk
