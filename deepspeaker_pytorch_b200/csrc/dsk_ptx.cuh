// sm_90a PTX wrappers used by the ResCNN kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma and its shared-memory
// descriptor encoding.
// Everything here is inline PTX; no CUTLASS/CuTe types.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace dsk {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of a fully converged warp.  TMA issue code sits under this predicate (not under `lane == 0`): ptxas then
// knows a single thread executes it and keeps descriptors in uniform registers.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  uint32_t laneid = 0;
  asm volatile(
      "{\n\t"
      ".reg .b32 %%rx;\n\t"
      ".reg .pred %%px;\n\t"
      "elect.sync %%rx|%%px, %2;\n\t"
      "@%%px mov.s32 %1, 1;\n\t"
      "mov.s32 %0, %%rx;\n\t"
      "}"
      : "+r"(laneid), "+r"(pred)
      : "r"(0xFFFFFFFF));
  return pred != 0;
}

// Programmatic dependent launch: every kernel of the forward chain lets its successor start launching at once and
// waits for its predecessor's memory only right before it first touches activations, so launch latency and the
// prologue (barrier init, scale/bias fetch) overlap the predecessor's tail.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2,
                                             int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2,
                                             int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): a warpgroup (4 consecutive warps, warp index % 4 == 0 first) multiplies a 64-row A slice by
// an N-column B tile from shared memory; the fp32 accumulator stays in the warpgroup's registers.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A * B, m64nNk16, fp16 or bf16 operands, fp32 accumulate.  TA / TB = 1: that operand is MN-major (transposed).
// Accumulator fragment: thread (warp w of the warpgroup, lane l) holds rows 16*(w%4) + l/4 and that + 8 of the 64; for
// each 8-column block i, d[4i], d[4i+1] = (row, 8i + 2*(l%4) + {0,1}) and d[4i+2], d[4i+3] = the same columns of row + 8.
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BF16) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
          "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
          "%32, %33, p, 1, 1, %35, %36;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
          : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  } else {
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
          "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
          "%32, %33, p, 1, 1, %35, %36;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
          : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
}

template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BF16) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
          "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
          "%64, %65, p, 1, 1, %67, %68;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
          : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  } else {
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
          "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
          "%64, %65, p, 1, 1, %67, %68;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
          : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
}

template <int N, bool BF16, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(N == 64 || N == 128, "wgmma N tile");
  if constexpr (N == 64) wgmma_m64n64<BF16, TA, TB>(d, da, db, scale_d);
  else wgmma_m64n128<BF16, TA, TB>(d, da, db, scale_d);
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptors
// ----------------------------------------------------------------------------------------------
// K-major operand tile stored as rows of 128 bytes (64 x 16-bit elements) with the 128-byte swizzle TMA writes
// (CU_TENSOR_MAP_SWIZZLE_128B; the tile base is 1024-byte aligned and the swizzle follows the address bits):
//   bits [0,14)  start address >> 4
//   bits [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1)
//   bits [32,46) stride byte offset >> 4 = distance between 8-row groups = 1024 B
//   bits [62,64) layout type: 1 = SWIZZLE_128B
// Advancing the start by 32 B moves 16 elements along K; by 128 B one row, by 8192 B 64 rows.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// The start-address field is in 16-byte units: descriptor offsets for one row / 64 rows of a K-major tile.
constexpr uint64_t kDescRow = 128 >> 4;
constexpr uint64_t kDescRows64 = 64 * kDescRow;

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------------------
// 16-bit operand helpers (fp16 or bf16 chosen at compile time)
// ----------------------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (BF16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}
// NaN-propagating fp32 max / min (max.NaN / min.NaN, FMNMX.NAN): NaN when either operand is NaN, as torch.clamp,
// Hardtanh and numpy.maximum give, where fmaxf / fminf return the other operand.  Otherwise the bits of fmaxf / fminf.
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float fmin_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// clamp(x, 0, hi), NaN in -> NaN out (the reference's Hardtanh(0, 20))
__device__ __forceinline__ float relu_clip(float x, float hi) { return fmin_nan(fmax_nan(x, 0.0f), hi); }
// clamp both 16-bit halves of a packed pair to [lo, hi] (lo / hi packed the same way).  Identical to clamping in fp32
// before the pack when lo and hi are exactly representable: rounding is monotonic, and like relu_clip the packed
// NaN-propagating min / max keep a NaN half NaN.
template <bool BF16>
__device__ __forceinline__ uint32_t clip2(uint32_t v, uint32_t lo, uint32_t hi) {
  if constexpr (BF16) {
    __nv_bfloat162 x = *reinterpret_cast<__nv_bfloat162*>(&v);
    x = __hmin2_nan(__hmax2_nan(x, *reinterpret_cast<__nv_bfloat162*>(&lo)), *reinterpret_cast<__nv_bfloat162*>(&hi));
    return *reinterpret_cast<uint32_t*>(&x);
  } else {
    __half2 x = *reinterpret_cast<__half2*>(&v);
    x = __hmin2_nan(__hmax2_nan(x, *reinterpret_cast<__half2*>(&lo)), *reinterpret_cast<__half2*>(&hi));
    return *reinterpret_cast<uint32_t*>(&x);
  }
}
// 16-byte shared-memory accesses through 32-bit shared-window addresses (no generic-address translation)
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

template <bool BF16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
  if constexpr (BF16) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
  } else {
    __half2 v = *reinterpret_cast<__half2*>(&u);
    return __half22float2(v);
  }
}
template <bool BF16>
__device__ __forceinline__ uint16_t to16(float a) {
  if constexpr (BF16) {
    __nv_bfloat16 v = __float2bfloat16_rn(a);
    return *reinterpret_cast<uint16_t*>(&v);
  } else {
    __half v = __float2half_rn(a);
    return *reinterpret_cast<uint16_t*>(&v);
  }
}
template <bool BF16>
__device__ __forceinline__ float from16(uint16_t u) {
  if constexpr (BF16) {
    return __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&u));
  } else {
    return __half2float(*reinterpret_cast<__half*>(&u));
  }
}

}  // namespace dsk
