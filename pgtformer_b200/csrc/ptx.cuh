// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
// Everything here is device-only and header-only.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>

#include <type_traits>

namespace pgt {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Non-blocking probe (no suspend): for issuers that poll several barriers.
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped launch (error code), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA stores (shared -> global, bulk async-group completion); out-of-bounds parts of the box are clipped.
// L2 prefetch of a tensor-map box (no smem, no barrier): issued a few tiles ahead so the later smem load is an L2 hit
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* m, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(m), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(m), "r"(c0), "r"(c1), "r"(c2),
               "r"(c3)
               : "memory");
}

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// A warpgroup (four consecutive warps 4k..4k+3) issues D[64 x N] (+)= A[64 x 16] * B[N x 16]^T with both operands read
// from shared memory through matrix descriptors and the fp32 accumulator D in registers: d[4j + e] of warp w, lane l
// holds row 16w + l/4 + 8 (e >> 1), column 8j + 2 (l % 4) + (e & 1).

// K-major, 128-byte-swizzled operand: rows of 128 B as TMA SWIZZLE_128B writes them, 8-row groups `sbo` bytes apart
// (1024 for a dense tile); LBO is unused for this layout.  Advancing the start address by 32 B steps K by 16.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t saddr, uint32_t sbo = 1024) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);          // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                        // leading byte offset (unused)
  d |= static_cast<uint64_t>((sbo >> 4) & 0x3FFF) << 32;      // stride byte offset [32,46)
  d |= static_cast<uint64_t>(1) << 62;                        // layout type SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// accumulator operand lists of the wrappers below: "+f"(d[i]) .. "+f"(d[i + n - 1])
#define PGT_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define PGT_D8(i) PGT_D4(i), PGT_D4(i + 4)
#define PGT_D24(i) PGT_D8(i), PGT_D8(i + 8), PGT_D8(i + 16)
#define PGT_D32(i) PGT_D8(i), PGT_D8(i + 8), PGT_D8(i + 16), PGT_D8(i + 24)
#define PGT_D64(i) PGT_D32(i), PGT_D32(i + 32)
#define PGT_D128(i) PGT_D64(i), PGT_D64(i + 64)
// m64nNk16, bf16 x bf16 -> fp32, both operands K-major from shared memory; acc == 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : PGT_D8(0)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_m64n48k16(float (&d)[24], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
      : PGT_D24(0)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : PGT_D32(0)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : PGT_D64(0)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : PGT_D128(0)
      : "l"(da), "l"(db), "r"(acc));
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (N == 16) wgmma_m64n16k16(d, da, db, acc);
  else if constexpr (N == 48) wgmma_m64n48k16(d, da, db, acc);
  else if constexpr (N == 64) wgmma_m64n64k16(d, da, db, acc);
  else if constexpr (N == 128) wgmma_m64n128k16(d, da, db, acc);
  else { static_assert(N == 256, "wgmma N"); wgmma_m64n256k16(d, da, db, acc); }
}

// m64n64k16 with A from registers and B MN-major (transposed) from shared memory.  a[0..3] = bf16 pairs (row g, k 2t..),
// (row g + 8, k 2t..), (row g, k 2t + 8..), (row g + 8, k 2t + 8..) with g = lane / 4, t = lane % 4 inside the warp's
// 16 rows — the layout of columns [16 i, 16 i + 16) of an fp32 accumulator fragment, so a softmax result feeds the next
// MMA without shared memory.
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : PGT_D32(0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}

// MN-major SW128 operand (rows = K, 64 MN-contiguous elements per 128-byte row; 8-row groups 1024 B apart): the B view
// of a row-major [keys x d] tile such as V.
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;                        // LBO: next 64-element atom along MN (unused: N <= 64)
  d |= static_cast<uint64_t>((1024 >> 4) & 0x3FFF) << 32;     // SBO: next 8 rows along K
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Columns [C0, C0 + C) of a warpgroup's m64 accumulator -> fp32 rows of `scratch` (pitch `ld` floats, column C0 stored
// at column 0, fragment row i at scratch row i).  The usual second half of a row-per-thread epilogue: after a barrier
// over the warpgroups that share the scratch, thread t reads row t.
template <int C0, int C, int R>
__device__ __forceinline__ void acc_to_smem(const float (&d)[R], float* scratch, int ld, int warp_in_wg, int lane) {
  static_assert(C0 % 8 == 0 && C % 8 == 0 && C0 + C <= 2 * R, "whole 8-column fragments inside D");
  const int row = 16 * warp_in_wg + (lane >> 2);
  float* p0 = scratch + row * ld + 2 * (lane & 3);
  float* p1 = p0 + 8 * ld;
#pragma unroll
  for (int j = 0; j < C / 8; ++j) {
    constexpr int f0 = C0 / 8;
    const int f = f0 + j;
    *reinterpret_cast<float2*>(p0 + 8 * j) = make_float2(d[4 * f + 0], d[4 * f + 1]);
    *reinterpret_cast<float2*>(p1 + 8 * j) = make_float2(d[4 * f + 2], d[4 * f + 3]);
  }
}

// compile-time loop (accumulator registers are only addressable with constant indices)
template <int I, int N, typename F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}

// 32 consecutive fp32 of one scratch row -> registers (the shape the epilogues consume)
__device__ __forceinline__ void smem_row_32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = reinterpret_cast<const float4*>(src)[q];
    v[4 * q + 0] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
    v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
  }
}

}  // namespace pgt
