// ptx.cuh -- thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the
// warpgroup MMA (wgmma.mma_async, uint8 -> int32).  No CUTLASS, no CuTe.
#pragma once
#include <cstdint>
#include <cuda.h>

namespace b2m {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
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

// ---- TMA ------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates (c0 = innermost/bytes-in-row, c1 = row).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ---- wgmma (Hopper warpgroup MMA) -------------------------------------------------------
// Shared-memory matrix descriptor for a K-major tile whose rows are exactly 128 bytes (= one SWIZZLE_128B
// atom, the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups are 1024 B apart (SBO), LBO
// unused (=1), layout type 1 (SWIZZLE_128B).  The tile base must be 1024-B aligned; a K step of 32 bytes
// is taken by adding 32 to the start address (+2 in the address >> 4 field).
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes & 0x3FFFF) >> 4);  // start address, bits [0,14)
  d |= static_cast<uint64_t>(1) << 16;                           // LBO (ignored for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                   // SBO = 1024 B
  d |= static_cast<uint64_t>(1) << 62;                           // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 128] (+)= A[64 x 32] * B[128 x 32]^T, uint8 x uint8 -> int32, both operands K-major in shared memory.
// Issued by all 128 threads of a warpgroup.  Thread t = 32 w + l holds rows 16 w + l / 4 (+ 8) and columns
// 8 j + 2 (l % 4) (+ 1): d[4 j + 2 i + e] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + e], j < 16.
__device__ __forceinline__ void wgmma_m64n128k32_u8(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// Keeps the compiler from moving accesses of the accumulators across the asynchronous MMA.
__device__ __forceinline__ void wgmma_fence_regs(uint32_t (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// One 64 x 128 tile over the full 128-byte descriptor: D = A[64 x 128] * B[128 x 128]^T, four k-steps, waited for.
// a_smem / b_smem: 1024-B aligned SWIZZLE_128B tiles (64 and 128 rows of 128 bytes).
__device__ __forceinline__ void wgmma_tile_u8(uint32_t (&d)[64], uint32_t a_smem, uint32_t b_smem) {
  const uint64_t adesc = make_wgmma_desc_sw128(a_smem), bdesc = make_wgmma_desc_sw128(b_smem);
  wgmma_fence_regs(d);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_m64n128k32_u8(d, adesc + 2 * k, bdesc + 2 * k, k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait_all();
  wgmma_fence_regs(d);
}

}  // namespace b2m
