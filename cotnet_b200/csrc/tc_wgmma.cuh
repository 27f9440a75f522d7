// wgmma (Hopper warpgroup MMA) PTX wrappers shared by the tensor-core kernels (tc_gemm.cu, tc_wgrad.cu), sm_90a.
//
// Every tensor-core kernel uses one instruction shape, m64n64k16 bf16 x bf16 -> fp32, with both operands read from shared memory
// through matrix descriptors.  A warpgroup owns a 64-row slice of the tile and keeps its accumulators in registers: 32 floats per
// thread per 64-column chunk, fragment layout (PTX ISA, wgmma "Matrix fragments for .m64nNk16"):
//   d[4 * i + 2 * h + e]  =  D[16 * (warp % 4) + lane / 4 + 8 * h][8 * i + 2 * (lane % 4) + e]      i = 0..7, h = 0..1, e = 0..1
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "tma.cuh"

namespace cotb200 {

// K-major, 128B-swizzled operand tile: rows of 128 B, 8-row atoms of 1024 B (SBO), LBO unused for swizzled K-major (=1),
// layout type 1 = 128B swizzle (bits 62-63).  The swizzle is a function of the absolute shared-memory address (that is how TMA
// wrote the tile), so a start address moved by whole 128-byte rows or by 32 bytes inside an atom addresses the same tile.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// MN-major, 128B-swizzled operand (canonical layout Swizzle<3,4,3> o ((64,m),(8,k)) : ((1,LBO),(64,SBO)) in elements): 64 MN elements
// (128 B) contiguous, 8 K rows of 128 B form a 1024-byte atom; SBO = bytes between consecutive 8-row K groups, LBO = bytes between
// consecutive 64-element MN blocks (an m64 / n64 instruction touches one MN block only).
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Keeps the compiler from moving accumulator reads or writes across an asynchronous wgmma (the registers change behind its back
// until wgmma_wait).
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// d (+)= A[64 x 16] * B[16 x 64]; TA / TB: 0 = K-major, 1 = MN-major operand; accumulate = 0 overwrites d
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

}  // namespace cotb200
